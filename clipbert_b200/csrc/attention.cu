// Fused self-attention for the cross-modal BertEncoder (reference: BertSelfAttention.forward,
// src/modeling/transformers.py:230-286): S = QK^T/sqrt(64) + additive mask, softmax (fp32),
// dropout on the probabilities, PV, heads merged in place. Probabilities never touch HBM: the
// backward recomputes them from Q, K and the saved log-sum-exp.
//
// Sequences on this path are short (L = Lt + 9 .. 521), head_dim is 64, and attention is < 1 % of
// the layer FLOPs at L = 41, so the kernel is a 64x64-tiled online-softmax CUDA-core kernel that
// packs a whole (sequence, head) into one or a few CTAs; it is latency- not FLOP-bound.
//
// By default every length runs on the tensor-core kernels of attention_tc.cu (L <= 64: one CTA per
// (sequence, head); longer: the flash forward and the two-kernel backward). The CUDA-core kernels
// here are the general path that cb_debug_attention_general(1) selects, and the reference the
// tensor-core kernels are tested against.
#include "common.cuh"
#include "host_util.h"

namespace cb {

constexpr int HD = 64;     // head dim
constexpr int TS = 64;     // tile size (queries / keys)
constexpr int LDS = 65;    // padded smem row stride (floats)
constexpr int ATT_THREADS = 256;
constexpr int TILE_FLOATS = TS * LDS;

using AttnDrop = DropCfg;   // (thresh, inv_keep, seed, device-side seed offset): drop_cfg.h

// load a [TS x 64] bf16 tile (rows r0.., row pitch ld elements) into fp32 smem; rows >= nrows are zero
__device__ __forceinline__ void load_tile(float* dst, const __nv_bfloat16* src, int64_t ld, int r0, int nrows) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    const int r = pass * 32 + (tid >> 3);
    const int c = (tid & 7) * 8;
    float f[8];
    if (r0 + r < nrows) {
      const uint4 u = *reinterpret_cast<const uint4*>(src + static_cast<int64_t>(r0 + r) * ld + c);
      float2 t;
      t = unpack_bf16x2(u.x); f[0] = t.x; f[1] = t.y;
      t = unpack_bf16x2(u.y); f[2] = t.x; f[3] = t.y;
      t = unpack_bf16x2(u.z); f[4] = t.x; f[5] = t.y;
      t = unpack_bf16x2(u.w); f[6] = t.x; f[7] = t.y;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) dst[r * LDS + c + j] = f[j];
  }
}
// store a [TS x 64] fp32 smem tile as bf16 rows (rows < nrows only)
__device__ __forceinline__ void store_tile(const float* src, __nv_bfloat16* dst, int64_t ld, int r0, int nrows) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    const int r = pass * 32 + (tid >> 3);
    const int c = (tid & 7) * 8;
    if (r0 + r < nrows) {
      const float* s = src + r * LDS + c;
      uint4 u;
      u.x = pack_bf16x2(s[0], s[1]); u.y = pack_bf16x2(s[2], s[3]);
      u.z = pack_bf16x2(s[4], s[5]); u.w = pack_bf16x2(s[6], s[7]);
      *reinterpret_cast<uint4*>(dst + static_cast<int64_t>(r0 + r) * ld + c) = u;
    }
  }
}

// acc[ii][jj] = sum_d A[4ty+ii][d] * B[tx+16jj][d]
__device__ __forceinline__ void mm_nt(const float* A, const float* B, int ty, int tx, float (&acc)[4][4]) {
#pragma unroll
  for (int ii = 0; ii < 4; ++ii)
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) acc[ii][jj] = 0.f;
#pragma unroll 8
  for (int d = 0; d < HD; ++d) {
    float a[4], b[4];
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) a[ii] = A[(4 * ty + ii) * LDS + d];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) b[jj] = B[(tx + 16 * jj) * LDS + d];
#pragma unroll
    for (int ii = 0; ii < 4; ++ii)
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) acc[ii][jj] = fmaf(a[ii], b[jj], acc[ii][jj]);
  }
}
// acc[ii][dd] += sum_j A[4ty+ii][j] * B[j][tx+16dd]
__device__ __forceinline__ void mm_nn(const float* A, const float* B, int ty, int tx, float (&acc)[4][4]) {
#pragma unroll 8
  for (int j = 0; j < TS; ++j) {
    float a[4], b[4];
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) a[ii] = A[(4 * ty + ii) * LDS + j];
#pragma unroll
    for (int dd = 0; dd < 4; ++dd) b[dd] = B[j * LDS + tx + 16 * dd];
#pragma unroll
    for (int ii = 0; ii < 4; ++ii)
#pragma unroll
      for (int dd = 0; dd < 4; ++dd) acc[ii][dd] = fmaf(a[ii], b[dd], acc[ii][dd]);
  }
}
// acc[jj][dd] += sum_i A[i][4ty+jj] * B[i][tx+16dd]
__device__ __forceinline__ void mm_tn(const float* A, const float* B, int ty, int tx, float (&acc)[4][4]) {
#pragma unroll 8
  for (int i = 0; i < TS; ++i) {
    float a[4], b[4];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) a[jj] = A[i * LDS + 4 * ty + jj];
#pragma unroll
    for (int dd = 0; dd < 4; ++dd) b[dd] = B[i * LDS + tx + 16 * dd];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
#pragma unroll
      for (int dd = 0; dd < 4; ++dd) acc[jj][dd] = fmaf(a[jj], b[dd], acc[jj][dd]);
  }
}

__device__ __forceinline__ float key_mask_add(const int64_t* text_mask, int b, int j, int Lt) {
  // hf get_extended_attention_mask: (1 - m) * -10000 ; visual tokens always attendable (modeling.py:217-227)
  if (j < Lt) return text_mask[static_cast<int64_t>(b) * Lt + j] != 0 ? 0.f : -10000.f;
  return 0.f;
}
__device__ __forceinline__ float red16_max(float v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float red16_sum(float v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(ATT_THREADS) attn_fwd_kernel(const __nv_bfloat16* __restrict__ q,
                                                               const __nv_bfloat16* __restrict__ k,
                                                               const __nv_bfloat16* __restrict__ v, int64_t ld_qkv,
                                                               const int64_t* __restrict__ text_mask,
                                                               __nv_bfloat16* __restrict__ ctx, int64_t ld_ctx,
                                                               float* __restrict__ lse, int L, int Lt, int H, float scale,
                                                               AttnDrop dc_in) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  const AttnDrop dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  extern __shared__ float sm[];
  float* Qs = sm;
  float* Ks = Qs + TILE_FLOATS;
  float* Vs = Ks + TILE_FLOATS;
  float* Ps = Vs + TILE_FLOATS;
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int64_t row0 = static_cast<int64_t>(b) * L;
  const __nv_bfloat16* qh = q + row0 * ld_qkv + h * HD;
  const __nv_bfloat16* kh = k + row0 * ld_qkv + h * HD;
  const __nv_bfloat16* vh = v + row0 * ld_qkv + h * HD;
  const int q0 = qb * TS;

  load_tile(Qs, qh, ld_qkv, q0, L);
  float m_i[4], l_i[4], o[4][4];
#pragma unroll
  for (int ii = 0; ii < 4; ++ii) {
    m_i[ii] = -INFINITY;
    l_i[ii] = 0.f;
#pragma unroll
    for (int dd = 0; dd < 4; ++dd) o[ii][dd] = 0.f;
  }
  const int nkb = (L + TS - 1) / TS;
  for (int kb = 0; kb < nkb; ++kb) {
    load_tile(Ks, kh, ld_qkv, kb * TS, L);
    load_tile(Vs, vh, ld_qkv, kb * TS, L);
    __syncthreads();
    float s[4][4];
    mm_nt(Qs, Ks, ty, tx, s);
    float madd[4];
    bool valid[4];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = kb * TS + tx + 16 * jj;
      valid[jj] = j < L;
      madd[jj] = valid[jj] ? key_mask_add(text_mask, b, j, Lt) : 0.f;
    }
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        s[ii][jj] = valid[jj] ? s[ii][jj] * scale + madd[jj] : -INFINITY;
        mx = fmaxf(mx, s[ii][jj]);
      }
      mx = red16_max(mx);
      const float m_new = fmaxf(m_i[ii], mx);
      const float corr = __expf(m_i[ii] - m_new);
      float rs = 0.f;
      const int i = q0 + 4 * ty + ii;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const float p = valid[jj] ? __expf(s[ii][jj] - m_new) : 0.f;
        rs += p;
        float pd = p;
        if (dc.thresh) {
          const int j = kb * TS + tx + 16 * jj;
          const uint64_t idx = ((static_cast<uint64_t>(b) * H + h) * L + i) * L + j;
          pd *= dropout_mult(dc.seed, idx, dc.thresh, dc.inv_keep);
        }
        Ps[(4 * ty + ii) * LDS + tx + 16 * jj] = pd;
      }
      rs = red16_sum(rs);
      l_i[ii] = l_i[ii] * corr + rs;
      m_i[ii] = m_new;
#pragma unroll
      for (int dd = 0; dd < 4; ++dd) o[ii][dd] *= corr;
    }
    __syncthreads();
    mm_nn(Ps, Vs, ty, tx, o);
    __syncthreads();
  }
  // normalise, stage through smem for coalesced bf16 stores
#pragma unroll
  for (int ii = 0; ii < 4; ++ii) {
    const float inv = 1.0f / l_i[ii];
#pragma unroll
    for (int dd = 0; dd < 4; ++dd) Ps[(4 * ty + ii) * LDS + tx + 16 * dd] = o[ii][dd] * inv;
    const int i = q0 + 4 * ty + ii;
    if (tx == 0 && i < L && lse) lse[(static_cast<int64_t>(b) * H + h) * L + i] = m_i[ii] + __logf(l_i[ii]);
  }
  __syncthreads();
  store_tile(Ps, ctx + row0 * ld_ctx + h * HD, ld_ctx, q0, L);
}

// ------------------------------------------------------------------------------------------------
// backward, shared pieces
// ------------------------------------------------------------------------------------------------
// Ds[i] = sum_d dO[i][d] * O[i][d] for the 64 query rows of a tile; lses[i] = saved log-sum-exp
__device__ __forceinline__ void load_row_stats(const float* dOs, const __nv_bfloat16* ctx_h, int64_t ld_ctx,
                                               const float* lse_bh, int q0, int L, float* Ds, float* lses) {
  const int tid = threadIdx.x;
  const int r = tid >> 2, part = tid & 3;
  float acc = 0.f;
  if (q0 + r < L) {
    const __nv_bfloat16* orow = ctx_h + static_cast<int64_t>(q0 + r) * ld_ctx + part * 16;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const uint4 u = *reinterpret_cast<const uint4*>(orow + half * 8);
      const float* d = dOs + r * LDS + part * 16 + half * 8;
      float2 t;
      t = unpack_bf16x2(u.x); acc += t.x * d[0] + t.y * d[1];
      t = unpack_bf16x2(u.y); acc += t.x * d[2] + t.y * d[3];
      t = unpack_bf16x2(u.z); acc += t.x * d[4] + t.y * d[5];
      t = unpack_bf16x2(u.w); acc += t.x * d[6] + t.y * d[7];
    }
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  if (part == 0) {
    Ds[r] = acc;
    lses[r] = (q0 + r < L) ? lse_bh[q0 + r] : 0.f;
  }
}

// computes for the (query tile, key tile) pair: Pd (dropped probs) and dS, written to smem
__device__ __forceinline__ void compute_p_ds(const float* Qs, const float* Ks, const float* Vs, const float* dOs,
                                             const float* Ds, const float* lses, const int64_t* text_mask, int b, int h,
                                             int H, int q0, int k0, int L, int Lt, float scale, const AttnDrop& dc,
                                             float* Pd_out, float* dS_out, int ty, int tx) {
  float s[4][4], dp[4][4];
  mm_nt(Qs, Ks, ty, tx, s);
  mm_nt(dOs, Vs, ty, tx, dp);
#pragma unroll
  for (int ii = 0; ii < 4; ++ii) {
    const int i = q0 + 4 * ty + ii;
    const float lse_i = lses[4 * ty + ii], D_i = Ds[4 * ty + ii];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = k0 + tx + 16 * jj;
      float p = 0.f, r = 1.f;
      if (i < L && j < L) {
        p = __expf(s[ii][jj] * scale + key_mask_add(text_mask, b, j, Lt) - lse_i);
        if (dc.thresh) {
          const uint64_t idx = ((static_cast<uint64_t>(b) * H + h) * L + i) * L + j;
          r = dropout_mult(dc.seed, idx, dc.thresh, dc.inv_keep);
        }
      }
      if (Pd_out) Pd_out[(4 * ty + ii) * LDS + tx + 16 * jj] = p * r;
      dS_out[(4 * ty + ii) * LDS + tx + 16 * jj] = p * (dp[ii][jj] * r - D_i);
    }
  }
}

// dK, dV for one key tile; loops over query tiles
__global__ void __launch_bounds__(ATT_THREADS) attn_bwd_kv_kernel(
    const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k, const __nv_bfloat16* __restrict__ v,
    int64_t ld_qkv, const int64_t* __restrict__ text_mask, const __nv_bfloat16* __restrict__ ctx,
    const __nv_bfloat16* __restrict__ dctx, int64_t ld_ctx, const float* __restrict__ lse, __nv_bfloat16* __restrict__ dk,
    __nv_bfloat16* __restrict__ dv, int64_t ld_dqkv, int L, int Lt, int H, float scale, AttnDrop dc_in) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  const AttnDrop dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  extern __shared__ float sm[];
  float* Ks = sm;
  float* Vs = Ks + TILE_FLOATS;
  float* Qs = Vs + TILE_FLOATS;
  float* dOs = Qs + TILE_FLOATS;
  float* Ps = dOs + TILE_FLOATS;
  float* dSs = Ps + TILE_FLOATS;
  float* Ds = dSs + TILE_FLOATS;
  float* lses = Ds + TS;
  const int kb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int64_t row0 = static_cast<int64_t>(b) * L;
  const int k0 = kb * TS;
  load_tile(Ks, k + row0 * ld_qkv + h * HD, ld_qkv, k0, L);
  load_tile(Vs, v + row0 * ld_qkv + h * HD, ld_qkv, k0, L);
  float dK[4][4], dV[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int c = 0; c < 4; ++c) dK[a][c] = dV[a][c] = 0.f;
  const int nqb = (L + TS - 1) / TS;
  for (int qb = 0; qb < nqb; ++qb) {
    const int q0 = qb * TS;
    load_tile(Qs, q + row0 * ld_qkv + h * HD, ld_qkv, q0, L);
    load_tile(dOs, dctx + row0 * ld_ctx + h * HD, ld_ctx, q0, L);
    __syncthreads();
    load_row_stats(dOs, ctx + row0 * ld_ctx + h * HD, ld_ctx, lse + (static_cast<int64_t>(b) * H + h) * L, q0, L, Ds, lses);
    __syncthreads();
    compute_p_ds(Qs, Ks, Vs, dOs, Ds, lses, text_mask, b, h, H, q0, k0, L, Lt, scale, dc, Ps, dSs, ty, tx);
    __syncthreads();
    mm_tn(Ps, dOs, ty, tx, dV);
    mm_tn(dSs, Qs, ty, tx, dK);
    __syncthreads();
  }
  // stage through smem for coalesced stores
#pragma unroll
  for (int jj = 0; jj < 4; ++jj)
#pragma unroll
    for (int dd = 0; dd < 4; ++dd) {
      Ps[(4 * ty + jj) * LDS + tx + 16 * dd] = dV[jj][dd];
      dSs[(4 * ty + jj) * LDS + tx + 16 * dd] = dK[jj][dd] * scale;
    }
  __syncthreads();
  store_tile(Ps, dv + row0 * ld_dqkv + h * HD, ld_dqkv, k0, L);
  store_tile(dSs, dk + row0 * ld_dqkv + h * HD, ld_dqkv, k0, L);
}

// dQ for one query tile; loops over key tiles
__global__ void __launch_bounds__(ATT_THREADS) attn_bwd_q_kernel(
    const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k, const __nv_bfloat16* __restrict__ v,
    int64_t ld_qkv, const int64_t* __restrict__ text_mask, const __nv_bfloat16* __restrict__ ctx,
    const __nv_bfloat16* __restrict__ dctx, int64_t ld_ctx, const float* __restrict__ lse, __nv_bfloat16* __restrict__ dq,
    int64_t ld_dqkv, int L, int Lt, int H, float scale, AttnDrop dc_in) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  const AttnDrop dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  extern __shared__ float sm[];
  float* Qs = sm;
  float* dOs = Qs + TILE_FLOATS;
  float* Ks = dOs + TILE_FLOATS;
  float* Vs = Ks + TILE_FLOATS;
  float* dSs = Vs + TILE_FLOATS;
  float* Ds = dSs + TILE_FLOATS;
  float* lses = Ds + TS;
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int64_t row0 = static_cast<int64_t>(b) * L;
  const int q0 = qb * TS;
  load_tile(Qs, q + row0 * ld_qkv + h * HD, ld_qkv, q0, L);
  load_tile(dOs, dctx + row0 * ld_ctx + h * HD, ld_ctx, q0, L);
  __syncthreads();
  load_row_stats(dOs, ctx + row0 * ld_ctx + h * HD, ld_ctx, lse + (static_cast<int64_t>(b) * H + h) * L, q0, L, Ds, lses);
  float dQ[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int c = 0; c < 4; ++c) dQ[a][c] = 0.f;
  const int nkb = (L + TS - 1) / TS;
  for (int kb = 0; kb < nkb; ++kb) {
    const int k0 = kb * TS;
    load_tile(Ks, k + row0 * ld_qkv + h * HD, ld_qkv, k0, L);
    load_tile(Vs, v + row0 * ld_qkv + h * HD, ld_qkv, k0, L);
    __syncthreads();
    compute_p_ds(Qs, Ks, Vs, dOs, Ds, lses, text_mask, b, h, H, q0, k0, L, Lt, scale, dc, nullptr, dSs, ty, tx);
    __syncthreads();
    mm_nn(dSs, Ks, ty, tx, dQ);
    __syncthreads();
  }
#pragma unroll
  for (int ii = 0; ii < 4; ++ii)
#pragma unroll
    for (int dd = 0; dd < 4; ++dd) dSs[(4 * ty + ii) * LDS + tx + 16 * dd] = dQ[ii][dd] * scale;
  __syncthreads();
  store_tile(dSs, dq + row0 * ld_dqkv + h * HD, ld_dqkv, q0, L);
}

static AttnDrop make_attn_drop(float p, uint64_t seed) { return make_drop(p, seed); }

template <typename K>
static int set_smem(K kern, int bytes) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) {
    set_error("cudaFuncSetAttribute(attention smem=%d): %s", bytes, cudaGetErrorString(e));
    return CB_ERR_CUDA;
  }
  return CB_OK;
}

// tensor-core fast path for l <= 64 (attention_tc.cu)
int attention_tc_fwd(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, void* ctx, int64_t ld_ctx, float* lse, int nseq, int l, int lt,
                     int heads, float dropout_p, uint64_t seed, cudaStream_t stream);
int attention_tc_bwd(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, const void* ctx, const void* dctx, int64_t ld_ctx,
                     const float* lse, void* dqkv, int64_t ld_dqkv, int nseq, int l, int lt, int heads, float dropout_p, uint64_t seed,
                     cudaStream_t stream);
int attention_tc_fwd_flash(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, void* ctx, int64_t ld_ctx, float* lse, int nseq, int l,
                           int lt, int heads, float dropout_p, uint64_t seed, cudaStream_t stream);
int attention_tc_bwd_long(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, const void* ctx, const void* dctx, int64_t ld_ctx,
                          const float* lse, void* dqkv, int64_t ld_dqkv, int nseq, int l, int lt, int heads, float dropout_p, uint64_t seed,
                          cudaStream_t stream);
void attention_tc_set_flash_pipe(int on);   // 1 (default): cp.async double-buffered key tiles in the long-sequence forward
void attention_tc_set_rows48(int on);   // 1 (default): sequences of up to 48 tokens on the 48-row / three-warp kernels
int g_attention_force_general = 0;   // test knob: 1 = always use the general (any L) kernels
int g_attention_flash = 1;           // 1 = forward of sequences longer than 64 tokens on the tensor-core online-softmax kernel
                                     // (attention_tc.cu)

}  // namespace cb

using namespace cb;

extern "C" {

void cb_debug_attention_general(int on) { cb::g_attention_force_general = on; }
void cb_debug_attention_flash(int on) { cb::g_attention_flash = on; }
void cb_debug_attention_rows48(int on) { cb::attention_tc_set_rows48(on); }
void cb_debug_attention_flash_pipe(int on) { cb::attention_tc_set_flash_pipe(on); }

/* qkv: bf16 [nseq*L, 3*heads*64] (Q | K | V); text_mask: int64 [nseq, Lt]; ctx: bf16 [nseq*L, heads*64];
 * lse: fp32 [nseq, heads, L] (saved for the backward; may be NULL for inference). */
int cb_attention_fwd(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, void* ctx, int64_t ld_ctx, float* lse,
                     int nseq, int l, int lt, int heads, int head_dim, float dropout_p, uint64_t seed, void* stream) {
  CB_REQUIRE(head_dim == HD, "cb_attention_fwd: head_dim %d unsupported (built for 64)", head_dim);
  CB_REQUIRE(qkv && text_mask && ctx && nseq > 0 && l > 0 && lt >= 0 && lt <= l && heads > 0, "cb_attention_fwd: bad arguments");
  CB_REQUIRE(ld_qkv % 8 == 0 && ld_ctx % 8 == 0, "cb_attention_fwd: row pitches must be multiples of 8");
  if (l <= 64 && !g_attention_force_general)
    return attention_tc_fwd(qkv, ld_qkv, text_mask, ctx, ld_ctx, lse, nseq, l, lt, heads, dropout_p, seed, static_cast<cudaStream_t>(stream));
  if (l > 64 && g_attention_flash && !g_attention_force_general)
    return attention_tc_fwd_flash(qkv, ld_qkv, text_mask, ctx, ld_ctx, lse, nseq, l, lt, heads, dropout_p, seed, static_cast<cudaStream_t>(stream));
  static bool once = false;
  const int smem = 4 * TILE_FLOATS * sizeof(float);
  if (!once) {
    int rc = set_smem(attn_fwd_kernel, smem);
    if (rc) return rc;
    once = true;
  }
  const __nv_bfloat16* base = static_cast<const __nv_bfloat16*>(qkv);
  const int hid = heads * HD;
  dim3 grid(ceil_div(l, TS), heads, nseq);
  launch_k(attn_fwd_kernel, grid, ATT_THREADS, smem, static_cast<cudaStream_t>(stream), 
      base, base + hid, base + 2 * hid, ld_qkv, text_mask, static_cast<__nv_bfloat16*>(ctx), ld_ctx, lse, l, lt, heads,
      0.125f, make_attn_drop(dropout_p, seed));
  return check_launch("cb_attention_fwd");
}

int cb_attention_bwd(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, const void* ctx, const void* dctx,
                     int64_t ld_ctx, const float* lse, void* dqkv, int64_t ld_dqkv, int nseq, int l, int lt, int heads,
                     int head_dim, float dropout_p, uint64_t seed, void* stream) {
  CB_REQUIRE(head_dim == HD, "cb_attention_bwd: head_dim %d unsupported (built for 64)", head_dim);
  CB_REQUIRE(qkv && text_mask && ctx && dctx && lse && dqkv && nseq > 0 && l > 0, "cb_attention_bwd: bad arguments");
  CB_REQUIRE(ld_qkv % 8 == 0 && ld_ctx % 8 == 0 && ld_dqkv % 8 == 0, "cb_attention_bwd: row pitches must be multiples of 8");
  if (l <= 64 && !g_attention_force_general)
    return attention_tc_bwd(qkv, ld_qkv, text_mask, ctx, dctx, ld_ctx, lse, dqkv, ld_dqkv, nseq, l, lt, heads, dropout_p, seed,
                            static_cast<cudaStream_t>(stream));
  if (l > 64 && !g_attention_force_general)
    return attention_tc_bwd_long(qkv, ld_qkv, text_mask, ctx, dctx, ld_ctx, lse, dqkv, ld_dqkv, nseq, l, lt, heads, dropout_p, seed,
                                 static_cast<cudaStream_t>(stream));
  static bool once = false;
  const int smem_kv = (6 * TILE_FLOATS + 2 * TS) * sizeof(float);
  const int smem_q = (5 * TILE_FLOATS + 2 * TS) * sizeof(float);
  if (!once) {
    int rc = set_smem(attn_bwd_kv_kernel, smem_kv);
    if (rc) return rc;
    rc = set_smem(attn_bwd_q_kernel, smem_q);
    if (rc) return rc;
    once = true;
  }
  const __nv_bfloat16* base = static_cast<const __nv_bfloat16*>(qkv);
  __nv_bfloat16* dbase = static_cast<__nv_bfloat16*>(dqkv);
  const int hid = heads * HD;
  const AttnDrop dc = make_attn_drop(dropout_p, seed);
  dim3 grid(ceil_div(l, TS), heads, nseq);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  launch_k(attn_bwd_kv_kernel, grid, ATT_THREADS, smem_kv, st, base, base + hid, base + 2 * hid, ld_qkv, text_mask,
                                                         static_cast<const __nv_bfloat16*>(ctx),
                                                         static_cast<const __nv_bfloat16*>(dctx), ld_ctx, lse, dbase + hid,
                                                         dbase + 2 * hid, ld_dqkv, l, lt, heads, 0.125f, dc);
  int rc = check_launch("cb_attention_bwd(kv)");
  if (rc) return rc;
  launch_k(attn_bwd_q_kernel, grid, ATT_THREADS, smem_q, st, base, base + hid, base + 2 * hid, ld_qkv, text_mask,
                                                       static_cast<const __nv_bfloat16*>(ctx),
                                                       static_cast<const __nv_bfloat16*>(dctx), ld_ctx, lse, dbase, ld_dqkv, l,
                                                       lt, heads, 0.125f, dc);
  return check_launch("cb_attention_bwd(q)");
}

}  // extern "C"
