// Tensor-core fast path of the fused self-attention for short sequences (L <= 64: every ClipBERT training
// configuration at 224 px, L = Lt + 9). One CTA = one (sequence, head); 4 warps x 16 query rows; Q, K, V (and dO)
// tiles live in shared memory as bf16, the 64x64x64 products run on mma.sync.m16n8k16 (bf16 in, fp32 accumulate)
// with ldmatrix operand fetches, softmax / dropout / dS stay in the accumulator registers (the S accumulator
// layout is reused as the A operand of the next product). Same math, masks, dropout stream and lse convention as
// csrc/attention.cu, whose CUDA-core kernels remain the general path (cb_debug_attention_general) and the test reference.
// Sequences longer than 64 tokens (448 / 768 px frames, 512-token inference) run the multi-tile kernels further down: the
// online-softmax forward (attn_tc_fwd_flash_kernel) and the backward pair attn_tc_bwd_kv_kernel / attn_tc_bwd_q_kernel.
//
// Why mma.sync and not wgmma here: a (sequence, head) problem is 41x41x64 - 0.9 % of the layer FLOPs; it is
// latency-bound, and a wgmma pipeline (warpgroup-wide 64-row tiles, TMA staging, mbarrier hand-offs) costs more than
// the whole product. All GEMM-shaped work of the path runs on wgmma (csrc/gemm.cu).
#include "common.cuh"
#include "host_util.h"

namespace cb {

constexpr int TC_LD = 72;                 // bf16 elements per smem row (144 B: 16 B aligned, conflict-free ldmatrix)
constexpr int TC_TILE = 64 * TC_LD;       // elements per 64-row tile
constexpr int TC_THREADS = 128;

using TcDrop = DropCfg;   // (thresh, inv_keep, seed, device-side seed offset): drop_cfg.h

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const __nv_bfloat16* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const __nv_bfloat16* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// global [rows, 64] bf16 (row pitch ld) -> smem tile [R][TC_LD], rows >= nrows zero-filled. R = 64, or 48 for the three-warp
// kernels of sequences up to 48 tokens (blockDim.x = 2 R threads)
template <int R = 64>
__device__ __forceinline__ void tc_load_tile(__nv_bfloat16* dst, const __nv_bfloat16* src, int64_t ld, int nrows) {
#pragma unroll
  for (int i = threadIdx.x; i < R * 8; i += 2 * R) {
    const int r = i >> 3, c = (i & 7) * 8;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (r < nrows) u = *reinterpret_cast<const uint4*>(src + static_cast<int64_t>(r) * ld + c);
    *reinterpret_cast<uint4*>(dst + r * TC_LD + c) = u;
  }
}
template <int R = 64>
__device__ __forceinline__ void tc_store_tile(const __nv_bfloat16* src, __nv_bfloat16* dst, int64_t ld, int nrows) {
#pragma unroll
  for (int i = threadIdx.x; i < R * 8; i += 2 * R) {
    const int r = i >> 3, c = (i & 7) * 8;
    if (r < nrows) *reinterpret_cast<uint4*>(dst + static_cast<int64_t>(r) * ld + c) = *reinterpret_cast<const uint4*>(src + r * TC_LD + c);
  }
}

// acc[j][4] (j = 8-wide column tile) = A(16 x 64 rows r0.. of As) * B^T where B rows are the OUTPUT columns
// (B stored [n][k] row-major, e.g. S = Q K^T with Bs = K, or dP = dO V^T with Bs = V)
// NJP = pairs of 8-wide output column tiles = rows of Bs / 16 (4: 64 keys, 3: 48 keys)
template <int NJP = 4>
__device__ __forceinline__ void tc_mm_abt(float (&acc)[2 * NJP][4], const __nv_bfloat16* As, const __nv_bfloat16* Bs, int r0, int lane) {
#pragma unroll
  for (int j = 0; j < 2 * NJP; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    uint32_t a[4];
    ldsm_x4(a, As + (r0 + (lane & 15)) * TC_LD + ks * 16 + (lane >> 4) * 8);
#pragma unroll
    for (int jp = 0; jp < NJP; ++jp) {     // two 8-column tiles per ldmatrix.x4
      uint32_t b[4];
      ldsm_x4(b, Bs + (jp * 16 + (lane & 7) + (lane >> 4) * 8) * TC_LD + ks * 16 + ((lane >> 3) & 1) * 8);
      mma16816(acc[2 * jp], a, b[0], b[1]);
      mma16816(acc[2 * jp + 1], a, b[2], b[3]);
    }
  }
}
// acc += A(16 x 64, given as register fragments afrag[ks]) * B where B is stored [k][n] row-major (e.g. O = P V, dQ = dS K)
// NKS = 16-row slabs of Bs contracted over (4: 64 keys, 3: 48 keys)
template <int NKS = 4>
__device__ __forceinline__ void tc_mm_ab_reg(float (&acc)[8][4], const uint32_t (&afrag)[NKS][4], const __nv_bfloat16* Bs, int lane) {
#pragma unroll
  for (int ks = 0; ks < NKS; ++ks) {
#pragma unroll
    for (int jp = 0; jp < 4; ++jp) {
      uint32_t b[4];
      ldsm_x4_t(b, Bs + (ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * TC_LD + jp * 16 + (lane >> 4) * 8);
      mma16816(acc[2 * jp], afrag[ks], b[0], b[1]);
      mma16816(acc[2 * jp + 1], afrag[ks], b[2], b[3]);
    }
  }
}
// acc = A^T-stored (As holds [k][m]: out rows m0.. come from As COLUMNS) * B ([k][n] row-major): dV = Pd^T dO, dK = dS^T Q
template <int NKS = 4>
__device__ __forceinline__ void tc_mm_atb(float (&acc)[8][4], const __nv_bfloat16* As, const __nv_bfloat16* Bs, int m0, int lane) {
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < NKS; ++ks) {
    uint32_t a[4];
    const int mi = lane >> 3;
    ldsm_x4_t(a, As + (ks * 16 + (lane & 7) + (mi >> 1) * 8) * TC_LD + m0 + (mi & 1) * 8);
#pragma unroll
    for (int jp = 0; jp < 4; ++jp) {
      uint32_t b[4];
      ldsm_x4_t(b, Bs + (ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * TC_LD + jp * 16 + (lane >> 4) * 8);
      mma16816(acc[2 * jp], a, b[0], b[1]);
      mma16816(acc[2 * jp + 1], a, b[2], b[3]);
    }
  }
}
// write a 16 x 64 accumulator (rows r0 + lane/4, +8) as bf16 into a smem tile
__device__ __forceinline__ void tc_acc_to_smem(const float (&acc)[8][4], __nv_bfloat16* dst, int r0, int lane, float mul) {
  const int r = r0 + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    *reinterpret_cast<uint32_t*>(dst + r * TC_LD + j * 8 + c) = pack_bf16x2(acc[j][0] * mul, acc[j][1] * mul);
    *reinterpret_cast<uint32_t*>(dst + (r + 8) * TC_LD + j * 8 + c) = pack_bf16x2(acc[j][2] * mul, acc[j][3] * mul);
  }
}

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// ------------------------------------------------------------------------------------------------ forward
// RT = 16-row tiles per (sequence, head): 4 (L <= 64, 128 threads) or 3 (L <= 48, 96 threads: every 224-px configuration has
// L = 41 - a quarter fewer warps, 44 % fewer MMAs and smaller tiles than padding to 64)
template <int RT>
__global__ void __launch_bounds__(RT * 32) attn_tc_fwd_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                                                 const __nv_bfloat16* __restrict__ v, int64_t ld_qkv,
                                                                 const int64_t* __restrict__ text_mask, __nv_bfloat16* __restrict__ ctx,
                                                                 int64_t ld_ctx, float* __restrict__ lse, int L, int Lt, int H, float scale,
                                                                 TcDrop dc_in) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  const TcDrop dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  extern __shared__ __align__(16) uint8_t tc_smem[];
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(tc_smem);
  constexpr int R = RT * 16, TILE = R * TC_LD;
  __nv_bfloat16* Ks = Qs + TILE;
  __nv_bfloat16* Vs = Ks + TILE;
  float* madd = reinterpret_cast<float*>(Vs + TILE);     // [R] additive key mask (-inf beyond L)
  const int h = blockIdx.x, b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row0 = static_cast<int64_t>(b) * L;
  tc_load_tile<R>(Qs, q + row0 * ld_qkv + h * 64, ld_qkv, L);
  tc_load_tile<R>(Ks, k + row0 * ld_qkv + h * 64, ld_qkv, L);
  tc_load_tile<R>(Vs, v + row0 * ld_qkv + h * 64, ld_qkv, L);
  if (threadIdx.x < R) {
    const int j = threadIdx.x;
    float m = -INFINITY;
    if (j < L) m = (j < Lt && text_mask[static_cast<int64_t>(b) * Lt + j] == 0) ? -10000.f : 0.f;
    madd[j] = m;
  }
  __syncthreads();
  const int r0 = warp * 16;
  float s[2 * RT][4];
  tc_mm_abt<RT>(s, Qs, Ks, r0, lane);
  const int rq = r0 + (lane >> 2), cq = 2 * (lane & 3);
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int j = 0; j < 2 * RT; ++j) {
    const float m0 = madd[j * 8 + cq], m1 = madd[j * 8 + cq + 1];
    s[j][0] = s[j][0] * scale + m0; s[j][1] = s[j][1] * scale + m1;
    s[j][2] = s[j][2] * scale + m0; s[j][3] = s[j][3] * scale + m1;
    mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1]));
    mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
  }
  mx0 = quad_max(mx0);
  mx1 = quad_max(mx1);
  float sum0 = 0.f, sum1 = 0.f;
  uint32_t pf[RT][4];     // P as A fragments for the P V product
#pragma unroll
  for (int j = 0; j < 2 * RT; ++j) {
    float p0 = __expf(s[j][0] - mx0), p1 = __expf(s[j][1] - mx0), p2 = __expf(s[j][2] - mx1), p3 = __expf(s[j][3] - mx1);
    sum0 += p0 + p1;
    sum1 += p2 + p3;
    if (dc.thresh) {
      const uint64_t base0 = ((static_cast<uint64_t>(b) * H + h) * L + rq) * L + j * 8 + cq;
      const uint64_t base1 = base0 + static_cast<uint64_t>(8) * L;
      { float m0_, m1_; dropout_mult2(dc.seed, base0, dc.thresh, dc.inv_keep, m0_, m1_); p0 *= m0_; p1 *= m1_; }
      { float m0_, m1_; dropout_mult2(dc.seed, base1, dc.thresh, dc.inv_keep, m0_, m1_); p2 *= m0_; p3 *= m1_; }
    }
    pf[j >> 1][(j & 1) * 2] = pack_bf16x2(p0, p1);
    pf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2, p3);
  }
  sum0 = quad_sum(sum0);
  sum1 = quad_sum(sum1);
  float o[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[j][e] = 0.f;
  tc_mm_ab_reg(o, pf, Vs, lane);
  const float i0 = 1.0f / sum0, i1 = 1.0f / sum1;
#pragma unroll
  for (int j = 0; j < 8; ++j) { o[j][0] *= i0; o[j][1] *= i0; o[j][2] *= i1; o[j][3] *= i1; }
  if (lse && (lane & 3) == 0) {
    float* lrow = lse + (static_cast<int64_t>(b) * H + h) * L;
    if (rq < L) lrow[rq] = mx0 + __logf(sum0);
    if (rq + 8 < L) lrow[rq + 8] = mx1 + __logf(sum1);
  }
  __syncthreads();                       // everyone is done reading Qs: reuse it to stage the output
  tc_acc_to_smem(o, Qs, r0, lane, 1.0f);
  __syncthreads();
  tc_store_tile<R>(Qs, ctx + row0 * ld_ctx + h * 64, ld_ctx, L);
}

// ------------------------------------------------------------------------------------------------ forward, any L
// The same tensor-core forward for sequences longer than one tile (448 px frames: L = 69; paragraph-retrieval inference:
// L = 512 + 9): one CTA = 64 query rows of one (sequence, head), looping over 64-key tiles with the online-softmax
// recurrence (running row max m, running sum, accumulator rescaled by exp(m_old - m_new)). Mask, dropout stream
// (index = ((b*H + h)*L + query)*L + key) and the saved log-sum-exp follow attn_fwd_kernel (attention.cu), so the general
// backward kernels consume its output unchanged. At L = 521 the CUDA-core kernel spends 0.83 GFLOP per (sequence, layer)
// on fp32 FMAs - more than the whole layer's GEMM time; this path puts those products on mma.sync.
// PIPE = true (default): the K / V / mask tiles are double-buffered and the next key tile travels global -> shared with cp.async
// (zero-filled beyond L) while the current one is multiplied; PIPE = false: the synchronous loads of the first version (A/B).
__device__ __forceinline__ void cp_async16_zfill(__nv_bfloat16* dst, const __nv_bfloat16* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// global [rows, 64] bf16 -> smem tile [64][TC_LD] with cp.async, rows >= nrows zero-filled (their source address is clamped to row 0)
__device__ __forceinline__ void tc_load_tile_async(__nv_bfloat16* dst, const __nv_bfloat16* src, int64_t ld, int nrows) {
#pragma unroll
  for (int i = threadIdx.x; i < 64 * 8; i += TC_THREADS) {
    const int r = i >> 3, c = (i & 7) * 8;
    const bool ok = r < nrows;
    cp_async16_zfill(dst + r * TC_LD + c, src + (ok ? static_cast<int64_t>(r) * ld : 0) + c, ok ? 16 : 0);
  }
}

template <bool PIPE>
__global__ void __launch_bounds__(TC_THREADS) attn_tc_fwd_flash_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                                                       const __nv_bfloat16* __restrict__ v, int64_t ld_qkv,
                                                                       const int64_t* __restrict__ text_mask, __nv_bfloat16* __restrict__ ctx,
                                                                       int64_t ld_ctx, float* __restrict__ lse, int L, int Lt, int H, float scale,
                                                                       TcDrop dc_in) {
  pdl_wait();
  const TcDrop dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  extern __shared__ __align__(16) uint8_t tc_smem[];
  constexpr int NBUF = PIPE ? 2 : 1;
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(tc_smem);
  __nv_bfloat16* Kbuf = Qs + TC_TILE;                        // [NBUF] K tiles
  __nv_bfloat16* Vbuf = Kbuf + NBUF * TC_TILE;               // [NBUF] V tiles
  float* mbuf = reinterpret_cast<float*>(Vbuf + NBUF * TC_TILE);   // [NBUF][64] additive key mask of a key tile (-inf beyond L)
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = qb * 64;
  const int64_t row0 = static_cast<int64_t>(b) * L;
  const int nkb = (L + 63) / 64;
  auto load_keys = [&](int kb, int buf) {                    // K, V and mask of key tile kb into buffer buf
    const int k0 = kb * 64;
    if (PIPE) {
      tc_load_tile_async(Kbuf + buf * TC_TILE, k + (row0 + k0) * ld_qkv + h * 64, ld_qkv, L - k0);
      tc_load_tile_async(Vbuf + buf * TC_TILE, v + (row0 + k0) * ld_qkv + h * 64, ld_qkv, L - k0);
      cp_async_commit();
    } else {
      tc_load_tile(Kbuf, k + (row0 + k0) * ld_qkv + h * 64, ld_qkv, L - k0);
      tc_load_tile(Vbuf, v + (row0 + k0) * ld_qkv + h * 64, ld_qkv, L - k0);
    }
    if (threadIdx.x < 64) {
      const int j = k0 + threadIdx.x;
      float m = -INFINITY;
      if (j < L) m = (j < Lt && text_mask[static_cast<int64_t>(b) * Lt + j] == 0) ? -10000.f : 0.f;
      mbuf[buf * 64 + threadIdx.x] = m;
    }
  };
  tc_load_tile(Qs, q + (row0 + q0) * ld_qkv + h * 64, ld_qkv, L - q0);
  if (PIPE) load_keys(0, 0);
  const int r0 = warp * 16;
  const int rq = r0 + (lane >> 2), cq = 2 * (lane & 3);
  float m0 = -INFINITY, m1 = -INFINITY, sum0 = 0.f, sum1 = 0.f;
  float o[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[j][e] = 0.f;
  for (int kb = 0; kb < nkb; ++kb) {
    const int k0 = kb * 64;
    const int buf = PIPE ? (kb & 1) : 0;
    __syncthreads();                     // the tile multiplied in the previous iteration (buffer buf ^ 1 / the only buffer) is free
    if (PIPE) {
      if (kb + 1 < nkb) {
        load_keys(kb + 1, buf ^ 1);      // travels while this tile is multiplied
        cp_async_wait<1>();              // every group but the one just committed: this thread's part of tile kb has landed
      } else {
        cp_async_wait<0>();
      }
    } else {
      load_keys(kb, 0);
    }
    __syncthreads();                     // tile kb (and Q, and its mask) visible to every warp
    const __nv_bfloat16* Ks = Kbuf + buf * TC_TILE;
    const __nv_bfloat16* Vs = Vbuf + buf * TC_TILE;
    const float* madd = mbuf + buf * 64;
    float s[8][4];
    tc_mm_abt(s, Qs, Ks, r0, lane);
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float a0 = madd[j * 8 + cq], a1 = madd[j * 8 + cq + 1];
      s[j][0] = s[j][0] * scale + a0; s[j][1] = s[j][1] * scale + a1;
      s[j][2] = s[j][2] * scale + a0; s[j][3] = s[j][3] * scale + a1;
      mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1]));
      mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
    }
    mx0 = quad_max(mx0);
    mx1 = quad_max(mx1);
    const float n0 = fmaxf(m0, mx0), n1 = fmaxf(m1, mx1);       // finite: every key tile holds at least one key < L
    const float c0 = __expf(m0 - n0), c1 = __expf(m1 - n1);     // exp(-inf) = 0 on the first tile
    float t0 = 0.f, t1 = 0.f;
    uint32_t pf[4][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float p0 = __expf(s[j][0] - n0), p1 = __expf(s[j][1] - n0), p2 = __expf(s[j][2] - n1), p3 = __expf(s[j][3] - n1);
      t0 += p0 + p1;
      t1 += p2 + p3;
      if (dc.thresh) {
        const uint64_t base0 = ((static_cast<uint64_t>(b) * H + h) * L + (q0 + rq)) * L + k0 + j * 8 + cq;
        const uint64_t base1 = base0 + static_cast<uint64_t>(8) * L;
        { float m0_, m1_; dropout_mult2(dc.seed, base0, dc.thresh, dc.inv_keep, m0_, m1_); p0 *= m0_; p1 *= m1_; }
        { float m0_, m1_; dropout_mult2(dc.seed, base1, dc.thresh, dc.inv_keep, m0_, m1_); p2 *= m0_; p3 *= m1_; }
      }
      pf[j >> 1][(j & 1) * 2] = pack_bf16x2(p0, p1);
      pf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2, p3);
    }
    t0 = quad_sum(t0);
    t1 = quad_sum(t1);
    sum0 = sum0 * c0 + t0;
    sum1 = sum1 * c1 + t1;
    m0 = n0;
    m1 = n1;
#pragma unroll
    for (int j = 0; j < 8; ++j) { o[j][0] *= c0; o[j][1] *= c0; o[j][2] *= c1; o[j][3] *= c1; }
    tc_mm_ab_reg(o, pf, Vs, lane);
  }
  const float i0 = 1.0f / sum0, i1 = 1.0f / sum1;
#pragma unroll
  for (int j = 0; j < 8; ++j) { o[j][0] *= i0; o[j][1] *= i0; o[j][2] *= i1; o[j][3] *= i1; }
  if (lse && (lane & 3) == 0) {
    float* lrow = lse + (static_cast<int64_t>(b) * H + h) * L;
    if (q0 + rq < L) lrow[q0 + rq] = m0 + __logf(sum0);
    if (q0 + rq + 8 < L) lrow[q0 + rq + 8] = m1 + __logf(sum1);
  }
  __syncthreads();                       // everyone is done reading Qs: reuse it to stage the output
  tc_acc_to_smem(o, Qs, r0, lane, 1.0f);
  __syncthreads();
  tc_store_tile(Qs, ctx + (row0 + q0) * ld_ctx + h * 64, ld_ctx, L - q0);
}

// ------------------------------------------------------------------------------------------------ backward
template <int RT>
__global__ void __launch_bounds__(RT * 32) attn_tc_bwd_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                                                 const __nv_bfloat16* __restrict__ v, int64_t ld_qkv,
                                                                 const int64_t* __restrict__ text_mask, const __nv_bfloat16* __restrict__ ctx,
                                                                 const __nv_bfloat16* __restrict__ dctx, int64_t ld_ctx,
                                                                 const float* __restrict__ lse, __nv_bfloat16* __restrict__ dq,
                                                                 __nv_bfloat16* __restrict__ dk, __nv_bfloat16* __restrict__ dv, int64_t ld_dqkv,
                                                                 int L, int Lt, int H, float scale, TcDrop dc_in) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  const TcDrop dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  extern __shared__ __align__(16) uint8_t tc_smem[];
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(tc_smem);
  constexpr int R = RT * 16, TILE = R * TC_LD;
  __nv_bfloat16* Ks = Qs + TILE;
  __nv_bfloat16* Vs = Ks + TILE;
  __nv_bfloat16* dOs = Vs + TILE;
  __nv_bfloat16* Ps = Vs;                // dropped probabilities [query][key]: take over the V tile once dP has been formed
  __nv_bfloat16* dSs = Ks;               // dS [query][key]: takes over the K tile once S and dQ have been formed
  __nv_bfloat16* dQs = dOs + TILE;       // dQ staged for the coalesced store (its own tile: written while K / V are still being read)
  float* madd = reinterpret_cast<float*>(dQs + TILE);
  float* Dv = madd + R;                  // D_i = sum_d dO[i][d] O[i][d]
  float* lses = Dv + R;
  const int h = blockIdx.x, b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row0 = static_cast<int64_t>(b) * L;
  tc_load_tile<R>(Qs, q + row0 * ld_qkv + h * 64, ld_qkv, L);
  tc_load_tile<R>(Ks, k + row0 * ld_qkv + h * 64, ld_qkv, L);
  tc_load_tile<R>(Vs, v + row0 * ld_qkv + h * 64, ld_qkv, L);
  tc_load_tile<R>(dOs, dctx + row0 * ld_ctx + h * 64, ld_ctx, L);
  if (threadIdx.x < R) {
    const int j = threadIdx.x;
    float m = -INFINITY;
    if (j < L) m = (j < Lt && text_mask[static_cast<int64_t>(b) * Lt + j] == 0) ? -10000.f : 0.f;
    madd[j] = m;
    lses[j] = j < L ? lse[(static_cast<int64_t>(b) * H + h) * L + j] : 0.f;
  }
  // D_i: 8 threads per row, 4 RT rows per pass, 4 passes
#pragma unroll
  for (int pass = 0; pass < 4; ++pass) {
    const int r = pass * (4 * RT) + (threadIdx.x >> 3), c = (threadIdx.x & 7) * 8;
    float acc = 0.f;
    if (r < L) {
      const uint4 uo = *reinterpret_cast<const uint4*>(ctx + (row0 + r) * ld_ctx + h * 64 + c);
      const uint4 ud = *reinterpret_cast<const uint4*>(dctx + (row0 + r) * ld_ctx + h * 64 + c);
      const uint32_t ov[4] = {uo.x, uo.y, uo.z, uo.w}, dvv[4] = {ud.x, ud.y, ud.z, ud.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 a = unpack_bf16x2(ov[e]), d = unpack_bf16x2(dvv[e]);
        acc += a.x * d.x + a.y * d.y;
      }
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    acc += __shfl_xor_sync(0xffffffffu, acc, 4);
    if ((threadIdx.x & 7) == 0) Dv[r] = acc;
  }
  __syncthreads();
  // ---- phase 1: this warp's 16 query rows: S, P, dP, dS, dQ ----
  const int r0 = warp * 16;
  const int rq = r0 + (lane >> 2), cq = 2 * (lane & 3);
  float s[2 * RT][4], dp[2 * RT][4];
  tc_mm_abt<RT>(s, Qs, Ks, r0, lane);
  tc_mm_abt<RT>(dp, dOs, Vs, r0, lane);
  const float l0 = lses[rq], l1 = lses[rq + 8], D0 = Dv[rq], D1 = Dv[rq + 8];
  const bool ok0 = rq < L, ok1 = rq + 8 < L;
  uint32_t dsf[RT][4], pdf[RT][4];      // dS and the dropped probabilities of this warp's rows, in the accumulator layout
#pragma unroll
  for (int j = 0; j < 2 * RT; ++j) {
    const float m0 = madd[j * 8 + cq], m1 = madd[j * 8 + cq + 1];
    float p0 = ok0 ? __expf(s[j][0] * scale + m0 - l0) : 0.f, p1 = ok0 ? __expf(s[j][1] * scale + m1 - l0) : 0.f;
    float p2 = ok1 ? __expf(s[j][2] * scale + m0 - l1) : 0.f, p3 = ok1 ? __expf(s[j][3] * scale + m1 - l1) : 0.f;
    float r_0 = 1.f, r_1 = 1.f, r_2 = 1.f, r_3 = 1.f;
    if (dc.thresh) {
      const uint64_t base0 = ((static_cast<uint64_t>(b) * H + h) * L + rq) * L + j * 8 + cq;
      const uint64_t base1 = base0 + static_cast<uint64_t>(8) * L;
      dropout_mult2(dc.seed, base0, dc.thresh, dc.inv_keep, r_0, r_1);
      dropout_mult2(dc.seed, base1, dc.thresh, dc.inv_keep, r_2, r_3);
    }
    const float ds0 = p0 * (dp[j][0] * r_0 - D0), ds1 = p1 * (dp[j][1] * r_1 - D0);
    const float ds2 = p2 * (dp[j][2] * r_2 - D1), ds3 = p3 * (dp[j][3] * r_3 - D1);
    pdf[j >> 1][(j & 1) * 2] = pack_bf16x2(p0 * r_0, p1 * r_1);
    pdf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2 * r_2, p3 * r_3);
    dsf[j >> 1][(j & 1) * 2] = pack_bf16x2(ds0, ds1);
    dsf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(ds2, ds3);
  }
  float acc[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;
  tc_mm_ab_reg(acc, dsf, Ks, lane);                  // dQ = dS K
  tc_acc_to_smem(acc, dQs, r0, lane, scale);
  __syncthreads();                                   // every warp is done reading Ks (S, dQ) and Vs (dP): both tiles are free
#pragma unroll
  for (int j = 0; j < 2 * RT; ++j) {                 // P -> the V tile, dS -> the K tile ([query][key], read transposed below)
    *reinterpret_cast<uint32_t*>(Ps + rq * TC_LD + j * 8 + cq) = pdf[j >> 1][(j & 1) * 2];
    *reinterpret_cast<uint32_t*>(Ps + (rq + 8) * TC_LD + j * 8 + cq) = pdf[j >> 1][(j & 1) * 2 + 1];
    *reinterpret_cast<uint32_t*>(dSs + rq * TC_LD + j * 8 + cq) = dsf[j >> 1][(j & 1) * 2];
    *reinterpret_cast<uint32_t*>(dSs + (rq + 8) * TC_LD + j * 8 + cq) = dsf[j >> 1][(j & 1) * 2 + 1];
  }
  __syncthreads();
  // ---- phase 2: this warp's 16 key rows: dV = Pd^T dO, dK = dS^T Q ----
  float dvacc[8][4], dkacc[8][4];
  tc_mm_atb<RT>(dvacc, Ps, dOs, r0, lane);
  tc_mm_atb<RT>(dkacc, dSs, Qs, r0, lane);
  __syncthreads();                                   // P, dS fully consumed: stage dV / dK in their tiles
  tc_acc_to_smem(dvacc, Ps, r0, lane, 1.0f);
  tc_acc_to_smem(dkacc, dSs, r0, lane, scale);
  __syncthreads();
  tc_store_tile<R>(dQs, dq + row0 * ld_dqkv + h * 64, ld_dqkv, L);
  tc_store_tile<R>(Ps, dv + row0 * ld_dqkv + h * 64, ld_dqkv, L);
  tc_store_tile<R>(dSs, dk + row0 * ld_dqkv + h * 64, ld_dqkv, L);
}

// ------------------------------------------------------------------------------------------------ backward, any L
// The tensor-core backward for sequences longer than one tile (448 px: L = 69 .. 149; 768 px: L = 130 .. 169; paragraph
// retrieval: L = 521). Two kernels, 4 warps each, grid (ceil(L / 64), heads, nseq), the split of attn_bwd_kv_kernel /
// attn_bwd_q_kernel (attention.cu): attn_tc_bwd_kv_kernel owns a 64-key tile and loops over query tiles (dK, dV), attn_tc_bwd_q_kernel
// owns a 64-query tile and loops over key tiles (dQ). Every output row is written by exactly one CTA, in a fixed order: no atomics,
// no workspace, bit-identical from run to run. Per (query tile, key tile) pair the math is phase 1 of attn_tc_bwd_kernel.
//
// Tail tiles: a 16-row slab that lies entirely beyond L costs no MMA. The helpers below are tc_mm_abt / tc_mm_ab_reg / tc_mm_atb
// with the output column pairs (abt) or the contraction slabs (ab_reg, atb) cut at a run-time count of live slabs; at L = 69 the
// second tile holds 5 live rows, and its products run over one slab instead of four.
__device__ __forceinline__ int tc_live_slabs(int nrows) { return min(4, (nrows + 15) >> 4); }

// acc = A(16 x 64 rows r0.. of As) * B^T, output columns [0, 16 njp) only (the others stay zero)
__device__ __forceinline__ void tc_mm_abt_live(float (&acc)[8][4], const __nv_bfloat16* As, const __nv_bfloat16* Bs, int r0, int lane, int njp) {
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    uint32_t a[4];
    ldsm_x4(a, As + (r0 + (lane & 15)) * TC_LD + ks * 16 + (lane >> 4) * 8);
#pragma unroll
    for (int jp = 0; jp < 4; ++jp) {
      if (jp < njp) {
        uint32_t b[4];
        ldsm_x4(b, Bs + (jp * 16 + (lane & 7) + (lane >> 4) * 8) * TC_LD + ks * 16 + ((lane >> 3) & 1) * 8);
        mma16816(acc[2 * jp], a, b[0], b[1]);
        mma16816(acc[2 * jp + 1], a, b[2], b[3]);
      }
    }
  }
}
// acc += A(16 x 64, register fragments afrag[ks]) * B ([k][n] row-major), contracted over the slabs ks < nks of Bs
__device__ __forceinline__ void tc_mm_ab_reg_live(float (&acc)[8][4], const uint32_t (&afrag)[4][4], const __nv_bfloat16* Bs, int lane, int nks) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    if (ks < nks) {
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {
        uint32_t b[4];
        ldsm_x4_t(b, Bs + (ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * TC_LD + jp * 16 + (lane >> 4) * 8);
        mma16816(acc[2 * jp], afrag[ks], b[0], b[1]);
        mma16816(acc[2 * jp + 1], afrag[ks], b[2], b[3]);
      }
    }
  }
}
// acc += A^T-stored (As holds [k][m]) * B ([k][n] row-major), contracted over the slabs ks < nks; accumulates (no zeroing), so
// dV / dK build up across query tiles
__device__ __forceinline__ void tc_mm_atb_live(float (&acc)[8][4], const __nv_bfloat16* As, const __nv_bfloat16* Bs, int m0, int lane, int nks) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    if (ks < nks) {
      uint32_t a[4];
      const int mi = lane >> 3;
      ldsm_x4_t(a, As + (ks * 16 + (lane & 7) + (mi >> 1) * 8) * TC_LD + m0 + (mi & 1) * 8);
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {
        uint32_t b[4];
        ldsm_x4_t(b, Bs + (ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * TC_LD + jp * 16 + (lane >> 4) * 8);
        mma16816(acc[2 * jp], a, b[0], b[1]);
        mma16816(acc[2 * jp + 1], a, b[2], b[3]);
      }
    }
  }
}

// additive key mask of the 64 keys k0.. (-10000 for masked text keys, -inf beyond L), and, for the 64 queries q0.., the saved
// log-sum-exp and D_i = sum_d dO[i][d] O[i][d] (8 threads per row, 16 rows per pass, 4 passes); rows beyond L get 0
__device__ __forceinline__ void tc_key_mask(float* madd, const int64_t* text_mask, int b, int k0, int L, int Lt) {
  if (threadIdx.x < 64) {
    const int j = k0 + threadIdx.x;
    float m = -INFINITY;
    if (j < L) m = (j < Lt && text_mask[static_cast<int64_t>(b) * Lt + j] == 0) ? -10000.f : 0.f;
    madd[threadIdx.x] = m;
  }
}
__device__ __forceinline__ void tc_row_stats(float* Dv, float* lses, const __nv_bfloat16* ctx_h, const __nv_bfloat16* dctx_h, int64_t ld_ctx,
                                             const float* lse_bh, int q0, int L) {
  if (threadIdx.x < 64) lses[threadIdx.x] = q0 + threadIdx.x < L ? lse_bh[q0 + threadIdx.x] : 0.f;
#pragma unroll
  for (int pass = 0; pass < 4; ++pass) {
    const int r = pass * 16 + (threadIdx.x >> 3), c = (threadIdx.x & 7) * 8;
    float acc = 0.f;
    if (q0 + r < L) {
      const uint4 uo = *reinterpret_cast<const uint4*>(ctx_h + static_cast<int64_t>(q0 + r) * ld_ctx + c);
      const uint4 ud = *reinterpret_cast<const uint4*>(dctx_h + static_cast<int64_t>(q0 + r) * ld_ctx + c);
      const uint32_t ov[4] = {uo.x, uo.y, uo.z, uo.w}, dvv[4] = {ud.x, ud.y, ud.z, ud.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 a = unpack_bf16x2(ov[e]), d = unpack_bf16x2(dvv[e]);
        acc += a.x * d.x + a.y * d.y;
      }
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    acc += __shfl_xor_sync(0xffffffffu, acc, 4);
    if ((threadIdx.x & 7) == 0) Dv[r] = acc;
  }
}

// P (dropped probabilities) and dS of a warp's 16 query rows against one 64-key tile, from the S and dP accumulators, in place:
// s[j] becomes P * dropout multiplier, dp[j] becomes dS. qrow = index of row rq within the sequence; rows >= L give P = dS = 0.
__device__ __forceinline__ void tc_p_ds(float (&s)[8][4], float (&dp)[8][4], const float* madd, float l0, float l1, float D0, float D1,
                                        bool ok0, bool ok1, int b, int h, int H, int L, int qrow, int k0, int cq, float scale, const TcDrop& dc) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float m0 = madd[j * 8 + cq], m1 = madd[j * 8 + cq + 1];
    float p0 = ok0 ? __expf(s[j][0] * scale + m0 - l0) : 0.f, p1 = ok0 ? __expf(s[j][1] * scale + m1 - l0) : 0.f;
    float p2 = ok1 ? __expf(s[j][2] * scale + m0 - l1) : 0.f, p3 = ok1 ? __expf(s[j][3] * scale + m1 - l1) : 0.f;
    float r_0 = 1.f, r_1 = 1.f, r_2 = 1.f, r_3 = 1.f;
    if (dc.thresh) {
      const uint64_t base0 = ((static_cast<uint64_t>(b) * H + h) * L + qrow) * L + k0 + j * 8 + cq;
      const uint64_t base1 = base0 + static_cast<uint64_t>(8) * L;
      dropout_mult2(dc.seed, base0, dc.thresh, dc.inv_keep, r_0, r_1);
      dropout_mult2(dc.seed, base1, dc.thresh, dc.inv_keep, r_2, r_3);
    }
    dp[j][0] = p0 * (dp[j][0] * r_0 - D0); dp[j][1] = p1 * (dp[j][1] * r_1 - D0);
    dp[j][2] = p2 * (dp[j][2] * r_2 - D1); dp[j][3] = p3 * (dp[j][3] * r_3 - D1);
    s[j][0] = p0 * r_0; s[j][1] = p1 * r_1; s[j][2] = p2 * r_2; s[j][3] = p3 * r_3;
  }
}

// dK, dV of one 64-key tile. K, V and the key mask stay in smem; per query tile: phase 1 (each warp: 16 query rows x 64 keys)
// forms P and dS and writes them to smem, phase 2 (each warp: 16 key rows) accumulates dV += Pd^T dO and dK += dS^T Q in registers.
__global__ void __launch_bounds__(TC_THREADS) attn_tc_bwd_kv_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                                                    const __nv_bfloat16* __restrict__ v, int64_t ld_qkv,
                                                                    const int64_t* __restrict__ text_mask, const __nv_bfloat16* __restrict__ ctx,
                                                                    const __nv_bfloat16* __restrict__ dctx, int64_t ld_ctx,
                                                                    const float* __restrict__ lse, __nv_bfloat16* __restrict__ dk,
                                                                    __nv_bfloat16* __restrict__ dv, int64_t ld_dqkv, int L, int Lt, int H,
                                                                    float scale, TcDrop dc_in) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  const TcDrop dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  extern __shared__ __align__(16) uint8_t tc_smem[];
  __nv_bfloat16* Ks = reinterpret_cast<__nv_bfloat16*>(tc_smem);
  __nv_bfloat16* Vs = Ks + TC_TILE;
  __nv_bfloat16* Qs = Vs + TC_TILE;
  __nv_bfloat16* dOs = Qs + TC_TILE;
  __nv_bfloat16* Ps = dOs + TC_TILE;     // dropped probabilities [query][key]
  __nv_bfloat16* dSs = Ps + TC_TILE;     // dS [query][key]
  float* madd = reinterpret_cast<float*>(dSs + TC_TILE);
  float* Dv = madd + 64;
  float* lses = Dv + 64;
  const int kb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = kb * 64;
  const int64_t row0 = static_cast<int64_t>(b) * L;
  const int nks = tc_live_slabs(L - k0);          // live 16-key slabs of this tile
  tc_load_tile(Ks, k + (row0 + k0) * ld_qkv + h * 64, ld_qkv, L - k0);
  tc_load_tile(Vs, v + (row0 + k0) * ld_qkv + h * 64, ld_qkv, L - k0);
  tc_key_mask(madd, text_mask, b, k0, L, Lt);
  const int r0 = warp * 16;
  const int rq = r0 + (lane >> 2), cq = 2 * (lane & 3);
  float dvacc[8][4], dkacc[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) dvacc[j][e] = dkacc[j][e] = 0.f;
  const int nqb = (L + 63) / 64;
  for (int qb = 0; qb < nqb; ++qb) {
    const int q0 = qb * 64;
    const int nqs = tc_live_slabs(L - q0);        // live 16-query slabs of this tile
    __syncthreads();                               // phase 2 of the previous query tile is done with Qs, dOs, Ps, dSs
    tc_load_tile(Qs, q + (row0 + q0) * ld_qkv + h * 64, ld_qkv, L - q0);
    tc_load_tile(dOs, dctx + (row0 + q0) * ld_ctx + h * 64, ld_ctx, L - q0);
    tc_row_stats(Dv, lses, ctx + row0 * ld_ctx + h * 64, dctx + row0 * ld_ctx + h * 64, ld_ctx, lse + (static_cast<int64_t>(b) * H + h) * L, q0, L);
    __syncthreads();
    // ---- phase 1: this warp's 16 query rows against the 64 keys: P, dS -> smem ----
    if (warp < nqs) {
      float s[8][4], dp[8][4];
      tc_mm_abt_live(s, Qs, Ks, r0, lane, nks);
      tc_mm_abt_live(dp, dOs, Vs, r0, lane, nks);
      tc_p_ds(s, dp, madd, lses[rq], lses[rq + 8], Dv[rq], Dv[rq + 8], q0 + rq < L, q0 + rq + 8 < L, b, h, H, L, q0 + rq, k0, cq, scale, dc);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        *reinterpret_cast<uint32_t*>(Ps + rq * TC_LD + j * 8 + cq) = pack_bf16x2(s[j][0], s[j][1]);
        *reinterpret_cast<uint32_t*>(Ps + (rq + 8) * TC_LD + j * 8 + cq) = pack_bf16x2(s[j][2], s[j][3]);
        *reinterpret_cast<uint32_t*>(dSs + rq * TC_LD + j * 8 + cq) = pack_bf16x2(dp[j][0], dp[j][1]);
        *reinterpret_cast<uint32_t*>(dSs + (rq + 8) * TC_LD + j * 8 + cq) = pack_bf16x2(dp[j][2], dp[j][3]);
      }
    } else {                                       // all 16 query rows beyond L: no products, P = dS = 0
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        *reinterpret_cast<uint32_t*>(Ps + rq * TC_LD + j * 8 + cq) = 0u;
        *reinterpret_cast<uint32_t*>(Ps + (rq + 8) * TC_LD + j * 8 + cq) = 0u;
        *reinterpret_cast<uint32_t*>(dSs + rq * TC_LD + j * 8 + cq) = 0u;
        *reinterpret_cast<uint32_t*>(dSs + (rq + 8) * TC_LD + j * 8 + cq) = 0u;
      }
    }
    __syncthreads();
    // ---- phase 2: this warp's 16 key rows: dV += Pd^T dO, dK += dS^T Q over the live query slabs ----
    if (warp < nks) {
      tc_mm_atb_live(dvacc, Ps, dOs, r0, lane, nqs);
      tc_mm_atb_live(dkacc, dSs, Qs, r0, lane, nqs);
    }
  }
  __syncthreads();                                 // P, dS fully consumed: stage dV / dK in their tiles
  tc_acc_to_smem(dvacc, Ps, r0, lane, 1.0f);
  tc_acc_to_smem(dkacc, dSs, r0, lane, scale);
  __syncthreads();
  tc_store_tile(Ps, dv + (row0 + k0) * ld_dqkv + h * 64, ld_dqkv, L - k0);
  tc_store_tile(dSs, dk + (row0 + k0) * ld_dqkv + h * 64, ld_dqkv, L - k0);
}

// dQ of one 64-query tile. Q, dO, lse and D stay in smem; per key tile each warp forms S and dP for its 16 query rows, turns them
// into dS in registers, and accumulates dQ += dS K with dS as the register-fragment A operand (dS never goes through smem).
__global__ void __launch_bounds__(TC_THREADS) attn_tc_bwd_q_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                                                   const __nv_bfloat16* __restrict__ v, int64_t ld_qkv,
                                                                   const int64_t* __restrict__ text_mask, const __nv_bfloat16* __restrict__ ctx,
                                                                   const __nv_bfloat16* __restrict__ dctx, int64_t ld_ctx,
                                                                   const float* __restrict__ lse, __nv_bfloat16* __restrict__ dq,
                                                                   int64_t ld_dqkv, int L, int Lt, int H, float scale, TcDrop dc_in) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  const TcDrop dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  extern __shared__ __align__(16) uint8_t tc_smem[];
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(tc_smem);
  __nv_bfloat16* dOs = Qs + TC_TILE;
  __nv_bfloat16* Ks = dOs + TC_TILE;
  __nv_bfloat16* Vs = Ks + TC_TILE;
  float* madd = reinterpret_cast<float*>(Vs + TC_TILE);
  float* Dv = madd + 64;
  float* lses = Dv + 64;
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = qb * 64;
  const int64_t row0 = static_cast<int64_t>(b) * L;
  const bool live = warp < tc_live_slabs(L - q0);  // this warp holds at least one query row < L
  tc_load_tile(Qs, q + (row0 + q0) * ld_qkv + h * 64, ld_qkv, L - q0);
  tc_load_tile(dOs, dctx + (row0 + q0) * ld_ctx + h * 64, ld_ctx, L - q0);
  tc_row_stats(Dv, lses, ctx + row0 * ld_ctx + h * 64, dctx + row0 * ld_ctx + h * 64, ld_ctx, lse + (static_cast<int64_t>(b) * H + h) * L, q0, L);
  const int r0 = warp * 16;
  const int rq = r0 + (lane >> 2), cq = 2 * (lane & 3);
  float acc[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;
  const int nkb = (L + 63) / 64;
  for (int kb = 0; kb < nkb; ++kb) {
    const int k0 = kb * 64;
    const int nks = tc_live_slabs(L - k0);        // live 16-key slabs of this tile
    __syncthreads();                               // every warp is done with the previous key tile
    tc_load_tile(Ks, k + (row0 + k0) * ld_qkv + h * 64, ld_qkv, L - k0);
    tc_load_tile(Vs, v + (row0 + k0) * ld_qkv + h * 64, ld_qkv, L - k0);
    tc_key_mask(madd, text_mask, b, k0, L, Lt);
    __syncthreads();
    if (live) {
      float s[8][4], dp[8][4];
      tc_mm_abt_live(s, Qs, Ks, r0, lane, nks);
      tc_mm_abt_live(dp, dOs, Vs, r0, lane, nks);
      tc_p_ds(s, dp, madd, lses[rq], lses[rq + 8], Dv[rq], Dv[rq + 8], q0 + rq < L, q0 + rq + 8 < L, b, h, H, L, q0 + rq, k0, cq, scale, dc);
      uint32_t dsf[4][4];                          // dS in the accumulator layout = the A fragments of dS K
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        dsf[j >> 1][(j & 1) * 2] = pack_bf16x2(dp[j][0], dp[j][1]);
        dsf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(dp[j][2], dp[j][3]);
      }
      tc_mm_ab_reg_live(acc, dsf, Ks, lane, nks);  // dQ += dS K
    }
  }
  __syncthreads();                                 // everyone is done reading Qs: reuse it to stage dQ
  tc_acc_to_smem(acc, Qs, r0, lane, scale);
  __syncthreads();
  tc_store_tile(Qs, dq + (row0 + q0) * ld_dqkv + h * 64, ld_dqkv, L - q0);
}

// ------------------------------------------------------------------------------------------------ probabilities
// attention_probs of BertSelfAttention (transformers.py:257-285), written to memory for output_attentions: P[i, j] =
// exp(S[i, j] - lse[i]) x dropout multiplier, from the log-sum-exp the forward saved (the P the backward kernels rebuild in
// tc_p_ds). One CTA = 64 query rows of one (sequence, head); per 64-key tile each warp forms S for its 16 rows on mma.sync.
// The kernel is bound by the bytes it writes (4 l^2 per (sequence, head)): each key tile is staged in shared memory as fp32
// and written out as 16-byte vectors. The output rows of a CTA are one contiguous run of memory, but a row segment starts at
// any 4-byte alignment (l is odd at 224 px), so each staged row is shifted by (its global element index) & 3: the aligned
// 16-byte groups of the segment are then aligned in shared memory too, and only the up to three elements at either end of a
// segment go out as scalar stores. Streaming stores (st.global.cs): P is written once and read by the host, not by a kernel.
constexpr int PR_LD = 72;                 // fp32 elements per staged row: 64 keys + up to 3 of shift, 16-byte aligned rows

// Writes the staged rows r < nq of one key tile (Ps row r: keys k0 .. k0 + nk - 1, shifted by the element index & 3 of its first
// key) to out viewed as [rows, L], row prow0 + r. 16 threads per row, 8 rows per pass; rows >= nq and keys >= nk are never
// written. ACC: each element becomes (its value in memory) + (the staged value), one fp32 add, the read through the same
// aligned vectors.
template <bool ACC>
__device__ __forceinline__ void tc_store_staged_rows(const float* Ps, float* __restrict__ out, uint64_t prow0, int L, int k0, int nq, int nk) {
  for (int r = threadIdx.x >> 4; r < nq; r += TC_THREADS / 16) {
    const uint64_t e = (prow0 + r) * L + k0;
    const int sh = static_cast<int>(e & 3), end = sh + nk;
    float* dst = out + (e - sh);       // 16-byte aligned
    const float* src = Ps + r * PR_LD;
    for (int c = (threadIdx.x & 15) * 4; c < end; c += 64) {
      const float4 v = *reinterpret_cast<const float4*>(src + c);
      if (c >= sh && c + 4 <= end) {
        if (ACC) {
          const float4 o = __ldcs(reinterpret_cast<const float4*>(dst + c));
          __stcs(reinterpret_cast<float4*>(dst + c), make_float4(o.x + v.x, o.y + v.y, o.z + v.z, o.w + v.w));
        } else {
          __stcs(reinterpret_cast<float4*>(dst + c), v);
        }
      } else {
        const float w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (c + i >= sh && c + i < end) __stcs(dst + c + i, ACC ? __ldcs(dst + c + i) + w[i] : w[i]);
      }
    }
  }
}

__global__ void __launch_bounds__(TC_THREADS) attn_tc_probs_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                                                   int64_t ld_qkv, const int64_t* __restrict__ text_mask,
                                                                   const float* __restrict__ lse, float* __restrict__ probs, int L, int Lt,
                                                                   int H, float scale, TcDrop dc_in) {
  pdl_wait();
  const TcDrop dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  extern __shared__ __align__(16) uint8_t tc_smem[];
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(tc_smem);
  __nv_bfloat16* Ks = Qs + TC_TILE;
  float* Ps = reinterpret_cast<float*>(Ks + TC_TILE);       // [64][PR_LD] staged probabilities of one key tile
  float* madd = Ps + 64 * PR_LD;
  float* lses = madd + 64;
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = qb * 64;
  const int nq = min(64, L - q0);
  const int64_t row0 = static_cast<int64_t>(b) * L;
  const uint64_t prow0 = (static_cast<uint64_t>(b) * H + h) * L + q0;   // row index of query q0 in probs viewed as [nseq*H*L, L]
  const bool live = warp < tc_live_slabs(nq);                          // this warp holds at least one query row < L
  tc_load_tile(Qs, q + (row0 + q0) * ld_qkv + h * 64, ld_qkv, nq);
  if (threadIdx.x < 64) lses[threadIdx.x] = threadIdx.x < nq ? lse[prow0 + threadIdx.x] : 0.f;
  const int r0 = warp * 16;
  const int rq = r0 + (lane >> 2), cq = 2 * (lane & 3);
  const int nkb = (L + 63) / 64;
  for (int kb = 0; kb < nkb; ++kb) {
    const int k0 = kb * 64, nk = min(64, L - k0);
    __syncthreads();                     // the previous tile has been written out: Ks, Ps and the mask are free
    tc_load_tile(Ks, k + (row0 + k0) * ld_qkv + h * 64, ld_qkv, nk);
    tc_key_mask(madd, text_mask, b, k0, L, Lt);
    __syncthreads();
    if (live) {
      float s[8][4];
      tc_mm_abt_live(s, Qs, Ks, r0, lane, tc_live_slabs(nk));
      const float l0 = lses[rq], l1 = lses[rq + 8];
      const uint64_t e0 = (prow0 + rq) * L + k0, e1 = e0 + static_cast<uint64_t>(8) * L;   // element index of (row, k0)
      float* d0 = Ps + rq * PR_LD + static_cast<int>(e0 & 3) + cq;
      float* d1 = Ps + (rq + 8) * PR_LD + static_cast<int>(e1 & 3) + cq;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float m0 = madd[j * 8 + cq], m1 = madd[j * 8 + cq + 1];
        float p0 = __expf(s[j][0] * scale + m0 - l0), p1 = __expf(s[j][1] * scale + m1 - l0);
        float p2 = __expf(s[j][2] * scale + m0 - l1), p3 = __expf(s[j][3] * scale + m1 - l1);
        if (dc.thresh) {
          float r_0, r_1, r_2, r_3;
          dropout_mult2(dc.seed, e0 + j * 8 + cq, dc.thresh, dc.inv_keep, r_0, r_1);
          dropout_mult2(dc.seed, e1 + j * 8 + cq, dc.thresh, dc.inv_keep, r_2, r_3);
          p0 *= r_0; p1 *= r_1; p2 *= r_2; p3 *= r_3;
        }
        d0[j * 8] = p0; d0[j * 8 + 1] = p1;
        d1[j * 8] = p2; d1[j * 8 + 1] = p3;
      }
    }
    __syncthreads();
    tc_store_staged_rows<false>(Ps, probs, prow0, L, k0, nq, nk);
  }
}

// The gradient the returned probabilities A receive from the context product ctx = A V (transformers.py:271-277):
// dA[s, h, i, j] = sum_d dO[s l + i, h 64 + d] V[s l + j, h 64 + d], for every i, j < l (padded keys, padded query rows and
// dropped positions included; A is post-dropout, so no dropout factor). One CTA = 64 query rows of one (sequence, head): the dO
// tile stays in shared memory, each 64-key V tile is loaded in turn, dO V^T is the Q K^T product shape of attn_tc_probs_kernel
// on mma.sync, and the tile leaves through the same staging and 16-byte streaming stores. ACC: added to the values in memory,
// one fp32 add per element; every element has one writer and a fixed order, so runs are bit-identical.
template <bool ACC>
__global__ void __launch_bounds__(TC_THREADS) attn_tc_dprobs_kernel(const __nv_bfloat16* __restrict__ v, int64_t ld_qkv,
                                                                    const __nv_bfloat16* __restrict__ dctx, int64_t ld_ctx,
                                                                    float* __restrict__ dprobs, int L, int H) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ __align__(16) uint8_t tc_smem[];
  __nv_bfloat16* dOs = reinterpret_cast<__nv_bfloat16*>(tc_smem);
  __nv_bfloat16* Vs = dOs + TC_TILE;
  float* Ps = reinterpret_cast<float*>(Vs + TC_TILE);       // [64][PR_LD] staged dA of one key tile
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = qb * 64;
  const int nq = min(64, L - q0);
  const int64_t row0 = static_cast<int64_t>(b) * L;
  const uint64_t prow0 = (static_cast<uint64_t>(b) * H + h) * L + q0;   // row index of query q0 in dprobs viewed as [nseq*H*L, L]
  const bool live = warp < tc_live_slabs(nq);
  tc_load_tile(dOs, dctx + (row0 + q0) * ld_ctx + h * 64, ld_ctx, nq);
  const int r0 = warp * 16;
  const int rq = r0 + (lane >> 2), cq = 2 * (lane & 3);
  const int nkb = (L + 63) / 64;
  for (int kb = 0; kb < nkb; ++kb) {
    const int k0 = kb * 64, nk = min(64, L - k0);
    __syncthreads();                     // the previous tile has been written out: Vs and Ps are free
    tc_load_tile(Vs, v + (row0 + k0) * ld_qkv + h * 64, ld_qkv, nk);
    __syncthreads();
    if (live) {
      float s[8][4];
      tc_mm_abt_live(s, dOs, Vs, r0, lane, tc_live_slabs(nk));
      const uint64_t e0 = (prow0 + rq) * L + k0, e1 = e0 + static_cast<uint64_t>(8) * L;
      float* d0 = Ps + rq * PR_LD + static_cast<int>(e0 & 3) + cq;
      float* d1 = Ps + (rq + 8) * PR_LD + static_cast<int>(e1 & 3) + cq;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        d0[j * 8] = s[j][0]; d0[j * 8 + 1] = s[j][1];
        d1[j * 8] = s[j][2]; d1[j * 8 + 1] = s[j][3];
      }
    }
    __syncthreads();
    tc_store_staged_rows<ACC>(Ps, dprobs, prow0, L, k0, nq, nk);
  }
}

// ------------------------------------------------------------------------------------------------ backward through the probabilities
// The gradient of a loss on the returned probabilities A = P r (output_attentions; G = dloss / dA, fp32 [nseq, heads, l, l]):
//   g = r G ;  D_i = sum_j P_ij g_ij ;  dS = P (g - D) ;  dQ += dS K / 8 ;  dK += dS^T Q / 8
// added to the dQ / dK cb_attention_bwd wrote. Two kernels on the grid (ceil(l / 64), heads, nseq), the split of the long
// backward: attn_tc_probs_bwd_q_kernel owns a 64-query tile (pass 1 over the key tiles: D, written to drow; pass 2: dS in
// registers, dQ += dS K), attn_tc_probs_bwd_k_kernel owns a 64-key tile and loops over the query tiles with D from drow
// (dS through shared memory, dK += dS^T Q). P is rebuilt from Q, K and the saved lse as attn_tc_probs_kernel forms it, never
// read from the returned tensor. Every output element has one writer and a fixed order: no atomics, bit-identical runs.
// G is read in the accumulator layout straight from global memory: a quad reads 8 consecutive floats of a row, and a row
// starts at any 4-byte alignment (l is odd at 224 px), so the reads are scalar; elements at or beyond l are never read.

// one 64-key tile of a warp's 16 query rows, from the S accumulator: ROWSUM: t0 / t1 += sum_j P r G over this thread's
// elements of rows rq / rq + 8 (s is left as is); else s[j] becomes dS = P (r G - D). e0 = element index of (row rq, key k0)
// in G viewed as [nseq*heads*l, l] (also the dropout index); rows with !ok and keys >= l give P = G = 0.
template <bool ROWSUM>
__device__ __forceinline__ void tc_probs_ds(float (&s)[8][4], const float* madd, float l0, float l1, float D0, float D1, bool ok0, bool ok1,
                                            const float* __restrict__ dprobs, uint64_t e0, int L, int k0, int cq, float scale, const TcDrop& dc,
                                            float& t0, float& t1) {
  const uint64_t e1 = e0 + static_cast<uint64_t>(8) * L;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = k0 + j * 8 + cq;
    const float m0 = madd[j * 8 + cq], m1 = madd[j * 8 + cq + 1];
    const float p0 = ok0 ? __expf(s[j][0] * scale + m0 - l0) : 0.f, p1 = ok0 ? __expf(s[j][1] * scale + m1 - l0) : 0.f;
    const float p2 = ok1 ? __expf(s[j][2] * scale + m0 - l1) : 0.f, p3 = ok1 ? __expf(s[j][3] * scale + m1 - l1) : 0.f;
    float g0 = 0.f, g1 = 0.f, g2 = 0.f, g3 = 0.f;
    if (ok0 && c < L) g0 = __ldg(dprobs + e0 + j * 8 + cq);
    if (ok0 && c + 1 < L) g1 = __ldg(dprobs + e0 + j * 8 + cq + 1);
    if (ok1 && c < L) g2 = __ldg(dprobs + e1 + j * 8 + cq);
    if (ok1 && c + 1 < L) g3 = __ldg(dprobs + e1 + j * 8 + cq + 1);
    if (dc.thresh) {
      float r_0, r_1, r_2, r_3;
      dropout_mult2(dc.seed, e0 + j * 8 + cq, dc.thresh, dc.inv_keep, r_0, r_1);
      dropout_mult2(dc.seed, e1 + j * 8 + cq, dc.thresh, dc.inv_keep, r_2, r_3);
      g0 *= r_0; g1 *= r_1; g2 *= r_2; g3 *= r_3;
    }
    if (ROWSUM) {
      t0 += p0 * g0 + p1 * g1;
      t1 += p2 * g2 + p3 * g3;
    } else {
      s[j][0] = p0 * (g0 - D0); s[j][1] = p1 * (g1 - D0);
      s[j][2] = p2 * (g2 - D1); s[j][3] = p3 * (g3 - D1);
    }
  }
}

// dst (bf16, 16 rows r0 + lane / 4, + 8 of a 64-column block, row pitch ld) += acc * mul, in fp32, rounded once; rows >= nrows
// are not touched
__device__ __forceinline__ void tc_acc_add_global(const float (&acc)[8][4], __nv_bfloat16* dst, int64_t ld, int r0, int lane, int nrows,
                                                  float mul) {
  const int r = r0 + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    if (r + 8 * half < nrows) {
      uint32_t* row = reinterpret_cast<uint32_t*>(dst + static_cast<int64_t>(r + 8 * half) * ld + c);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 o = unpack_bf16x2(row[j * 4]);
        row[j * 4] = pack_bf16x2(o.x + acc[j][2 * half] * mul, o.y + acc[j][2 * half + 1] * mul);
      }
    }
  }
}

// dst (bf16, 16 rows r0 + lane / 4, + 8 of a 64-column block, row pitch ld) = acc * mul, rounded once; rows >= nrows are not
// touched and nothing is read
__device__ __forceinline__ void tc_acc_store_global(const float (&acc)[8][4], __nv_bfloat16* dst, int64_t ld, int r0, int lane, int nrows,
                                                    float mul) {
  const int r = r0 + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    if (r + 8 * half < nrows) {
      uint32_t* row = reinterpret_cast<uint32_t*>(dst + static_cast<int64_t>(r + 8 * half) * ld + c);
#pragma unroll
      for (int j = 0; j < 8; ++j) row[j * 4] = pack_bf16x2(acc[j][2 * half] * mul, acc[j][2 * half + 1] * mul);
    }
  }
}

// dQ of one 64-query tile; writes D of its rows to drow [nseq, heads, l]. STORE: dQ is written, not added (a fresh dqkv)
template <bool STORE>
__global__ void __launch_bounds__(TC_THREADS) attn_tc_probs_bwd_q_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                                                         int64_t ld_qkv, const int64_t* __restrict__ text_mask,
                                                                         const float* __restrict__ lse, const float* __restrict__ dprobs,
                                                                         float* __restrict__ drow, __nv_bfloat16* __restrict__ dq, int64_t ld_dqkv,
                                                                         int L, int Lt, int H, float scale, TcDrop dc_in) {
  pdl_wait();
  const TcDrop dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  extern __shared__ __align__(16) uint8_t tc_smem[];
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(tc_smem);
  __nv_bfloat16* Ks = Qs + TC_TILE;
  float* madd = reinterpret_cast<float*>(Ks + TC_TILE);
  float* lses = madd + 64;
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = qb * 64;
  const int nq = min(64, L - q0);
  const int64_t row0 = static_cast<int64_t>(b) * L;
  const uint64_t prow0 = (static_cast<uint64_t>(b) * H + h) * L + q0;   // row of query q0 in G viewed as [nseq*H*L, L]
  const bool live = warp < tc_live_slabs(nq);                          // this warp holds at least one query row < L
  tc_load_tile(Qs, q + (row0 + q0) * ld_qkv + h * 64, ld_qkv, nq);
  if (threadIdx.x < 64) lses[threadIdx.x] = threadIdx.x < nq ? lse[prow0 + threadIdx.x] : 0.f;
  const int r0 = warp * 16;
  const int rq = r0 + (lane >> 2), cq = 2 * (lane & 3);
  const bool ok0 = rq < nq, ok1 = rq + 8 < nq;
  const int nkb = (L + 63) / 64;
  float D0 = 0.f, D1 = 0.f;
  float acc[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;
  // pass 0: D_i = sum_j P_ij r_ij G_ij; pass 1: dQ += dS K
  for (int pass = 0; pass < 2; ++pass) {
    for (int kb = 0; kb < nkb; ++kb) {
      const int k0 = kb * 64, nks = tc_live_slabs(L - k0);
      __syncthreads();                   // every warp is done with the previous key tile
      tc_load_tile(Ks, k + (row0 + k0) * ld_qkv + h * 64, ld_qkv, L - k0);
      tc_key_mask(madd, text_mask, b, k0, L, Lt);
      __syncthreads();
      if (live) {
        float s[8][4];
        tc_mm_abt_live(s, Qs, Ks, r0, lane, nks);
        const uint64_t e0 = (prow0 + rq) * L + k0;
        if (pass == 0) {
          tc_probs_ds<true>(s, madd, lses[rq], lses[rq + 8], 0.f, 0.f, ok0, ok1, dprobs, e0, L, k0, cq, scale, dc, D0, D1);
        } else {
          float u0, u1;
          tc_probs_ds<false>(s, madd, lses[rq], lses[rq + 8], D0, D1, ok0, ok1, dprobs, e0, L, k0, cq, scale, dc, u0, u1);
          uint32_t dsf[4][4];              // dS in the accumulator layout = the A fragments of dS K
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            dsf[j >> 1][(j & 1) * 2] = pack_bf16x2(s[j][0], s[j][1]);
            dsf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(s[j][2], s[j][3]);
          }
          tc_mm_ab_reg_live(acc, dsf, Ks, lane, nks);
        }
      }
    }
    if (pass == 0) {
      D0 = quad_sum(D0);
      D1 = quad_sum(D1);
      if ((lane & 3) == 0) {
        if (ok0) drow[prow0 + rq] = D0;
        if (ok1) drow[prow0 + rq + 8] = D1;
      }
    }
  }
  if (live) {
    if (STORE)
      tc_acc_store_global(acc, dq + (row0 + q0) * ld_dqkv + h * 64, ld_dqkv, r0, lane, nq, scale);
    else
      tc_acc_add_global(acc, dq + (row0 + q0) * ld_dqkv + h * 64, ld_dqkv, r0, lane, nq, scale);
  }
}

// dK of one 64-key tile, with D from drow. STORE: dK is written, not added
template <bool STORE>
__global__ void __launch_bounds__(TC_THREADS) attn_tc_probs_bwd_k_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                                                         int64_t ld_qkv, const int64_t* __restrict__ text_mask,
                                                                         const float* __restrict__ lse, const float* __restrict__ dprobs,
                                                                         const float* __restrict__ drow, __nv_bfloat16* __restrict__ dk,
                                                                         int64_t ld_dqkv, int L, int Lt, int H, float scale, TcDrop dc_in) {
  pdl_wait();      // drow is written by attn_tc_probs_bwd_q_kernel, the launch before this one
  const TcDrop dc = drop_resolve(dc_in);
  pdl_trigger();
  extern __shared__ __align__(16) uint8_t tc_smem[];
  __nv_bfloat16* Ks = reinterpret_cast<__nv_bfloat16*>(tc_smem);
  __nv_bfloat16* Qs = Ks + TC_TILE;
  __nv_bfloat16* dSs = Qs + TC_TILE;     // dS [query][key]
  float* madd = reinterpret_cast<float*>(dSs + TC_TILE);
  float* lses = madd + 64;
  float* Ds = lses + 64;
  const int kb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = kb * 64;
  const int nk = min(64, L - k0), nks = tc_live_slabs(nk);
  const int64_t row0 = static_cast<int64_t>(b) * L;
  const uint64_t bh0 = (static_cast<uint64_t>(b) * H + h) * L;         // row of query 0 in G viewed as [nseq*H*L, L]
  tc_load_tile(Ks, k + (row0 + k0) * ld_qkv + h * 64, ld_qkv, nk);
  tc_key_mask(madd, text_mask, b, k0, L, Lt);
  const int r0 = warp * 16;
  const int rq = r0 + (lane >> 2), cq = 2 * (lane & 3);
  float dkacc[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) dkacc[j][e] = 0.f;
  const int nqb = (L + 63) / 64;
  for (int qb = 0; qb < nqb; ++qb) {
    const int q0 = qb * 64, nq = min(64, L - q0);
    const int nqs = tc_live_slabs(nq);
    __syncthreads();                     // the previous query tile's dK products are done with Qs and dSs
    tc_load_tile(Qs, q + (row0 + q0) * ld_qkv + h * 64, ld_qkv, nq);
    if (threadIdx.x < 64) {
      const bool ok = static_cast<int>(threadIdx.x) < nq;
      lses[threadIdx.x] = ok ? lse[bh0 + q0 + threadIdx.x] : 0.f;
      Ds[threadIdx.x] = ok ? drow[bh0 + q0 + threadIdx.x] : 0.f;
    }
    __syncthreads();
    if (warp < nqs) {
      float s[8][4], u0, u1;
      tc_mm_abt_live(s, Qs, Ks, r0, lane, nks);
      tc_probs_ds<false>(s, madd, lses[rq], lses[rq + 8], Ds[rq], Ds[rq + 8], rq < nq, rq + 8 < nq, dprobs, (bh0 + q0 + rq) * L + k0, L,
                         k0, cq, scale, dc, u0, u1);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        *reinterpret_cast<uint32_t*>(dSs + rq * TC_LD + j * 8 + cq) = pack_bf16x2(s[j][0], s[j][1]);
        *reinterpret_cast<uint32_t*>(dSs + (rq + 8) * TC_LD + j * 8 + cq) = pack_bf16x2(s[j][2], s[j][3]);
      }
    } else {                             // all 16 query rows beyond L: dS = 0
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        *reinterpret_cast<uint32_t*>(dSs + rq * TC_LD + j * 8 + cq) = 0u;
        *reinterpret_cast<uint32_t*>(dSs + (rq + 8) * TC_LD + j * 8 + cq) = 0u;
      }
    }
    __syncthreads();
    if (warp < nks) tc_mm_atb_live(dkacc, dSs, Qs, r0, lane, nqs);   // this warp's 16 key rows: dK += dS^T Q
  }
  if (warp < nks) {
    if (STORE)
      tc_acc_store_global(dkacc, dk + (row0 + k0) * ld_dqkv + h * 64, ld_dqkv, r0, lane, nk, scale);
    else
      tc_acc_add_global(dkacc, dk + (row0 + k0) * ld_dqkv + h * 64, ld_dqkv, r0, lane, nk, scale);
  }
}

// ------------------------------------------------------------------------------------------------ dV alone
// dV_j = sum_i P_ij r_ij dO_i of one 64-key tile, for the backward split at a differentiable attention map (the context product's
// share of the attention backward; dQ / dK come from the map's gradient through cb_attention_probs_bwd_store). P is rebuilt from
// Q, K and the saved lse as attn_tc_probs_kernel forms it, with the forward's dropout multipliers r; the returned map is never
// read. The layout of attn_tc_bwd_kv_kernel without dS: K and the key mask stay in smem; per query tile, phase 1 (each warp: 16
// query rows x 64 keys) forms P r and stages it as bf16, phase 2 (each warp: 16 key rows) accumulates dV += (P r)^T dO in
// registers. dV is written once to the V block: one writer per element, no atomics.
__global__ void __launch_bounds__(TC_THREADS) attn_tc_bwd_dv_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                                                    int64_t ld_qkv, const int64_t* __restrict__ text_mask,
                                                                    const __nv_bfloat16* __restrict__ dctx, int64_t ld_ctx,
                                                                    const float* __restrict__ lse, __nv_bfloat16* __restrict__ dv,
                                                                    int64_t ld_dqkv, int L, int Lt, int H, float scale, TcDrop dc_in) {
  pdl_wait();
  const TcDrop dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  extern __shared__ __align__(16) uint8_t tc_smem[];
  __nv_bfloat16* Ks = reinterpret_cast<__nv_bfloat16*>(tc_smem);
  __nv_bfloat16* Qs = Ks + TC_TILE;
  __nv_bfloat16* dOs = Qs + TC_TILE;
  __nv_bfloat16* Ps = dOs + TC_TILE;     // dropped probabilities [query][key], then the dV tile
  float* madd = reinterpret_cast<float*>(Ps + TC_TILE);
  float* lses = madd + 64;
  const int kb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = kb * 64;
  const int nk = min(64, L - k0), nks = tc_live_slabs(nk);
  const int64_t row0 = static_cast<int64_t>(b) * L;
  const uint64_t bh0 = (static_cast<uint64_t>(b) * H + h) * L;         // row of query 0 in P viewed as [nseq*H*L, L]
  tc_load_tile(Ks, k + (row0 + k0) * ld_qkv + h * 64, ld_qkv, nk);
  tc_key_mask(madd, text_mask, b, k0, L, Lt);
  const int r0 = warp * 16;
  const int rq = r0 + (lane >> 2), cq = 2 * (lane & 3);
  float dvacc[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) dvacc[j][e] = 0.f;
  const int nqb = (L + 63) / 64;
  for (int qb = 0; qb < nqb; ++qb) {
    const int q0 = qb * 64, nq = min(64, L - q0);
    const int nqs = tc_live_slabs(nq);
    __syncthreads();                     // phase 2 of the previous query tile is done with Qs, dOs and Ps
    tc_load_tile(Qs, q + (row0 + q0) * ld_qkv + h * 64, ld_qkv, nq);
    tc_load_tile(dOs, dctx + (row0 + q0) * ld_ctx + h * 64, ld_ctx, nq);
    if (threadIdx.x < 64) lses[threadIdx.x] = static_cast<int>(threadIdx.x) < nq ? lse[bh0 + q0 + threadIdx.x] : 0.f;
    __syncthreads();
    if (warp < nqs) {
      float s[8][4];
      tc_mm_abt_live(s, Qs, Ks, r0, lane, nks);
      const bool ok0 = rq < nq, ok1 = rq + 8 < nq;
      const float l0 = lses[rq], l1 = lses[rq + 8];
      const uint64_t e0 = (bh0 + q0 + rq) * L + k0, e1 = e0 + static_cast<uint64_t>(8) * L;   // dropout index of (row, k0)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float m0 = madd[j * 8 + cq], m1 = madd[j * 8 + cq + 1];
        float p0 = ok0 ? __expf(s[j][0] * scale + m0 - l0) : 0.f, p1 = ok0 ? __expf(s[j][1] * scale + m1 - l0) : 0.f;
        float p2 = ok1 ? __expf(s[j][2] * scale + m0 - l1) : 0.f, p3 = ok1 ? __expf(s[j][3] * scale + m1 - l1) : 0.f;
        if (dc.thresh) {
          float r_0, r_1, r_2, r_3;
          dropout_mult2(dc.seed, e0 + j * 8 + cq, dc.thresh, dc.inv_keep, r_0, r_1);
          dropout_mult2(dc.seed, e1 + j * 8 + cq, dc.thresh, dc.inv_keep, r_2, r_3);
          p0 *= r_0; p1 *= r_1; p2 *= r_2; p3 *= r_3;
        }
        *reinterpret_cast<uint32_t*>(Ps + rq * TC_LD + j * 8 + cq) = pack_bf16x2(p0, p1);
        *reinterpret_cast<uint32_t*>(Ps + (rq + 8) * TC_LD + j * 8 + cq) = pack_bf16x2(p2, p3);
      }
    } else {                             // all 16 query rows beyond L: P = 0
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        *reinterpret_cast<uint32_t*>(Ps + rq * TC_LD + j * 8 + cq) = 0u;
        *reinterpret_cast<uint32_t*>(Ps + (rq + 8) * TC_LD + j * 8 + cq) = 0u;
      }
    }
    __syncthreads();
    if (warp < nks) tc_mm_atb_live(dvacc, Ps, dOs, r0, lane, nqs);   // this warp's 16 key rows: dV += (P r)^T dO
  }
  __syncthreads();                       // P fully consumed: stage dV in its tile
  tc_acc_to_smem(dvacc, Ps, r0, lane, 1.0f);
  __syncthreads();
  tc_store_tile(Ps, dv + (row0 + k0) * ld_dqkv + h * 64, ld_dqkv, nk);
}

static TcDrop make_tc_drop(float p, uint64_t seed) { return make_drop(p, seed); }

// called from cb_attention_fwd / cb_attention_bwd (attention.cu) when l <= 64
template <int RT>
static int launch_tc_fwd(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, void* ctx, int64_t ld_ctx, float* lse, int nseq, int l, int lt,
                         int heads, float dropout_p, uint64_t seed, cudaStream_t stream) {
  constexpr int R = RT * 16;
  const int smem = 3 * R * TC_LD * 2 + R * 4;
  static bool once = false;
  if (!once) {
    cudaError_t e = cudaFuncSetAttribute(attn_tc_fwd_kernel<RT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { set_error("attention_tc_fwd smem: %s", cudaGetErrorString(e)); return CB_ERR_CUDA; }
    once = true;
  }
  const __nv_bfloat16* base = static_cast<const __nv_bfloat16*>(qkv);
  const int hid = heads * 64;
  launch_k(attn_tc_fwd_kernel<RT>, dim3(heads, nseq), RT * 32, smem, stream, base, base + hid, base + 2 * hid, ld_qkv, text_mask,
           static_cast<__nv_bfloat16*>(ctx), ld_ctx, lse, l, lt, heads, 0.125f, make_tc_drop(dropout_p, seed));
  return check_launch("cb_attention_fwd(tc)");
}

static int g_tc_rows48 = 1;      // 0: sequences of up to 48 tokens also run the 64-row kernels (A/B)
void attention_tc_set_rows48(int on) { g_tc_rows48 = on; }

int attention_tc_fwd(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, void* ctx, int64_t ld_ctx, float* lse, int nseq, int l, int lt,
                     int heads, float dropout_p, uint64_t seed, cudaStream_t stream) {
  if (l <= 48 && g_tc_rows48) return launch_tc_fwd<3>(qkv, ld_qkv, text_mask, ctx, ld_ctx, lse, nseq, l, lt, heads, dropout_p, seed, stream);
  return launch_tc_fwd<4>(qkv, ld_qkv, text_mask, ctx, ld_ctx, lse, nseq, l, lt, heads, dropout_p, seed, stream);
}

// called from cb_attention_fwd (attention.cu) for l > 64 when the tensor-core path for long sequences is enabled
template <bool PIPE>
static int launch_tc_fwd_flash(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, void* ctx, int64_t ld_ctx, float* lse, int nseq, int l,
                               int lt, int heads, float dropout_p, uint64_t seed, cudaStream_t stream) {
  constexpr int NBUF = PIPE ? 2 : 1;
  const int smem = (1 + 2 * NBUF) * TC_TILE * 2 + NBUF * 64 * 4;
  static bool once = false;
  if (!once) {
    cudaError_t e = cudaFuncSetAttribute(attn_tc_fwd_flash_kernel<PIPE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { set_error("attention_tc_fwd_flash smem: %s", cudaGetErrorString(e)); return CB_ERR_CUDA; }
    once = true;
  }
  const __nv_bfloat16* base = static_cast<const __nv_bfloat16*>(qkv);
  const int hid = heads * 64;
  launch_k(attn_tc_fwd_flash_kernel<PIPE>, dim3(ceil_div(l, 64), heads, nseq), TC_THREADS, smem, stream, base, base + hid, base + 2 * hid, ld_qkv,
           text_mask, static_cast<__nv_bfloat16*>(ctx), ld_ctx, lse, l, lt, heads, 0.125f, make_tc_drop(dropout_p, seed));
  return check_launch("cb_attention_fwd(tc, flash)");
}

static int g_tc_flash_pipe = 1;      // 0: synchronous key-tile loads (A/B)
void attention_tc_set_flash_pipe(int on) { g_tc_flash_pipe = on; }

int attention_tc_fwd_flash(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, void* ctx, int64_t ld_ctx, float* lse, int nseq, int l,
                           int lt, int heads, float dropout_p, uint64_t seed, cudaStream_t stream) {
  if (g_tc_flash_pipe) return launch_tc_fwd_flash<true>(qkv, ld_qkv, text_mask, ctx, ld_ctx, lse, nseq, l, lt, heads, dropout_p, seed, stream);
  return launch_tc_fwd_flash<false>(qkv, ld_qkv, text_mask, ctx, ld_ctx, lse, nseq, l, lt, heads, dropout_p, seed, stream);
}

template <int RT>
static int launch_tc_bwd(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, const void* ctx, const void* dctx, int64_t ld_ctx,
                         const float* lse, void* dqkv, int64_t ld_dqkv, int nseq, int l, int lt, int heads, float dropout_p, uint64_t seed,
                         cudaStream_t stream) {
  constexpr int R = RT * 16;
  const int smem = 5 * R * TC_LD * 2 + 3 * R * 4;
  static bool once = false;
  if (!once) {
    cudaError_t e = cudaFuncSetAttribute(attn_tc_bwd_kernel<RT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { set_error("attention_tc_bwd smem: %s", cudaGetErrorString(e)); return CB_ERR_CUDA; }
    once = true;
  }
  const __nv_bfloat16* base = static_cast<const __nv_bfloat16*>(qkv);
  __nv_bfloat16* dbase = static_cast<__nv_bfloat16*>(dqkv);
  const int hid = heads * 64;
  launch_k(attn_tc_bwd_kernel<RT>, dim3(heads, nseq), RT * 32, smem, stream, base, base + hid, base + 2 * hid, ld_qkv, text_mask,
           static_cast<const __nv_bfloat16*>(ctx), static_cast<const __nv_bfloat16*>(dctx), ld_ctx, lse, dbase, dbase + hid,
           dbase + 2 * hid, ld_dqkv, l, lt, heads, 0.125f, make_tc_drop(dropout_p, seed));
  return check_launch("cb_attention_bwd(tc)");
}

int attention_tc_bwd(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, const void* ctx, const void* dctx, int64_t ld_ctx,
                     const float* lse, void* dqkv, int64_t ld_dqkv, int nseq, int l, int lt, int heads, float dropout_p, uint64_t seed,
                     cudaStream_t stream) {
  if (l <= 48 && g_tc_rows48)
    return launch_tc_bwd<3>(qkv, ld_qkv, text_mask, ctx, dctx, ld_ctx, lse, dqkv, ld_dqkv, nseq, l, lt, heads, dropout_p, seed, stream);
  return launch_tc_bwd<4>(qkv, ld_qkv, text_mask, ctx, dctx, ld_ctx, lse, dqkv, ld_dqkv, nseq, l, lt, heads, dropout_p, seed, stream);
}

// called from cb_attention_bwd (attention.cu) for l > 64. kv kernel: K, V, Q, dO, P, dS tiles + three 64-float vectors = 55 KB;
// q kernel: Q, dO, K, V tiles + the same vectors = 37 KB; both leave room for several CTAs per SM.
int attention_tc_bwd_long(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, const void* ctx, const void* dctx, int64_t ld_ctx,
                          const float* lse, void* dqkv, int64_t ld_dqkv, int nseq, int l, int lt, int heads, float dropout_p, uint64_t seed,
                          cudaStream_t stream) {
  const int smem_kv = 6 * TC_TILE * 2 + 3 * 64 * 4;
  const int smem_q = 4 * TC_TILE * 2 + 3 * 64 * 4;
  static bool once = false;
  if (!once) {
    cudaError_t e = cudaFuncSetAttribute(attn_tc_bwd_kv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_kv);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(attn_tc_bwd_q_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_q);
    if (e != cudaSuccess) { set_error("attention_tc_bwd_long smem: %s", cudaGetErrorString(e)); return CB_ERR_CUDA; }
    once = true;
  }
  const __nv_bfloat16* base = static_cast<const __nv_bfloat16*>(qkv);
  __nv_bfloat16* dbase = static_cast<__nv_bfloat16*>(dqkv);
  const int hid = heads * 64;
  const TcDrop dc = make_tc_drop(dropout_p, seed);
  const dim3 grid(ceil_div(l, 64), heads, nseq);
  launch_k(attn_tc_bwd_kv_kernel, grid, TC_THREADS, smem_kv, stream, base, base + hid, base + 2 * hid, ld_qkv, text_mask,
           static_cast<const __nv_bfloat16*>(ctx), static_cast<const __nv_bfloat16*>(dctx), ld_ctx, lse, dbase + hid, dbase + 2 * hid,
           ld_dqkv, l, lt, heads, 0.125f, dc);
  int rc = check_launch("cb_attention_bwd(tc, kv)");
  if (rc) return rc;
  launch_k(attn_tc_bwd_q_kernel, grid, TC_THREADS, smem_q, stream, base, base + hid, base + 2 * hid, ld_qkv, text_mask,
           static_cast<const __nv_bfloat16*>(ctx), static_cast<const __nv_bfloat16*>(dctx), ld_ctx, lse, dbase, ld_dqkv, l, lt, heads,
           0.125f, dc);
  return check_launch("cb_attention_bwd(tc, q)");
}

}  // namespace cb

extern "C" int cb_attention_probs(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, const float* lse, float* probs, int nseq, int l,
                                  int lt, int heads, int head_dim, float dropout_p, uint64_t seed, void* stream) {
  using namespace cb;
  CB_REQUIRE(head_dim == 64, "cb_attention_probs: head_dim %d unsupported (built for 64)", head_dim);
  CB_REQUIRE(qkv && text_mask && lse && probs && nseq > 0 && l > 0 && lt >= 0 && lt <= l && heads > 0 && nseq <= 65535 && heads <= 65535,
             "cb_attention_probs: bad arguments");
  CB_REQUIRE(ld_qkv % 8 == 0 && ld_qkv >= 3 * heads * 64, "cb_attention_probs: qkv row pitch must be a multiple of 8 and hold Q | K | V");
  CB_REQUIRE(reinterpret_cast<uintptr_t>(qkv) % 16 == 0 && reinterpret_cast<uintptr_t>(probs) % 16 == 0,
             "cb_attention_probs: qkv and probs must be 16-byte aligned");
  const int smem = 2 * TC_TILE * 2 + (64 * PR_LD + 2 * 64) * 4;   // Q, K tiles (bf16) + staged P, key mask, lse (fp32): 37 KB
  const __nv_bfloat16* base = static_cast<const __nv_bfloat16*>(qkv);
  const int hid = heads * 64;
  launch_k(attn_tc_probs_kernel, dim3(ceil_div(l, 64), heads, nseq), TC_THREADS, smem, static_cast<cudaStream_t>(stream), base, base + hid,
           ld_qkv, text_mask, lse, probs, l, lt, heads, 0.125f, make_tc_drop(dropout_p, seed));
  return check_launch("cb_attention_probs");
}

namespace cb {
// cb_attention_probs_bwd (STORE = false: added to dQ / dK) and cb_attention_probs_bwd_store (written)
template <bool STORE>
static int attention_probs_bwd(const char* name, const void* qkv, int64_t ld_qkv, const int64_t* text_mask, const float* lse,
                               const float* dprobs, float* drow, void* dqkv, int64_t ld_dqkv, int nseq, int l, int lt, int heads,
                               int head_dim, float dropout_p, uint64_t seed, void* stream) {
  CB_REQUIRE(head_dim == 64, "%s: head_dim %d unsupported (built for 64)", name, head_dim);
  CB_REQUIRE(qkv && text_mask && lse && dprobs && drow && dqkv && nseq > 0 && l > 0 && lt >= 0 && lt <= l && heads > 0 && nseq <= 65535 &&
                 heads <= 65535,
             "%s: bad arguments", name);
  CB_REQUIRE(ld_qkv % 8 == 0 && ld_dqkv % 8 == 0 && ld_qkv >= 3 * static_cast<int64_t>(heads) * 64 &&
                 ld_dqkv >= 3 * static_cast<int64_t>(heads) * 64,
             "%s: row pitches must be multiples of 8 and hold Q | K | V", name);
  CB_REQUIRE(reinterpret_cast<uintptr_t>(qkv) % 16 == 0 && reinterpret_cast<uintptr_t>(dqkv) % 16 == 0 &&
                 reinterpret_cast<uintptr_t>(dprobs) % 16 == 0,
             "%s: qkv, dqkv and dprobs must be 16-byte aligned", name);
  // q kernel: Q, K tiles + key mask, lse = 18.5 KB; k kernel: K, Q, dS tiles + key mask, lse, D = 27.8 KB
  const int smem_q = 2 * TC_TILE * 2 + 2 * 64 * 4;
  const int smem_k = 3 * TC_TILE * 2 + 3 * 64 * 4;
  const __nv_bfloat16* base = static_cast<const __nv_bfloat16*>(qkv);
  __nv_bfloat16* dbase = static_cast<__nv_bfloat16*>(dqkv);
  const int hid = heads * 64;
  const TcDrop dc = make_tc_drop(dropout_p, seed);
  const dim3 grid(ceil_div(l, 64), heads, nseq);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  launch_k(attn_tc_probs_bwd_q_kernel<STORE>, grid, TC_THREADS, smem_q, st, base, base + hid, ld_qkv, text_mask, lse, dprobs, drow, dbase,
           ld_dqkv, l, lt, heads, 0.125f, dc);
  int rc = check_launch(STORE ? "cb_attention_probs_bwd_store(q)" : "cb_attention_probs_bwd(q)");
  if (rc) return rc;
  launch_k(attn_tc_probs_bwd_k_kernel<STORE>, grid, TC_THREADS, smem_k, st, base, base + hid, ld_qkv, text_mask, lse, dprobs,
           static_cast<const float*>(drow), dbase + hid, ld_dqkv, l, lt, heads, 0.125f, dc);
  return check_launch(STORE ? "cb_attention_probs_bwd_store(k)" : "cb_attention_probs_bwd(k)");
}
}  // namespace cb

extern "C" int cb_attention_probs_bwd(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, const float* lse, const float* dprobs,
                                      float* drow, void* dqkv, int64_t ld_dqkv, int nseq, int l, int lt, int heads, int head_dim,
                                      float dropout_p, uint64_t seed, void* stream) {
  return cb::attention_probs_bwd<false>("cb_attention_probs_bwd", qkv, ld_qkv, text_mask, lse, dprobs, drow, dqkv, ld_dqkv, nseq, l, lt,
                                        heads, head_dim, dropout_p, seed, stream);
}

extern "C" int cb_attention_probs_bwd_store(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, const float* lse,
                                            const float* dprobs, float* drow, void* dqkv, int64_t ld_dqkv, int nseq, int l, int lt,
                                            int heads, int head_dim, float dropout_p, uint64_t seed, void* stream) {
  return cb::attention_probs_bwd<true>("cb_attention_probs_bwd_store", qkv, ld_qkv, text_mask, lse, dprobs, drow, dqkv, ld_dqkv, nseq, l,
                                       lt, heads, head_dim, dropout_p, seed, stream);
}

extern "C" int cb_attention_bwd_dv(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, const float* lse, const void* dctx,
                                   int64_t ld_ctx, void* dqkv, int64_t ld_dqkv, int nseq, int l, int lt, int heads, int head_dim,
                                   float dropout_p, uint64_t seed, void* stream) {
  using namespace cb;
  CB_REQUIRE(head_dim == 64, "cb_attention_bwd_dv: head_dim %d unsupported (built for 64)", head_dim);
  CB_REQUIRE(qkv && text_mask && lse && dctx && dqkv && nseq > 0 && l > 0 && lt >= 0 && lt <= l && heads > 0 && nseq <= 65535 &&
                 heads <= 65535,
             "cb_attention_bwd_dv: bad arguments");
  CB_REQUIRE(ld_qkv % 8 == 0 && ld_ctx % 8 == 0 && ld_dqkv % 8 == 0 && ld_qkv >= 3 * static_cast<int64_t>(heads) * 64 &&
                 ld_dqkv >= 3 * static_cast<int64_t>(heads) * 64 && ld_ctx >= static_cast<int64_t>(heads) * 64,
             "cb_attention_bwd_dv: row pitches must be multiples of 8 and hold Q | K | V and the merged heads");
  CB_REQUIRE(reinterpret_cast<uintptr_t>(qkv) % 16 == 0 && reinterpret_cast<uintptr_t>(dctx) % 16 == 0 &&
                 reinterpret_cast<uintptr_t>(dqkv) % 16 == 0,
             "cb_attention_bwd_dv: qkv, dctx and dqkv must be 16-byte aligned");
  const int smem = 4 * TC_TILE * 2 + 2 * 64 * 4;                  // K, Q, dO, P tiles (bf16) + key mask, lse (fp32): 37 KB
  const __nv_bfloat16* base = static_cast<const __nv_bfloat16*>(qkv);
  const int hid = heads * 64;
  launch_k(attn_tc_bwd_dv_kernel, dim3(ceil_div(l, 64), heads, nseq), TC_THREADS, smem, static_cast<cudaStream_t>(stream), base,
           base + hid, ld_qkv, text_mask, static_cast<const __nv_bfloat16*>(dctx), ld_ctx, lse,
           static_cast<__nv_bfloat16*>(dqkv) + 2 * hid, ld_dqkv, l, lt, heads, 0.125f, make_tc_drop(dropout_p, seed));
  return check_launch("cb_attention_bwd_dv");
}

extern "C" int cb_attention_dprobs(const void* qkv, int64_t ld_qkv, const void* dctx, int64_t ld_ctx, float* dprobs, int accumulate,
                                   int nseq, int l, int heads, int head_dim, void* stream) {
  using namespace cb;
  CB_REQUIRE(head_dim == 64, "cb_attention_dprobs: head_dim %d unsupported (built for 64)", head_dim);
  CB_REQUIRE(qkv && dctx && dprobs && (accumulate == 0 || accumulate == 1) && nseq > 0 && l > 0 && heads > 0 && nseq <= 65535 &&
                 heads <= 65535,
             "cb_attention_dprobs: bad arguments");
  CB_REQUIRE(ld_qkv % 8 == 0 && ld_ctx % 8 == 0 && ld_qkv >= 3 * static_cast<int64_t>(heads) * 64 &&
                 ld_ctx >= static_cast<int64_t>(heads) * 64,
             "cb_attention_dprobs: row pitches must be multiples of 8 and hold Q | K | V and the merged heads");
  CB_REQUIRE(reinterpret_cast<uintptr_t>(qkv) % 16 == 0 && reinterpret_cast<uintptr_t>(dctx) % 16 == 0 &&
                 reinterpret_cast<uintptr_t>(dprobs) % 16 == 0,
             "cb_attention_dprobs: qkv, dctx and dprobs must be 16-byte aligned");
  const int smem = 2 * TC_TILE * 2 + 64 * PR_LD * 4;             // dO, V tiles (bf16) + staged dA (fp32): 36 KB
  const __nv_bfloat16* v = static_cast<const __nv_bfloat16*>(qkv) + 2 * heads * 64;
  const __nv_bfloat16* d = static_cast<const __nv_bfloat16*>(dctx);
  const dim3 grid(ceil_div(l, 64), heads, nseq);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (accumulate)
    launch_k(attn_tc_dprobs_kernel<true>, grid, TC_THREADS, smem, st, v, ld_qkv, d, ld_ctx, dprobs, l, heads);
  else
    launch_k(attn_tc_dprobs_kernel<false>, grid, TC_THREADS, smem, st, v, ld_qkv, d, ld_ctx, dprobs, l, heads);
  return check_launch("cb_attention_dprobs");
}
