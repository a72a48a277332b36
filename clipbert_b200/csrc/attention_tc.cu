// Tensor-core fast path of the fused self-attention for short sequences (L <= 64: every ClipBERT training
// configuration at 224 px, L = Lt + 9). One CTA = one (sequence, head); 4 warps x 16 query rows; Q, K, V (and dO)
// tiles live in shared memory as bf16, the 64x64x64 products run on mma.sync.m16n8k16 (bf16 in, fp32 accumulate)
// with ldmatrix operand fetches, softmax / dropout / dS stay in the accumulator registers (the S accumulator
// layout is reused as the A operand of the next product). Same math, masks, dropout stream and lse convention as
// csrc/attention.cu, which remains the path for L > 64 (448 px frames, 512-token inference).
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

}  // namespace cb
