// Memory-bound BERT-side kernels: LayerNorm fwd/bwd, text / visual embedding (+LN) fwd/bwd,
// bias-gradient column sums, dropout, small casts. One warp per 768-wide row, 128-bit loads,
// fp32 statistics via warp shuffles (the reference path is apex FusedLayerNorm + ATen
// elementwise kernels: src/modeling/transformers.py:172-199,297-301,377-381; modeling.py:62-101).
#include "common.cuh"
#include "host_util.h"

namespace cb {

constexpr int HID = 768;          // hidden size (src/configs/base_model.json)
constexpr int CH = HID / 256;     // uint4 (8 x bf16) chunks per lane
constexpr int ROWS_PER_BLOCK = 4; // one warp per row

// lane-local view of one row: element (c, j) is column c*256 + lane*8 + j
__device__ __forceinline__ void load_row_bf16(const __nv_bfloat16* row, int lane, float (&x)[CH][8]) {
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const uint4 u = *reinterpret_cast<const uint4*>(row + c * 256 + lane * 8);
    float2 t;
    t = unpack_bf16x2(u.x); x[c][0] = t.x; x[c][1] = t.y;
    t = unpack_bf16x2(u.y); x[c][2] = t.x; x[c][3] = t.y;
    t = unpack_bf16x2(u.z); x[c][4] = t.x; x[c][5] = t.y;
    t = unpack_bf16x2(u.w); x[c][6] = t.x; x[c][7] = t.y;
  }
}
__device__ __forceinline__ void load_row_f32(const float* row, int lane, float (&x)[CH][8]) {
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(row + c * 256 + lane * 8));
    const float4 b = __ldg(reinterpret_cast<const float4*>(row + c * 256 + lane * 8 + 4));
    x[c][0] = a.x; x[c][1] = a.y; x[c][2] = a.z; x[c][3] = a.w;
    x[c][4] = b.x; x[c][5] = b.y; x[c][6] = b.z; x[c][7] = b.w;
  }
}
__device__ __forceinline__ void store_row_bf16(__nv_bfloat16* row, int lane, const float (&x)[CH][8]) {
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    uint4 u;
    u.x = pack_bf16x2(x[c][0], x[c][1]);
    u.y = pack_bf16x2(x[c][2], x[c][3]);
    u.z = pack_bf16x2(x[c][4], x[c][5]);
    u.w = pack_bf16x2(x[c][6], x[c][7]);
    *reinterpret_cast<uint4*>(row + c * 256 + lane * 8) = u;
  }
}
__device__ __forceinline__ void store_row_f32(float* row, int lane, const float (&x)[CH][8]) {
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    *reinterpret_cast<float4*>(row + c * 256 + lane * 8) = make_float4(x[c][0], x[c][1], x[c][2], x[c][3]);
    *reinterpret_cast<float4*>(row + c * 256 + lane * 8 + 4) = make_float4(x[c][4], x[c][5], x[c][6], x[c][7]);
  }
}

// y = (x - mean) * rstd * gamma + beta ; returns mean / rstd (fp32, biased variance like F.layer_norm)
__device__ __forceinline__ void ln_forward_row(float (&x)[CH][8], const float* gamma, const float* beta,
                                               float eps, int lane, float& mean, float& rstd) {
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) s += x[c][j];
  mean = warp_sum(s) * (1.0f / HID);
  float v = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float d = x[c][j] - mean;
      v += d * d;
    }
  rstd = rsqrtf(warp_sum(v) * (1.0f / HID) + eps);
  float g[CH][8], b[CH][8];
  load_row_f32(gamma, lane, g);
  load_row_f32(beta, lane, b);
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) x[c][j] = (x[c][j] - mean) * rstd * g[c][j] + b[c][j];
}

__device__ __forceinline__ void apply_dropout_row(float (&x)[CH][8], const DropCfg& dc, int64_t row, int lane) {
  if (dc.thresh == 0) return;
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; j += 4) {      // 4-aligned runs: one hash per four elements
      float m[4];
      dropout_mult4(dc.seed, static_cast<uint64_t>(row) * HID + c * 256 + lane * 8 + j, dc.thresh, dc.inv_keep, m);
#pragma unroll
      for (int t = 0; t < 4; ++t) x[c][j + t] *= m[t];
    }
}

// dx = rstd * (g - mean(g) - xhat * mean(g * xhat)), g = dy * gamma. On return x holds xhat, dy holds dx.
__device__ __forceinline__ void ln_backward_row(float (&dy)[CH][8], float (&x)[CH][8], const float (&gam)[CH][8],
                                                float mean, float rstd) {
  float c1 = 0.f, c2 = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      x[c][j] = (x[c][j] - mean) * rstd;
      const float g = dy[c][j] * gam[c][j];
      c1 += g;
      c2 += g * x[c][j];
    }
  c1 = warp_sum(c1) * (1.0f / HID);
  c2 = warp_sum(c2) * (1.0f / HID);
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) dy[c][j] = rstd * (dy[c][j] * gam[c][j] - c1 - x[c][j] * c2);
}

// block-level reduction of per-warp [CH][8] partials into global fp32 vectors via atomics
__device__ __forceinline__ void block_accumulate(float (&acc)[CH][8], float* smem_buf /*[ROWS][HID]*/, float* gdst,
                                                 int warp, int lane) {
  store_row_f32(smem_buf + warp * HID, lane, acc);
  __syncthreads();
  if ((reinterpret_cast<uintptr_t>(gdst) & 15) == 0) {      // every vector of the flat gradient buffer: 16-byte reductions
    for (int i = threadIdx.x * 4; i < HID; i += blockDim.x * 4) {
      float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int w = 0; w < ROWS_PER_BLOCK; ++w) {
        const float4 v = *reinterpret_cast<const float4*>(smem_buf + w * HID + i);
        s.x += v.x, s.y += v.y, s.z += v.z, s.w += v.w;
      }
      if (s.x != 0.f || s.y != 0.f || s.z != 0.f || s.w != 0.f) red_add_f32x4(gdst + i, s);
    }
  } else {
    for (int i = threadIdx.x; i < HID; i += blockDim.x) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < ROWS_PER_BLOCK; ++w) s += smem_buf[w * HID + i];
      if (s != 0.f) atomicAdd(gdst + i, s);
    }
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// LayerNorm over rows of a [M, 768] bf16 matrix
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) ln_fwd_kernel(const __nv_bfloat16* __restrict__ x, const float* gamma,
                                                     const float* beta, __nv_bfloat16* __restrict__ y,
                                                     float* __restrict__ stats, int M, float eps) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t m = static_cast<int64_t>(blockIdx.x) * ROWS_PER_BLOCK + warp;
  if (m >= M) return;
  float v[CH][8];
  load_row_bf16(x + m * HID, lane, v);
  float mean, rstd;
  ln_forward_row(v, gamma, beta, eps, lane, mean, rstd);
  store_row_bf16(y + m * HID, lane, v);
  if (lane == 0 && stats) {
    stats[2 * m] = mean;
    stats[2 * m + 1] = rstd;
  }
}

// grid-stride over rows; per-warp dgamma / dbeta / dbias partials, reduced per block
__global__ void __launch_bounds__(128) ln_bwd_kernel(const __nv_bfloat16* __restrict__ dy,
                                                     const __nv_bfloat16* __restrict__ x,
                                                     const float* __restrict__ stats, const float* gamma,
                                                     __nv_bfloat16* __restrict__ dx, __nv_bfloat16* __restrict__ dx_drop,
                                                     float* dgamma, float* dbeta, float* dbias_drop, int M, DropCfg dc_in) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  const DropCfg dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  __shared__ __align__(16) float red[ROWS_PER_BLOCK * HID];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float gam[CH][8];
  load_row_f32(gamma, lane, gam);
  float ag[CH][8], ab[CH][8], ad[CH][8];
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) ag[c][j] = ab[c][j] = ad[c][j] = 0.f;

  for (int64_t m = static_cast<int64_t>(blockIdx.x) * ROWS_PER_BLOCK + warp; m < M;
       m += static_cast<int64_t>(gridDim.x) * ROWS_PER_BLOCK) {
    float g[CH][8], xv[CH][8];
    load_row_bf16(dy + m * HID, lane, g);
    load_row_bf16(x + m * HID, lane, xv);
    const float mean = stats[2 * m], rstd = stats[2 * m + 1];
#pragma unroll
    for (int c = 0; c < CH; ++c)
#pragma unroll
      for (int j = 0; j < 8; ++j) ab[c][j] += g[c][j];
    float gsave[CH][8];
#pragma unroll
    for (int c = 0; c < CH; ++c)
#pragma unroll
      for (int j = 0; j < 8; ++j) gsave[c][j] = g[c][j];
    ln_backward_row(g, xv, gam, mean, rstd);  // g <- dx, xv <- xhat
#pragma unroll
    for (int c = 0; c < CH; ++c)
#pragma unroll
      for (int j = 0; j < 8; ++j) ag[c][j] += gsave[c][j] * xv[c][j];
    store_row_bf16(dx + m * HID, lane, g);
    if (dx_drop) {
      apply_dropout_row(g, dc, m, lane);
      store_row_bf16(dx_drop + m * HID, lane, g);
    }
    if (dbias_drop) {
      // gradient of the bias of the dense layer feeding this LN (after its dropout): column sum of
      // the bf16-rounded tensor the wgrad GEMM will read
#pragma unroll
      for (int c = 0; c < CH; ++c)
#pragma unroll
        for (int j = 0; j < 8; ++j) ad[c][j] += __bfloat162float(__float2bfloat16(g[c][j]));
    }
  }
  if (dgamma) block_accumulate(ag, red, dgamma, warp, lane);
  if (dbeta) block_accumulate(ab, red, dbeta, warp, lane);
  if (dbias_drop) block_accumulate(ad, red, dbias_drop, warp, lane);
}

// ------------------------------------------------------------------------------------------------
// Text embeddings: out[b*L + t] = dropout(LN(word[id] + pos[t] + type[0]))   (t < Lt)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) embed_text_fwd_kernel(const int64_t* __restrict__ ids, const float* word,
                                                             const float* pos, const float* type0,
                                                             const float* gamma, const float* beta,
                                                             __nv_bfloat16* __restrict__ out, float* __restrict__ stats,
                                                             int nseq, int Lt, int L, int vocab, float eps, DropCfg dc_in) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  const DropCfg dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t r = static_cast<int64_t>(blockIdx.x) * ROWS_PER_BLOCK + warp;
  if (r >= static_cast<int64_t>(nseq) * Lt) return;
  const int b = static_cast<int>(r / Lt), t = static_cast<int>(r - static_cast<int64_t>(b) * Lt);
  int64_t id = ids[r];
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  float v[CH][8], p[CH][8], ty[CH][8];
  load_row_f32(word + id * HID, lane, v);
  load_row_f32(pos + static_cast<int64_t>(t) * HID, lane, p);
  load_row_f32(type0, lane, ty);
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) v[c][j] = v[c][j] + p[c][j] + ty[c][j];
  float mean, rstd;
  ln_forward_row(v, gamma, beta, eps, lane, mean, rstd);
  const int64_t orow = static_cast<int64_t>(b) * L + t;
  apply_dropout_row(v, dc, orow, lane);
  store_row_bf16(out + orow * HID, lane, v);
  if (lane == 0) {
    stats[2 * r] = mean;
    stats[2 * r + 1] = rstd;
  }
}

// grid = (blocks per position, Lt): every block works on ONE text position t, so the position-embedding gradient is summed in
// registers / shared memory and leaves the block as 768 atomics (it was one atomic per element per row: 64-way contention on the
// Lt rows of dpos made this kernel 82 us at 64 sequences); the word rows go out as 16-byte reductions.
__global__ void __launch_bounds__(128) embed_text_bwd_kernel(const __nv_bfloat16* __restrict__ dh,
                                                             const int64_t* __restrict__ ids, const float* word,
                                                             const float* pos, const float* type0, const float* gamma,
                                                             const float* __restrict__ stats, float* dword, float* dpos,
                                                             float* dtype0, float* dgamma, float* dbeta, int nseq, int Lt,
                                                             int L, int vocab, DropCfg dc_in) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  const DropCfg dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  __shared__ __align__(16) float red[ROWS_PER_BLOCK * HID];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.y;
  float gam[CH][8], p[CH][8], ty[CH][8];
  load_row_f32(gamma, lane, gam);
  load_row_f32(pos + static_cast<int64_t>(t) * HID, lane, p);
  load_row_f32(type0, lane, ty);
  float ag[CH][8], ab[CH][8], at[CH][8];
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      ag[c][j] = ab[c][j] = at[c][j] = 0.f;
      p[c][j] += ty[c][j];
    }
  for (int b = blockIdx.x * ROWS_PER_BLOCK + warp; b < nseq; b += gridDim.x * ROWS_PER_BLOCK) {
    const int64_t r = static_cast<int64_t>(b) * Lt + t;
    int64_t id = ids[r];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    const int64_t orow = static_cast<int64_t>(b) * L + t;
    float g[CH][8], e[CH][8];
    load_row_bf16(dh + orow * HID, lane, g);
    apply_dropout_row(g, dc, orow, lane);
    load_row_f32(word + id * HID, lane, e);
#pragma unroll
    for (int c = 0; c < CH; ++c)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        e[c][j] += p[c][j];
        ab[c][j] += g[c][j];
      }
    float gsave[CH][8];
#pragma unroll
    for (int c = 0; c < CH; ++c)
#pragma unroll
      for (int j = 0; j < 8; ++j) gsave[c][j] = g[c][j];
    ln_backward_row(g, e, gam, stats[2 * r], stats[2 * r + 1]);
#pragma unroll
    for (int c = 0; c < CH; ++c) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        ag[c][j] += gsave[c][j] * e[c][j];
        at[c][j] += g[c][j];
      }
      float* wrow = dword + id * HID + c * 256 + lane * 8;
      red_add_f32x4(wrow, make_float4(g[c][0], g[c][1], g[c][2], g[c][3]));
      red_add_f32x4(wrow + 4, make_float4(g[c][4], g[c][5], g[c][6], g[c][7]));
    }
  }
  block_accumulate(ag, red, dgamma, warp, lane);
  block_accumulate(ab, red, dbeta, warp, lane);
  block_accumulate(at, red, dtype0, warp, lane);
  block_accumulate(at, red, dpos + static_cast<int64_t>(t) * HID, warp, lane);      // d pos[t] = d type[0] restricted to this position
}

// ------------------------------------------------------------------------------------------------
// Visual embeddings: out[b'*L + Lt + j] = dropout(LN(mean_t grid[vid(b'), t, j] + row[j/w] + col[j%w] + type[0]))
// vid(b') = b' / n_ex (uniform) or looked up in seq2vid (ragged n_examples_list).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) embed_visual_fwd_kernel(const __nv_bfloat16* __restrict__ grid,
                                                               const int32_t* __restrict__ seq2vid, int n_ex,
                                                               const float* rowemb, const float* colemb,
                                                               const float* type0, const float* gamma, const float* beta,
                                                               __nv_bfloat16* __restrict__ out, float* __restrict__ stats,
                                                               int nseq, int T, int gh, int gw, int Lt, int L, float eps,
                                                               DropCfg dc_in) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  const DropCfg dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int Lv = gh * gw;
  const int64_t r = static_cast<int64_t>(blockIdx.x) * ROWS_PER_BLOCK + warp;
  if (r >= static_cast<int64_t>(nseq) * Lv) return;
  const int b = static_cast<int>(r / Lv), j = static_cast<int>(r - static_cast<int64_t>(b) * Lv);
  const int vid = seq2vid ? seq2vid[b] : b / n_ex;
  float v[CH][8];
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int q = 0; q < 8; ++q) v[c][q] = 0.f;
  for (int t = 0; t < T; ++t) {
    float f[CH][8];
    load_row_bf16(grid + ((static_cast<int64_t>(vid) * T + t) * Lv + j) * HID, lane, f);
#pragma unroll
    for (int c = 0; c < CH; ++c)
#pragma unroll
      for (int q = 0; q < 8; ++q) v[c][q] += f[c][q];
  }
  const float invT = 1.0f / T;
  float re[CH][8], ce[CH][8], ty[CH][8];
  load_row_f32(rowemb + static_cast<int64_t>(j / gw) * HID, lane, re);
  load_row_f32(colemb + static_cast<int64_t>(j % gw) * HID, lane, ce);
  load_row_f32(type0, lane, ty);
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int q = 0; q < 8; ++q) v[c][q] = v[c][q] * invT + re[c][q] + ce[c][q] + ty[c][q];
  float mean, rstd;
  ln_forward_row(v, gamma, beta, eps, lane, mean, rstd);
  const int64_t orow = static_cast<int64_t>(b) * L + Lt + j;
  apply_dropout_row(v, dc, orow, lane);
  store_row_bf16(out + orow * HID, lane, v);
  if (lane == 0) {
    stats[2 * r] = mean;
    stats[2 * r + 1] = rstd;
  }
}

// pass 1: LN backward per (b', j); writes dv (fp32) to tmp and accumulates parameter gradients
__global__ void __launch_bounds__(128) embed_visual_bwd_kernel(const __nv_bfloat16* __restrict__ dh,
                                                               const __nv_bfloat16* __restrict__ grid,
                                                               const int32_t* __restrict__ seq2vid, int n_ex,
                                                               const float* rowemb, const float* colemb,
                                                               const float* type0, const float* gamma,
                                                               const float* __restrict__ stats, float* __restrict__ dv_tmp,
                                                               float* drow, float* dcol, float* dtype0, float* dgamma,
                                                               float* dbeta, int nseq, int T, int gh, int gw, int Lt, int L,
                                                               DropCfg dc_in) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  const DropCfg dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  __shared__ __align__(16) float red[ROWS_PER_BLOCK * HID];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int Lv = gh * gw;
  float gam[CH][8];
  load_row_f32(gamma, lane, gam);
  float ag[CH][8], ab[CH][8], at[CH][8];
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int q = 0; q < 8; ++q) ag[c][q] = ab[c][q] = at[c][q] = 0.f;
  // grid = (blocks per grid cell, Lv): a block works on ONE visual position j, so d row[j / gw], d col[j % gw] (and d type[0])
  // leave it as one reduced vector each instead of one atomic per element per row
  const int j = blockIdx.y;
  for (int b = blockIdx.x * ROWS_PER_BLOCK + warp; b < nseq; b += gridDim.x * ROWS_PER_BLOCK) {
    const int64_t r = static_cast<int64_t>(b) * Lv + j;
    const int vid = seq2vid ? seq2vid[b] : b / n_ex;
    const int64_t orow = static_cast<int64_t>(b) * L + Lt + j;
    float g[CH][8], v[CH][8];
    load_row_bf16(dh + orow * HID, lane, g);
    apply_dropout_row(g, dc, orow, lane);
#pragma unroll
    for (int c = 0; c < CH; ++c)
#pragma unroll
      for (int q = 0; q < 8; ++q) v[c][q] = 0.f;
    for (int t = 0; t < T; ++t) {
      float f[CH][8];
      load_row_bf16(grid + ((static_cast<int64_t>(vid) * T + t) * Lv + j) * HID, lane, f);
#pragma unroll
      for (int c = 0; c < CH; ++c)
#pragma unroll
        for (int q = 0; q < 8; ++q) v[c][q] += f[c][q];
    }
    const float invT = 1.0f / T;
    float re[CH][8], ce[CH][8], ty[CH][8];
    load_row_f32(rowemb + static_cast<int64_t>(j / gw) * HID, lane, re);
    load_row_f32(colemb + static_cast<int64_t>(j % gw) * HID, lane, ce);
    load_row_f32(type0, lane, ty);
    float gsave[CH][8];
#pragma unroll
    for (int c = 0; c < CH; ++c)
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        v[c][q] = v[c][q] * invT + re[c][q] + ce[c][q] + ty[c][q];
        ab[c][q] += g[c][q];
        gsave[c][q] = g[c][q];
      }
    ln_backward_row(g, v, gam, stats[2 * r], stats[2 * r + 1]);
    store_row_f32(dv_tmp + r * HID, lane, g);
#pragma unroll
    for (int c = 0; c < CH; ++c)
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        ag[c][q] += gsave[c][q] * v[c][q];
        at[c][q] += g[c][q];
      }
  }
  block_accumulate(ag, red, dgamma, warp, lane);
  block_accumulate(ab, red, dbeta, warp, lane);
  block_accumulate(at, red, dtype0, warp, lane);
  block_accumulate(at, red, drow + static_cast<int64_t>(j / gw) * HID, warp, lane);
  block_accumulate(at, red, dcol + static_cast<int64_t>(j % gw) * HID, warp, lane);
}

// pass 2: dgrid[vid, t, j] = (1/T) * sum_{b' -> vid} dv[b', j]   (backward of repeat_tensor_rows + frame mean)
__global__ void __launch_bounds__(128) embed_visual_bwd_reduce_kernel(const float* __restrict__ dv_tmp,
                                                                      const int32_t* __restrict__ vid_start, int n_ex,
                                                                      __nv_bfloat16* __restrict__ dgrid, int nvid, int T,
                                                                      int Lv) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t r = static_cast<int64_t>(blockIdx.x) * ROWS_PER_BLOCK + warp;
  if (r >= static_cast<int64_t>(nvid) * Lv) return;
  const int vid = static_cast<int>(r / Lv), j = static_cast<int>(r - static_cast<int64_t>(vid) * Lv);
  const int s0 = vid_start ? vid_start[vid] : vid * n_ex;
  const int s1 = vid_start ? vid_start[vid + 1] : (vid + 1) * n_ex;
  float acc[CH][8];
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[c][q] = 0.f;
  for (int s = s0; s < s1; ++s) {
    float f[CH][8];
    load_row_f32(dv_tmp + (static_cast<int64_t>(s) * Lv + j) * HID, lane, f);
#pragma unroll
    for (int c = 0; c < CH; ++c)
#pragma unroll
      for (int q = 0; q < 8; ++q) acc[c][q] += f[c][q];
  }
  const float invT = 1.0f / T;
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[c][q] *= invT;
  for (int t = 0; t < T; ++t) store_row_bf16(dgrid + ((static_cast<int64_t>(vid) * T + t) * Lv + j) * HID, lane, acc);
}

// ------------------------------------------------------------------------------------------------
// column sums (bias gradients): db[n] += sum_m dY[m, n]
// ------------------------------------------------------------------------------------------------
// block = 8 warps x 32 lanes: a lane owns 8 columns (one 128-bit load per row), warps stride the rows of a
// 128-row slab; partials are combined across warps in smem so that each block issues ONE atomic per column
__global__ void __launch_bounds__(256) colsum_kernel(const __nv_bfloat16* __restrict__ x, int64_t ld, float* __restrict__ out, int M,
                                                     int N) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  __shared__ float red[8][256 + 8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = blockIdx.x * 256 + lane * 8;
  const int m0 = blockIdx.y * 128;
  const int m1 = min(M, m0 + 128);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (col < N) {
#pragma unroll 4
    for (int m = m0 + warp; m < m1; m += 8) {
      const uint4 u = *reinterpret_cast<const uint4*>(x + static_cast<int64_t>(m) * ld + col);
      float2 t;
      t = unpack_bf16x2(u.x); acc[0] += t.x; acc[1] += t.y;
      t = unpack_bf16x2(u.y); acc[2] += t.x; acc[3] += t.y;
      t = unpack_bf16x2(u.z); acc[4] += t.x; acc[5] += t.y;
      t = unpack_bf16x2(u.w); acc[6] += t.x; acc[7] += t.y;
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[warp][lane * 8 + j] = acc[j];
  __syncthreads();
  const int c = threadIdx.x;           // 256 threads <-> 256 columns
  if (blockIdx.x * 256 + c < N) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][c];
    atomicAdd(out + blockIdx.x * 256 + c, s);
  }
}

// ------------------------------------------------------------------------------------------------
// small elementwise helpers
// ------------------------------------------------------------------------------------------------
__global__ void dropout_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int64_t n, DropCfg dc_in) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  const DropCfg dc = drop_resolve(dc_in);   // seed + device-side offset (read after the wait)
  pdl_trigger();
  const int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
  if (i >= n) return;
  const uint4 u = *reinterpret_cast<const uint4*>(x + i);
  float f[8];
  float2 t;
  t = unpack_bf16x2(u.x); f[0] = t.x; f[1] = t.y;
  t = unpack_bf16x2(u.y); f[2] = t.x; f[3] = t.y;
  t = unpack_bf16x2(u.z); f[4] = t.x; f[5] = t.y;
  t = unpack_bf16x2(u.w); f[6] = t.x; f[7] = t.y;
#pragma unroll
  for (int j = 0; j < 8; j += 4) {
    float m[4];
    dropout_mult4(dc.seed, static_cast<uint64_t>(i + j), dc.thresh, dc.inv_keep, m);
#pragma unroll
    for (int t = 0; t < 4; ++t) f[j + t] *= m[t];
  }
  uint4 o;
  o.x = pack_bf16x2(f[0], f[1]); o.y = pack_bf16x2(f[2], f[3]);
  o.z = pack_bf16x2(f[4], f[5]); o.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(y + i) = o;
}

// dx = dy * gelu'(u)  (backward of the MLM-head transform activation, transformers.py:486-495)
__global__ void gelu_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ u,
                                __nv_bfloat16* __restrict__ dx, int64_t n8) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= n8) return;
  const uint4 a = reinterpret_cast<const uint4*>(dy)[t], b = reinterpret_cast<const uint4*>(u)[t];
  const uint32_t av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
  uint32_t o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 g = unpack_bf16x2(av[j]), x = unpack_bf16x2(bv[j]);
    o[j] = pack_bf16x2(g.x * gelu_erf_grad(x.x), g.y * gelu_erf_grad(x.y));
  }
  reinterpret_cast<uint4*>(dx)[t] = make_uint4(o[0], o[1], o[2], o[3]);
}

// out[r, 0:cpad] (bf16) = in[r, 0:c] (fp32) zero-padded ; used for dlogits -> padded classifier grad
__global__ void pad_cast_kernel(const float* __restrict__ in, int64_t in_ld, __nv_bfloat16* __restrict__ out, int rows,
                                int c, int cpad) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<int64_t>(rows) * cpad) return;
  const int r = static_cast<int>(i / cpad), j = static_cast<int>(i - static_cast<int64_t>(r) * cpad);
  out[i] = __float2bfloat16(j < c ? in[static_cast<int64_t>(r) * in_ld + j] : 0.0f);
}

// fp32 -> bf16 (weight packing), optional per-row scale (FrozenBN fold: row = element / row_len)
__global__ void cast_scale_kernel(const float* __restrict__ in, const float* __restrict__ rowscale, int64_t row_len,
                                  __nv_bfloat16* __restrict__ out, int64_t n) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  const int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (i >= n) return;
  if (i + 4 <= n) {
    const float4 v = *reinterpret_cast<const float4*>(in + i);
    float s0 = 1.f, s1 = 1.f, s2 = 1.f, s3 = 1.f;
    if (rowscale) {
      s0 = rowscale[i / row_len]; s1 = rowscale[(i + 1) / row_len];
      s2 = rowscale[(i + 2) / row_len]; s3 = rowscale[(i + 3) / row_len];
    }
    uint2 o;
    o.x = pack_bf16x2(v.x * s0, v.y * s1);
    o.y = pack_bf16x2(v.z * s2, v.w * s3);
    *reinterpret_cast<uint2*>(out + i) = o;
  } else {
    for (int64_t k = i; k < n; ++k) out[k] = __float2bfloat16(in[k] * (rowscale ? rowscale[k / row_len] : 1.f));
  }
}

// bf16 -> fp32 (gradients back from the bf16 wire format of the data-parallel exchange)
__global__ void cast_bf16_f32_kernel(const __nv_bfloat16* __restrict__ in, float* __restrict__ out, int64_t n) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  const int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
  if (i >= n) return;
  if (i + 8 <= n) {
    const uint4 u = *reinterpret_cast<const uint4*>(in + i);
    const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    *reinterpret_cast<float4*>(out + i) = make_float4(a.x, a.y, b.x, b.y);
    *reinterpret_cast<float4*>(out + i + 4) = make_float4(c.x, c.y, d.x, d.y);
  } else {
    for (int64_t k = i; k < n; ++k) out[k] = __bfloat162float(in[k]);
  }
}

// all conv weights of the backbone in ONE launch: segment g (blockIdx.y) = one conv's KRSC block, scaled per output row
__global__ void cast_scale_segments_kernel(const float* __restrict__ master, __nv_bfloat16* __restrict__ packed,
                                           const int64_t* __restrict__ seg /*[nseg][4]: offset, numel, row_len, scale_off (-1: none)*/,
                                           const float* __restrict__ scales) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  const int64_t* sg = seg + 4 * blockIdx.y;
  const int64_t off = sg[0], n = sg[1], row_len = sg[2], soff = sg[3];
  for (int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 4; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x * 4) {
    if (i + 4 <= n) {
      const float4 v = *reinterpret_cast<const float4*>(master + off + i);
      float s0 = 1.f, s1 = 1.f, s2 = 1.f, s3 = 1.f;
      if (soff >= 0) {
        s0 = scales[soff + i / row_len]; s1 = scales[soff + (i + 1) / row_len];
        s2 = scales[soff + (i + 2) / row_len]; s3 = scales[soff + (i + 3) / row_len];
      }
      uint2 o;
      o.x = pack_bf16x2(v.x * s0, v.y * s1);
      o.y = pack_bf16x2(v.z * s2, v.w * s3);
      *reinterpret_cast<uint2*>(packed + off + i) = o;
    } else {
      for (int64_t k = i; k < n; ++k) packed[off + k] = __float2bfloat16(master[off + k] * (soff >= 0 ? scales[soff + k / row_len] : 1.f));
    }
  }
}

}  // namespace cb

// ================================================================================================
// C ABI
// ================================================================================================
using namespace cb;

extern "C" {

int cb_layernorm_fwd(const void* x, const float* gamma, const float* beta, void* y, float* stats, int m, int hidden,
                     float eps, void* stream) {
  CB_REQUIRE(hidden == HID, "cb_layernorm_fwd: hidden size %d unsupported (built for %d)", hidden, HID);
  CB_REQUIRE(x && gamma && beta && y && m > 0, "cb_layernorm_fwd: bad arguments");
  launch_k(ln_fwd_kernel, ceil_div(m, ROWS_PER_BLOCK), 128, 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(x), gamma, beta, static_cast<__nv_bfloat16*>(y), stats, m, eps);
  return check_launch("cb_layernorm_fwd");
}

int cb_layernorm_bwd(const void* dy, const void* x, const float* stats, const float* gamma, void* dx, void* dx_drop,
                     float* dgamma, float* dbeta, float* dbias_drop, int m, int hidden, float dropout_p,
                     uint64_t dropout_seed, void* stream) {
  CB_REQUIRE(hidden == HID, "cb_layernorm_bwd: hidden size %d unsupported", hidden);
  CB_REQUIRE(dy && x && stats && gamma && dx && m > 0, "cb_layernorm_bwd: bad arguments");
  // the dgamma / dbeta / dbias atomics contend once per block and column: a few rows per warp, not one
  const int blocks = max(1, min(ceil_div(m, ROWS_PER_BLOCK), 132 * 2));   // two CTAs per H100 SM
  launch_k(ln_bwd_kernel, blocks, 128, 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(dy), static_cast<const __nv_bfloat16*>(x), stats, gamma,
      static_cast<__nv_bfloat16*>(dx), static_cast<__nv_bfloat16*>(dx_drop), dgamma, dbeta, dbias_drop, m,
      make_drop(dropout_p, dropout_seed));
  return check_launch("cb_layernorm_bwd");
}

int cb_embed_text_fwd(const int64_t* ids, const float* word, const float* pos, const float* type0, const float* gamma,
                      const float* beta, void* out, float* stats, int nseq, int lt, int l, int vocab, int hidden,
                      float eps, float dropout_p, uint64_t seed, void* stream) {
  CB_REQUIRE(hidden == HID, "cb_embed_text_fwd: hidden size %d unsupported", hidden);
  CB_REQUIRE(ids && word && pos && type0 && out && stats && nseq > 0 && lt > 0 && l >= lt, "cb_embed_text_fwd: bad arguments");
  launch_k(embed_text_fwd_kernel, ceil_div(static_cast<int64_t>(nseq) * lt, ROWS_PER_BLOCK), 128, 0, static_cast<cudaStream_t>(stream), 
      ids, word, pos, type0, gamma, beta, static_cast<__nv_bfloat16*>(out), stats, nseq, lt, l, vocab, eps,
      make_drop(dropout_p, seed));
  return check_launch("cb_embed_text_fwd");
}

int cb_embed_text_bwd(const void* dh, const int64_t* ids, const float* word, const float* pos, const float* type0,
                      const float* gamma, const float* stats, float* dword, float* dpos, float* dtype0, float* dgamma,
                      float* dbeta, int nseq, int lt, int l, int vocab, int hidden, float dropout_p, uint64_t seed,
                      void* stream) {
  CB_REQUIRE(hidden == HID, "cb_embed_text_bwd: hidden size %d unsupported", hidden);
  CB_REQUIRE(dh && ids && dword && dpos && dtype0 && dgamma && dbeta, "cb_embed_text_bwd: bad arguments");
  CB_REQUIRE(nseq > 0 && lt > 0 && lt <= 65535, "cb_embed_text_bwd: bad sizes");
  const int per_pos = max(1, min(ceil_div(nseq, 2 * ROWS_PER_BLOCK), 32));      // two (up to five at 640 sequences) rows per warp
  launch_k(embed_text_bwd_kernel, dim3(per_pos, lt), 128, 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(dh), ids, word, pos, type0, gamma, stats, dword, dpos, dtype0, dgamma, dbeta,
      nseq, lt, l, vocab, make_drop(dropout_p, seed));
  return check_launch("cb_embed_text_bwd");
}

int cb_embed_visual_fwd(const void* grid, const int32_t* seq2vid, int n_ex, const float* rowemb, const float* colemb,
                        const float* type0, const float* gamma, const float* beta, void* out, float* stats, int nseq,
                        int t, int gh, int gw, int lt, int l, int hidden, float eps, float dropout_p, uint64_t seed,
                        void* stream) {
  CB_REQUIRE(hidden == HID, "cb_embed_visual_fwd: hidden size %d unsupported", hidden);
  CB_REQUIRE(grid && out && stats && nseq > 0 && t > 0 && gh > 0 && gw > 0 && l == lt + gh * gw, "cb_embed_visual_fwd: bad arguments");
  CB_REQUIRE(seq2vid || n_ex > 0, "cb_embed_visual_fwd: need seq2vid or uniform n_ex");
  launch_k(embed_visual_fwd_kernel, ceil_div(static_cast<int64_t>(nseq) * gh * gw, ROWS_PER_BLOCK), 128, 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(grid), seq2vid, n_ex, rowemb, colemb, type0, gamma, beta,
      static_cast<__nv_bfloat16*>(out), stats, nseq, t, gh, gw, lt, l, eps, make_drop(dropout_p, seed));
  return check_launch("cb_embed_visual_fwd");
}

int cb_embed_visual_bwd(const void* dh, const void* grid, const int32_t* seq2vid, const int32_t* vid_start, int n_ex,
                        const float* rowemb, const float* colemb, const float* type0, const float* gamma,
                        const float* stats, float* dv_tmp, void* dgrid, float* drow, float* dcol, float* dtype0,
                        float* dgamma, float* dbeta, int nseq, int nvid, int t, int gh, int gw, int lt, int l, int hidden,
                        float dropout_p, uint64_t seed, void* stream) {
  CB_REQUIRE(hidden == HID, "cb_embed_visual_bwd: hidden size %d unsupported", hidden);
  CB_REQUIRE(dh && grid && dv_tmp && drow && dcol && dtype0 && dgamma && dbeta, "cb_embed_visual_bwd: bad arguments");
  CB_REQUIRE((seq2vid && vid_start) || n_ex > 0, "cb_embed_visual_bwd: need seq2vid+vid_start or uniform n_ex");
  const int Lv = gh * gw;
  CB_REQUIRE(Lv <= 65535, "cb_embed_visual_bwd: grid of %d cells unsupported", Lv);
  const int per_pos = max(1, min(ceil_div(nseq, 2 * ROWS_PER_BLOCK), 32));
  launch_k(embed_visual_bwd_kernel, dim3(per_pos, Lv), 128, 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(dh), static_cast<const __nv_bfloat16*>(grid), seq2vid, n_ex, rowemb, colemb,
      type0, gamma, stats, dv_tmp, drow, dcol, dtype0, dgamma, dbeta, nseq, t, gh, gw, lt, l, make_drop(dropout_p, seed));
  int rc = check_launch("cb_embed_visual_bwd");
  if (rc != CB_OK) return rc;
  if (dgrid) {
    launch_k(embed_visual_bwd_reduce_kernel, ceil_div(static_cast<int64_t>(nvid) * Lv, ROWS_PER_BLOCK), 128, 0, static_cast<cudaStream_t>(stream), dv_tmp, vid_start, n_ex,
                                                                          static_cast<__nv_bfloat16*>(dgrid), nvid, t, Lv);
    rc = check_launch("cb_embed_visual_bwd(reduce)");
  }
  return rc;
}

int cb_colsum(const void* x, int64_t ld, float* out, int m, int n, void* stream) {
  CB_REQUIRE(x && out && m > 0 && n > 0 && n % 8 == 0 && ld % 8 == 0, "cb_colsum: bad arguments (n, ld must be multiples of 8)");
  dim3 grid(ceil_div(n, 256), ceil_div(m, 128));
  launch_k(colsum_kernel, grid, 256, 0, static_cast<cudaStream_t>(stream), static_cast<const __nv_bfloat16*>(x), ld, out, m, n);
  return check_launch("cb_colsum");
}

int cb_dropout(const void* x, void* y, int64_t n, float p, uint64_t seed, void* stream) {
  CB_REQUIRE(x && y && n > 0 && n % 8 == 0, "cb_dropout: n must be a positive multiple of 8");
  launch_k(dropout_kernel, ceil_div(n / 8, 256), 256, 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), n, make_drop(p, seed));
  return check_launch("cb_dropout");
}

int cb_gelu_bwd(const void* dy, const void* u, void* dx, int64_t n, void* stream) {
  CB_REQUIRE(dy && u && dx && n > 0 && n % 8 == 0, "cb_gelu_bwd: n must be a positive multiple of 8");
  launch_k(gelu_bwd_kernel, ceil_div(n / 8, 256), 256, 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(dy), static_cast<const __nv_bfloat16*>(u), static_cast<__nv_bfloat16*>(dx), n / 8);
  return check_launch("cb_gelu_bwd");
}

int cb_pad_cast(const float* in, int64_t in_ld, void* out, int rows, int c, int cpad, void* stream) {
  CB_REQUIRE(in && out && rows > 0 && c > 0 && cpad >= c, "cb_pad_cast: bad arguments");
  launch_k(pad_cast_kernel, ceil_div(static_cast<int64_t>(rows) * cpad, 256), 256, 0, static_cast<cudaStream_t>(stream), 
      in, in_ld, static_cast<__nv_bfloat16*>(out), rows, c, cpad);
  return check_launch("cb_pad_cast");
}

int cb_cast_scale_segments(const float* master, void* packed, const int64_t* segments, int nseg, const float* scales, void* stream) {
  CB_REQUIRE(master && packed && segments && nseg > 0, "cb_cast_scale_segments: bad arguments");
  CB_REQUIRE((reinterpret_cast<uintptr_t>(master) & 15) == 0 && (reinterpret_cast<uintptr_t>(packed) & 7) == 0, "cb_cast_scale_segments: misaligned");
  dim3 grid(64, nseg);
  launch_k(cast_scale_segments_kernel, grid, 256, 0, static_cast<cudaStream_t>(stream), master, static_cast<__nv_bfloat16*>(packed), segments, scales);
  return check_launch("cb_cast_scale_segments");
}

int cb_cast_scale(const float* in, const float* rowscale, int64_t row_len, void* out, int64_t n, void* stream) {
  CB_REQUIRE(in && out && n > 0 && (!rowscale || row_len > 0), "cb_cast_scale: bad arguments");
  CB_REQUIRE((reinterpret_cast<uintptr_t>(in) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0, "cb_cast_scale: misaligned");
  launch_k(cast_scale_kernel, ceil_div(ceil_div(n, 4), 256), 256, 0, static_cast<cudaStream_t>(stream), 
      in, rowscale, row_len, static_cast<__nv_bfloat16*>(out), n);
  return check_launch("cb_cast_scale");
}

int cb_cast_bf16_f32(const void* in, float* out, int64_t n, void* stream) {
  CB_REQUIRE(in && out && n > 0, "cb_cast_bf16_f32: bad arguments");
  CB_REQUIRE((reinterpret_cast<uintptr_t>(in) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0, "cb_cast_bf16_f32: misaligned");
  launch_k(cast_bf16_f32_kernel, ceil_div(ceil_div(n, 8), 256), 256, 0, static_cast<cudaStream_t>(stream), static_cast<const __nv_bfloat16*>(in), out, n);
  return check_launch("cb_cast_bf16_f32");
}

}  // extern "C"
