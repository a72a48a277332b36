// Memory-bound CNN-side kernels for the GridFeat ResNet-50 path (reference call sites:
// src/modeling/grid_feat.py:89-105 -> detectron2 BasicStem / BottleneckBlock / MaxPool, and the
// grid_encoder MaxPool2d+ReLU at grid_feat.py:43-48). Activations are NHWC bf16; every thread moves
// 8 channels with one 128-bit access. All convolution FLOPs run in gemm.cu (wgmma).
#include <cuda_fp16.h>

#include "common.cuh"
#include "host_util.h"

namespace cb {

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  float2 t;
  t = unpack_bf16x2(u.x); f[0] = t.x; f[1] = t.y;
  t = unpack_bf16x2(u.y); f[2] = t.x; f[3] = t.y;
  t = unpack_bf16x2(u.z); f[4] = t.x; f[5] = t.y;
  t = unpack_bf16x2(u.w); f[6] = t.x; f[7] = t.y;
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
  return u;
}

// ------------------------------------------------------------------------------------------------
// Stem im2col: fp32 NCHW RGB (mean-subtracted, 0..255 scale) -> bf16 [N*Ho*Wo, KP] rows of the
// 7x7/s2/p3 patches, K index = (r*7 + s)*3 + c with c in BGR order (the x[:, [2,1,0]] flip of
// grid_feat.py:92-94 is folded into the gather). KP = 152 (147 zero-padded to a multiple of 8).
// ------------------------------------------------------------------------------------------------
// One block per (image, output row): the 7 input rows it needs are staged once in shared memory as PIXEL-INTERLEAVED BGR
// rows [r][x][c] (coalesced planar reads, mean subtraction + bf16 rounding + BGR flip applied there, zero padding
// materialised). With that layout the 21 K-elements (s, c) of tap row r of output pixel ox are ONE contiguous run
// srow[r][6*ox .. 6*ox + 21), so a warp's 16-byte output chunks gather from consecutive shared-memory words (the planar
// layout of the first version cost an ~8-way bank conflict per element and ran at 1.1 TB/s); the 19 x Wo 128-bit patch
// chunks of the output row are written fully coalesced.
template <typename TIn>
__global__ void __launch_bounds__(256) stem_im2col_kernel(const TIn* __restrict__ x, __nv_bfloat16* __restrict__ out, int N, int H, int W,
                                                          int Ho, int Wo, int KP, float m0, float m1, float m2) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  extern __shared__ __nv_bfloat16 srow[];          // [7 rows][W + 6 pixels][3 channels, BGR]
  const int oy = blockIdx.x % Ho, n = blockIdx.x / Ho;
  const int WP = W + 6;
  const int RP = WP * 3;                           // row pitch in elements
  const float mean_rgb[3] = {m0, m1, m2};
  for (int i = threadIdx.x; i < 21 * WP; i += blockDim.x) {
    const int xp = i % WP, rp = i / WP;            // rp = r * 3 + plane: consecutive threads read consecutive x of one plane row
    const int plane = rp % 3, r = rp / 3;
    const int iy = oy * 2 - 3 + r, ix = xp - 3;
    float v = 0.f;
    if (iy >= 0 && iy < H && ix >= 0 && ix < W)
      v = static_cast<float>(x[((static_cast<int64_t>(n) * 3 + plane) * H + iy) * W + ix]) - mean_rgb[plane];
    srow[r * RP + xp * 3 + (2 - plane)] = __float2bfloat16(v);     // BGR channel c is RGB plane 2-c
  }
  __syncthreads();
  const int chunks = KP / 8;
  __nv_bfloat16* orow = out + (static_cast<int64_t>(n) * Ho + oy) * Wo * KP;
  for (int i = threadIdx.x; i < Wo * chunks; i += blockDim.x) {
    const int chunk = i % chunks, ox = i / chunks;
    const int k0 = chunk * 8;
    int r = k0 / 21, off = k0 - r * 21;            // K index k = r * 21 + (s * 3 + c)
    const __nv_bfloat16* src = srow + r * RP + ox * 6;
    __align__(16) __nv_bfloat16 v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      v[j] = (k0 + j < 147) ? src[off] : __float2bfloat16(0.f);
      if (++off == 21) { off = 0; src += RP; }
    }
    *reinterpret_cast<uint4*>(orow + static_cast<int64_t>(ox) * KP + chunk * 8) = *reinterpret_cast<const uint4*>(v);
  }
}

// ------------------------------------------------------------------------------------------------
// Stem without an im2col buffer: space-to-depth(2) of the zero-padded frame.
//   S[n, Y, X, (dy*2 + dx)*4 + c] = padded[n, c(BGR), 2Y + dy, 2X + dx],  c = 3 is a zero lane, padded = 3 zero rows / columns
//   on the top / left (and whatever is needed bottom / right), Y < Ho + 3, X < Wo + 3.
// The 7x7/s2/p3 conv, its kernel zero-extended to 8x8, is then a 4-row-tap contraction: tap r' of output pixel (oy, ox) is
// the 64 CONTIGUOUS bf16 of S pixels (oy + r', ox .. ox + 3), i.e. row (m + r'*(Wo+3)) of a matrix whose rows OVERLAP
// (row pitch = 16 elements, row length 64): one TMA tensor map, four row-shifted K-slabs, exactly like the 3x3 convs.
// `ld` = 16 writes S itself (54 MB per 128 frames instead of the 488 MB patch matrix); `ld` = 64 writes every row's
// 4-pixel window explicitly (for drivers that reject overlapping tensor-map rows).
// ------------------------------------------------------------------------------------------------
template <typename TIn>
__global__ void __launch_bounds__(256) stem_s2d_kernel(const TIn* __restrict__ x, __nv_bfloat16* __restrict__ out, int N, int H, int W,
                                                       int Hs, int Ws, int ld, float m0, float m1, float m2) {
  pdl_wait();
  pdl_trigger();
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t total = static_cast<int64_t>(N) * Hs * Ws;
  if (t >= total) return;
  const int X = static_cast<int>(t % Ws), Y = static_cast<int>((t / Ws) % Hs);
  const int n = static_cast<int>(t / (static_cast<int64_t>(Ws) * Hs));
  const float mean_bgr[3] = {m2, m1, m0};
  __align__(16) __nv_bfloat16 v[16];
#pragma unroll
  for (int dy = 0; dy < 2; ++dy)
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      const int iy = 2 * Y + dy - 3, ix = 2 * X + dx - 3;
      const bool in = iy >= 0 && iy < H && ix >= 0 && ix < W;
#pragma unroll
      for (int c = 0; c < 3; ++c) {      // BGR channel c is RGB plane 2-c (the flip of grid_feat.py:92-94)
        float f = 0.f;
        if (in) f = static_cast<float>(x[((static_cast<int64_t>(n) * 3 + (2 - c)) * H + iy) * W + ix]) - mean_bgr[c];
        v[(dy * 2 + dx) * 4 + c] = __float2bfloat16(f);
      }
      v[(dy * 2 + dx) * 4 + 3] = __float2bfloat16(0.f);
    }
  const uint4 lo = *reinterpret_cast<const uint4*>(v), hi = *reinterpret_cast<const uint4*>(v + 8);
  if (ld == 16) {
    uint4* o = reinterpret_cast<uint4*>(out + t * 16);
    o[0] = lo; o[1] = hi;
  } else {                                // row (n, Y, X - j) holds this pixel in its j-th 16-channel slot
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (X - j < 0) continue;
      uint4* o = reinterpret_cast<uint4*>(out + (t - j) * 64 + j * 16);
      o[0] = lo; o[1] = hi;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Frame resize + pad of the data pipeline (src/datasets/data_utils.py:202-234 ImageResize = F.interpolate(mode="bilinear",
// align_corners=False) to (nh, nw) with the longer side = max_size, :136-160 ImagePad = F.pad with zeros at the bottom / right
// up to max_size x max_size; dataset_base.py:191-195). NCHW in (uint8 or fp32), fp32 NCHW out [n, c, S, S].
// Source coordinate of output pixel o: max(0, (o + 0.5) * in / out - 0.5) (ATen area_pixel_compute_source_index).
// ------------------------------------------------------------------------------------------------
// The source taps of output pixel (oy, ox) of an H x W frame (sh = H / nh, sw = W / nw in fp32): rows y0 <= y1 with weights
// 1 - ly and ly, columns alike. At the top / left edge the coordinate clamps to 0, so ly = 0 and y0 takes weight 1; at the
// bottom / right y1 = y0 = H - 1 and the two weights land on one pixel. cb_resize_pad and its adjoint both call this, so they
// agree on every tap and weight. (The two axes stay in one function: with them written in this order resize_pad_kernel
// compiles to the same instructions as when it carried these lines itself.)
__device__ __forceinline__ void resize_taps(int oy, int ox, float sh, float sw, int H, int W, int& y0, int& x0, int& y1, int& x1,
                                            float& ly, float& lx) {
  const float fy = fmaxf((oy + 0.5f) * sh - 0.5f, 0.f), fx = fmaxf((ox + 0.5f) * sw - 0.5f, 0.f);
  y0 = min(static_cast<int>(fy), H - 1), x0 = min(static_cast<int>(fx), W - 1);
  y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
  ly = fy - y0, lx = fx - x0;
}

// One axis of resize_taps (the other axis' results are unused and compiled away).
__device__ __forceinline__ void resize_taps_1d(int o, float scale, int n, int& i0, int& i1, float& l) {
  int j0, j1;
  float m;
  resize_taps(o, o, scale, scale, n, n, i0, j0, i1, j1, l, m);
}

template <typename TIn>
__global__ void __launch_bounds__(256) resize_pad_kernel(const TIn* __restrict__ x, float* __restrict__ y, int NC, int H, int W, int nh, int nw,
                                                         int S, float sh, float sw) {
  pdl_wait();
  pdl_trigger();
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<int64_t>(NC) * S * S) return;
  const int ox = static_cast<int>(t % S), oy = static_cast<int>((t / S) % S);
  const int64_t plane = t / (static_cast<int64_t>(S) * S);
  float v = 0.f;
  if (oy < nh && ox < nw) {
    int y0, x0, y1, x1;
    float ly, lx;
    resize_taps(oy, ox, sh, sw, H, W, y0, x0, y1, x1, ly, lx);
    const TIn* p = x + plane * H * W;
    const float a = static_cast<float>(p[static_cast<int64_t>(y0) * W + x0]), b = static_cast<float>(p[static_cast<int64_t>(y0) * W + x1]);
    const float c = static_cast<float>(p[static_cast<int64_t>(y1) * W + x0]), d = static_cast<float>(p[static_cast<int64_t>(y1) * W + x1]);
    v = (1.f - ly) * ((1.f - lx) * a + lx * b) + ly * ((1.f - lx) * c + lx * d);
  }
  y[t] = v;
}

// The output indices o in [0, n_out) whose taps include input index i: those with i0(o) in {i - 1, i}. i0 does not decrease with
// o, so they form one range [lo, hi] (lo > hi: none). Start from the real-valued inverse of (o + 0.5) * scale - 0.5 and correct
// it against resize_taps itself, so that fp32 rounding and the edge clamps cannot put a tap outside the range.
__device__ __forceinline__ int2 resize_tap_range(int i, float scale, float inv_scale, int n_in, int n_out) {
  auto first = [&](int o) {
    int i0, i1;
    float l;
    resize_taps_1d(o, scale, n_in, i0, i1, l);
    return i0;
  };
  int lo = min(max(static_cast<int>(ceilf((i - 0.5f) * inv_scale - 0.5f)), 0), n_out);
  while (lo > 0 && first(lo - 1) >= i - 1) --lo;
  while (lo < n_out && first(lo) < i - 1) ++lo;
  int hi = min(max(static_cast<int>(ceilf((i + 1.5f) * inv_scale - 0.5f)) - 1, -1), n_out - 1);
  while (hi < n_out - 1 && first(hi + 1) <= i) ++hi;
  while (hi >= 0 && first(hi) > i) --hi;
  return make_int2(lo, hi);
}

// Adjoint of resize_pad_kernel in gather form: dx[y, x] = sum over the output rows oy that tap y, in ascending order, of
// w_y(oy) * (sum over the output columns ox that tap x, ascending, of w_x(ox) * dy[oy, ox]), with the forward's weights (1 - l on
// the first tap, l on the second, both when they land on one pixel). The pad region (oy >= nh or ox >= nw) taps nothing. One
// writer per element, fp32, a fixed order: the same bits on every run. A CTA covers a 32 x 32 tile of one plane (a warp per row,
// 4 rows per thread); the output ranges of its rows and columns, and the taps of those outputs, are computed once into shared
// memory (recomputed instead when an extreme upscale makes a tile's span longer than the table).
constexpr int kResizeBwdTile = 32;
constexpr int kResizeBwdTaps = 512;

__global__ void __launch_bounds__(256) resize_pad_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, int H, int W, int nh, int nw,
                                                             int S, float sh, float sw, float inv_sh, float inv_sw, int tiles_w, int tiles_h,
                                                             int accumulate) {
  __shared__ int2 col_range[kResizeBwdTile], row_range[kResizeBwdTile];
  __shared__ int2 xtap[kResizeBwdTaps], ytap[kResizeBwdTaps];     // {i0, l as bits} of output column ox_lo + j / row oy_lo + j
  pdl_wait();
  pdl_trigger();
  const int tile = blockIdx.x % (tiles_w * tiles_h);
  const int64_t plane = blockIdx.x / (tiles_w * tiles_h);
  const int cx = (tile % tiles_w) * kResizeBwdTile, cy = (tile / tiles_w) * kResizeBwdTile;
  const int ncols = min(kResizeBwdTile, W - cx), nrows = min(kResizeBwdTile, H - cy);
  const int tid = threadIdx.x;
  if (tid < kResizeBwdTile)
    col_range[tid] = tid < ncols ? resize_tap_range(cx + tid, sw, inv_sw, W, nw) : make_int2(0, -1);
  else if (tid >= 128 && tid < 128 + kResizeBwdTile)
    row_range[tid - 128] = tid - 128 < nrows ? resize_tap_range(cy + tid - 128, sh, inv_sh, H, nh) : make_int2(0, -1);
  __syncthreads();
  // every column's range lies inside [first column's lo, last column's hi] (both ends are monotone); rows alike
  const int ox_lo = col_range[0].x, nx = col_range[ncols - 1].y - ox_lo + 1;
  const int oy_lo = row_range[0].x, ny = row_range[nrows - 1].y - oy_lo + 1;
  const bool xtab = nx <= kResizeBwdTaps, ytab = ny <= kResizeBwdTaps;
  for (int j = tid; j < kResizeBwdTaps && (j < nx || j < ny); j += blockDim.x) {
    int i0, i1;
    float l;
    if (xtab && j < nx) {
      resize_taps_1d(ox_lo + j, sw, W, i0, i1, l);
      xtap[j] = make_int2(i0, __float_as_int(l));
    }
    if (ytab && j < ny) {
      resize_taps_1d(oy_lo + j, sh, H, i0, i1, l);
      ytap[j] = make_int2(i0, __float_as_int(l));
    }
  }
  __syncthreads();
  const int col = tid % kResizeBwdTile;
  if (col >= ncols) return;
  const int x = cx + col;
  const int2 xr = col_range[col];
  const float* plane_dy = dy + plane * S * S;
  for (int row = tid / kResizeBwdTile; row < nrows; row += 256 / kResizeBwdTile) {
    const int y = cy + row;
    const int2 yr = row_range[row];
    float acc = 0.f;
    for (int oy = yr.x; oy <= yr.y; ++oy) {
      int y0, y1;
      float ly;
      if (ytab) {
        const int2 e = ytap[oy - oy_lo];
        y0 = e.x, ly = __int_as_float(e.y), y1 = min(y0 + 1, H - 1);
      } else {
        resize_taps_1d(oy, sh, H, y0, y1, ly);
      }
      const float* dy_row = plane_dy + static_cast<int64_t>(oy) * S;
      float r = 0.f;
      for (int ox = xr.x; ox <= xr.y; ++ox) {
        int x0, x1;
        float lx;
        if (xtab) {
          const int2 e = xtap[ox - ox_lo];
          x0 = e.x, lx = __int_as_float(e.y), x1 = min(x0 + 1, W - 1);
        } else {
          resize_taps_1d(ox, sw, W, x0, x1, lx);
        }
        const float g = __ldg(dy_row + ox);
        if (x0 == x) r += (1.f - lx) * g;
        if (x1 == x) r += lx * g;
      }
      if (y0 == y) acc += (1.f - ly) * r;
      if (y1 == y) acc += ly * r;
    }
    float* o = dx + (plane * H + y) * W + x;
    *o = accumulate ? *o + acc : acc;
  }
}

// ATen's max-pool update (max_pool2d_with_indices): a value replaces the running maximum when it is larger or NaN, so NaN
// propagates (fmaxf would drop it) and, among equal maxima, the first one in window order stays
__device__ __forceinline__ bool pool_takes(float v, float best) { return v > best || v != v; }

// 3x3 stride-2 pad-1 max pool, NHWC
__global__ void maxpool3x3s2_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int N, int H, int W,
                                    int C, int Ho, int Wo, int64_t row_pitch /* pixels */, int64_t img_pitch /* pixels */) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  const int c8n = C / 8;
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<int64_t>(N) * Ho * Wo * c8n) return;
  const int c8 = static_cast<int>(t % c8n);
  const int64_t pix = t / c8n;
  const int ox = static_cast<int>(pix % Wo), oy = static_cast<int>((pix / Wo) % Ho);
  const int n = static_cast<int>(pix / (static_cast<int64_t>(Wo) * Ho));
  float m[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) m[j] = -INFINITY;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const int iy = oy * 2 - 1 + r;
    if (iy < 0 || iy >= H) continue;
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      const int ix = ox * 2 - 1 + s;
      if (ix < 0 || ix >= W) continue;
      float f[8];
      unpack8(*reinterpret_cast<const uint4*>(x + (static_cast<int64_t>(n) * img_pitch + iy * row_pitch + ix) * C + c8 * 8), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) m[j] = pool_takes(f[j], m[j]) ? f[j] : m[j];
    }
  }
  *reinterpret_cast<uint4*>(y + pix * C + c8 * 8) = pack8(m);
}

// Backward of the 3x3 stride-2 pad-1 max pool above fused with the stem's ReLU' (BasicStem relu_ -> max_pool2d(3, 2, 1)), in
// gather form: every input element visits the <= 4 windows that contain it, recomputes each window's arg-max with the forward's
// rule (pool_takes: first maximum in window order, last NaN; an all -inf window picks its first pixel, as ATen), sums in fp32 the
// window gradients that pick it (oy, then ox ascending), rounds once and applies ReLU' = (x > 0). One writer per element.
// x: the pool input on its (row_pitch, img_pitch) grid; dy: compact [N, Ho, Wo, C]; dx: compact [N, H, W, C].
__global__ void maxpool3x3s2_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                        __nv_bfloat16* __restrict__ dx, int N, int H, int W, int C, int Ho, int Wo, int64_t row_pitch,
                                        int64_t img_pitch) {
  pdl_wait();
  pdl_trigger();
  const int c8n = C / 8;
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<int64_t>(N) * H * W * c8n) return;
  const int c8 = static_cast<int>(t % c8n);
  const int64_t pix = t / c8n;
  const int xx = static_cast<int>(pix % W), yy = static_cast<int>((pix / W) % H);
  const int n = static_cast<int>(pix / (static_cast<int64_t>(W) * H));
  const __nv_bfloat16* xn = x + static_cast<int64_t>(n) * img_pitch * C + c8 * 8;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  // windows (oy, ox) with 2 oy - 1 <= yy <= 2 oy + 1
  const int oy0 = yy / 2, oy1 = min((yy + 1) / 2, Ho - 1);
  const int ox0 = xx / 2, ox1 = min((xx + 1) / 2, Wo - 1);
  for (int oy = oy0; oy <= oy1; ++oy)
    for (int ox = ox0; ox <= ox1; ++ox) {
      float best[8];
      int arg[8];
      const int ry0 = max(2 * oy - 1, 0), rx0 = max(2 * ox - 1, 0);
#pragma unroll
      for (int j = 0; j < 8; ++j) { best[j] = -INFINITY; arg[j] = ry0 * W + rx0; }
      for (int iy = ry0; iy <= min(2 * oy + 1, H - 1); ++iy)
        for (int ix = rx0; ix <= min(2 * ox + 1, W - 1); ++ix) {
          float f[8];
          unpack8(*reinterpret_cast<const uint4*>(xn + (iy * row_pitch + ix) * C), f);
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (pool_takes(f[j], best[j])) { best[j] = f[j]; arg[j] = iy * W + ix; }
        }
      float g[8];
      unpack8(*reinterpret_cast<const uint4*>(dy + ((static_cast<int64_t>(n) * Ho + oy) * Wo + ox) * C + c8 * 8), g);
      const int me = yy * W + xx;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (arg[j] == me) acc[j] += g[j];
    }
  float a[8];
  unpack8(*reinterpret_cast<const uint4*>(xn + (yy * row_pitch + xx) * C), a);
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = a[j] > 0.f ? acc[j] : 0.f;
  *reinterpret_cast<uint4*>(dx + pix * C + c8 * 8) = pack8(acc);
}

// ------------------------------------------------------------------------------------------------
// Stem input gradient (BasicStem conv1 7x7/s2/p3 of grid_feat.py:92-95, backward to the frames): the transposed convolution
//   dX_bgr[n, c, y, x] = sum_{k, r, s} dc1[n, (y+3-r)/2, (x+3-s)/2, k] * W'[k, (r*7 + s)*3 + c]
// over the taps where both halves are integers inside the conv output, written as fp32 NCHW in RGB order (plane 2 - c).
// Output pixel x = 2i + px takes the taps s = px^1, px^1 + 2, ... at dc1 column ox = i + o, o = (px + 3 - s) / 2 in {-1, 0, 1, 2}
// (px = 0: s = 5, 3, 1; px = 1: s = 6, 4, 2, 0), rows alike. So for one output row y, one 16-pixel tile of i and one kernel row r,
// the four dc1 tiles at column offsets o = -1 .. 2 each feed one m16n8k16 product per 16-channel k-step for both phases
// (o = 2 only px = 1): A = 16 dc1 pixels x 16 channels, B = 16 channels x 8 (BGR + 5 zero columns), fp32 accumulators D0 / D1
// for px = 0 / 1. A comes straight from global memory (L1 / L2: neighbouring warps read the same dc1 rows) with the k index
// permuted so that lane (g, t) reads channels 16t .. 16t+15 of its two rows as two 16-byte loads: mma k = 2t, 2t+1, 2t+8, 2t+9 of
// k-step q are channels 16t + 4q + 0, 1, 2, 3 (the contraction is order-free in k; B uses the same permutation). B fragments of
// all 49 taps live in shared memory (18.8 KB). Every output element has one writer and a fixed summation order (r, o, q).
// One warp per (frame, output row, 16-pixel tile), eight warps per CTA; CTAs stride over the tiles.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

constexpr int kStemDgradWarps = 8;
constexpr int kStemTaps = 49;

__global__ void __launch_bounds__(kStemDgradWarps * 32) stem_dgrad_kernel(const __nv_bfloat16* __restrict__ dc1,
                                                                          const __nv_bfloat16* __restrict__ w, int w_ld,
                                                                          float* __restrict__ dx, int N, int H, int W, int Ho, int Wo,
                                                                          int tiles) {
  // B fragments: wf[((tap * 4 + q) * 4 + t) * 3 + g] = {W'[16t+4q+0][tap*3+g], W'[+1]}, {W'[+2], W'[+3]} (bf16 pairs, low = lower k)
  __shared__ uint2 wf[kStemTaps * 4 * 4 * 3];
  pdl_wait();
  pdl_trigger();
  for (int i = threadIdx.x; i < kStemTaps * 4 * 4 * 3; i += blockDim.x) {
    const int g = i % 3, t = (i / 3) % 4, q = (i / 12) % 4, tap = i / 48;
    const int ch = 16 * t + 4 * q, col = tap * 3 + g;
    __nv_bfloat162 p0, p1;
    p0.x = w[(ch + 0) * w_ld + col]; p0.y = w[(ch + 1) * w_ld + col];
    p1.x = w[(ch + 2) * w_ld + col]; p1.y = w[(ch + 3) * w_ld + col];
    wf[i] = make_uint2(*reinterpret_cast<uint32_t*>(&p0), *reinterpret_cast<uint32_t*>(&p1));
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int64_t total = static_cast<int64_t>(N) * H * tiles;
  for (int64_t task = static_cast<int64_t>(blockIdx.x) * kStemDgradWarps + (threadIdx.x >> 5); task < total;
       task += static_cast<int64_t>(gridDim.x) * kStemDgradWarps) {
    const int tile = static_cast<int>(task % tiles);
    const int y = static_cast<int>((task / tiles) % H);
    const int n = static_cast<int>(task / (static_cast<int64_t>(tiles) * H));
    const int i0 = tile * 16;
    float d0[4] = {0.f, 0.f, 0.f, 0.f}, d1[4] = {0.f, 0.f, 0.f, 0.f};
    for (int r = (y + 3) & 1; r < 7; r += 2) {
      const int oy = (y + 3 - r) >> 1;
      if (oy < 0 || oy >= Ho) continue;
      const __nv_bfloat16* row = dc1 + (static_cast<int64_t>(n) * Ho + oy) * Wo * 64 + 16 * t;
#pragma unroll
      for (int o = -1; o <= 2; ++o) {
        uint4 lo[2], hi[2];       // rows g and g + 8 of the tile: channels 16t .. 16t+7 and 16t+8 .. 16t+15
        const int oxg = i0 + g + o, oxh = oxg + 8;
        const uint4 z = make_uint4(0, 0, 0, 0);
        const bool vg = oxg >= 0 && oxg < Wo, vh = oxh >= 0 && oxh < Wo;
        lo[0] = vg ? __ldg(reinterpret_cast<const uint4*>(row + static_cast<int64_t>(oxg) * 64)) : z;
        lo[1] = vg ? __ldg(reinterpret_cast<const uint4*>(row + static_cast<int64_t>(oxg) * 64 + 8)) : z;
        hi[0] = vh ? __ldg(reinterpret_cast<const uint4*>(row + static_cast<int64_t>(oxh) * 64)) : z;
        hi[1] = vh ? __ldg(reinterpret_cast<const uint4*>(row + static_cast<int64_t>(oxh) * 64 + 8)) : z;
        const uint32_t* wg = reinterpret_cast<const uint32_t*>(lo);
        const uint32_t* wh = reinterpret_cast<const uint32_t*>(hi);
        const int s0 = 3 - 2 * o, s1 = 4 - 2 * o;       // px = 0 / px = 1 tap column of this dc1 offset
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint32_t a[4] = {wg[2 * q], wh[2 * q], wg[2 * q + 1], wh[2 * q + 1]};
          if (o <= 1) {
            uint2 b = make_uint2(0, 0);
            if (g < 3) b = wf[(((r * 7 + s0) * 4 + q) * 4 + t) * 3 + g];
            mma_bf16_16816(d0, a, b.x, b.y);
          }
          uint2 b = make_uint2(0, 0);
          if (g < 3) b = wf[(((r * 7 + s1) * 4 + q) * 4 + t) * 3 + g];
          mma_bf16_16816(d1, a, b.x, b.y);
        }
      }
    }
    // D[row][col]: c[0], c[1] = row g, cols 2t, 2t+1; c[2], c[3] = row g+8. col = BGR channel -> RGB plane 2 - col
    if (t < 2) {
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int i = i0 + g + 8 * half;
#pragma unroll
        for (int cc = 0; cc < 2; ++cc) {
          const int c = 2 * t + cc;
          if (c > 2) continue;
          float* o = dx + ((static_cast<int64_t>(n) * 3 + (2 - c)) * H + y) * W;
          if (2 * i < W) o[2 * i] = d0[2 * half + cc];
          if (2 * i + 1 < W) o[2 * i + 1] = d1[2 * half + cc];
        }
      }
    }
  }
}

// stride-2 pixel subsample (input of a stride-2 1x1 conv): y[n, oy, ox] = x[n, 2oy, 2ox]
__global__ void subsample2_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int N, int H, int W,
                                  int C, int Ho, int Wo) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  const int c8n = C / 8;
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<int64_t>(N) * Ho * Wo * c8n) return;
  const int c8 = static_cast<int>(t % c8n);
  const int64_t pix = t / c8n;
  const int ox = static_cast<int>(pix % Wo), oy = static_cast<int>((pix / Wo) % Ho);
  const int n = static_cast<int>(pix / (static_cast<int64_t>(Wo) * Ho));
  *reinterpret_cast<uint4*>(y + pix * C + c8 * 8) =
      *reinterpret_cast<const uint4*>(x + ((static_cast<int64_t>(n) * H + 2 * oy) * W + 2 * ox) * C + c8 * 8);
}

// backward of subsample2 fused with the ReLU mask of the producer of x:
//   dx[n,y,x] = (y,x even ? dsub[n,y/2,x/2] : 0) * (act[n,y,x] > 0)
__global__ void unsubsample2_mask_kernel(const __nv_bfloat16* __restrict__ dsub, const __nv_bfloat16* __restrict__ act,
                                         __nv_bfloat16* __restrict__ dx, int N, int H, int W, int C, int Ho, int Wo) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  const int c8n = C / 8;
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<int64_t>(N) * H * W * c8n) return;
  const int c8 = static_cast<int>(t % c8n);
  const int64_t pix = t / c8n;
  const int xx = static_cast<int>(pix % W), yy = static_cast<int>((pix / W) % H);
  const int n = static_cast<int>(pix / (static_cast<int64_t>(W) * H));
  uint4 o = make_uint4(0, 0, 0, 0);
  if ((yy & 1) == 0 && (xx & 1) == 0) {
    float g[8], a[8];
    unpack8(*reinterpret_cast<const uint4*>(dsub + ((static_cast<int64_t>(n) * Ho + yy / 2) * Wo + xx / 2) * C + c8 * 8), g);
    unpack8(*reinterpret_cast<const uint4*>(act + pix * C + c8 * 8), a);
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] = a[j] > 0.f ? g[j] : 0.f;
    o = pack8(g);
  }
  *reinterpret_cast<uint4*>(dx + pix * C + c8 * 8) = o;
}

// the mask-free form of the above (act == NULL): dx[n,y,x] = (y,x even ? dsub[n,y/2,x/2] : 0). A kernel of its own so that the
// masked one keeps its instructions.
__global__ void unsubsample2_kernel(const __nv_bfloat16* __restrict__ dsub, __nv_bfloat16* __restrict__ dx, int N, int H, int W,
                                    int C, int Ho, int Wo) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  const int c8n = C / 8;
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<int64_t>(N) * H * W * c8n) return;
  const int c8 = static_cast<int>(t % c8n);
  const int64_t pix = t / c8n;
  const int xx = static_cast<int>(pix % W), yy = static_cast<int>((pix / W) % H);
  const int n = static_cast<int>(pix / (static_cast<int64_t>(W) * H));
  uint4 o = make_uint4(0, 0, 0, 0);
  if ((yy & 1) == 0 && (xx & 1) == 0)
    o = *reinterpret_cast<const uint4*>(dsub + ((static_cast<int64_t>(n) * Ho + yy / 2) * Wo + xx / 2) * C + c8 * 8);
  *reinterpret_cast<uint4*>(dx + pix * C + c8 * 8) = o;
}

// ---- cb_nhwc_intake: a strided (n, c, h, w) tensor into the engine's NHWC bf16 layout, optionally masked by (act > 0) ----
template <typename T>
__device__ __forceinline__ float intake_ld(const T* p);
template <>
__device__ __forceinline__ float intake_ld<float>(const float* p) { return __ldg(p); }
template <>
__device__ __forceinline__ float intake_ld<__half>(const __half* p) { return __half2float(__ldg(p)); }
template <>
__device__ __forceinline__ float intake_ld<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(__ldg(p)); }

// 8 contiguous channels as fp32
__device__ __forceinline__ void intake_ld8(const float* p, float (&v)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void intake_ld8(const __nv_bfloat16* p, float (&v)[8]) { unpack8(__ldg(reinterpret_cast<const uint4*>(p)), v); }
__device__ __forceinline__ void intake_ld8(const __half* p, float (&v)[8]) {
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = __half22float2(h2[j]);
    v[2 * j] = f.x;
    v[2 * j + 1] = f.y;
  }
}

// the engine row of pixel (n, y, x): compact, or the interior of the zero-bordered [n, h+2, w+2] grid
__device__ __forceinline__ int64_t intake_row(int64_t pix, int H, int W, bool bordered) {
  if (!bordered) return pix;
  const int64_t xx = pix % W, r = pix / W;
  const int64_t yy = r % H, n = r / H;
  return (n * (H + 2) + yy + 1) * (W + 2) + xx + 1;
}

// 8 channels of one pixel: mask (act > 0 ? v : +0), one rounding to bf16, one 16-byte store
__device__ __forceinline__ void intake_store8(float (&v)[8], const __nv_bfloat16* __restrict__ act, bool act_bordered,
                                              __nv_bfloat16* __restrict__ out, bool out_bordered, int64_t pix, int c, int H, int W,
                                              int C) {
  if (act != nullptr) {
    float a[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(act + intake_row(pix, H, W, act_bordered) * C + c)), a);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = a[j] > 0.f ? v[j] : 0.f;
  }
  *reinterpret_cast<uint4*>(out + intake_row(pix, H, W, out_bordered) * C + c) = pack8(v);
}

// one thread per (pixel, 8 channels). kVec: the 8 channels are contiguous and 16-byte aligned (channels-last input)
template <typename T, bool kVec>
__global__ void nhwc_intake_kernel(const T* __restrict__ x, int64_t sn, int64_t sc, int64_t sh, int64_t sw,
                                   const __nv_bfloat16* __restrict__ act, int act_bordered, __nv_bfloat16* __restrict__ out,
                                   int out_bordered, int N, int C, int H, int W) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  const int c8n = C / 8;
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<int64_t>(N) * H * W * c8n) return;
  const int c = static_cast<int>(t % c8n) * 8;
  const int64_t pix = t / c8n;
  const int64_t xx = pix % W, yy = (pix / W) % H, n = pix / (static_cast<int64_t>(W) * H);
  const T* p = x + n * sn + yy * sh + xx * sw + c * sc;
  float v[8];
  if (kVec) {
    intake_ld8(p, v);
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = intake_ld(p + j * sc);
  }
  intake_store8(v, act, act_bordered, out, out_bordered, pix, c, H, W, C);
}

// contiguous NCHW planes (sw = 1, sh = w, sc = h * w): a 32-channel x 64-pixel tile through shared memory, so that the loads run
// along pixels and the 16-byte stores along channels
constexpr int kIntakeTileP = 64, kIntakeTileC = 32;
template <typename T>
__global__ void __launch_bounds__(256) nhwc_intake_nchw_kernel(const T* __restrict__ x, int64_t sn, const __nv_bfloat16* __restrict__ act,
                                                               int act_bordered, __nv_bfloat16* __restrict__ out, int out_bordered, int C,
                                                               int H, int W) {
  __shared__ float tile[kIntakeTileC][kIntakeTileP + 1];
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  const int64_t hw = static_cast<int64_t>(H) * W;
  const int64_t p0 = static_cast<int64_t>(blockIdx.x) * kIntakeTileP;
  const int c0 = blockIdx.y * kIntakeTileC, n = blockIdx.z;
  const int tp = threadIdx.x % kIntakeTileP, tc = threadIdx.x / kIntakeTileP;     // 64 pixels x 4 channel rows per pass
  const T* xn = x + n * sn;
#pragma unroll
  for (int j = 0; j < kIntakeTileC / 4; ++j) {
    const int c = c0 + tc + 4 * j;
    const int64_t p = p0 + tp;
    tile[tc + 4 * j][tp] = (c < C && p < hw) ? intake_ld(xn + c * hw + p) : 0.f;
  }
  __syncthreads();
  const int op = threadIdx.x / 4, oc = (threadIdx.x % 4) * 8;      // each thread: one pixel, 8 channels
  const int64_t p = p0 + op;
  if (p < hw && c0 + oc < C) {
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = tile[oc + j][op];
    intake_store8(v, act, act_bordered, out, out_bordered, n * hw + p, c0 + oc, H, W, C);
  }
}

template <typename T>
static void launch_intake(const void* xv, int64_t sn, int64_t sc, int64_t sh, int64_t sw, const __nv_bfloat16* act, int act_bordered,
                          __nv_bfloat16* out, int out_bordered, int n, int c, int h, int w, cudaStream_t st) {
  const T* x = static_cast<const T*>(xv);
  const bool aligned = (reinterpret_cast<uintptr_t>(x) & 15) == 0;
  if (sc == 1 && aligned && sn % 8 == 0 && sh % 8 == 0 && sw % 8 == 0) {
    const int64_t total = static_cast<int64_t>(n) * h * w * (c / 8);
    launch_k(nhwc_intake_kernel<T, true>, ceil_div(total, 256), 256, 0, st, x, sn, sc, sh, sw, act, act_bordered, out, out_bordered, n, c,
             h, w);
  } else if (sw == 1 && sh == w && sc == static_cast<int64_t>(h) * w && n <= 65535) {
    const dim3 grid(static_cast<unsigned>(ceil_div(static_cast<int64_t>(h) * w, kIntakeTileP)), ceil_div(c, kIntakeTileC), n);
    launch_k(nhwc_intake_nchw_kernel<T>, grid, 256, 0, st, x, sn, act, act_bordered, out, out_bordered, c, h, w);
  } else {
    const int64_t total = static_cast<int64_t>(n) * h * w * (c / 8);
    launch_k(nhwc_intake_kernel<T, false>, ceil_div(total, 256), 256, 0, st, x, sn, sc, sh, sw, act, act_bordered, out, out_bordered, n,
             c, h, w);
  }
}

// grid_encoder tail: MaxPool2d(2,2) (floor) then ReLU, NHWC compact -> NHWC compact
__global__ void maxpool2x2_relu_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int N, int H,
                                           int W, int C, int Ho, int Wo) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  const int c8n = C / 8;
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<int64_t>(N) * Ho * Wo * c8n) return;
  const int c8 = static_cast<int>(t % c8n);
  const int64_t pix = t / c8n;
  const int ox = static_cast<int>(pix % Wo), oy = static_cast<int>((pix / Wo) % Ho);
  const int n = static_cast<int>(pix / (static_cast<int64_t>(Wo) * Ho));
  float m[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) m[j] = 0.f;  // ReLU folded: max(+0, window max); a window of zeros / -0 gives +0, a NaN gives NaN
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      float f[8];
      unpack8(*reinterpret_cast<const uint4*>(x + ((static_cast<int64_t>(n) * H + 2 * oy + r) * W + 2 * ox + s) * C + c8 * 8), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) m[j] = pool_takes(f[j], m[j]) ? f[j] : m[j];
    }
  *reinterpret_cast<uint4*>(y + pix * C + c8 * 8) = pack8(m);
}

// backward of the above into the zero-bordered ("padded") layout the 3x3 dgrad / wgrad GEMMs read.
// Writes EVERY element of dx_pad [N, H+2, W+2, C] (zeros on the border and on non-argmax pixels).
__global__ void maxpool2x2_relu_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                           __nv_bfloat16* __restrict__ dx_pad, int N, int H, int W, int C, int Ho, int Wo) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  const int c8n = C / 8;
  const int Hp = H + 2, Wp = W + 2;
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<int64_t>(N) * Hp * Wp * c8n) return;
  const int c8 = static_cast<int>(t % c8n);
  const int64_t pix = t / c8n;
  const int xp = static_cast<int>(pix % Wp), yp = static_cast<int>((pix / Wp) % Hp);
  const int n = static_cast<int>(pix / (static_cast<int64_t>(Wp) * Hp));
  uint4 o = make_uint4(0, 0, 0, 0);
  const int yy = yp - 1, xx = xp - 1;
  if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
    const int oy = yy / 2, ox = xx / 2;
    if (oy < Ho && ox < Wo) {
      float best[8];
      int arg[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) { best[j] = -INFINITY; arg[j] = 0; }
#pragma unroll
      for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          float f[8];
          unpack8(*reinterpret_cast<const uint4*>(x + ((static_cast<int64_t>(n) * H + 2 * oy + r) * W + 2 * ox + s) * C + c8 * 8), f);
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (pool_takes(f[j], best[j])) { best[j] = f[j]; arg[j] = r * 2 + s; }  // ATen's arg-max: first maximum, last NaN
        }
      const int me = (yy - 2 * oy) * 2 + (xx - 2 * ox);
      float g[8];
      unpack8(*reinterpret_cast<const uint4*>(dy + ((static_cast<int64_t>(n) * Ho + oy) * Wo + ox) * C + c8 * 8), g);
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] = (arg[j] == me && best[j] > 0.f) ? g[j] : 0.f;   // ReLU' = (max > 0), as every mask here
      o = pack8(g);
    }
  }
  *reinterpret_cast<uint4*>(dx_pad + pix * C + c8 * 8) = o;
}

// y = dy * (act > 0), both compact: ReLU backward where no GEMM epilogue can carry it
__global__ void relu_mask_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ act,
                                 __nv_bfloat16* __restrict__ dx, int64_t n8) {
  pdl_wait();      // PDL: everything above ran while the previous kernel drained; no global access before this
  pdl_trigger();
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= n8) return;
  float g[8], a[8];
  unpack8(reinterpret_cast<const uint4*>(dy)[t], g);
  unpack8(reinterpret_cast<const uint4*>(act)[t], a);
#pragma unroll
  for (int j = 0; j < 8; ++j) g[j] = a[j] > 0.f ? g[j] : 0.f;
  reinterpret_cast<uint4*>(dx)[t] = pack8(g);
}

}  // namespace cb

using namespace cb;

extern "C" {

/* in_dtype: 0 = fp32 (already mean-subtracted: pass mean = 0), 1 = uint8 (mean subtracted here, as
 * ImageNorm does: src/datasets/data_utils.py:256-276). x is NCHW RGB; out is bf16 [n*ho*wo, kp]. */
int cb_stem_im2col(const void* x, int in_dtype, void* out, int n, int h, int w, int kp, float mean_r, float mean_g,
                   float mean_b, void* stream) {
  CB_REQUIRE(x && out && n > 0 && h > 0 && w > 0, "cb_stem_im2col: bad arguments");
  CB_REQUIRE(kp >= 152 && kp % 8 == 0, "cb_stem_im2col: kp must be a multiple of 8 and >= 152");
  const int ho = (h + 6 - 7) / 2 + 1, wo = (w + 6 - 7) / 2 + 1;
  const int smem = 21 * (w + 6) * 2;
  CB_REQUIRE(smem <= 48 * 1024, "cb_stem_im2col: frame width %d too large for the row staging buffer", w);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (in_dtype == 0)
    launch_k(stem_im2col_kernel<float>, n * ho, 256, smem, st, static_cast<const float*>(x), static_cast<__nv_bfloat16*>(out), n, h, w, ho, wo, kp,
                                                         mean_r, mean_g, mean_b);
  else if (in_dtype == 1)
    launch_k(stem_im2col_kernel<uint8_t>, n * ho, 256, smem, st, static_cast<const uint8_t*>(x), static_cast<__nv_bfloat16*>(out), n, h, w, ho, wo,
                                                           kp, mean_r, mean_g, mean_b);
  else
    CB_REQUIRE(false, "cb_stem_im2col: in_dtype must be 0 (fp32) or 1 (uint8)");
  return check_launch("cb_stem_im2col");
}

#define CB_NHWC_CHECK(name) \
  CB_REQUIRE(x && y && n > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0, name ": bad arguments (c must be a multiple of 8)")

int cb_maxpool3x3s2_strided(const void* x, void* y, int n, int h, int w, int c, int64_t row_pitch, int64_t img_pitch, void* stream) {
  CB_NHWC_CHECK("cb_maxpool3x3s2");
  CB_REQUIRE(row_pitch >= w && img_pitch >= static_cast<int64_t>(h) * row_pitch, "cb_maxpool3x3s2: pitches smaller than the image");
  const int ho = (h + 2 - 3) / 2 + 1, wo = (w + 2 - 3) / 2 + 1;
  const int64_t total = static_cast<int64_t>(n) * ho * wo * (c / 8);
  launch_k(maxpool3x3s2_kernel, ceil_div(total, 256), 256, 0, static_cast<cudaStream_t>(stream),
           static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), n, h, w, c, ho, wo, row_pitch, img_pitch);
  return check_launch("cb_maxpool3x3s2");
}

int cb_maxpool3x3s2(const void* x, void* y, int n, int h, int w, int c, void* stream) {
  return cb_maxpool3x3s2_strided(x, y, n, h, w, c, w, static_cast<int64_t>(h) * w, stream);
}

int cb_maxpool3x3s2_bwd_strided(const void* dy, const void* x, void* dx, int n, int h, int w, int c, int64_t row_pitch,
                                int64_t img_pitch, void* stream) {
  CB_REQUIRE(dy && x && dx && n > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0,
             "cb_maxpool3x3s2_bwd: bad arguments (c must be a multiple of 8)");
  CB_REQUIRE(row_pitch >= w && img_pitch >= static_cast<int64_t>(h) * row_pitch, "cb_maxpool3x3s2_bwd: pitches smaller than the image");
  const int ho = (h + 2 - 3) / 2 + 1, wo = (w + 2 - 3) / 2 + 1;
  const int64_t total = static_cast<int64_t>(n) * h * w * (c / 8);
  launch_k(maxpool3x3s2_bwd_kernel, ceil_div(total, 256), 256, 0, static_cast<cudaStream_t>(stream), static_cast<const __nv_bfloat16*>(dy),
           static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(dx), n, h, w, c, ho, wo, row_pitch, img_pitch);
  return check_launch("cb_maxpool3x3s2_bwd");
}

int cb_maxpool3x3s2_bwd(const void* dy, const void* x, void* dx, int n, int h, int w, int c, void* stream) {
  return cb_maxpool3x3s2_bwd_strided(dy, x, dx, n, h, w, c, w, static_cast<int64_t>(h) * w, stream);
}

int cb_stem_dgrad(const void* dc1, const void* w, int w_ld, float* dx, int n, int h, int w_img, void* stream) {
  CB_REQUIRE(dc1 && w && dx && n > 0 && h > 0 && w_img > 0, "cb_stem_dgrad: bad arguments");
  CB_REQUIRE(w_ld >= 147, "cb_stem_dgrad: w_ld must be >= 147 (the 7x7x3 taps of one output channel)");
  CB_REQUIRE((reinterpret_cast<uintptr_t>(dc1) & 15) == 0, "cb_stem_dgrad: dc1 must be 16-byte aligned");
  const int ho = (h - 1) / 2 + 1, wo = (w_img - 1) / 2 + 1;
  const int tiles = ((w_img + 1) / 2 + 15) / 16;
  const int64_t warps = static_cast<int64_t>(n) * h * tiles;
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  const int grid = static_cast<int>(std::min<int64_t>(ceil_div(warps, kStemDgradWarps), static_cast<int64_t>(sms) * 4));
  launch_k(stem_dgrad_kernel, grid, kStemDgradWarps * 32, 0, static_cast<cudaStream_t>(stream), static_cast<const __nv_bfloat16*>(dc1),
           static_cast<const __nv_bfloat16*>(w), w_ld, dx, n, h, w_img, ho, wo, tiles);
  return check_launch("cb_stem_dgrad");
}

int cb_stem_s2d(const void* x, int in_dtype, void* out, int n, int h, int w, int ld, float mean_r, float mean_g, float mean_b,
                void* stream) {
  CB_REQUIRE(x && out && n > 0 && h > 0 && w > 0, "cb_stem_s2d: bad arguments");
  CB_REQUIRE(ld == 16 || ld == 64, "cb_stem_s2d: ld must be 16 (overlapping rows) or 64 (explicit 4-pixel windows)");
  CB_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, "cb_stem_s2d: out must be 16-byte aligned");
  const int ho = (h + 6 - 7) / 2 + 1, wo = (w + 6 - 7) / 2 + 1;
  const int64_t total = static_cast<int64_t>(n) * (ho + 3) * (wo + 3);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (in_dtype == 0)
    launch_k(stem_s2d_kernel<float>, ceil_div(total, 256), 256, 0, st, static_cast<const float*>(x), static_cast<__nv_bfloat16*>(out), n, h, w,
             ho + 3, wo + 3, ld, mean_r, mean_g, mean_b);
  else if (in_dtype == 1)
    launch_k(stem_s2d_kernel<uint8_t>, ceil_div(total, 256), 256, 0, st, static_cast<const uint8_t*>(x), static_cast<__nv_bfloat16*>(out), n, h,
             w, ho + 3, wo + 3, ld, mean_r, mean_g, mean_b);
  else
    CB_REQUIRE(false, "cb_stem_s2d: in_dtype must be 0 (fp32) or 1 (uint8)");
  return check_launch("cb_stem_s2d");
}

int cb_resize_pad(const void* x, int in_dtype, float* y, int planes, int h, int w, int new_h, int new_w, int max_size, void* stream) {
  CB_REQUIRE(x && y && planes > 0 && h > 0 && w > 0, "cb_resize_pad: bad arguments");
  CB_REQUIRE(new_h > 0 && new_w > 0 && new_h <= max_size && new_w <= max_size, "cb_resize_pad: resized frame %d x %d must fit %d x %d", new_h,
             new_w, max_size, max_size);
  const int64_t total = static_cast<int64_t>(planes) * max_size * max_size;
  const float sh = static_cast<float>(h) / new_h, sw = static_cast<float>(w) / new_w;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (in_dtype == 0)
    launch_k(resize_pad_kernel<float>, ceil_div(total, 256), 256, 0, st, static_cast<const float*>(x), y, planes, h, w, new_h, new_w, max_size, sh, sw);
  else if (in_dtype == 1)
    launch_k(resize_pad_kernel<uint8_t>, ceil_div(total, 256), 256, 0, st, static_cast<const uint8_t*>(x), y, planes, h, w, new_h, new_w, max_size,
             sh, sw);
  else
    CB_REQUIRE(false, "cb_resize_pad: in_dtype must be 0 (fp32) or 1 (uint8)");
  return check_launch("cb_resize_pad");
}

int cb_resize_pad_bwd(const float* dy, float* dx, int planes, int h, int w, int new_h, int new_w, int max_size, int accumulate,
                      void* stream) {
  CB_REQUIRE(dy && dx && planes > 0 && h > 0 && w > 0, "cb_resize_pad_bwd: bad arguments");
  CB_REQUIRE(new_h > 0 && new_w > 0 && new_h <= max_size && new_w <= max_size, "cb_resize_pad_bwd: resized frame %d x %d must fit %d x %d",
             new_h, new_w, max_size, max_size);
  CB_REQUIRE(accumulate == 0 || accumulate == 1, "cb_resize_pad_bwd: accumulate must be 0 or 1");
  const int tiles_w = ceil_div(w, kResizeBwdTile), tiles_h = ceil_div(h, kResizeBwdTile);
  const int64_t blocks = static_cast<int64_t>(planes) * tiles_w * tiles_h;
  CB_REQUIRE(blocks <= INT32_MAX, "cb_resize_pad_bwd: %lld tiles of 32 x 32 pixels exceed one launch", static_cast<long long>(blocks));
  const float sh = static_cast<float>(h) / new_h, sw = static_cast<float>(w) / new_w;
  launch_k(resize_pad_bwd_kernel, static_cast<int>(blocks), 256, 0, static_cast<cudaStream_t>(stream), dy, dx, h, w, new_h, new_w, max_size, sh,
           sw, static_cast<float>(new_h) / h, static_cast<float>(new_w) / w, tiles_w, tiles_h, accumulate);
  return check_launch("cb_resize_pad_bwd");
}

int cb_subsample2(const void* x, void* y, int n, int h, int w, int c, void* stream) {
  CB_NHWC_CHECK("cb_subsample2");
  const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1;
  const int64_t total = static_cast<int64_t>(n) * ho * wo * (c / 8);
  launch_k(subsample2_kernel, ceil_div(total, 256), 256, 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), n, h, w, c, ho, wo);
  return check_launch("cb_subsample2");
}

/* dsub: [n, ho, wo, c]; act, dx: [n, h, w, c] */
int cb_unsubsample2_mask(const void* dsub, const void* act, void* dx, int n, int h, int w, int c, void* stream) {
  CB_REQUIRE(dsub && dx && n > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0, "cb_unsubsample2_mask: bad arguments");
  const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1;
  const int64_t total = static_cast<int64_t>(n) * h * w * (c / 8);
  if (act == nullptr)
    launch_k(unsubsample2_kernel, ceil_div(total, 256), 256, 0, static_cast<cudaStream_t>(stream), static_cast<const __nv_bfloat16*>(dsub),
             static_cast<__nv_bfloat16*>(dx), n, h, w, c, ho, wo);
  else
    launch_k(unsubsample2_mask_kernel, ceil_div(total, 256), 256, 0, static_cast<cudaStream_t>(stream),
        static_cast<const __nv_bfloat16*>(dsub), static_cast<const __nv_bfloat16*>(act), static_cast<__nv_bfloat16*>(dx), n, h, w, c,
        ho, wo);
  return check_launch("cb_unsubsample2_mask");
}

int cb_nhwc_intake(const void* x, int in_dtype, int64_t sn, int64_t sc, int64_t sh, int64_t sw, int n, int c, int h, int w, const void* act,
                   int act_bordered, void* out, int out_bordered, void* stream) {
  CB_REQUIRE(x && out && n > 0 && c > 0 && h > 0 && w > 0 && c % 8 == 0, "cb_nhwc_intake: bad arguments (c must be a multiple of 8)");
  CB_REQUIRE(sn >= 0 && sc >= 0 && sh >= 0 && sw >= 0, "cb_nhwc_intake: negative stride");
  CB_REQUIRE((act_bordered == 0 || act_bordered == 1) && (out_bordered == 0 || out_bordered == 1),
             "cb_nhwc_intake: act_bordered and out_bordered must be 0 or 1");
  CB_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0 && (reinterpret_cast<uintptr_t>(act) & 15) == 0,
             "cb_nhwc_intake: out and act must be 16-byte aligned");
  const __nv_bfloat16* a = static_cast<const __nv_bfloat16*>(act);
  __nv_bfloat16* o = static_cast<__nv_bfloat16*>(out);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (in_dtype == 0)
    launch_intake<float>(x, sn, sc, sh, sw, a, act_bordered, o, out_bordered, n, c, h, w, st);
  else if (in_dtype == 2)
    launch_intake<__nv_bfloat16>(x, sn, sc, sh, sw, a, act_bordered, o, out_bordered, n, c, h, w, st);
  else if (in_dtype == 3)
    launch_intake<__half>(x, sn, sc, sh, sw, a, act_bordered, o, out_bordered, n, c, h, w, st);
  else
    CB_REQUIRE(false, "cb_nhwc_intake: in_dtype must be 0 (fp32), 2 (bf16) or 3 (fp16)");
  return check_launch("cb_nhwc_intake");
}

int cb_maxpool2x2_relu_fwd(const void* x, void* y, int n, int h, int w, int c, void* stream) {
  CB_NHWC_CHECK("cb_maxpool2x2_relu_fwd");
  CB_REQUIRE(h >= 2 && w >= 2, "cb_maxpool2x2_relu_fwd: spatial size must be >= 2");
  const int ho = h / 2, wo = w / 2;
  const int64_t total = static_cast<int64_t>(n) * ho * wo * (c / 8);
  launch_k(maxpool2x2_relu_fwd_kernel, ceil_div(total, 256), 256, 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), n, h, w, c, ho, wo);
  return check_launch("cb_maxpool2x2_relu_fwd");
}

/* dy: [n, h/2, w/2, c]; x: conv output [n, h, w, c]; dx_pad: [n, h+2, w+2, c] fully overwritten */
int cb_maxpool2x2_relu_bwd(const void* dy, const void* x, void* dx_pad, int n, int h, int w, int c, void* stream) {
  CB_REQUIRE(dy && x && dx_pad && n > 0 && h >= 2 && w >= 2 && c > 0 && c % 8 == 0, "cb_maxpool2x2_relu_bwd: bad arguments");
  const int64_t total = static_cast<int64_t>(n) * (h + 2) * (w + 2) * (c / 8);
  launch_k(maxpool2x2_relu_bwd_kernel, ceil_div(total, 256), 256, 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(dy), static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(dx_pad), n, h, w, c,
      h / 2, w / 2);
  return check_launch("cb_maxpool2x2_relu_bwd");
}

int cb_relu_mask(const void* dy, const void* act, void* dx, int64_t n, void* stream) {
  CB_REQUIRE(dy && act && dx && n > 0 && n % 8 == 0, "cb_relu_mask: n must be a positive multiple of 8");
  launch_k(relu_mask_kernel, ceil_div(n / 8, 256), 256, 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(dy), static_cast<const __nv_bfloat16*>(act), static_cast<__nv_bfloat16*>(dx), n / 8);
  return check_launch("cb_relu_mask");
}

}  // extern "C"
