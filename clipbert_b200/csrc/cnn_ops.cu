// Memory-bound CNN-side kernels for the GridFeat ResNet-50 path (reference call sites:
// src/modeling/grid_feat.py:89-105 -> detectron2 BasicStem / BottleneckBlock / MaxPool, and the
// grid_encoder MaxPool2d+ReLU at grid_feat.py:43-48). Activations are NHWC bf16; every thread moves
// 8 channels with one 128-bit access. All convolution FLOPs run in gemm.cu (wgmma).
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
    const float fy = fmaxf((oy + 0.5f) * sh - 0.5f, 0.f), fx = fmaxf((ox + 0.5f) * sw - 0.5f, 0.f);
    const int y0 = min(static_cast<int>(fy), H - 1), x0 = min(static_cast<int>(fx), W - 1);
    const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
    const float ly = fy - y0, lx = fx - x0;
    const TIn* p = x + plane * H * W;
    const float a = static_cast<float>(p[static_cast<int64_t>(y0) * W + x0]), b = static_cast<float>(p[static_cast<int64_t>(y0) * W + x1]);
    const float c = static_cast<float>(p[static_cast<int64_t>(y1) * W + x0]), d = static_cast<float>(p[static_cast<int64_t>(y1) * W + x1]);
    v = (1.f - ly) * ((1.f - lx) * a + lx * b) + ly * ((1.f - lx) * c + lx * d);
  }
  y[t] = v;
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
  CB_REQUIRE(dsub && act && dx && n > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0, "cb_unsubsample2_mask: bad arguments");
  const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1;
  const int64_t total = static_cast<int64_t>(n) * h * w * (c / 8);
  launch_k(unsubsample2_mask_kernel, ceil_div(total, 256), 256, 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(dsub), static_cast<const __nv_bfloat16*>(act), static_cast<__nv_bfloat16*>(dx), n, h, w, c,
      ho, wo);
  return check_launch("cb_unsubsample2_mask");
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
