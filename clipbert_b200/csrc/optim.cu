// Fused optimizer step over the flat parameter buffers (SURVEY.md section 8 f2).
//
// Replaces, for the ClipBERT training loop (src/tasks/run_video_retrieval.py:477-487):
//   clip_grad_norm_(amp.master_params(optimizer), cfg.grad_norm)     -> cb_sumsq + the clip coefficient inside cb_adamw_step
//   AdamW.step()   (src/optimization/adamw.py:40-103)                -> cb_adamw_step
//   optimizer.zero_grad()                                            -> zero_grad flag of cb_adamw_step
//   apex amp O2 master -> model weight copy (run_video_retrieval.py:307-309) -> the bf16 "packed" tensor-core operand
//       (FrozenBN scale folded in for conv weights) is written by the same kernel, so the next forward needs no re-cast.
// One launch per flat buffer (transformer, CNN): every parameter element is read once (master, grad, exp_avg, exp_avg_sq:
// 16 B) and written once (master, exp_avg, exp_avg_sq, grad = 0, packed: 18 B) - HBM-bound, 34 B per element.
#include "common.cuh"
#include "host_util.h"

namespace cb {

// chunk table row: offset, numel (<= 65536, multiple of 4 except the tail of a parameter), group, row_len (0: no row scale),
// scale_off (index into scales of the chunk's FIRST element's parameter, -1: none), flags (bit 0: emit bf16 packed copy),
// elem0 (index of the chunk's first element inside its parameter: row = (elem0 + i) / row_len)
constexpr int CHUNK_COLS = 8;
// hyper table row (floats): lr, step_size, weight_decay, beta1, beta2, eps, 0, 0
constexpr int HYPER_COLS = 8;

__device__ __forceinline__ void block_atomic_sum(float acc, float* out) {
  acc = warp_sum(acc);
  __shared__ float red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 8) {
    float v = red[threadIdx.x];
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) v += __shfl_xor_sync(0xffu, v, o);
    if (threadIdx.x == 0) atomicAdd(out, v);
  }
}

// out += sum(x^2) over x[0, n): grid-stride float4 loads, warp shuffle + shared reduction, one atomicAdd per block
__global__ void __launch_bounds__(256) sumsq_kernel(const float* __restrict__ x, int64_t n, float* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  float acc = 0.f;
  const int64_t n4 = n >> 2;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    acc = fmaf(v.x, v.x, acc); acc = fmaf(v.y, v.y, acc); acc = fmaf(v.z, v.z, acc); acc = fmaf(v.w, v.w, acc);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0)
    for (int64_t i = n4 << 2; i < n; ++i) acc = fmaf(x[i], x[i], acc);
  block_atomic_sum(acc, out);
}

// out += sum of x^2 over the chunk table's elements only: alignment padding between parameters and the zero-padded
// classifier rows belong to no parameter and must not enter the gradient norm
__global__ void __launch_bounds__(256) sumsq_chunks_kernel(const float* __restrict__ x, const int64_t* __restrict__ chunks, float* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  const int64_t* ch = chunks + static_cast<int64_t>(blockIdx.x) * CHUNK_COLS;
  const int64_t off = ch[0], n = ch[1];
  float acc = 0.f;
  for (int64_t i = static_cast<int64_t>(threadIdx.x) * 4; i < n; i += 256 * 4) {
    if (i + 4 <= n) {
      const float4 v = *reinterpret_cast<const float4*>(x + off + i);
      acc = fmaf(v.x, v.x, acc); acc = fmaf(v.y, v.y, acc); acc = fmaf(v.z, v.z, acc); acc = fmaf(v.w, v.w, acc);
    } else {
      for (int64_t k = i; k < n; ++k) acc = fmaf(x[off + k], x[off + k], acc);
    }
  }
  block_atomic_sum(acc, out);
}

__global__ void __launch_bounds__(256) adamw_kernel(float* __restrict__ master, float* __restrict__ grad, float* __restrict__ exp_avg,
                                                    float* __restrict__ exp_avg_sq, __nv_bfloat16* __restrict__ packed,
                                                    const int64_t* __restrict__ chunks, const float* __restrict__ hyper,
                                                    const float* __restrict__ scales, const float* __restrict__ grad_sumsq,
                                                    float max_norm, int zero_grad) {
  pdl_wait();
  pdl_trigger();
  const int64_t* ch = chunks + static_cast<int64_t>(blockIdx.x) * CHUNK_COLS;
  const int64_t off = ch[0], n = ch[1], row_len = ch[3], soff = ch[4], flags = ch[5], elem0 = ch[6];
  const float* hp = hyper + ch[2] * HYPER_COLS;
  const float lr = hp[0], step_size = hp[1], wd = hp[2], b1 = hp[3], b2 = hp[4], eps = hp[5];
  // clip_grad_norm_: coef = max_norm / (total_norm + 1e-6), applied only when < 1 (torch.nn.utils.clip_grad_norm_)
  float coef = 1.0f;
  if (grad_sumsq != nullptr && max_norm > 0.0f) coef = fminf(1.0f, max_norm / (sqrtf(*grad_sumsq) + 1e-6f));
  const bool emit = (flags & 1) && packed != nullptr;
  auto update = [&](float p, float g, float& m, float& v) {
    g *= coef;
    m = m * b1 + (1.0f - b1) * g;                       // exp_avg.mul_(beta1).add_(1 - beta1, grad)        adamw.py:76
    v = v * b2 + (1.0f - b2) * g * g;                   // exp_avg_sq.mul_(beta2).addcmul_(1 - beta2, g, g) adamw.py:77
    const float denom = sqrtf(v) + eps;                 // denom = exp_avg_sq.sqrt().add_(eps)              adamw.py:78
    p = p - step_size * (m / denom);                    // p.addcdiv_(-step_size, exp_avg, denom)           adamw.py:87
    if (wd > 0.0f) p = p - lr * wd * p;                 // p.add_(-lr * wd, p) AFTER the Adam update        adamw.py:98-99
    return p;
  };
  for (int64_t i = static_cast<int64_t>(threadIdx.x) * 4; i < n; i += 256 * 4) {
    const int64_t a = off + i;
    if (i + 4 <= n) {
      float4 p = *reinterpret_cast<const float4*>(master + a);
      const float4 g = *reinterpret_cast<const float4*>(grad + a);
      float4 m = *reinterpret_cast<const float4*>(exp_avg + a);
      float4 v = *reinterpret_cast<const float4*>(exp_avg_sq + a);
      p.x = update(p.x, g.x, m.x, v.x); p.y = update(p.y, g.y, m.y, v.y);
      p.z = update(p.z, g.z, m.z, v.z); p.w = update(p.w, g.w, m.w, v.w);
      *reinterpret_cast<float4*>(master + a) = p;
      *reinterpret_cast<float4*>(exp_avg + a) = m;
      *reinterpret_cast<float4*>(exp_avg_sq + a) = v;
      if (zero_grad) *reinterpret_cast<float4*>(grad + a) = make_float4(0.f, 0.f, 0.f, 0.f);
      if (emit) {
        float s0 = 1.f, s1 = 1.f, s2 = 1.f, s3 = 1.f;
        if (soff >= 0) {
          const int64_t e = elem0 + i;
          s0 = scales[soff + e / row_len]; s1 = scales[soff + (e + 1) / row_len];
          s2 = scales[soff + (e + 2) / row_len]; s3 = scales[soff + (e + 3) / row_len];
        }
        uint2 o;
        o.x = pack_bf16x2(p.x * s0, p.y * s1);
        o.y = pack_bf16x2(p.z * s2, p.w * s3);
        *reinterpret_cast<uint2*>(packed + a) = o;
      }
    } else {
      for (int64_t k = i; k < n; ++k) {
        float m = exp_avg[off + k], v = exp_avg_sq[off + k];
        const float p = update(master[off + k], grad[off + k], m, v);
        master[off + k] = p; exp_avg[off + k] = m; exp_avg_sq[off + k] = v;
        if (zero_grad) grad[off + k] = 0.f;
        if (emit) packed[off + k] = __float2bfloat16(p * (soff >= 0 ? scales[soff + (elem0 + k) / row_len] : 1.f));
      }
    }
  }
}

}  // namespace cb

extern "C" {
using namespace cb;

int cb_sumsq(const float* x, int64_t n, const int64_t* chunks, int nchunks, float* out, void* stream) {
  CB_REQUIRE(x && out && (chunks ? nchunks > 0 : n > 0), "cb_sumsq: bad arguments");
  CB_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, "cb_sumsq: x must be 16-byte aligned");
  if (chunks) {
    launch_k(sumsq_chunks_kernel, nchunks, 256, 0, static_cast<cudaStream_t>(stream), x, chunks, out);
    return check_launch("cb_sumsq");
  }
  const int64_t want = (n / 4 + 255) / 256;
  const int grid = static_cast<int>(want < 1 ? 1 : (want > 132 * 8 ? 132 * 8 : want));   // 8 resident 256-thread CTAs per H100 SM
  launch_k(sumsq_kernel, grid, 256, 0, static_cast<cudaStream_t>(stream), x, n, out);
  return check_launch("cb_sumsq");
}

int cb_adamw_step(float* master, float* grad, float* exp_avg, float* exp_avg_sq, void* packed, const int64_t* chunks, int nchunks,
                  const float* hyper, const float* scales, const float* grad_sumsq, float max_norm, int zero_grad, void* stream) {
  CB_REQUIRE(master && grad && exp_avg && exp_avg_sq && chunks && hyper && nchunks > 0, "cb_adamw_step: bad arguments");
  CB_REQUIRE(((reinterpret_cast<uintptr_t>(master) | reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(exp_avg) |
               reinterpret_cast<uintptr_t>(exp_avg_sq)) & 15) == 0 && (reinterpret_cast<uintptr_t>(packed) & 7) == 0,
             "cb_adamw_step: buffers must be 16-byte aligned (packed: 8)");
  launch_k(adamw_kernel, nchunks, 256, 0, static_cast<cudaStream_t>(stream), master, grad, exp_avg, exp_avg_sq,
           static_cast<__nv_bfloat16*>(packed), chunks, hyper, scales, grad_sumsq, max_norm, zero_grad);
  return check_launch("cb_adamw_step");
}

}  // extern "C"
