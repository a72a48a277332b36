// Clip-level score aggregation + loss of the training loops, pool_method "lse"
// (src/tasks/run_video_retrieval.py:404-422, src/tasks/run_video_qa.py:484-501):
//     logits = stack(per-clip logits).permute(1, 0, 2)                        (B', n_clips, C)
//     out    = logsumexp(logits.view(B', -1), -1, keepdim) - logsumexp(logits, dim=1)   (B', C)
//     loss   = gather(out, -1, labels).mean()
// and its backward, in ONE launch: the reference spends ~45 ATen launches (two logsumexp, gather, mean and their autograd
// nodes) on a (n_clips, B', C) fp32 tensor of a few hundred values; inside the step's CUDA graph those are ~45 dependent
// nodes of 2-4 us each on the critical path between the last forward kernel and the first backward kernel.
//     d loss / d z[k, b, c] = (1 / B') * ( softmax over all (k', c') of example b  -  [c == y_b] * softmax over k' of z[:, b, y_b] )
#include "common.cuh"
#include "host_util.h"

namespace cb {

// the block's share of the mean: one atomic per block, or (DET) a plain store to part[blockIdx.x] summed in block order afterwards
template <bool DET>
__device__ __forceinline__ void block_loss_sum(float l, float inv_n, float* loss, float* part) {
  l = warp_sum(l);
  __shared__ float red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = l;
  __syncthreads();
  if (threadIdx.x < 8) {
    float v = red[threadIdx.x];
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) v += __shfl_xor_sync(0xffu, v, o);
    if (threadIdx.x == 0) {
      if constexpr (DET) part[blockIdx.x] = v * inv_n;
      else atomicAdd(loss, v * inv_n);
    }
  }
}

template <bool DET>
__global__ void __launch_bounds__(256) clip_lse_loss_kernel(const float* __restrict__ logits, const int64_t* __restrict__ labels,
                                                            float* __restrict__ loss, float* __restrict__ dlogits, int n_clips,
                                                            int nseq, int ncls, float inv_n, float grad_scale, float* part) {
  pdl_wait();
  pdl_trigger();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  float l = 0.f;
  if (b < nseq) {
    const int64_t y64 = labels[b];
    const int y = static_cast<int>(y64 < 0 ? 0 : (y64 >= ncls ? ncls - 1 : y64));   // torch.gather would raise; stay in bounds
    const int64_t clip_pitch = static_cast<int64_t>(nseq) * ncls;
    const float* z = logits + static_cast<int64_t>(b) * ncls;
    float m_all = -INFINITY, m_y = -INFINITY;
    for (int k = 0; k < n_clips; ++k) {
      for (int c = 0; c < ncls; ++c) m_all = fmaxf(m_all, z[k * clip_pitch + c]);
      m_y = fmaxf(m_y, z[k * clip_pitch + y]);
    }
    float s_all = 0.f, s_y = 0.f;
    for (int k = 0; k < n_clips; ++k) {
      for (int c = 0; c < ncls; ++c) s_all += expf(z[k * clip_pitch + c] - m_all);
      s_y += expf(z[k * clip_pitch + y] - m_y);
    }
    const float lse_all = m_all + logf(s_all), lse_y = m_y + logf(s_y);
    l = lse_all - lse_y;
    if (dlogits != nullptr) {
      float* d = dlogits + static_cast<int64_t>(b) * ncls;
      const float gs = inv_n * grad_scale;
      for (int k = 0; k < n_clips; ++k)
        for (int c = 0; c < ncls; ++c) {
          const float v = z[k * clip_pitch + c];
          float g = expf(v - lse_all);
          if (c == y) g -= expf(v - lse_y);
          d[k * clip_pitch + c] = g * gs;
        }
    }
  }
  block_loss_sum<DET>(l, inv_n, loss, part);
}

// ------------------------------------------------------------------------------------------------
// Clip pooling "mean" / "max" followed by cross entropy (run_video_retrieval.py:405-408,419-420 / run_video_qa.py:485-488,498-499:
// logits.mean(0) or logits.max(0)[0], then calc_loss -> F.cross_entropy(reduction="none") -> .mean()), forward + backward.
//   mean: d z[k, b, c] = (softmax_c(mean_k z) - onehot) / (n_clips * B')      max: the gradient goes to the arg-max clip only
// ------------------------------------------------------------------------------------------------
template <bool DET>
__global__ void __launch_bounds__(256) clip_pool_ce_kernel(const float* __restrict__ logits, const int64_t* __restrict__ labels,
                                                           float* __restrict__ loss, float* __restrict__ dlogits, int n_clips, int nseq,
                                                           int ncls, int pool_max, float inv_n, float grad_scale, float* part) {
  pdl_wait();
  pdl_trigger();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  float l = 0.f;
  if (b < nseq) {
    const int64_t y64 = labels[b];
    const int y = static_cast<int>(y64 < 0 ? 0 : (y64 >= ncls ? ncls - 1 : y64));
    const int64_t clip_pitch = static_cast<int64_t>(nseq) * ncls;
    const float* z = logits + static_cast<int64_t>(b) * ncls;
    auto pooled = [&](int c, int* arg) {
      float v = pool_max ? -INFINITY : 0.f;
      int a = 0;
      for (int k = 0; k < n_clips; ++k) {
        const float x = z[k * clip_pitch + c];
        if (pool_max) { if (x > v) { v = x; a = k; } }
        else v += x;
      }
      if (arg) *arg = a;
      return pool_max ? v : v / n_clips;
    };
    float m = -INFINITY;
    for (int c = 0; c < ncls; ++c) m = fmaxf(m, pooled(c, nullptr));
    float sum = 0.f;
    for (int c = 0; c < ncls; ++c) sum += expf(pooled(c, nullptr) - m);
    const float lse = m + logf(sum);
    l = lse - pooled(y, nullptr);
    if (dlogits != nullptr) {
      float* d = dlogits + static_cast<int64_t>(b) * ncls;
      const float gs = inv_n * grad_scale;
      for (int c = 0; c < ncls; ++c) {
        int a = 0;
        const float g = (expf(pooled(c, &a) - lse) - (c == y ? 1.f : 0.f)) * gs;
        for (int k = 0; k < n_clips; ++k) d[k * clip_pitch + c] = pool_max ? (k == a ? g : 0.f) : g / n_clips;
      }
    }
  }
  block_loss_sum<DET>(l, inv_n, loss, part);
}

// ------------------------------------------------------------------------------------------------
// F.cross_entropy(logits, labels, reduction="none") and its backward for wide rows - the masked-LM loss over the 30 522-word
// vocabulary (src/modeling/modeling.py:286-299: B' * Lt rows), the 5-way / 2-way heads (:560-580). One block per row:
//   forward : ONE read of the row (online max / sum-of-exp per thread, block reduction), loss[r] = lse - z[y] (0 for
//             ignore_index), lse[r] stashed;
//   backward: d z[r, c] = g[r] * (exp(z - lse[r]) - [c == y]), one read + one write.
// ATen makes a log_softmax tensor of the size of the logits plus nll_loss (3 passes forward, 2 backward).
// ------------------------------------------------------------------------------------------------
constexpr int CE_THREADS = 256;
__global__ void __launch_bounds__(CE_THREADS) ce_fwd_kernel(const float* __restrict__ logits, int64_t ld, const int64_t* __restrict__ labels,
                                                            float* __restrict__ loss, float* __restrict__ lse_out, int ncls, int64_t ignore_index) {
  pdl_wait();
  pdl_trigger();
  const int64_t r = blockIdx.x;
  const float* z = logits + r * ld;
  float m = -INFINITY, s = 0.f;
  for (int c = threadIdx.x; c < ncls; c += CE_THREADS) {      // online softmax statistics: one pass over the row
    const float v = z[c];
    if (v > m) { s = s * __expf(m - v) + 1.f; m = v; }
    else if (v != -INFINITY) s += __expf(v - m);   // (a -inf logit adds exp(-inf) = 0; while m is still -inf, exp(-inf + inf) is NaN)
  }
  __shared__ float sm[CE_THREADS / 32], ss[CE_THREADS / 32];
  const float wm = warp_max(m);
  s = warp_sum(m == -INFINITY ? 0.f : s * __expf(m - wm));      // (threads / warps beyond a short row hold (-inf, 0): exp(-inf + inf) is NaN)
  if ((threadIdx.x & 31) == 0) { sm[threadIdx.x >> 5] = wm; ss[threadIdx.x >> 5] = s; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float bm = -INFINITY, bs = 0.f;
    for (int i = 0; i < CE_THREADS / 32; ++i) bm = fmaxf(bm, sm[i]);
    for (int i = 0; i < CE_THREADS / 32; ++i) bs += sm[i] == -INFINITY ? 0.f : ss[i] * __expf(sm[i] - bm);
    const float lse = bm + __logf(bs);
    const int64_t y = labels[r];
    lse_out[r] = lse;
    loss[r] = (y == ignore_index || y < 0 || y >= ncls) ? 0.f : lse - z[y];
  }
}
__global__ void __launch_bounds__(CE_THREADS) ce_bwd_kernel(const float* __restrict__ logits, int64_t ld, const int64_t* __restrict__ labels,
                                                            const float* __restrict__ lse, const float* __restrict__ gloss,
                                                            float* __restrict__ dlogits, int64_t dld, int ncls, int64_t ignore_index) {
  pdl_wait();
  pdl_trigger();
  const int64_t r = blockIdx.x;
  const int64_t y = labels[r];
  const bool ignored = (y == ignore_index || y < 0 || y >= ncls);
  const float g = ignored ? 0.f : gloss[r];
  const float l = lse[r];
  const float* z = logits + r * ld;
  float* d = dlogits + r * dld;
  for (int c = threadIdx.x; c < ncls; c += CE_THREADS) d[c] = ignored ? 0.f : g * (__expf(z[c] - l) - (c == y ? 1.f : 0.f));
}

}  // namespace cb

using namespace cb;

extern "C" int cb_cross_entropy_fwd(const float* logits, int64_t ld, const int64_t* labels, float* loss, float* lse, int64_t rows, int ncls,
                                    int64_t ignore_index, void* stream) {
  CB_REQUIRE(logits && labels && loss && lse, "cb_cross_entropy_fwd: null pointer");
  CB_REQUIRE(rows > 0 && ncls > 0 && ld >= ncls && rows < (1ll << 31), "cb_cross_entropy_fwd: bad shape (rows=%lld ncls=%d ld=%lld)",
             static_cast<long long>(rows), ncls, static_cast<long long>(ld));
  launch_k(ce_fwd_kernel, static_cast<int>(rows), CE_THREADS, 0, static_cast<cudaStream_t>(stream), logits, ld, labels, loss, lse, ncls, ignore_index);
  return check_launch("cb_cross_entropy_fwd");
}

extern "C" int cb_cross_entropy_bwd(const float* logits, int64_t ld, const int64_t* labels, const float* lse, const float* grad_loss,
                                    float* dlogits, int64_t dld, int64_t rows, int ncls, int64_t ignore_index, void* stream) {
  CB_REQUIRE(logits && labels && lse && grad_loss && dlogits, "cb_cross_entropy_bwd: null pointer");
  CB_REQUIRE(rows > 0 && ncls > 0 && ld >= ncls && dld >= ncls && rows < (1ll << 31), "cb_cross_entropy_bwd: bad shape");
  launch_k(ce_bwd_kernel, static_cast<int>(rows), CE_THREADS, 0, static_cast<cudaStream_t>(stream), logits, ld, labels, lse, grad_loss, dlogits, dld,
           ncls, ignore_index);
  return check_launch("cb_cross_entropy_bwd");
}

// pool 0 = lse (clip_lse_loss_kernel), 1 / 2 = mean / max (clip_pool_ce_kernel); scratch != nullptr: deterministic launch
static int clip_loss(const char* name, const float* logits, const int64_t* labels, float* loss, float* dlogits, int n_clips, int nseq,
                     int ncls, int pool, float grad_scale, float* scratch, int64_t scratch_bytes, void* stream) {
  CB_REQUIRE(logits && labels && loss, "%s: null pointer", name);
  CB_REQUIRE(n_clips > 0 && nseq > 0 && ncls > 0, "%s: empty problem (n_clips=%d nseq=%d ncls=%d)", name, n_clips, nseq, ncls);
  const int blocks = ceil_div(nseq, 256);
  if (scratch == nullptr)
    CB_REQUIRE(!g_det.load(std::memory_order_relaxed), "%s: deterministic mode is on; call %s_det with its scratch", name, name);
  else
    CB_REQUIRE(scratch_bytes >= 4ll * blocks, "%s: needs a scratch of %lld bytes", name, 4ll * blocks);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(loss, 0, sizeof(float), st);
  if (e != cudaSuccess) {
    set_error("%s: memset failed: %s", name, cudaGetErrorString(e));
    return CB_ERR_CUDA;
  }
  if (pool == 0) {
    if (scratch) launch_k(clip_lse_loss_kernel<true>, blocks, 256, 0, st, logits, labels, loss, dlogits, n_clips, nseq, ncls, 1.0f / nseq, grad_scale, scratch);
    else launch_k(clip_lse_loss_kernel<false>, blocks, 256, 0, st, logits, labels, loss, dlogits, n_clips, nseq, ncls, 1.0f / nseq, grad_scale, scratch);
  } else {
    if (scratch) launch_k(clip_pool_ce_kernel<true>, blocks, 256, 0, st, logits, labels, loss, dlogits, n_clips, nseq, ncls, pool == 2 ? 1 : 0,
                          1.0f / nseq, grad_scale, scratch);
    else launch_k(clip_pool_ce_kernel<false>, blocks, 256, 0, st, logits, labels, loss, dlogits, n_clips, nseq, ncls, pool == 2 ? 1 : 0,
                  1.0f / nseq, grad_scale, scratch);
  }
  const int rc = check_launch(name);
  if (rc != CB_OK || scratch == nullptr) return rc;
  return launch_ordered_sum(scratch, blocks, loss, st, name);
}

extern "C" int cb_clip_pool_ce_loss(const float* logits, const int64_t* labels, float* loss, float* dlogits, int n_clips, int nseq, int ncls,
                                    int pool, float grad_scale, void* stream) {
  CB_REQUIRE(pool == 1 || pool == 2, "cb_clip_pool_ce_loss: pool must be 1 (mean) or 2 (max); lse is cb_clip_lse_loss");
  return clip_loss("cb_clip_pool_ce_loss", logits, labels, loss, dlogits, n_clips, nseq, ncls, pool, grad_scale, nullptr, 0, stream);
}

extern "C" int cb_clip_lse_loss(const float* logits, const int64_t* labels, float* loss, float* dlogits, int n_clips, int nseq,
                                int ncls, float grad_scale, void* stream) {
  return clip_loss("cb_clip_lse_loss", logits, labels, loss, dlogits, n_clips, nseq, ncls, 0, grad_scale, nullptr, 0, stream);
}

extern "C" int64_t cb_clip_loss_scratch_bytes(int nseq) { return nseq > 0 ? 4ll * ceil_div(nseq, 256) : 0; }

extern "C" int cb_clip_lse_loss_det(const float* logits, const int64_t* labels, float* loss, float* dlogits, int n_clips, int nseq,
                                    int ncls, float grad_scale, float* scratch, int64_t scratch_bytes, void* stream) {
  CB_REQUIRE(scratch != nullptr, "cb_clip_lse_loss_det: needs a scratch of %lld bytes", static_cast<long long>(cb_clip_loss_scratch_bytes(nseq)));
  return clip_loss("cb_clip_lse_loss_det", logits, labels, loss, dlogits, n_clips, nseq, ncls, 0, grad_scale, scratch, scratch_bytes, stream);
}

extern "C" int cb_clip_pool_ce_loss_det(const float* logits, const int64_t* labels, float* loss, float* dlogits, int n_clips, int nseq,
                                        int ncls, int pool, float grad_scale, float* scratch, int64_t scratch_bytes, void* stream) {
  CB_REQUIRE(pool == 1 || pool == 2, "cb_clip_pool_ce_loss_det: pool must be 1 (mean) or 2 (max); lse is cb_clip_lse_loss_det");
  CB_REQUIRE(scratch != nullptr, "cb_clip_pool_ce_loss_det: needs a scratch of %lld bytes",
             static_cast<long long>(cb_clip_loss_scratch_bytes(nseq)));
  return clip_loss("cb_clip_pool_ce_loss_det", logits, labels, loss, dlogits, n_clips, nseq, ncls, pool, grad_scale, scratch, scratch_bytes,
                   stream);
}
