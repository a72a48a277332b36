// Hand-written all-reduce of a flat fp32 gradient buffer through the NVSwitch (NVLink SHARP, "NVLS") - the NVSwitch-native form of
// the data-parallel exchange that Horovod + NCCL perform for the reference (src/tasks/run_video_retrieval.py:299-301,432).
//
// Every rank allocates the buffer as symmetric memory and maps it at a MULTICAST address (torch.distributed._symmetric_memory:
// rendezvous(...).multicast_ptr). Rank r owns the r-th 1/world slice of the element range:
//     multimem.ld_reduce.add.f32  pulls the slice through the switch, which sums the copies of ALL ranks in flight,
//     (x scale: 1/world for the average),
//     multimem.st                 writes the result back through the switch into EVERY rank's copy.
// Per rank that is n/world elements pulled and n/world pushed - the reduce-scatter + all-gather traffic of a ring, without the
// ring: no per-hop latency, no staging buffers, and only as many CTAs as the caller allows (NCCL's all-reduce kernel pins its
// CTAs for the whole exchange, which with this library's persistent one-CTA-per-SM GEMMs costs a second wave).
// The caller brackets the launch with cross-rank barriers (all gradients written before; all slices stored after).
#include "common.cuh"
#include "host_util.h"

namespace cb {

// 128-thread CTAs with ~30 registers per thread: small enough to share an SM with one of this library's persistent GEMM CTAs
// (608 threads x 96 registers), so the exchange pins no SM of its own. Four independent 16-byte multicast loads are in flight
// per thread before the first dependent store (the loads cross the NVSwitch: ~2-3 us each).
constexpr int NVLS_THREADS = 128;
constexpr int NVLS_UNROLL = 4;

__device__ __forceinline__ float4 mc_ld_reduce(const float* p) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void mc_st(float* p, float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

__global__ void __launch_bounds__(NVLS_THREADS) nvls_allreduce_f32_kernel(float* __restrict__ mc, int64_t v4_begin, int64_t v4_end, float scale) {
  pdl_wait();
  pdl_trigger();
  const int64_t stride = static_cast<int64_t>(gridDim.x) * NVLS_THREADS;
  for (int64_t i0 = v4_begin + static_cast<int64_t>(blockIdx.x) * NVLS_THREADS + threadIdx.x; i0 < v4_end; i0 += stride * NVLS_UNROLL) {
    float4 v[NVLS_UNROLL];
#pragma unroll
    for (int u = 0; u < NVLS_UNROLL; ++u) {
      const int64_t i = i0 + u * stride;
      if (i < v4_end) v[u] = mc_ld_reduce(mc + i * 4);
    }
#pragma unroll
    for (int u = 0; u < NVLS_UNROLL; ++u) {
      const int64_t i = i0 + u * stride;
      if (i < v4_end) {
        v[u].x *= scale; v[u].y *= scale; v[u].z *= scale; v[u].w *= scale;
        mc_st(mc + i * 4, v[u]);
      }
    }
  }
}

}  // namespace cb

using namespace cb;

extern "C" int cb_nvls_allreduce_f32(void* multicast_ptr, int64_t n, int rank, int world, float scale, int max_ctas, void* stream) {
  CB_REQUIRE(multicast_ptr != nullptr, "cb_nvls_allreduce_f32: null multicast pointer (no NVLS mapping)");
  CB_REQUIRE((reinterpret_cast<uintptr_t>(multicast_ptr) & 15) == 0 && n > 0 && n % 4 == 0,
             "cb_nvls_allreduce_f32: pointer must be 16-byte aligned and n a positive multiple of 4 (got %lld)", static_cast<long long>(n));
  CB_REQUIRE(world >= 1 && rank >= 0 && rank < world, "cb_nvls_allreduce_f32: bad rank %d / world %d", rank, world);
  const int64_t v4 = n / 4;
  const int64_t per = (v4 + world - 1) / world;
  const int64_t begin = rank * per < v4 ? rank * per : v4;
  const int64_t end = begin + per < v4 ? begin + per : v4;
  if (end <= begin) return CB_OK;                      // nothing in this rank's slice (tiny buffers)
  int grid = ceil_div(end - begin, static_cast<int64_t>(NVLS_THREADS) * NVLS_UNROLL);
  const int cap = max_ctas > 0 ? max_ctas : 64;
  if (grid > cap) grid = cap;
  launch_k(nvls_allreduce_f32_kernel, grid, NVLS_THREADS, 0, static_cast<cudaStream_t>(stream), static_cast<float*>(multicast_ptr), begin, end, scale);
  return check_launch("cb_nvls_allreduce_f32");
}
