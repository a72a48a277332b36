// Host-side helpers shared by the C-ABI translation units: error reporting, launch counting,
// TMA tensor-map encoding (driver entry point fetched at run time, no link-time libcuda).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <utility>

#include "../../include/clipbert_b200.h"

namespace cb {

void set_error(const char* fmt, ...);
extern std::atomic<int64_t> g_launches;

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return CB_ERR_CUDA;
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return CB_OK;
}

// Programmatic dependent launch (PDL). Every kernel of this library starts with griddepcontrol.wait (all of its global
// memory traffic comes after it) and griddepcontrol.launch_dependents, and is launched with the programmatic-stream-
// serialization attribute: the next kernel's CTAs are scheduled while this one drains and run their prologue (barrier
// init, descriptor prefetch) under its tail. A step is ~500-900 dependent launches of 5-60 us, so the
// ~2-4 us launch + prologue bubble between them is a double-digit share of the step. Works inside CUDA-graph capture
// (programmatic dependency edges). OFF by default (cb_set_pdl(1) / CB_PDL=1 enables): it can defeat the two-stream wgrad
// overlap, see include/clipbert_b200.h.
extern std::atomic<int> g_pdl;

// deterministic mode (cb_set_deterministic): accumulations run in a fixed order; see include/clipbert_b200.h
extern std::atomic<int> g_det;
// out[0] += sum of part[0, n) in a fixed order (bert_ops.cu: ordered_sum_kernel), one launch on `stream`
int launch_ordered_sum(const float* part, int n, float* out, cudaStream_t stream, const char* what);

// g_pdl: 0 off, 1 every kernel, 2 every kernel EXCEPT the persistent GEMMs (their early-launched CTAs would hold ~200 KB
// of shared memory per SM while they wait; an LN / attention / column-sum CTA holds a few KB)
template <bool kGemm, typename... KArgs, typename... Args>
inline void launch_k_impl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  const int mode = g_pdl.load(std::memory_order_relaxed);
  cfg.numAttrs = (mode == 1 || (mode == 2 && !kGemm)) ? 1 : 0;
  (void)cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);   // errors are picked up by check_launch()
}
template <typename... KArgs, typename... Args>
inline void launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  launch_k_impl<false>(kern, grid, block, smem, stream, std::forward<Args>(args)...);
}
template <typename... KArgs, typename... Args>
inline void launch_gemm_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  launch_k_impl<true>(kern, grid, block, smem, stream, std::forward<Args>(args)...);
}

// 2D bf16 row-major tensor [rows, inner] (row pitch ld elements), 128B-swizzled boxes.
// Cached; the encoded map is COPIED into *out (the caller owns its copy). Returns false (and sets the error) on failure.
bool get_tmap_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t rows, uint64_t ld,
                 uint32_t box_inner, uint32_t box_rows);

// the same matrix as {64, rows, cols / 64}: one box = nblk swizzled [box_rows x 64] slabs (MN-major wgmma operands)
bool get_tmap_3d_mn(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t ld, uint32_t box_rows, uint32_t nblk);

#define CB_REQUIRE(cond, ...)        \
  do {                               \
    if (!(cond)) {                   \
      cb::set_error(__VA_ARGS__);    \
      return CB_ERR_INVALID;         \
    }                                \
  } while (0)

inline int ceil_div(int64_t a, int64_t b) { return static_cast<int>((a + b - 1) / b); }

}  // namespace cb
