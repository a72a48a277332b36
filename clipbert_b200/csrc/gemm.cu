// wgmma tensor-core contraction for every dense op on the ClipBERT path (see cb_gemm in
// include/clipbert_b200.h). One persistent, warp-specialised kernel, three operand modes:
//   MODE 0 (TN)    : A [rows, K] and B [N, K] both K-major; optional 9-tap row-shifted K loop
//                    (3x3 conv over a zero-bordered NHWC activation); fused epilogue.
//   MODE 2 (NN)    : as TN but B [K, ntaps*N] is read MN-major (dgrad straight from the forward weight).
//   MODE 1 (WGRAD) : dW = dY^T X with both operands read MN-major from the activation layout,
//                    split over the pixel/token dimension, fp32 red.global accumulation.
//
// Structure (persistent CTAs, grid = min(#tiles, #SMs x CTAs per SM), static round-robin tile schedule):
//   warp 8      TMA producer   : smem ring of STAGES x (A 128x64 | B BNx64) bf16 tiles, 128B swizzle
//   warps 0..7  two consumer warpgroups: warpgroup g multiplies rows 64g .. 64g+63 of the tile with wgmma m64nBNk16 into
//               registers, hands every smem stage back as soon as the products that read it have retired (one stage of
//               wgmma stays in flight), then runs the epilogue of its rows while the producer already fills the ring
//               with the next tile's operands.
//   Epilogue (TN / NN): each warp owns 16 rows of the tile. Per 32-column slice it moves its accumulator fragment through a
//               small per-warp fp32 staging tile so that every lane holds 16 consecutive columns of one row, applies the
//               fused epilogue (bias / FrozenBN shift, residual, dropout, activation, stashes) and writes 16-byte vectors,
//               re-mapping the output row (zero-bordered <-> compact pixel rows) where asked.
//   Epilogue (WGRAD): red.global.add.v2.f32 straight from the fragment (four lanes cover 32 contiguous bytes of a row).
#include "common.cuh"
#include "host_util.h"

namespace cb {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int CONSUMER_WARPS = 8;                          // two warpgroups of 64 tile rows each
constexpr int GEMM_THREADS = (CONSUMER_WARPS + 1) * 32;    // + the TMA producer warp
// (Nine warps put three on each SM sub-partition, which caps a thread at 168 registers: the 128 x 256 tiles of the TN / NN
// epilogue spill at that budget, so the launch model only picks them for the weight gradients, whose epilogue is lean.)
constexpr int MAX_STAGES = 8;
constexpr int SMEM_LIMIT = 232448;              // 227 KB opt-in limit per CTA
constexpr int SMEM_LIMIT_OCC2 = 113 * 1024;     // two CTAs per SM: (228 KB - 2 x 1 KB reserved) / 2
constexpr int STG_PITCH = 36;                   // fp32 staging row pitch in floats (32 + 4: conflict-free 16-byte row reads)
constexpr int STG_WARP_FLOATS = 16 * STG_PITCH; // one warp: 16 rows x 32 columns
constexpr int EPI_BYTES = CONSUMER_WARPS * STG_WARP_FLOATS * 4;

struct GemmEpi {
  const float* scale;
  const float* shift;
  const __nv_bfloat16* residual;
  int64_t res_ld;
  const __nv_bfloat16* aux;
  int64_t aux_ld;
  int aux_mode;
  int act;
  void* out;
  int64_t out_ld;
  int out_fp32;
  __nv_bfloat16* out2;
  int64_t out2_ld;
  int rowmap, H, W;
  uint32_t drop_thresh;
  float drop_inv_keep;
  uint64_t seed;
  const uint64_t* seed_off;   // device word folded into the seed at run time (cb_dropout_offset_bind), or nullptr
  int mn3d;         // MN-major operands (B of NN mode, A and B of WGRAD mode) arrive as ONE 3-D TMA box per k-chunk instead of
                    // BN/64 (BM/64) 2-D boxes: tmA / tmB are then the {64, rows, cols/64} maps of get_tmap_3d_mn
  long long* dbg;   // optional in-kernel clock64 timeline, 32 slots per CTA (bring-up / tuning only; NULL in production)
};

// bring-up / tuning only: clock64 stamps of EVERY CTA (32 slots per CTA; slots 12 / 13 = %globaltimer at entry / exit so that
// the per-SM cycle counters can be laid on one time axis)
__device__ __forceinline__ void dbg_stamp(const GemmEpi& epi, int slot) {
  if (epi.dbg) {
    epi.dbg[blockIdx.x * 32 + slot] = clock64();
    if (slot == 0 || slot == 11) {
      unsigned long long ns;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ns));
      epi.dbg[blockIdx.x * 32 + (slot == 0 ? 12 : 13)] = static_cast<long long>(ns);
    }
  }
}

template <int BN>
struct GemmCfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int BAR_BYTES = 256;
};

// ---- epilogue arithmetic on NC consecutive columns [nb, nb+NC) of one output row ------------------------------------------------
// shv[] holds the NC shift values (bias / FrozenBN shift) of these columns when has_shift. One function per epilogue KIND of the
// step: the kind is fixed per launch and selected by ONE uniform branch per 16 columns - a single generic body with run-time
// tests of every optional stage was if-converted by the compiler into straight-line code that evaluated gelu / gelu' / tanh
// under predicates for every element whatever the launch asked for (~2.4 k cycles per 16 columns for a bare multiply).
enum { EK_GENERIC = 0, EK_SHIFT_ACT = 1, EK_RELU_MASK = 2, EK_DROP_RES = 3, EK_GELU_STASH = 4, EK_AUX_MUL = 5 };

template <int NC>
__device__ __forceinline__ void add_shift(float (&f)[NC], const float (&shv)[NC]) {
#pragma unroll
  for (int j = 0; j < NC; ++j) f[j] += shv[j];
}
template <int NC>
__device__ __forceinline__ void add_residual(float (&f)[NC], const uint32_t (&res16)[NC / 2]) {
#pragma unroll
  for (int j = 0; j < NC / 2; ++j) {
    const float2 r2 = unpack_bf16x2(res16[j]);
    f[2 * j] += r2.x;
    f[2 * j + 1] += r2.y;
  }
}
//   EK_SHIFT_ACT : v = v (+ shift) (+ residual) -> ReLU / none      conv + FrozenBN shift (+ shortcut), Linear + bias, plain dgrad (+ residual)
template <int NC>
__device__ __forceinline__ void epilogue_shift_act(float (&f)[NC], const float (&shv)[NC], bool has_shift, const uint32_t (&res16)[NC / 2], bool has_res,
                                                   bool relu) {
  if (has_shift) add_shift<NC>(f, shv);
  if (has_res) add_residual<NC>(f, res16);
  if (relu) {
#pragma unroll
    for (int j = 0; j < NC; ++j) f[j] = fmaxf(f[j], 0.0f);
  }
}
//   EK_RELU_MASK : v = (v (+ residual)) * (aux > 0)                dgrad through a ReLU (CB_AUX_RELU_MASK)
template <int NC>
__device__ __forceinline__ void epilogue_relu_mask(float (&f)[NC], const uint32_t (&res16)[NC / 2], bool has_res, const uint32_t (&aux16)[NC / 2]) {
  if (has_res) add_residual<NC>(f, res16);
#pragma unroll
  for (int j = 0; j < NC / 2; ++j) {     // bf16 > 0  <=>  sign bit clear and magnitude non-zero, tested on the packed halves
    const uint32_t a = aux16[j];
    f[2 * j] = ((a & 0x8000u) == 0u && (a & 0x7fffu) != 0u) ? f[2 * j] : 0.0f;
    f[2 * j + 1] = ((a & 0x80000000u) == 0u && (a & 0x7fff0000u) != 0u) ? f[2 * j + 1] : 0.0f;
  }
}
//   EK_DROP_RES  : v = dropout(v + shift) + residual               BertSelfOutput / BertOutput dense (transformers.py:297-301,377-381)
template <int NC>
__device__ __forceinline__ void epilogue_drop_res(float (&f)[NC], const float (&shv)[NC], bool has_shift, const uint32_t (&res16)[NC / 2], bool has_res,
                                                  uint64_t dseed, uint64_t didx, uint32_t thresh, float inv_keep) {
  if (has_shift) add_shift<NC>(f, shv);
#pragma unroll
  for (int j = 0; j < NC; j += 4) {       // didx is a multiple of 4 (N % 8 == 0, 16-column runs): one hash per four columns
    float m[4];
    dropout_mult4(dseed, didx + j, thresh, inv_keep, m);
    f[j] *= m[0]; f[j + 1] *= m[1]; f[j + 2] *= m[2]; f[j + 3] *= m[3];
  }
  if (has_res) add_residual<NC>(f, res16);
}
//   EK_GELU_STASH: out = gelu(v + shift), out2 = gelu'(v + shift)  BertIntermediate (transformers.py:363-366) with the derivative stashed
template <int NC>
__device__ __forceinline__ void epilogue_gelu_stash(float (&f)[NC], const float (&shv)[NC], bool has_shift, uint32_t (&o2_16)[NC / 2]) {
  if (has_shift) add_shift<NC>(f, shv);
#pragma unroll
  for (int j = 0; j < NC / 2; ++j) {
    float y0, g0, y1, g1;
    gelu_erf_and_grad(f[2 * j], y0, g0);
    gelu_erf_and_grad(f[2 * j + 1], y1, g1);
    f[2 * j] = y0;
    f[2 * j + 1] = y1;
    o2_16[j] = pack_bf16x2(g0, g1);
  }
}
//   EK_AUX_MUL   : v = (v (+ residual)) * aux                      dgrad through the stashed gelu'
template <int NC>
__device__ __forceinline__ void epilogue_aux_mul(float (&f)[NC], const uint32_t (&res16)[NC / 2], bool has_res, const uint32_t (&aux16)[NC / 2]) {
  if (has_res) add_residual<NC>(f, res16);
#pragma unroll
  for (int j = 0; j < NC / 2; ++j) {
    const float2 a2 = unpack_bf16x2(aux16[j]);
    f[2 * j] *= a2.x;
    f[2 * j + 1] *= a2.y;
  }
}
//   EK_GENERIC   : every optional stage under run-time tests (heads, pooler tanh, ragged N): rare and tiny launches. GUARD: N is
//   not a multiple of 64, the per-column scale vector is read under per-float4 column checks (out-of-range outputs are dropped
//   by the caller). The activation / aux alternatives sit in separate switch arms so that only the requested one executes.
template <int NC, bool GUARD>
__device__ __forceinline__ void epilogue_math(float (&f)[NC], const GemmEpi& epi, const float (&shv)[NC], bool has_shift, uint64_t dseed, int nb, int N,
                                              int64_t orow, const uint32_t (&res16)[NC / 2], bool has_res, const uint32_t (&aux16)[NC / 2], bool has_aux,
                                              uint32_t (&o2_16)[NC / 2], bool has_out2) {
  if (GUARD && nb >= N) return;
  if (epi.scale) {
#pragma unroll
    for (int j = 0; j < NC; j += 4) {
      if (!GUARD || nb + j + 4 <= N) {
        const float4 s4 = __ldg(reinterpret_cast<const float4*>(epi.scale + nb + j));
        f[j] *= s4.x; f[j + 1] *= s4.y; f[j + 2] *= s4.z; f[j + 3] *= s4.w;
      }
    }
  }
  if (has_shift) add_shift<NC>(f, shv);
  if (epi.drop_thresh) {
    const uint64_t base = static_cast<uint64_t>(orow) * static_cast<uint64_t>(N) + nb;
#pragma unroll
    for (int j = 0; j < NC; j += 4) {
      float m[4];
      dropout_mult4(dseed, base + j, epi.drop_thresh, epi.drop_inv_keep, m);
      f[j] *= m[0]; f[j + 1] *= m[1]; f[j + 2] *= m[2]; f[j + 3] *= m[3];
    }
  }
  if (has_res) add_residual<NC>(f, res16);
  if (epi.act == CB_ACT_GELU_STASH_GRAD) {      // out = gelu(v), out2 = gelu'(v): one erf for both
#pragma unroll
    for (int j = 0; j < NC / 2; ++j) {
      float y0, g0, y1, g1;
      gelu_erf_and_grad(f[2 * j], y0, g0);
      gelu_erf_and_grad(f[2 * j + 1], y1, g1);
      f[2 * j] = y0;
      f[2 * j + 1] = y1;
      if (has_out2) o2_16[j] = pack_bf16x2(g0, g1);
    }
  } else if (has_out2) {
#pragma unroll
    for (int j = 0; j < NC / 2; ++j) o2_16[j] = pack_bf16x2(f[2 * j], f[2 * j + 1]);
  }
  switch (epi.act) {
    case CB_ACT_RELU:
#pragma unroll
      for (int j = 0; j < NC; ++j) f[j] = fmaxf(f[j], 0.0f);
      break;
    case CB_ACT_GELU:
#pragma unroll
      for (int j = 0; j < NC; ++j) f[j] = gelu_erf(f[j]);
      break;
    case CB_ACT_TANH:
#pragma unroll
      for (int j = 0; j < NC; ++j) f[j] = tanhf(f[j]);
      break;
    default: break;
  }
  if (has_aux) {
    switch (epi.aux_mode) {
      case CB_AUX_RELU_MASK:
#pragma unroll
        for (int j = 0; j < NC / 2; ++j) {
          const float2 a2 = unpack_bf16x2(aux16[j]);
          f[2 * j] = a2.x > 0.0f ? f[2 * j] : 0.0f;
          f[2 * j + 1] = a2.y > 0.0f ? f[2 * j + 1] : 0.0f;
        }
        break;
      case CB_AUX_GELU_GRAD:
#pragma unroll
        for (int j = 0; j < NC / 2; ++j) {
          const float2 a2 = unpack_bf16x2(aux16[j]);
          f[2 * j] *= gelu_erf_grad(a2.x);
          f[2 * j + 1] *= gelu_erf_grad(a2.y);
        }
        break;
      case CB_AUX_TANH_GRAD:
#pragma unroll
        for (int j = 0; j < NC / 2; ++j) {
          const float2 a2 = unpack_bf16x2(aux16[j]);
          f[2 * j] *= (1.0f - a2.x * a2.x);
          f[2 * j + 1] *= (1.0f - a2.y * a2.y);
        }
        break;
      case CB_AUX_MUL:
#pragma unroll
        for (int j = 0; j < NC / 2; ++j) {
          const float2 a2 = unpack_bf16x2(aux16[j]);
          f[2 * j] *= a2.x;
          f[2 * j + 1] *= a2.y;
        }
        break;
      default: break;
    }
  }
}

struct TileInfo {
  int m0, n0, nb0, tap, it_begin, n_iters;
};

// tile index -> coordinates; n-tiles are fastest so that concurrently running CTAs share the A rows.
template <int BN, int MODE>
__device__ __forceinline__ TileInfo decode_tile(int tile, int tiles_m, int tiles_n, int K, int ntaps, int iters_per_split) {
  TileInfo t;
  const int nt = tile % tiles_n;
  int r = tile / tiles_n;
  const int mt = r % tiles_m;
  r /= tiles_m;
  t.m0 = mt * BM;
  t.n0 = nt * BN;
  t.nb0 = t.n0;
  const int kc = (K + BK - 1) / BK;
  if (MODE == 1) {
    t.tap = r % ntaps;
    const int split = r / ntaps;
    t.it_begin = split * iters_per_split;
    t.n_iters = min(kc, t.it_begin + iters_per_split) - t.it_begin;
  } else {
    t.tap = 0;
    t.it_begin = 0;
    t.n_iters = ntaps * kc;
  }
  return t;
}

// ---- consumer side of the operand ring ------------------------------------------------------------------------------------------
// One tile's main loop of a consumer warpgroup: n_iters 64-deep k-chunks, KCH per ring stage. The wgmma of a stage are committed
// as one group; once the NEXT stage's group is issued, the previous group is waited for and its stage handed back to the producer
// (every consumer warp arrives on the stage's empty barrier). On return every product of the tile has landed in acc.
template <int BN, int TA, int TB>
__device__ __forceinline__ void mma_tile(float (&acc)[BN / 2], uint32_t smem0, int stage_bytes, int KCH, int STAGES, int n_iters, int wg,
                                         int lane, int& s, uint32_t& ph, uint64_t* full_bar, uint64_t* empty_bar) {
  using Cfg = GemmCfg<BN>;
  int prev = -1;
  for (int i = 0; i < n_iters; i += KCH) {
    const int nch = min(KCH, n_iters - i);
    mbar_wait(&full_bar[s], ph);
    __syncwarp();
    wgmma_fence();
    wgmma_fence_acc(acc);
    for (int ch = 0; ch < nch; ++ch) {
      // this warpgroup's 64 A rows: K-major, 64 rows x 128 B further on; MN-major, the second 64-row box (8 KB) - the same offset
      const uint32_t a_addr = smem0 + s * stage_bytes + ch * Cfg::STAGE_BYTES + wg * (64 * 128);
      const uint32_t b_addr = smem0 + s * stage_bytes + ch * Cfg::STAGE_BYTES + Cfg::A_BYTES;
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t ad = TA ? gmma_desc(a_addr + k * 2048, BK * 128, 1024) : gmma_desc(a_addr + k * 32, 16, 1024);
        const uint64_t bd = TB ? gmma_desc(b_addr + k * 2048, BK * 128, 1024) : gmma_desc(b_addr + k * 32, 16, 1024);
        wgmma_bf16<BN, TA, TB>(acc, ad, bd, (i > 0 || ch > 0 || k > 0) ? 1u : 0u);
      }
    }
    wgmma_commit();
    wgmma_wait<1>();
    wgmma_fence_acc(acc);
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
    }
    prev = s;
    if (++s == STAGES) { s = 0; ph ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_fence_acc(acc);
  if (prev >= 0) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[prev]);
  }
}

// ---- weight-gradient epilogue: out[tap * N + n] of rows m += acc * scale[m], straight from the wgmma fragment ----------------------
// Fragment layout of m64nNk16 (f32): warp w of the warpgroup holds rows 16w + lane/4 (d[4j], d[4j+1]) and 16w + lane/4 + 8
// (d[4j+2], d[4j+3]) at columns 8j + 2 (lane % 4) + {0, 1}.
template <int BN>
__device__ __forceinline__ void wgrad_epilogue(const float (&acc)[BN / 2], float* obase, int64_t out_ld, const float* scale, int M, int N, int r0,
                                               int n0, int lane) {
  const int r1 = r0 + 8;
  const float rs0 = (r0 < M && scale) ? scale[r0] : 1.0f;
  const float rs1 = (r1 < M && scale) ? scale[r1] : 1.0f;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int n = n0 + j * 8 + 2 * (lane & 3);
    if (n < N) {     // N % 8 == 0: the pair n, n + 1 is inside
      if (r0 < M) red_add_f32x2(obase + static_cast<int64_t>(r0) * out_ld + n, acc[4 * j] * rs0, acc[4 * j + 1] * rs0);
      if (r1 < M) red_add_f32x2(obase + static_cast<int64_t>(r1) * out_ld + n, acc[4 * j + 2] * rs1, acc[4 * j + 3] * rs1);
    }
  }
}

template <int BN, int MODE, int OCC>
__global__ void __launch_bounds__(GEMM_THREADS, OCC)
    gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int M, int N, int K, int ntaps, int tap_w,
                int tap_sign, int iters_per_split, int tiles_m, int tiles_n, int total_tiles, int STAGES, int KCH, int epi_bytes, GemmEpi epi) {
  using Cfg = GemmCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const int stage_bytes = KCH * Cfg::STAGE_BYTES;           // a stage holds KCH consecutive 64-deep k-chunks (one barrier round trip)
  uint8_t* stg_base = smem + STAGES * stage_bytes;          // epilogue staging (TN / NN)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stg_base + epi_bytes);
  uint64_t* empty_bar = full_bar + MAX_STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int unit = blockIdx.x;                                          // persistent work unit
  const int n_units = gridDim.x;
  if (threadIdx.x == 0) dbg_stamp(epi, 0);   // (debug-only buffer, not produced by any kernel: safe before pdl_wait)
  pdl_trigger();   // PDL: let the next kernel's CTAs take this SM as soon as this CTA leaves it
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  __syncthreads();
  const int kc_per_tap = (K + BK - 1) / BK;
  // PDL: barrier init and descriptor prefetch above overlapped the previous kernel's tail; from here on this kernel touches
  // global memory (TMA loads, epilogue loads/stores), so its producers must have completed.
  pdl_wait();
  if (threadIdx.x == 0) dbg_stamp(epi, 1);

  if (warp >= CONSUMER_WARPS) {
    // ===================== TMA producer =====================
    // One elected lane owns the barriers and issues the TMA boxes of a stage (KCH chunks x {A boxes, B boxes}).
    if (warp == CONSUMER_WARPS && lane == 0) {
      constexpr int A_BOXES = (MODE == 1) ? BM / 64 : 1;
      constexpr int B_BOXES = (MODE == 0) ? 1 : BN / 64;
      int s = 0;        // smem ring position / phase, carried across tiles
      uint32_t ph = 0;
      for (int tile = unit; tile < total_tiles; tile += n_units) {
        const TileInfo t = decode_tile<BN, MODE>(tile, tiles_m, tiles_n, K, ntaps, iters_per_split);
        for (int i = 0; i < t.n_iters; i += KCH) {
          const int nch = min(KCH, t.n_iters - i);
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_expect_tx(&full_bar[s], nch * Cfg::STAGE_BYTES);
          auto load = [&](void* dst, const CUtensorMap* map, int c0, int c1) { tma_load_2d(dst, map, &full_bar[s], c0, c1); };
          // the producer thread is issue-bound: per-chunk index math is done once, box loops are fully unrolled
          int kit = t.it_begin + i;
          int tp = 0, kc = kit;
          if (MODE != 1 && ntaps > 1) { tp = kit / kc_per_tap; kc = kit - tp * kc_per_tap; }
          for (int ch = 0; ch < nch; ++ch, ++kit) {
            uint8_t* sa = smem + s * stage_bytes + ch * Cfg::STAGE_BYTES;
            uint8_t* sb = sa + Cfg::A_BYTES;
            if (MODE == 1) {
              int shift = 0;
              if (ntaps == 9) shift = tap_sign * ((t.tap / 3 - 1) * tap_w + (t.tap % 3 - 1));
              const int p = kit * BK;
              if (epi.mn3d) {
                tma_load_3d(sa, &tmA, &full_bar[s], 0, p, t.m0 >> 6);
                tma_load_3d(sb, &tmB, &full_bar[s], 0, p + shift, t.nb0 >> 6);
              } else {
#pragma unroll
                for (int j = 0; j < A_BOXES; ++j) load(sa + j * (BK * 128), &tmA, t.m0 + j * 64, p);
#pragma unroll
                for (int j = 0; j < B_BOXES; ++j) load(sb + j * (BK * 128), &tmB, t.nb0 + j * 64, p + shift);
              }
            } else {
              int shift = 0;
              if (ntaps == 9) shift = tap_sign * ((tp / 3 - 1) * tap_w + (tp % 3 - 1));
              else if (ntaps > 1) shift = tap_sign * tp * tap_w;        // row taps (space-to-depth stem): tap t reads row m + t * tap_w
              load(sa, &tmA, kc * BK, t.m0 + shift);
              if (MODE == 0) {
                load(sb, &tmB, tp * K + kc * BK, t.nb0);
              } else if (epi.mn3d) {
                tma_load_3d(sb, &tmB, &full_bar[s], 0, kc * BK, (tp * N + t.nb0) >> 6);
              } else {
#pragma unroll
                for (int j = 0; j < B_BOXES; ++j) load(sb + j * (BK * 128), &tmB, tp * N + t.nb0 + j * 64, kc * BK);
              }
              if (++kc == kc_per_tap) { kc = 0; ++tp; }
            }
          }
          if (++s == STAGES) { s = 0; ph ^= 1; }
          if (i == 0 && tile == unit) dbg_stamp(epi, 2);
        }
      }
      dbg_stamp(epi, 3);
    }
    return;
  }

  // ===================== consumer warpgroups: wgmma main loop + epilogue =====================
  const int wg = warp >> 2;                 // rows wg * 64 .. wg * 64 + 63 of the tile
  const int wrow = wg * 64 + (warp & 3) * 16;   // first of this warp's 16 rows
  const uint32_t smem0 = smem_u32(smem);
  const uint64_t dseed = epi.drop_thresh ? drop_seed(epi.seed, epi.seed_off) : 0ull;   // after pdl_wait: the word is device data
  float acc[BN / 2];
  int s = 0;
  uint32_t ph = 0;
  int local = 0;

  // TN / NN epilogue: lane (er, eh) handles row er of the warp's 16, columns eh * 16 .. eh * 16 + 15 of each 32-column slice
  const int er = lane & 15, eh = lane >> 4;
  float* stg = reinterpret_cast<float*>(stg_base) + warp * STG_WARP_FLOATS;
  const bool has_out2 = epi.out2 != nullptr;
  const bool has_res = epi.residual != nullptr, has_aux = epi.aux != nullptr;
  const bool has_shift = epi.shift != nullptr;
  // epilogue kind, fixed for the launch (see the EK_* functions)
  const bool full = (N & 15) == 0 && epi.scale == nullptr;
  const bool drop = epi.drop_thresh != 0;
  int kind = EK_GENERIC;
  if (full) {
    if (!drop && !has_out2 && !has_aux && (epi.act == CB_ACT_NONE || epi.act == CB_ACT_RELU)) kind = EK_SHIFT_ACT;
    else if (!drop && !has_out2 && !has_shift && has_aux && epi.aux_mode == CB_AUX_RELU_MASK && epi.act == CB_ACT_NONE) kind = EK_RELU_MASK;
    else if (drop && !has_out2 && !has_aux && epi.act == CB_ACT_NONE) kind = EK_DROP_RES;
    else if (!drop && has_out2 && !has_aux && !has_res && epi.act == CB_ACT_GELU_STASH_GRAD) kind = EK_GELU_STASH;
    else if (!drop && !has_out2 && !has_shift && has_aux && epi.aux_mode == CB_AUX_MUL && epi.act == CB_ACT_NONE) kind = EK_AUX_MUL;
  }
  const bool kind_relu = epi.act == CB_ACT_RELU;
  const bool guard = (N & 15) != 0;                 // ragged last 16 columns: per-vector column checks in the generic epilogue

  for (int tile = unit; tile < total_tiles; tile += n_units, ++local) {
    const TileInfo t = decode_tile<BN, MODE>(tile, tiles_m, tiles_n, K, ntaps, iters_per_split);
    if (local == 0 && warp == 0 && lane == 0) dbg_stamp(epi, 4);
    mma_tile<BN, MODE == 1, MODE != 0>(acc, smem0, stage_bytes, KCH, STAGES, t.n_iters, wg, lane, s, ph, full_bar, empty_bar);
    if (local == 0 && warp == 0 && lane == 0) dbg_stamp(epi, 5);

    if (MODE == 1) {
      wgrad_epilogue<BN>(acc, reinterpret_cast<float*>(epi.out) + static_cast<int64_t>(t.tap) * N, epi.out_ld, epi.scale, M, N,
                         t.m0 + wrow + (lane >> 2), t.n0, lane);
      continue;
    }

    // ---- this lane's row: A-row space m (residual / aux), output row orow (re-mapped), row_ok ----
    const int m = t.m0 + wrow + er;
    bool row_ok = m < M;
    int64_t orow = m;
    if (epi.rowmap == CB_ROWMAP_PAD) {
      const int hw = epi.H * epi.W;
      const int img = m / hw;
      const int r = m - img * hw;
      const int y = r / epi.W, x = r - y * epi.W;
      orow = (static_cast<int64_t>(img) * (epi.H + 2) + y + 1) * (epi.W + 2) + x + 1;
    } else if (epi.rowmap == CB_ROWMAP_UNPAD) {
      const int wp = epi.W + 2, hp = epi.H + 2;
      const int img = m / (hp * wp);
      const int r = m - img * (hp * wp);
      const int y = r / wp, x = r - y * wp;
      row_ok = row_ok && y >= 1 && y <= epi.H && x >= 1 && x <= epi.W;
      orow = (static_cast<int64_t>(img) * epi.H + (y - 1)) * epi.W + (x - 1);
    }
#pragma unroll
    for (int sc = 0; sc < BN / 32; ++sc) {
      // fragment -> staging: this warp's 16 rows x 32 columns, then one row segment per lane
      __syncwarp();
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = sc * 4 + jj;
        float* p = stg + (lane >> 2) * STG_PITCH + jj * 8 + 2 * (lane & 3);
        *reinterpret_cast<float2*>(p) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(p + 8 * STG_PITCH) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
      __syncwarp();
      const int nb = t.n0 + sc * 32 + eh * 16;        // global column of f[0]
      if (!row_ok || nb >= N) continue;
      constexpr int NC = 16;
      float f[NC];
      const uint32_t srow = smem_u32(stg + er * STG_PITCH + eh * 16);
#pragma unroll
      for (int j = 0; j < NC / 4; ++j) {
        const uint4 u = lds128(srow + j * 16);
        f[4 * j] = __uint_as_float(u.x); f[4 * j + 1] = __uint_as_float(u.y);
        f[4 * j + 2] = __uint_as_float(u.z); f[4 * j + 3] = __uint_as_float(u.w);
      }
      uint32_t res16[NC / 2], aux16[NC / 2];
      if (has_res) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          uint4 u = make_uint4(0, 0, 0, 0);
          if (nb + 8 * j + 8 <= N) u = __ldg(reinterpret_cast<const uint4*>(epi.residual + static_cast<int64_t>(m) * epi.res_ld + nb + 8 * j));
          res16[4 * j] = u.x; res16[4 * j + 1] = u.y; res16[4 * j + 2] = u.z; res16[4 * j + 3] = u.w;
        }
      }
      if (has_aux) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          uint4 u = make_uint4(0, 0, 0, 0);
          if (nb + 8 * j + 8 <= N) u = __ldg(reinterpret_cast<const uint4*>(epi.aux + static_cast<int64_t>(m) * epi.aux_ld + nb + 8 * j));
          aux16[4 * j] = u.x; aux16[4 * j + 1] = u.y; aux16[4 * j + 2] = u.z; aux16[4 * j + 3] = u.w;
        }
      }
      float shv[NC];                                  // shift (bias / FrozenBN shift) of these columns
      if (has_shift) {
#pragma unroll
        for (int j = 0; j < NC; j += 4) {
          float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
          if (nb + j + 4 <= N) s4 = __ldg(reinterpret_cast<const float4*>(epi.shift + nb + j));
          shv[j] = s4.x; shv[j + 1] = s4.y; shv[j + 2] = s4.z; shv[j + 3] = s4.w;
        }
      }
      uint32_t o2_16[NC / 2];
      switch (kind) {
        case EK_SHIFT_ACT: epilogue_shift_act<NC>(f, shv, has_shift, res16, has_res, kind_relu); break;
        case EK_RELU_MASK: epilogue_relu_mask<NC>(f, res16, has_res, aux16); break;
        case EK_DROP_RES:
          epilogue_drop_res<NC>(f, shv, has_shift, res16, has_res, dseed, static_cast<uint64_t>(orow) * static_cast<uint64_t>(N) + nb, epi.drop_thresh,
                                epi.drop_inv_keep);
          break;
        case EK_GELU_STASH: epilogue_gelu_stash<NC>(f, shv, has_shift, o2_16); break;
        case EK_AUX_MUL: epilogue_aux_mul<NC>(f, res16, has_res, aux16); break;
        default:
          if (guard) epilogue_math<NC, true>(f, epi, shv, has_shift, dseed, nb, N, orow, res16, has_res, aux16, has_aux, o2_16, has_out2);
          else epilogue_math<NC, false>(f, epi, shv, has_shift, dseed, nb, N, orow, res16, has_res, aux16, has_aux, o2_16, has_out2);
      }
      if (epi.out_fp32) {
        float* o = reinterpret_cast<float*>(epi.out) + orow * epi.out_ld + nb;
#pragma unroll
        for (int j = 0; j < NC; j += 4)
          if (nb + j + 4 <= N) *reinterpret_cast<float4*>(o + j) = make_float4(f[j], f[j + 1], f[j + 2], f[j + 3]);
      } else {
        __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(epi.out) + orow * epi.out_ld + nb;
#pragma unroll
        for (int j = 0; j < 2; ++j)
          if (nb + 8 * j + 8 <= N)
            *reinterpret_cast<uint4*>(o + 8 * j) = make_uint4(pack_bf16x2(f[8 * j], f[8 * j + 1]), pack_bf16x2(f[8 * j + 2], f[8 * j + 3]),
                                                              pack_bf16x2(f[8 * j + 4], f[8 * j + 5]), pack_bf16x2(f[8 * j + 6], f[8 * j + 7]));
      }
      if (has_out2) {
        __nv_bfloat16* o = epi.out2 + orow * epi.out2_ld + nb;
#pragma unroll
        for (int j = 0; j < 2; ++j)
          if (nb + 8 * j + 8 <= N) *reinterpret_cast<uint4*>(o + 8 * j) = make_uint4(o2_16[4 * j], o2_16[4 * j + 1], o2_16[4 * j + 2], o2_16[4 * j + 3]);
      }
    }
    if (local == 0 && warp == 0 && lane == 0) dbg_stamp(epi, 8);
  }
  if (threadIdx.x == 0) dbg_stamp(epi, 11);
}

static int g_sm_limit = 0;    // tuning hook: cap on the persistent grid (0 = every SM). A long-running co-resident kernel (an NCCL
                              // all-reduce overlapped with the backward pass) pins some SMs for its whole duration; with the static
                              // round-robin tile schedule the CTAs that cannot be placed run as a second wave. Capping the grid at
                              // the SM count minus the co-resident kernel's CTAs avoids the second wave.
static int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return (g_sm_limit > 0 && g_sm_limit < n) ? g_sm_limit : n;
}

static long long* g_gemm_timeline = nullptr;
static int g_force_kch = 0;   // tuning hook: chunks per stage (0 = automatic)
static int g_mn3d = 1;        // 1 (default) = MN-major operands through one 3-D TMA box per k-chunk (GemmEpi::mn3d); cb_debug_gemm_mn3d

// Shared-memory plan of one launch: the epilogue staging (TN / NN: 16 x 32 fp32 per consumer warp; WGRAD: none), then as many
// 64-deep operand chunks as fit, grouped KCH per stage. Every stage costs one full / empty barrier round trip whatever its size,
// so deep stages are preferred to many shallow ones.
struct SmemPlan {
  int epi_bytes, kch, stages, chunk_bytes;
};
static SmemPlan plan_smem(int bn, bool staging, int kiters, int force_kch = 0, int occ = 1) {
  SmemPlan p;
  const int limit = occ == 2 ? SMEM_LIMIT_OCC2 : SMEM_LIMIT;
  p.chunk_bytes = BM * BK * 2 + bn * BK * 2;
  p.epi_bytes = staging ? EPI_BYTES : 0;
  const int chunks_fit = (limit - 1024 - GemmCfg<64>::BAR_BYTES - p.epi_bytes) / p.chunk_bytes;
  p.kch = 1;
  if (force_kch > 0) p.kch = force_kch;
  else if (g_force_kch > 0) p.kch = g_force_kch;
  else if (kiters >= 4 && chunks_fit >= 8) p.kch = 4;
  else if (kiters >= 2 && chunks_fit >= 4) p.kch = 2;
  if (p.kch > kiters) p.kch = kiters;
  if (p.kch > 1 && chunks_fit / p.kch < 2) p.kch = 1;
  p.stages = chunks_fit / p.kch;
  if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
  const int stage_iters = ceil_div(kiters, p.kch);
  if (p.stages > stage_iters + 1) p.stages = stage_iters + 1 > 2 ? stage_iters + 1 : 2;   // no ring deeper than the K loop
  return p;
}

template <int BN, int MODE, int OCC = 1>
static int launch_gemm(const cb_gemm_desc& d, const GemmEpi& epi_in, cudaStream_t stream) {
  GemmEpi epi = epi_in;
  using Cfg = GemmCfg<BN>;
  constexpr int LIMIT = OCC == 2 ? SMEM_LIMIT_OCC2 : SMEM_LIMIT;
  static bool attr_set = false;
  auto kern = gemm_kernel<BN, MODE, OCC>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, LIMIT);
    if (e == cudaSuccess && OCC == 2)   // both CTAs of an SM need their 113 KB: ask for the full shared-memory carve-out
      e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(smem=%d): %s", LIMIT, cudaGetErrorString(e));
      return CB_ERR_CUDA;
    }
    attr_set = true;
  }
  // Tensor maps are copied out of the cache into this frame (and from here into the kernel's parameter space)
  alignas(64) CUtensorMap ta, tb;
  bool mn3d = false;
  int iters_per_split = 0;
  const int tiles_m = ceil_div(d.m, BM), tiles_n = ceil_div(d.n, BN);
  int total = tiles_m * tiles_n;
  int kiters;
  bool ok;
  if (MODE == 0) {
    ok = get_tmap_2d(&ta, d.a, d.k, d.a_rows, d.a_ld, BK, BM) &&
         get_tmap_2d(&tb, d.b, static_cast<uint64_t>(d.k) * d.ntaps, d.b_rows, d.b_ld, BK, BN);
    kiters = ceil_div(d.k, BK) * d.ntaps;
  } else if (MODE == 2) {
    ok = get_tmap_2d(&ta, d.a, d.k, d.a_rows, d.a_ld, BK, BM);
    mn3d = g_mn3d && d.n % 64 == 0 &&
           get_tmap_3d_mn(&tb, d.b, static_cast<uint64_t>(d.n) * d.ntaps, d.b_rows, d.b_ld, BK, BN / 64);
    // not asked for, or the driver refused the 3-D view: the 2-D boxes always work
    if (!mn3d) ok = ok && get_tmap_2d(&tb, d.b, static_cast<uint64_t>(d.n) * d.ntaps, d.b_rows, d.b_ld, 64, BK);
    kiters = ceil_div(d.k, BK) * d.ntaps;
  } else {
    mn3d = g_mn3d && d.m % 64 == 0 && d.n % 64 == 0 && get_tmap_3d_mn(&ta, d.a, d.m, d.a_rows, d.a_ld, BK, BM / 64) &&
           get_tmap_3d_mn(&tb, d.b, d.n, d.b_rows, d.b_ld, BK, BN / 64);
    ok = mn3d || (get_tmap_2d(&ta, d.a, d.m, d.a_rows, d.a_ld, 64, BK) && get_tmap_2d(&tb, d.b, d.n, d.b_rows, d.b_ld, 64, BK));
    const int kc = ceil_div(d.k, BK);
    int splits = d.split_k < 1 ? 1 : d.split_k;
    if (splits > kc) splits = kc;
    iters_per_split = ceil_div(kc, splits);
    splits = ceil_div(kc, iters_per_split);   // every split is non-empty
    total *= splits * d.ntaps;
    kiters = iters_per_split;
  }
  if (!ok) return CB_ERR_CUDA;
  epi.mn3d = mn3d ? 1 : 0;
  const SmemPlan sp = plan_smem(BN, MODE != 1, kiters, (d.reserved >> 8) & 15, OCC);
  const int epi_bytes = sp.epi_bytes, kch = sp.kch, stages = sp.stages;
  if (stages < 2) {
    set_error("cb_gemm: not enough shared memory for a 2-stage pipeline (BN=%d, epilogue %d B, %d CTA(s) per SM)", BN, epi_bytes, OCC);
    return CB_ERR_INVALID;
  }
  const int smem_bytes = stages * kch * Cfg::STAGE_BYTES + epi_bytes + Cfg::BAR_BYTES + 1024;
  const int units = sm_count() * OCC;
  const int grid = total < units ? total : units;
  launch_gemm_k(kern, grid, GEMM_THREADS, smem_bytes, stream, ta, tb, d.m, d.n, d.k, d.ntaps, d.tap_w, d.tap_sign, iters_per_split, tiles_m,
                tiles_n, total, stages, kch, epi_bytes, epi);
  return check_launch("cb_gemm");
}

// ------------------------------------------------------------------------------------------------
// Launch configuration: an analytic model picks the tile width (and the wgrad K-split). A persistent CTA's main loop costs about
// (k-iterations x stage bytes) / (operand ingest rate) plus a barrier round trip per stage, and the launch is done when the
// busiest SM is; a per-tile epilogue term is added.
// ------------------------------------------------------------------------------------------------
struct LaunchCfg {
  int bn, splits;
};

// Two CTAs per SM (the OCC = 2 instantiations: 128 x 64 tiles, <= 113 KB of shared memory and <= 96 registers per thread
// each). One CTA's epilogue runs under the other's main loop. g_occ2_mode: 0 = never, 1 = only launches that ask for it
// (cb_gemm_desc.reserved bit 5), 2 = every eligible launch whose work is at most g_occ2_max_gflop (0 = no limit).
static int g_occ2_mode = 1;
static double g_occ2_max_gflop = 0.0;

static LaunchCfg choose_config(const cb_gemm_desc& d, int occ = 1) {
  const int units = sm_count() * occ;
  const int kc = ceil_div(d.k, BK);
  const bool wgrad = d.mode == CB_GEMM_WGRAD;
  static const int cand[3] = {64, 128, 256};
  LaunchCfg best = {0, 1};      // bn = 0: no candidate fits (only possible with occ = 2)
  double best_cost = 1e30;
  for (int c = 0; c < 3; ++c) {
    const int bn = cand[c];
    if (occ == 2 && bn > 64) continue;
    if (d.block_n && bn != d.block_n) continue;
    if (!d.block_n && !wgrad && bn == 256) continue;      // see GEMM_THREADS
    if (bn > 64 && d.n <= bn / 2) continue;               // mostly padding
    const int64_t base = static_cast<int64_t>(ceil_div(d.m, BM)) * ceil_div(d.n, bn) * (wgrad ? d.ntaps : 1);
    const int max_split = wgrad ? (d.split_k > 0 ? d.split_k : (kc < 32 ? kc : 32)) : 1;
    for (int sp = (wgrad && d.split_k > 0) ? d.split_k : 1; sp <= max_split; ++sp) {
      const int ips = ceil_div(wgrad ? kc : kc * d.ntaps, sp);
      const int real_sp = wgrad ? ceil_div(kc, ips) : 1;
      const int64_t tiles = base * real_sp;
      const double rounds = static_cast<double>((tiles + units - 1) / units);
      const SmemPlan pl = plan_smem(bn, !wgrad, ips, (d.reserved >> 8) & 15, occ);
      if (pl.stages < 2) continue;
      // a ring of 2 chunks cannot cover the TMA round trip of a long K loop
      const double shallow = (pl.stages * pl.kch < 3 && ips > 2) ? 3.0 : 1.0;
      // per stage: ~450-cycle barrier round trip + bytes at ~60 B/clk (shared by the CTAs of an SM); per tile: epilogue
      const double stage_cost = 450.0 + pl.kch * pl.chunk_bytes / (60.0 / occ);
      const double epi = wgrad ? bn * 24.0 : bn * 30.0;
      const double cost = rounds * (ceil_div(ips, pl.kch) * stage_cost * shallow + epi) + 2500.0;
      if (cost < best_cost) {
        best_cost = cost;
        best = {bn, real_sp};
      }
    }
  }
  if (best.bn == 0 && occ == 1) best = {64, 1};
  return best;
}

// ------------------------------------------------------------------------------------------------
// Grouped weight gradients: ONE persistent launch walks the tiles of several independent dW = dY^T X problems (the four
// Linear layers of a BertLayer, the three / four convs of a bottleneck block). The problems of a group share the reduction
// length (tokens / pixels), so their tiles cost the same and the static round-robin schedule stays balanced; what the group buys
// is one prologue + one tail instead of four, tiles of all problems filling the SMs together, and - because four problems
// together have enough tiles - no K-split, i.e. half the fp32 red.global traffic of the single launches. Same warp roles, ring
// and red.add epilogue as gemm_kernel<BN, MODE 1>; the problem descriptors (tensor maps included) travel in the kernel's
// parameter space.
// ------------------------------------------------------------------------------------------------
constexpr int WG_MAX_PROBLEMS = 8;
struct WgradProblem {
  CUtensorMap tmA, tmB;       // dY [P, M] and X [P, N] as MN-major operands: 2-D {64, BK} boxes or the 3-D {64, BK, cols / 64} view
  float* out;                 // fp32 [M, ntaps * N] (+= accumulation)
  const float* scale;         // optional per-output-row scale (FrozenBN fold), or nullptr
  int64_t out_ld;
  int M, N, K;                // output rows (= dY columns), output columns per tap, reduction length P
  int ntaps, tap_w, tap_sign;
  int iters_per_split, tiles_m, tiles_n;
  int tile_begin;             // first tile of this problem in the group's tile list
  int mn3d;
};
struct WgradGroup {
  int nprob, total_tiles;
  WgradProblem p[WG_MAX_PROBLEMS];
};
struct WgTile {
  int pi, m0, n0, tap, it_begin, n_iters;
};
__device__ __forceinline__ WgTile wg_decode(const WgradGroup& g, int tile) {
  WgTile t;
  int pi = 0;
  while (pi + 1 < g.nprob && tile >= g.p[pi + 1].tile_begin) ++pi;
  const WgradProblem& P = g.p[pi];
  int r = tile - P.tile_begin;
  const int nt = r % P.tiles_n;
  r /= P.tiles_n;
  const int mt = r % P.tiles_m;
  r /= P.tiles_m;
  t.pi = pi;
  t.m0 = mt * BM;
  t.tap = r % P.ntaps;
  const int split = r / P.ntaps;
  const int kc = (P.K + BK - 1) / BK;
  t.it_begin = split * P.iters_per_split;
  t.n_iters = min(kc, t.it_begin + P.iters_per_split) - t.it_begin;
  t.n0 = nt;      // (tile column index; multiplied by BN by the caller, which knows BN)
  return t;
}

template <int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    wgrad_group_kernel(const __grid_constant__ WgradGroup g, int STAGES, int KCH) {
  using Cfg = GemmCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const int stage_bytes = KCH * Cfg::STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * stage_bytes);
  uint64_t* empty_bar = full_bar + MAX_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int unit = blockIdx.x, n_units = gridDim.x;
  pdl_trigger();
  if (threadIdx.x == 0) {
    for (int i = 0; i < g.nprob; ++i) {
      tma_prefetch_desc(&g.p[i].tmA);
      tma_prefetch_desc(&g.p[i].tmB);
    }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp >= CONSUMER_WARPS) {
    // ===================== TMA producer =====================
    if (warp == CONSUMER_WARPS && lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int tile = unit; tile < g.total_tiles; tile += n_units) {
        const WgTile t = wg_decode(g, tile);
        const WgradProblem& P = g.p[t.pi];
        const int n0 = t.n0 * BN;
        int shift = 0;
        if (P.ntaps == 9) shift = P.tap_sign * ((t.tap / 3 - 1) * P.tap_w + (t.tap % 3 - 1));
        for (int i = 0; i < t.n_iters; i += KCH) {
          const int nch = min(KCH, t.n_iters - i);
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_expect_tx(&full_bar[s], nch * Cfg::STAGE_BYTES);
          int kit = t.it_begin + i;
          for (int ch = 0; ch < nch; ++ch, ++kit) {
            uint8_t* sa = smem + s * stage_bytes + ch * Cfg::STAGE_BYTES;
            uint8_t* sb = sa + Cfg::A_BYTES;
            const int p = kit * BK;
            if (P.mn3d) {
              tma_load_3d(sa, &P.tmA, &full_bar[s], 0, p, t.m0 >> 6);
              tma_load_3d(sb, &P.tmB, &full_bar[s], 0, p + shift, n0 >> 6);
            } else {
#pragma unroll
              for (int j = 0; j < BM / 64; ++j) tma_load_2d(sa + j * (BK * 128), &P.tmA, &full_bar[s], t.m0 + j * 64, p);
#pragma unroll
              for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * (BK * 128), &P.tmB, &full_bar[s], n0 + j * 64, p + shift);
            }
          }
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  const int wg = warp >> 2;
  const int wrow = wg * 64 + (warp & 3) * 16;
  const uint32_t smem0 = smem_u32(smem);
  float acc[BN / 2];
  int s = 0;
  uint32_t ph = 0;
  for (int tile = unit; tile < g.total_tiles; tile += n_units) {
    const WgTile t = wg_decode(g, tile);
    const WgradProblem& P = g.p[t.pi];
    mma_tile<BN, 1, 1>(acc, smem0, stage_bytes, KCH, STAGES, t.n_iters, wg, lane, s, ph, full_bar, empty_bar);
    wgrad_epilogue<BN>(acc, P.out + static_cast<int64_t>(t.tap) * P.N, P.out_ld, P.scale, P.M, P.N, t.m0 + wrow + (lane >> 2), t.n0 * BN, lane);
  }
}

template <int BN>
static int launch_wgrad_group(const cb_gemm_desc* descs, int n, int splits, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  static bool attr_set = false;
  auto kern = wgrad_group_kernel<BN>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(smem=%d): %s", SMEM_LIMIT, cudaGetErrorString(e));
      return CB_ERR_CUDA;
    }
    attr_set = true;
  }
  alignas(64) WgradGroup g;
  g.nprob = n;
  int total = 0, max_iters = 0;
  for (int i = 0; i < n; ++i) {
    const cb_gemm_desc& d = descs[i];
    WgradProblem& P = g.p[i];
    const bool mn3d = g_mn3d && d.m % 64 == 0 && d.n % 64 == 0 && get_tmap_3d_mn(&P.tmA, d.a, d.m, d.a_rows, d.a_ld, BK, BM / 64) &&
                      get_tmap_3d_mn(&P.tmB, d.b, d.n, d.b_rows, d.b_ld, BK, BN / 64);
    if (!mn3d && !(get_tmap_2d(&P.tmA, d.a, d.m, d.a_rows, d.a_ld, 64, BK) && get_tmap_2d(&P.tmB, d.b, d.n, d.b_rows, d.b_ld, 64, BK)))
      return CB_ERR_CUDA;
    P.mn3d = mn3d ? 1 : 0;
    P.out = static_cast<float*>(d.out);
    P.scale = d.scale;
    P.out_ld = d.out_ld;
    P.M = d.m; P.N = d.n; P.K = d.k;
    P.ntaps = d.ntaps; P.tap_w = d.tap_w; P.tap_sign = d.tap_sign;
    const int kc = ceil_div(d.k, BK);
    int sp = splits < 1 ? 1 : (splits > kc ? kc : splits);
    P.iters_per_split = ceil_div(kc, sp);
    sp = ceil_div(kc, P.iters_per_split);
    P.tiles_m = ceil_div(d.m, BM);
    P.tiles_n = ceil_div(d.n, BN);
    P.tile_begin = total;
    total += P.tiles_m * P.tiles_n * d.ntaps * sp;
    if (P.iters_per_split > max_iters) max_iters = P.iters_per_split;
  }
  g.total_tiles = total;
  const SmemPlan sp = plan_smem(BN, false, max_iters, 0, 1);
  if (sp.stages < 2) {
    set_error("cb_gemm_wgrad_group: not enough shared memory for a 2-stage pipeline (BN=%d)", BN);
    return CB_ERR_INVALID;
  }
  const int smem_bytes = sp.stages * sp.kch * Cfg::STAGE_BYTES + Cfg::BAR_BYTES + 1024;
  const int units = sm_count();
  launch_gemm_k(kern, total < units ? total : units, GEMM_THREADS, smem_bytes, stream, g, sp.stages, sp.kch);
  return check_launch("cb_gemm_wgrad_group");
}

}  // namespace cb

/* bring-up / tuning hook (not part of the public header): device buffer of >= 32 x grid int64 receiving clock64() stamps of every CTA */
extern "C" void cb_debug_gemm_timeline(void* device_buf) { cb::g_gemm_timeline = static_cast<long long*>(device_buf); }
extern "C" void cb_debug_gemm_kch(int kch) { cb::g_force_kch = kch; }
extern "C" void cb_debug_gemm_mn3d(int on) { cb::g_mn3d = on ? 1 : 0; }
extern "C" void cb_debug_gemm_occ2(int mode, double max_gflop) {
  cb::g_occ2_mode = mode < 0 ? 0 : (mode > 2 ? 2 : mode);
  cb::g_occ2_max_gflop = max_gflop;
}
extern "C" void cb_debug_gemm_sm_limit(int n) { cb::g_sm_limit = n > 0 ? n : 0; }

extern "C" int cb_gemm(const cb_gemm_desc* dp, void* stream_v) {
  using namespace cb;
  CB_REQUIRE(dp != nullptr, "cb_gemm: null descriptor");
  const cb_gemm_desc& d = *dp;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  CB_REQUIRE(d.a && d.b && d.out, "cb_gemm: null operand pointer");
  CB_REQUIRE(d.m > 0 && d.n > 0 && d.k > 0, "cb_gemm: empty problem m=%d n=%d k=%d", d.m, d.n, d.k);
  CB_REQUIRE(d.ntaps == 1 || d.ntaps == 9 || (d.ntaps == 4 && d.mode == CB_GEMM_TN),
             "cb_gemm: ntaps must be 1, 9 (3x3 conv) or 4 (row taps, TN only) (got %d)", d.ntaps);
  CB_REQUIRE(d.mode == CB_GEMM_TN || d.mode == CB_GEMM_WGRAD || d.mode == CB_GEMM_NN, "cb_gemm: bad mode %d", d.mode);
  CB_REQUIRE(d.dropout_p >= 0.0f && d.dropout_p < 1.0f, "cb_gemm: dropout_p out of range");

  GemmEpi epi;
  epi.scale = d.scale;
  epi.shift = d.shift;
  epi.residual = static_cast<const __nv_bfloat16*>(d.residual);
  epi.res_ld = d.res_ld;
  epi.aux = static_cast<const __nv_bfloat16*>(d.aux);
  epi.aux_ld = d.aux_ld;
  epi.aux_mode = d.aux ? d.aux_mode : CB_AUX_NONE;
  epi.act = d.act;
  epi.out = d.out;
  epi.out_ld = d.out_ld;
  epi.out_fp32 = d.out_fp32;
  epi.out2 = static_cast<__nv_bfloat16*>(d.out2);
  epi.out2_ld = d.out2_ld;
  epi.rowmap = d.rowmap;
  epi.H = d.map_h;
  epi.W = d.map_w;
  epi.seed = d.dropout_seed;
  epi.dbg = g_gemm_timeline;
  epi.mn3d = 0;
  {
    const DropCfg dc = make_drop(d.dropout_p, d.dropout_seed);
    epi.drop_thresh = dc.thresh;
    epi.drop_inv_keep = dc.inv_keep;
    epi.seed_off = dc.offset;
  }
  const double gflop = 2.0e-9 * d.m * d.n * d.k * d.ntaps;
  const bool want_occ2 = (d.reserved & 64) == 0 && (!d.block_n || d.block_n == 64) &&
                         ((d.reserved & 32) ? g_occ2_mode >= 1 : (g_occ2_mode == 2 && (g_occ2_max_gflop <= 0.0 || gflop <= g_occ2_max_gflop)));

  if (d.mode == CB_GEMM_TN || d.mode == CB_GEMM_NN) {
    const bool nn = d.mode == CB_GEMM_NN;
    CB_REQUIRE(d.n % 8 == 0, "cb_gemm(TN): n must be a multiple of 8 (got %d)", d.n);
    CB_REQUIRE(d.k % 8 == 0, "cb_gemm(TN): k must be a multiple of 8 (got %d)", d.k);
    CB_REQUIRE(d.out_ld % 8 == 0, "cb_gemm(TN): out_ld must be a multiple of 8");
    CB_REQUIRE(!d.residual || d.res_ld % 8 == 0, "cb_gemm(TN): res_ld must be a multiple of 8");
    CB_REQUIRE(!d.aux || d.aux_ld % 8 == 0, "cb_gemm(TN): aux_ld must be a multiple of 8");
    CB_REQUIRE(!d.out2 || d.out2_ld % 8 == 0, "cb_gemm(TN): out2_ld must be a multiple of 8");
    CB_REQUIRE(!(d.out2 && d.out_fp32), "cb_gemm(TN): out2 requires a bf16 primary output");
    CB_REQUIRE(d.rowmap == CB_ROWMAP_NONE || (d.map_h > 0 && d.map_w > 0), "cb_gemm: rowmap needs map_h/map_w");
    CB_REQUIRE(d.ntaps == 1 || d.tap_w > 2, "cb_gemm: tap modes need tap_w (padded row pitch in pixels)");
    if (want_occ2) {
      const LaunchCfg l2 = choose_config(d, 2);
      if (l2.bn == 64) return nn ? launch_gemm<64, 2, 2>(d, epi, stream) : launch_gemm<64, 0, 2>(d, epi, stream);
    }
    const LaunchCfg lc = choose_config(d);
    switch (lc.bn) {
      case 64: return nn ? launch_gemm<64, 2>(d, epi, stream) : launch_gemm<64, 0>(d, epi, stream);
      case 128: return nn ? launch_gemm<128, 2>(d, epi, stream) : launch_gemm<128, 0>(d, epi, stream);
      case 256: return nn ? launch_gemm<256, 2>(d, epi, stream) : launch_gemm<256, 0>(d, epi, stream);
      default: CB_REQUIRE(false, "cb_gemm: block_n must be 0, 64, 128 or 256 (got %d)", lc.bn);
    }
  } else {
    CB_REQUIRE(d.out_fp32 == 1, "cb_gemm(WGRAD): output must be fp32");
    CB_REQUIRE(d.m % 8 == 0 && d.n % 8 == 0, "cb_gemm(WGRAD): m, n must be multiples of 8 (got %d, %d)", d.m, d.n);
    CB_REQUIRE(d.out_ld % 4 == 0, "cb_gemm(WGRAD): out_ld must be a multiple of 4");
    CB_REQUIRE((reinterpret_cast<uintptr_t>(d.out) & 15) == 0, "cb_gemm(WGRAD): out must be 16-byte aligned");
    if (want_occ2) {
      const LaunchCfg l2 = choose_config(d, 2);
      cb_gemm_desc d2 = d;
      d2.split_k = l2.splits;
      if (l2.bn == 64) return launch_gemm<64, 1, 2>(d2, epi, stream);
    }
    const LaunchCfg lc = choose_config(d);
    cb_gemm_desc d2 = d;
    d2.split_k = lc.splits;
    switch (lc.bn) {
      case 64: return launch_gemm<64, 1>(d2, epi, stream);
      case 128: return launch_gemm<128, 1>(d2, epi, stream);
      case 256: return launch_gemm<256, 1>(d2, epi, stream);
      default: CB_REQUIRE(false, "cb_gemm(WGRAD): block_n must be 0, 64, 128 or 256 (got %d)", lc.bn);
    }
  }
  return CB_ERR_INVALID;
}

/* Several independent weight-gradient problems (CB_GEMM_WGRAD descriptors with the same reduction length) in ONE persistent launch. */
extern "C" int cb_gemm_wgrad_group(const cb_gemm_desc* descs, int n, void* stream_v) {
  using namespace cb;
  CB_REQUIRE(descs != nullptr && n >= 1, "cb_gemm_wgrad_group: no problems");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  bool groupable = n >= 2 && n <= WG_MAX_PROBLEMS;
  for (int i = 0; i < n; ++i) {
    const cb_gemm_desc& d = descs[i];
    CB_REQUIRE(d.mode == CB_GEMM_WGRAD && d.out_fp32 == 1, "cb_gemm_wgrad_group: problem %d is not an fp32 WGRAD descriptor", i);
    CB_REQUIRE(d.a && d.b && d.out && d.m > 0 && d.n > 0 && d.k > 0, "cb_gemm_wgrad_group: problem %d: null operand / empty shape", i);
    CB_REQUIRE(d.m % 8 == 0 && d.n % 8 == 0 && d.out_ld % 4 == 0 && (reinterpret_cast<uintptr_t>(d.out) & 15) == 0,
               "cb_gemm_wgrad_group: problem %d: m, n multiples of 8, out 16-byte aligned, out_ld a multiple of 4", i);
    CB_REQUIRE(d.ntaps == 1 || d.ntaps == 9, "cb_gemm_wgrad_group: problem %d: ntaps must be 1 or 9", i);
    // one schedule for all: reduction lengths within 2 x of each other, otherwise the round-robin tiles are unbalanced
    if (d.k * 2 < descs[0].k || descs[0].k * 2 < d.k) groupable = false;
  }
  if (!groupable) {      // a single problem, too many, or very different reduction lengths: the ordinary launches
    for (int i = 0; i < n; ++i) {
      const int rc = cb_gemm(&descs[i], stream_v);
      if (rc != CB_OK) return rc;
    }
    return CB_OK;
  }
  // tile width: the widest that does not mostly pad; K-split: fewest fp32 red.add passes that fill the SMs (one split if the group
  // already has >= 1 wave of tiles)
  int min_n = descs[0].n;
  for (int i = 1; i < n; ++i) min_n = descs[i].n < min_n ? descs[i].n : min_n;
  const int bn = min_n >= 192 ? 256 : (min_n >= 96 ? 128 : 64);
  int64_t base = 0;
  int kc_min = 1 << 30;
  for (int i = 0; i < n; ++i) {
    base += static_cast<int64_t>(ceil_div(descs[i].m, BM)) * ceil_div(descs[i].n, bn) * descs[i].ntaps;
    const int kc = ceil_div(descs[i].k, BK);
    kc_min = kc < kc_min ? kc : kc_min;
  }
  const int sms = sm_count();
  int best_split = 1;
  double best_cost = 1e30;
  for (int sp = 1; sp <= 8 && sp <= kc_min; ++sp) {
    const double waves = static_cast<double>((base * sp + sms - 1) / sms);
    const double cost = waves / sp + 0.06 * sp;      // main-loop time ~ waves / split; every split adds a red.add pass over the output
    if (cost < best_cost) { best_cost = cost; best_split = sp; }
  }
  if (bn == 256) return launch_wgrad_group<256>(descs, n, best_split, stream);
  if (bn == 128) return launch_wgrad_group<128>(descs, n, best_split, stream);
  return launch_wgrad_group<64>(descs, n, best_split, stream);
}
