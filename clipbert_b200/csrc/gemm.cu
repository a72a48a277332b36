// wgmma tensor-core contraction for every dense op on the ClipBERT path (see cb_gemm in
// include/clipbert_b200.h). One persistent, warp-specialised kernel, three operand modes:
//   MODE 0 (TN)    : A [rows, K] and B [N, K] both K-major; optional 9-tap row-shifted K loop
//                    (3x3 conv over a zero-bordered NHWC activation); fused epilogue.
//   MODE 2 (NN)    : as TN but B [K, ntaps*N] is read MN-major (dgrad straight from the forward weight).
//   MODE 1 (WGRAD) : dW = dY^T X with both operands read MN-major from the activation layout,
//                    optionally split over the pixel/token dimension, fp32 red.global accumulation.
//
// Every kernel is persistent (grid = min(#tiles, #SMs x CTAs per SM), static round-robin tile schedule) and fills a shared-memory
// ring of STAGES x KCH x (A 128x64 | B BNx64) bf16 k-chunks, 128B swizzle, from ONE elected TMA producer lane.
//
// TN / NN: gemm_pingpong_kernel, 384 threads = three warpgroups, one CTA per SM.
//   warpgroup 0   TMA producer. Its warps give registers back (setmaxnreg.dec 40); one lane issues the operand boxes and the
//                 epilogue-input boxes in tile order.
//   warpgroups 1, 2  consumers (setmaxnreg.inc 232). Each owns WHOLE 128 x BN tiles (BN = 64 / 128): per k16 step two wgmma
//                 m64nBNk16, rows 0-63 and 64-127, into BN fp32 accumulators per thread. A CTA's local tile j belongs to
//                 consumer j & 1 ("ping-pong"). The main loops run in tile order: a consumer starts tile j's main loop when the
//                 other one has issued the last wgmma of tile j-1 (named barrier per consumer); the other consumer then runs
//                 tile j-1's epilogue while this one's wgmma run. So a tile's epilogue - fused
//                 arithmetic and 16-byte stores, which at K = 64 takes several times as long as the main loop - overlaps the
//                 next tile's main loop and, when it is the longer part, the other consumer's epilogue. Both consumers walk the
//                 one operand ring, each skipping the other's stages (n_iters is the same for every TN / NN tile). A stage is
//                 read by one consumer, so its empty barrier counts that consumer's four warps.
//   Epilogue:     each warp owns rows 16w .. 16w+15 of both 64-row halves of its tile. Per half and 32-column slice it moves its
//                 accumulator fragment through a small per-warp fp32 staging tile so that every lane holds 16 consecutive
//                 columns of one row, applies the fused epilogue (bias / FrozenBN shift, residual, dropout, activation,
//                 stashes) and writes 16-byte vectors, re-mapping the output row (zero-bordered <-> compact pixel rows) where
//                 asked. The residual / aux tiles (bf16, rows m0 .. m0+127 of the A-row space in every row-map mode; with UNPAD
//                 that includes the zero-border rows the epilogue then drops) arrive by TMA in 128B-swizzled [128 x 64] boxes:
//                 into one of N_IN epilogue-input buffers with their own full / empty barrier pair (with two buffers, each
//                 consumer has its own), or, for K loops longer than four chunks, into the operand ring stage after the
//                 tile's operands (plan_smem). Reading them with per-lane global loads inside the epilogue left four dependent
//                 HBM round trips per tile and warp exposed on the one-chunk main loops of the HBM-bound 1x1 convs.
//
// TN / NN 128 x 256: gemm_coop_kernel, the same three warpgroups, both consumers on rows 0-63 / 64-127 of ONE tile (see there);
//   choose_config picks it for long tensor-bound K loops where it about halves the wave count.
//
// WGRAD: wgrad_group_kernel, 288 threads, one CTA per SM. It walks the tiles of a group of problems; a single weight gradient
//   (cb_gemm) is a group of one. Warp 8 is the TMA producer, warps 0..7 two consumer warpgroups that multiply rows
//   64g .. 64g+63 of one 128 x BN tile (BN up to 256) with wgmma m64nBNk16, hand every ring stage back as soon as the products
//   that read it have retired (one stage of wgmma stays in flight), then add the tile into the fp32 output with
//   red.global.add.v2.f32 straight from the fragment (four lanes cover 32 contiguous bytes of a row).
#include <algorithm>

#include "common.cuh"
#include "host_util.h"

namespace cb {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int CONSUMER_WARPS = 8;                          // WGRAD: two warpgroups of 64 tile rows each
constexpr int GEMM_THREADS = (CONSUMER_WARPS + 1) * 32;    // + the TMA producer warp
// (Nine warps put three on each SM sub-partition, which caps a thread at 168 registers; the lean red.add epilogue of the weight
// gradients fits 128 x 256 tiles in that budget.)
constexpr int PP_THREADS = 3 * 128;                        // TN / NN: producer warpgroup + two consumer warpgroups
constexpr int PP_PRODUCER_REGS = 40;                       // 128 x 40 + 256 x 232 = 64512 = 384 x 168, the entry budget
constexpr int PP_CONSUMER_REGS = 232;
constexpr int PP_BAR_TURN = 1;                             // named barriers 1, 2: consumer 0 / 1 may start its next main loop
constexpr int MAX_STAGES = 8;
constexpr int SMEM_LIMIT = 232448;              // 227 KB opt-in limit per CTA
constexpr int STG_PITCH = 36;                   // fp32 staging row pitch in floats (32 + 4: conflict-free 16-byte row reads)
constexpr int STG_WARP_FLOATS = 16 * STG_PITCH; // one warp: 16 rows x 32 columns
constexpr int EPI_BYTES = CONSUMER_WARPS * STG_WARP_FLOATS * 4;
constexpr int IN_BOX_BYTES = BM * 64 * 2;       // one epilogue-input box: 128 rows x 64 bf16 columns, 128B swizzle

struct GemmEpi {
  const float* scale;
  const float* shift;
  const __nv_bfloat16* residual;   // (read through the tmR / tmX tensor maps; the pointers only say which inputs exist)
  const __nv_bfloat16* aux;
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
  int mn3d;         // the MN-major B operand of NN mode arrives as ONE 3-D TMA box per k-chunk instead of BN/64 2-D boxes:
                    // tmB is then the {64, rows, cols/64} map of get_tmap_3d_mn
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

// ReLU of the epilogue: NaN propagates (as ATen's relu; fmaxf would return 0) and a -0 pre-activation gives +0. One FSETP.GTU +
// FSEL per element.
__device__ __forceinline__ float relu_nan(float v) { return !(v <= 0.0f) ? v : 0.0f; }
// ReLU' of a bf16 activation, tested on its bits (lo: the low half of x): > 0 for a positive normal number or +inf. A NaN,
// a zero of either sign and a subnormal give 0 - the same answer as the flush-to-zero float compare (act > 0) of the library's
// other ReLU backwards, whatever the packing.
__device__ __forceinline__ bool bf16_relu_pos(uint32_t x, bool lo) {
  const uint32_t b = lo ? (x & 0xffffu) : (x >> 16);
  return b - 0x0080u <= 0x7f80u - 0x0080u;
}

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
    for (int j = 0; j < NC; ++j) f[j] = relu_nan(f[j]);
  }
}
//   EK_RELU_MASK : v = (aux > 0) ? v (+ residual) : 0              dgrad through a ReLU (CB_AUX_RELU_MASK), a select
template <int NC>
__device__ __forceinline__ void epilogue_relu_mask(float (&f)[NC], const uint32_t (&res16)[NC / 2], bool has_res, const uint32_t (&aux16)[NC / 2]) {
  if (has_res) add_residual<NC>(f, res16);
#pragma unroll
  for (int j = 0; j < NC / 2; ++j) {     // tested on the packed halves
    f[2 * j] = bf16_relu_pos(aux16[j], true) ? f[2 * j] : 0.0f;
    f[2 * j + 1] = bf16_relu_pos(aux16[j], false) ? f[2 * j + 1] : 0.0f;
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
      for (int j = 0; j < NC; ++j) f[j] = relu_nan(f[j]);
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
        for (int j = 0; j < NC / 2; ++j) {        // as EK_RELU_MASK
          f[2 * j] = bf16_relu_pos(aux16[j], true) ? f[2 * j] : 0.0f;
          f[2 * j + 1] = bf16_relu_pos(aux16[j], false) ? f[2 * j + 1] : 0.0f;
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
  int m0, n0;
};

// TN / NN tile index -> coordinates; n-tiles are fastest so that concurrently running CTAs share the A rows.
template <int BN>
__device__ __forceinline__ TileInfo decode_tile(int tile, int tiles_m, int tiles_n) {
  TileInfo t;
  t.m0 = (tile / tiles_n) % tiles_m * BM;
  t.n0 = tile % tiles_n * BN;
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

// The same for one consumer warpgroup of the ping-pong kernel, which owns the whole 128-row tile: per k16 step one wgmma for rows
// 0-63 (acc[0]) and one for rows 64-127 (acc[1]), so every accumulator sees its k steps in the order of mma_tile. Once the last
// wgmma group of the tile is committed, the other consumer may start its main loop (pass_bar, 0 = no next tile); in_stage: the
// tile's epilogue inputs follow its operands in the ring, and have landed before the turn passes.
template <int BN, int TB>
__device__ __forceinline__ void mma_tile_pp(float (&acc)[2][BN / 2], uint32_t smem0, int stage_bytes, int KCH, int STAGES, int n_iters,
                                            int lane, int& s, uint32_t& ph, uint64_t* full_bar, uint64_t* empty_bar, int pass_bar,
                                            bool in_stage) {
  using Cfg = GemmCfg<BN>;
  int prev = -1;
  for (int i = 0; i < n_iters; i += KCH) {
    const int nch = min(KCH, n_iters - i);
    mbar_wait_unguarded(&full_bar[s], ph);
    __syncwarp();
    wgmma_fence();
    wgmma_fence_acc(acc[0]);
    wgmma_fence_acc(acc[1]);
    for (int ch = 0; ch < nch; ++ch) {
      const uint32_t a_addr = smem0 + s * stage_bytes + ch * Cfg::STAGE_BYTES;
      const uint32_t b_addr = a_addr + Cfg::A_BYTES;
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t bd = TB ? gmma_desc(b_addr + k * 2048, BK * 128, 1024) : gmma_desc(b_addr + k * 32, 16, 1024);
        const uint32_t accum = (i > 0 || ch > 0 || k > 0) ? 1u : 0u;
#pragma unroll
        for (int h = 0; h < 2; ++h) wgmma_bf16<BN, 0, TB>(acc[h], gmma_desc(a_addr + h * (64 * 128) + k * 32, 16, 1024), bd, accum);
      }
    }
    wgmma_commit();
    wgmma_wait<1>();
    wgmma_fence_acc(acc[0]);
    wgmma_fence_acc(acc[1]);
    if (prev >= 0) {
      __syncwarp();
      mbar_arrive_if(&empty_bar[prev], lane == 0);
    }
    prev = s;
    if (++s == STAGES) { s = 0; ph ^= 1; }
    if (pass_bar && i + KCH >= n_iters) {
      // the tile's inputs in the ring stage after its operands (see the consumer loop of gemm_pingpong_kernel): that stage's
      // slot was last held by an operand stage of this tile that has just been handed back, so the producer can fill it
      if (in_stage) mbar_wait_unguarded(&full_bar[s], ph);
      named_bar_arrive(pass_bar, 2 * 128);
    }
  }
  wgmma_wait<0>();
  wgmma_fence_acc(acc[0]);
  wgmma_fence_acc(acc[1]);
  if (prev >= 0) {
    __syncwarp();
    mbar_arrive_if(&empty_bar[prev], lane == 0);
  }
}

// ---- weight-gradient epilogue: out[tap * N + n] of rows m += acc * scale[m], straight from the wgmma fragment ----------------------
// Fragment layout of m64nNk16 (f32): warp w of the warpgroup holds rows 16w + lane/4 (d[4j], d[4j+1]) and 16w + lane/4 + 8
// (d[4j+2], d[4j+3]) at columns 8j + 2 (lane % 4) + {0, 1}.
// STORE (deterministic mode, K split): the scaled partial goes to the split's own workspace plane with plain stores instead; the
// planes are added into out in split order by wgrad_split_reduce_kernel.
template <int BN, bool STORE = false>
__device__ __forceinline__ void wgrad_epilogue(const float (&acc)[BN / 2], float* obase, int64_t out_ld, const float* scale, int M, int N, int r0,
                                               int n0, int lane) {
  const int r1 = r0 + 8;
  const float rs0 = (r0 < M && scale) ? scale[r0] : 1.0f;
  const float rs1 = (r1 < M && scale) ? scale[r1] : 1.0f;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int n = n0 + j * 8 + 2 * (lane & 3);
    if (n < N) {     // N % 8 == 0: the pair n, n + 1 is inside
      if constexpr (STORE) {
        if (r0 < M) *reinterpret_cast<float2*>(obase + static_cast<int64_t>(r0) * out_ld + n) = make_float2(acc[4 * j] * rs0, acc[4 * j + 1] * rs0);
        if (r1 < M) *reinterpret_cast<float2*>(obase + static_cast<int64_t>(r1) * out_ld + n) = make_float2(acc[4 * j + 2] * rs1, acc[4 * j + 3] * rs1);
      } else {
        if (r0 < M) red_add_f32x2(obase + static_cast<int64_t>(r0) * out_ld + n, acc[4 * j] * rs0, acc[4 * j + 1] * rs0);
        if (r1 < M) red_add_f32x2(obase + static_cast<int64_t>(r1) * out_ld + n, acc[4 * j + 2] * rs1, acc[4 * j + 3] * rs1);
      }
    }
  }
}

// Shared-memory address of 16 bytes (8 bf16 columns, chunk q = 0..7 of the 128-byte row) in row r of a 128B-swizzled TMA box
// (1024-byte aligned): the 16-byte chunks of a row are permuted by r % 8, so the 8 consecutive rows a quarter-warp reads at the
// same logical chunk fall into 8 different bank groups.
__device__ __forceinline__ uint32_t swz128(uint32_t box, int r, int q) { return box + r * 128 + ((q ^ (r & 7)) << 4); }

// ---- TN / NN producer: one ring stage of a tile ----------------------------------------------------------------------------------
// k-chunks i .. i + nch - 1 of the tile at (m0, n0) into `stage`: the A rows shifted by the chunk's tap (9 taps of a 3x3 conv over a
// zero-bordered activation, or row taps), B K-major (TN) or MN-major (NN: one 3-D box or BN / 64 2-D boxes per chunk).
template <int BN, int MODE>
__device__ __forceinline__ void load_operand_stage(uint8_t* stage, const CUtensorMap* tmA, const CUtensorMap* tmB, uint64_t* bar, TileInfo t, int i,
                                                   int nch, int kc_per_tap, int K, int N, int ntaps, int tap_w, int tap_sign, int mn3d) {
  using Cfg = GemmCfg<BN>;
  constexpr int B_BOXES = (MODE == 0) ? 1 : BN / 64;
  // the producer thread is issue-bound: per-chunk index math is done once, box loops are fully unrolled
  int tp = 0, kc = i;
  if (ntaps > 1) { tp = i / kc_per_tap; kc = i - tp * kc_per_tap; }
  for (int ch = 0; ch < nch; ++ch) {
    uint8_t* sa = stage + ch * Cfg::STAGE_BYTES;
    uint8_t* sb = sa + Cfg::A_BYTES;
    int shift = 0;
    if (ntaps == 9) shift = tap_sign * ((tp / 3 - 1) * tap_w + (tp % 3 - 1));
    else if (ntaps > 1) shift = tap_sign * tp * tap_w;        // row taps (space-to-depth stem): tap t reads row m + t * tap_w
    tma_load_2d(sa, tmA, bar, kc * BK, t.m0 + shift);
    if (MODE == 0) {
      tma_load_2d(sb, tmB, bar, tp * K + kc * BK, t.n0);
    } else if (mn3d) {
      tma_load_3d(sb, tmB, bar, 0, kc * BK, (tp * N + t.n0) >> 6);
    } else {
#pragma unroll
      for (int j = 0; j < B_BOXES; ++j) tma_load_2d(sb + j * (BK * 128), tmB, bar, tp * N + t.n0 + j * 64, kc * BK);
    }
    if (++kc == kc_per_tap) { kc = 0; ++tp; }
  }
}

// ---- TN / NN epilogue -------------------------------------------------------------------------------------------------------------
// Output row of A-row m: re-mapped between zero-bordered and compact pixel rows where asked; -1 = not written (m >= M, or a border
// row under UNPAD). Output rows are int: cb_gemm's row counts are.
__device__ __forceinline__ int output_row(const GemmEpi& epi, int m, int M) {
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
  return row_ok ? static_cast<int>(orow) : -1;
}

// The launch's epilogue kind (see the EK_* functions) and switches, fixed per launch.
struct EpiKind {
  int kind;
  bool relu, guard, has_res, has_aux, has_shift, has_out2;
};
__device__ __forceinline__ EpiKind epilogue_kind(const GemmEpi& epi, int N) {
  EpiKind k;
  k.has_res = epi.residual != nullptr;
  k.has_aux = epi.aux != nullptr;
  k.has_shift = epi.shift != nullptr;
  k.has_out2 = epi.out2 != nullptr;
  const bool full = (N & 15) == 0 && epi.scale == nullptr;
  const bool drop = epi.drop_thresh != 0;
  k.kind = EK_GENERIC;
  if (full) {
    if (!drop && !k.has_out2 && !k.has_aux && (epi.act == CB_ACT_NONE || epi.act == CB_ACT_RELU)) k.kind = EK_SHIFT_ACT;
    else if (!drop && !k.has_out2 && !k.has_shift && k.has_aux && epi.aux_mode == CB_AUX_RELU_MASK && epi.act == CB_ACT_NONE) k.kind = EK_RELU_MASK;
    else if (drop && !k.has_out2 && !k.has_aux && epi.act == CB_ACT_NONE) k.kind = EK_DROP_RES;
    else if (!drop && k.has_out2 && !k.has_aux && !k.has_res && epi.act == CB_ACT_GELU_STASH_GRAD) k.kind = EK_GELU_STASH;
    else if (!drop && !k.has_out2 && !k.has_shift && k.has_aux && epi.aux_mode == CB_AUX_MUL && epi.act == CB_ACT_NONE) k.kind = EK_AUX_MUL;
  }
  k.relu = epi.act == CB_ACT_RELU;
  k.guard = (N & 15) != 0;                 // ragged last 16 columns: per-vector column checks in the generic epilogue
  return k;
}

// One lane's 16 columns [nb, nb + 16) of output row orow (nb < N): the fp32 values from its staging row at srow, the residual /
// aux 16-byte chunks q, q + 1 of row brow of their 128B-swizzled [128 x 64] boxes (zeros beyond N), the fused epilogue, 16-byte
// stores.
__device__ __forceinline__ void epilogue_store16(const GemmEpi& epi, const EpiKind& ek, uint64_t dseed, uint32_t srow, int64_t orow, int nb, int N,
                                                 uint32_t res_box, uint32_t aux_box, int brow, int q) {
  constexpr int NC = 16;
  float f[NC];
#pragma unroll
  for (int j = 0; j < NC / 4; ++j) {
    const uint4 u = lds128(srow + j * 16);
    f[4 * j] = __uint_as_float(u.x); f[4 * j + 1] = __uint_as_float(u.y);
    f[4 * j + 2] = __uint_as_float(u.z); f[4 * j + 3] = __uint_as_float(u.w);
  }
  uint32_t res16[NC / 2], aux16[NC / 2];
  if (ek.has_res) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const uint4 u = lds128(swz128(res_box, brow, q + j));
      res16[4 * j] = u.x; res16[4 * j + 1] = u.y; res16[4 * j + 2] = u.z; res16[4 * j + 3] = u.w;
    }
  }
  if (ek.has_aux) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const uint4 u = lds128(swz128(aux_box, brow, q + j));
      aux16[4 * j] = u.x; aux16[4 * j + 1] = u.y; aux16[4 * j + 2] = u.z; aux16[4 * j + 3] = u.w;
    }
  }
  float shv[NC];                                  // shift (bias / FrozenBN shift) of these columns
  if (ek.has_shift) {
#pragma unroll
    for (int j = 0; j < NC; j += 4) {
      float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
      if (nb + j + 4 <= N) s4 = __ldg(reinterpret_cast<const float4*>(epi.shift + nb + j));
      shv[j] = s4.x; shv[j + 1] = s4.y; shv[j + 2] = s4.z; shv[j + 3] = s4.w;
    }
  }
  uint32_t o2_16[NC / 2];
  switch (ek.kind) {
    case EK_SHIFT_ACT: epilogue_shift_act<NC>(f, shv, ek.has_shift, res16, ek.has_res, ek.relu); break;
    case EK_RELU_MASK: epilogue_relu_mask<NC>(f, res16, ek.has_res, aux16); break;
    case EK_DROP_RES:
      epilogue_drop_res<NC>(f, shv, ek.has_shift, res16, ek.has_res, dseed, static_cast<uint64_t>(orow) * static_cast<uint64_t>(N) + nb,
                            epi.drop_thresh, epi.drop_inv_keep);
      break;
    case EK_GELU_STASH: epilogue_gelu_stash<NC>(f, shv, ek.has_shift, o2_16); break;
    case EK_AUX_MUL: epilogue_aux_mul<NC>(f, res16, ek.has_res, aux16); break;
    default:
      if (ek.guard) epilogue_math<NC, true>(f, epi, shv, ek.has_shift, dseed, nb, N, orow, res16, ek.has_res, aux16, ek.has_aux, o2_16, ek.has_out2);
      else epilogue_math<NC, false>(f, epi, shv, ek.has_shift, dseed, nb, N, orow, res16, ek.has_res, aux16, ek.has_aux, o2_16, ek.has_out2);
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
  if (ek.has_out2) {
    __nv_bfloat16* o = epi.out2 + orow * epi.out2_ld + nb;
#pragma unroll
    for (int j = 0; j < 2; ++j)
      if (nb + 8 * j + 8 <= N) *reinterpret_cast<uint4*>(o + 8 * j) = make_uint4(o2_16[4 * j], o2_16[4 * j + 1], o2_16[4 * j + 2], o2_16[4 * j + 3]);
  }
}

// ===================================== TN / NN: ping-pong consumers =====================================
template <int BN, int MODE>
__global__ void __launch_bounds__(PP_THREADS, 1)
    gemm_pingpong_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmR,
                         const __grid_constant__ CUtensorMap tmX, int M, int N, int K, int ntaps, int tap_w, int tap_sign, int tiles_m,
                         int tiles_n, int total_tiles, int STAGES, int KCH, int N_IN, GemmEpi epi) {
  static_assert(MODE != 1 && BN <= 128, "TN / NN tiles of 128 x 64 or 128 x 128");
  using Cfg = GemmCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const int stage_bytes = KCH * Cfg::STAGE_BYTES;           // a stage holds KCH consecutive 64-deep k-chunks (one barrier round trip)
  // epilogue inputs of one tile: the residual boxes, then the aux boxes, BN / 64 of each. N_IN = 2: one dedicated buffer per
  // consumer; N_IN = 1: one buffer the consumers take in turn; N_IN = 0 with inputs: they occupy the ring stage after the
  // tile's operands (in_bytes <= stage_bytes), so that a long K loop keeps the whole ring for its operands
  const bool has_res = epi.residual != nullptr, has_aux = epi.aux != nullptr;
  constexpr int IN_TILE_BYTES = (BN / 64) * IN_BOX_BYTES;
  const int in_bytes = (has_res + has_aux) * IN_TILE_BYTES;
  uint8_t* in_base = smem + STAGES * stage_bytes;           // (1024-byte aligned: stage sizes are multiples of 8 KB)
  uint8_t* stg_base = in_base + N_IN * in_bytes;            // epilogue staging
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stg_base + EPI_BYTES);
  uint64_t* empty_bar = full_bar + MAX_STAGES;
  uint64_t* in_full = empty_bar + MAX_STAGES;               // [consumer]: that consumer's tile inputs have landed
  uint64_t* in_empty = in_full + 2;                         // [buffer]: its consumer is done with it

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);   // warp-uniform for the compiler
  const int lane = threadIdx.x & 31;
  const int unit = blockIdx.x;                                          // persistent work unit
  const int n_units = gridDim.x;
  if (threadIdx.x == 0) dbg_stamp(epi, 0);   // (debug-only buffer, not produced by any kernel: safe before pdl_wait)
  pdl_trigger();   // PDL: let the next kernel's CTAs take this SM as soon as this CTA leaves it
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (has_res) tma_prefetch_desc(&tmR);
    if (has_aux) tma_prefetch_desc(&tmX);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);            // a stage is read by ONE consumer warpgroup
    }
    for (int b = 0; b < 2; ++b) {
      mbar_init(&in_full[b], 1);
      mbar_init(&in_empty[b], 4);
    }
    fence_mbar_init();
  }
  __syncthreads();
  const int kc_per_tap = (K + BK - 1) / BK;
  const int n_iters = ntaps * kc_per_tap;                       // the same for every tile
  const bool in_stage = in_bytes && !N_IN;
  const int tile_stages = (n_iters + KCH - 1) / KCH + (in_stage ? 1 : 0);   // ring stages one tile takes
  // PDL: barrier init and descriptor prefetch above overlapped the previous kernel's tail; from here on this kernel touches
  // global memory (TMA loads, epilogue loads/stores), so its producers must have completed.
  pdl_wait();
  if (threadIdx.x == 0) dbg_stamp(epi, 1);

  if (warp < 4) {
    // ===================== TMA producer warpgroup =====================
    setmaxnreg_dec<PP_PRODUCER_REGS>();
    if (warp == 0 && lane == 0) {
      int s = 0;        // smem ring position / phase, carried across tiles
      uint32_t ph = 0;
      // residual / aux boxes of a tile into its input buffer, or into the next ring stage (N_IN = 0); rows and columns outside
      // [M, N] arrive as zeros
      auto load_inputs = [&](int tile) {
        const TileInfo t = decode_tile<BN>(tile, tiles_m, tiles_n);
        uint64_t* bar;
        uint8_t* dst;
        if (N_IN) {
          const int local = (tile - unit) / n_units;
          const int b = N_IN == 2 ? (local & 1) : 0;
          const int uses = N_IN == 2 ? (local >> 1) : local;     // earlier tiles of this buffer
          mbar_wait(&in_empty[b], (static_cast<uint32_t>(uses) & 1u) ^ 1u);
          bar = &in_full[local & 1];
          dst = in_base + b * in_bytes;
        } else {
          mbar_wait(&empty_bar[s], ph ^ 1);
          bar = &full_bar[s];
          dst = smem + s * stage_bytes;
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
        mbar_expect_tx(bar, in_bytes);
        if (has_res) {
#pragma unroll
          for (int j = 0; j < BN / 64; ++j) tma_load_2d(dst + j * IN_BOX_BYTES, &tmR, bar, t.n0 + j * 64, t.m0);
          dst += IN_TILE_BYTES;
        }
        if (has_aux) {
#pragma unroll
          for (int j = 0; j < BN / 64; ++j) tma_load_2d(dst + j * IN_BOX_BYTES, &tmX, bar, t.n0 + j * 64, t.m0);
        }
      };
      int pend = -1;    // tile whose inputs wait for the next tile's operands
      for (int tile = unit; tile < total_tiles; tile += n_units) {
        const TileInfo t = decode_tile<BN>(tile, tiles_m, tiles_n);
        // A CTA's first N_IN tiles find their input buffer free: their inputs go out ahead of the operands. A later tile's
        // inputs wait for the buffer (the epilogue N_IN tiles back), so they go out after the NEXT tile's operands: that wait
        // never holds back operands the ring has room for, and the inputs still land under the tile's own main loop. In the
        // ring (N_IN = 0) they take the stage after the tile's operands.
        const bool inputs_first = tile < unit + N_IN * n_units;
        if (in_bytes && N_IN && inputs_first) load_inputs(tile);
        for (int i = 0; i < n_iters; i += KCH) {
          const int nch = min(KCH, n_iters - i);
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_expect_tx(&full_bar[s], nch * Cfg::STAGE_BYTES);
          load_operand_stage<BN, MODE>(smem + s * stage_bytes, &tmA, &tmB, &full_bar[s], t, i, nch, kc_per_tap, K, N, ntaps, tap_w, tap_sign,
                                       epi.mn3d);
          if (++s == STAGES) { s = 0; ph ^= 1; }
          if (i == 0 && tile == unit) dbg_stamp(epi, 2);
        }
        if (in_stage) load_inputs(tile);
        if (pend >= 0) load_inputs(pend);
        pend = (in_bytes && N_IN && !inputs_first) ? tile : -1;
      }
      if (pend >= 0) load_inputs(pend);
      dbg_stamp(epi, 3);
    }
    return;
  }

  // ===================== consumer warpgroups: wgmma main loop + epilogue, ping-pong over the CTA's tiles =====================
  setmaxnreg_inc<PP_CONSUMER_REGS>();
  const int wg = (warp >> 2) - 1;           // consumer 0 / 1: local tiles 0, 2, 4, ... / 1, 3, 5, ...
  const int wq = warp & 3;                  // rows 16 wq .. 16 wq + 15 of each 64-row half of the tile
  const uint32_t smem0 = smem_u32(smem);
  const uint64_t dseed = epi.drop_thresh ? drop_seed(epi.seed, epi.seed_off) : 0ull;   // after pdl_wait: the word is device data
  float acc[2][BN / 2];
  // ring position / phase: a consumer reads its own tiles' stages and steps over the other consumer's (tile_stages each).
  // A wait on a stage never runs two phases ahead of it: the turn barrier orders this consumer's main loop after the other's
  // wait on every stage of the previous tile (its inputs included, see mma_tile_pp).
  int s = 0;
  uint32_t ph = 0;
  auto ring_skip = [&](int n) {
    s += n;
    while (s >= STAGES) { s -= STAGES; ph ^= 1; }
  };
  if (wg == 1) ring_skip(tile_stages);

  // epilogue: lane (er, eh) handles row er of the warp's 16, columns eh * 16 .. eh * 16 + 15 of each 32-column slice
  const int er = lane & 15, eh = lane >> 4;
  float* stg = reinterpret_cast<float*>(stg_base) + (warp - 4) * STG_WARP_FLOATS;
  const EpiKind ek = epilogue_kind(epi, N);

  for (int local = wg, tile = unit + wg * n_units; tile < total_tiles; local += 2, tile += 2 * n_units) {
    const TileInfo t = decode_tile<BN>(tile, tiles_m, tiles_n);
    if (local > 0) named_bar_sync(PP_BAR_TURN + wg, 2 * 128);         // the other consumer has issued tile local - 1
    const int pass = tile + n_units < total_tiles ? PP_BAR_TURN + (wg ^ 1) : 0;
    mma_tile_pp<BN, MODE != 0>(acc, smem0, stage_bytes, KCH, STAGES, n_iters, lane, s, ph, full_bar, empty_bar, pass, in_stage);

    // this tile's epilogue inputs (residual boxes, then aux boxes): this consumer's buffer (N_IN = 2), the shared one (N_IN = 1),
    // or the ring stage after the tile's operands (N_IN = 0)
    const uint32_t in_buf = N_IN ? smem_u32(in_base) + (N_IN == 2 ? wg : 0) * in_bytes : smem0 + s * stage_bytes;
    if (in_bytes) {
      if (N_IN) mbar_wait_unguarded(&in_full[wg], static_cast<uint32_t>(local >> 1) & 1u);
      else mbar_wait_unguarded(&full_bar[s], ph);
    }
    // this lane's row in each 64-row half: A-row space m (residual / aux) -> output row (re-mapped; -1 = not written)
    int orow_half[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) orow_half[h] = output_row(epi, t.m0 + h * 64 + wq * 16 + er, M);
    // per 32-column slice, the staging pass of each half: rows wrow .. wrow + 15 of the tile from accumulator half h
#pragma unroll
    for (int sc = 0; sc < BN / 32; ++sc) {
      // (not unrolled: two interleaved copies of the fused epilogue would not fit the consumer's registers beside the
      // accumulators; the half is picked per element with a select)
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        const int wrow = h * 64 + wq * 16;
        // fragment -> staging: this warp's 16 rows x 32 columns, then one row segment per lane
        __syncwarp();
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int j = sc * 4 + jj;
          float* p = stg + (lane >> 2) * STG_PITCH + jj * 8 + 2 * (lane & 3);
          const bool h1 = h != 0;
          *reinterpret_cast<float2*>(p) = make_float2(h1 ? acc[1][4 * j] : acc[0][4 * j], h1 ? acc[1][4 * j + 1] : acc[0][4 * j + 1]);
          *reinterpret_cast<float2*>(p + 8 * STG_PITCH) =
              make_float2(h1 ? acc[1][4 * j + 2] : acc[0][4 * j + 2], h1 ? acc[1][4 * j + 3] : acc[0][4 * j + 3]);
        }
        __syncwarp();
        const int nb = t.n0 + sc * 32 + eh * 16;        // global column of f[0]
        const int64_t orow = h ? orow_half[1] : orow_half[0];
        if (orow < 0 || nb >= N) continue;
        // residual / aux of these 16 columns: box (tile column / 64)
        const int tc = sc * 32 + eh * 16;               // tile column of f[0]
        const uint32_t res_box = in_buf + (tc >> 6) * IN_BOX_BYTES;
        epilogue_store16(epi, ek, dseed, smem_u32(stg + er * STG_PITCH + eh * 16), orow, nb, N, res_box,
                         res_box + (has_res ? IN_TILE_BYTES : 0), wrow + er, (tc & 63) >> 3);
      }
    }
    if (in_bytes) {                                 // this warp is done with the tile's inputs: hand the buffer / stage back
      __syncwarp();
      if (lane == 0) mbar_arrive(N_IN ? &in_empty[N_IN == 2 ? wg : 0] : &empty_bar[s]);
      if (!N_IN && ++s == STAGES) { s = 0; ph ^= 1; }
    }
    ring_skip(tile_stages);                         // past the other consumer's next tile
  }
  if (threadIdx.x == 4 * 32) dbg_stamp(epi, 11);
}

// ===================================== TN / NN: one 128 x 256 tile on both consumers =====================================
// Warpgroup 0 is the TMA producer as in gemm_pingpong_kernel; consumer warpgroup g multiplies rows 64g .. 64g + 63 of the CTA's
// current tile with one wgmma m64n256k16 per k16 step (mma_tile, 128 accumulators per thread) and runs their epilogue, one tile at
// a time: only the producer's run-ahead into the next tile overlaps an epilogue. A stage is read by both consumers, so its empty
// barrier counts all eight consumer warps. The epilogue inputs (residual / aux, four [128 x 64] boxes each, 64 KB per input) fit
// neither one ring stage nor a buffer beside a ring of four 48 KB stages, and three stages leave the main loop short of operands
// (H100: 0.9 against 0.6 us per k-chunk). So they travel through the ring itself: after a tile's last operand stage the producer
// fills one ring stage per 64 output columns with that column block's residual box and aux box, and the consumer warps hand the
// stage back once both 32-column slices of the block are written. Those stages load under the end of the tile's main loop, and
// the next tile's operands follow as the epilogue frees them.
template <int MODE>
__global__ void __launch_bounds__(PP_THREADS, 1)
    gemm_coop_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmR,
                     const __grid_constant__ CUtensorMap tmX, int M, int N, int K, int ntaps, int tap_w, int tap_sign, int tiles_m, int tiles_n,
                     int total_tiles, int STAGES, int KCH, GemmEpi epi) {
  static_assert(MODE != 1, "TN / NN only");
  constexpr int BN = 256;
  using Cfg = GemmCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const int stage_bytes = KCH * Cfg::STAGE_BYTES;
  const bool has_res = epi.residual != nullptr, has_aux = epi.aux != nullptr;
  const int n_in = has_res + has_aux;                       // input boxes per 64 columns (one ring stage)
  uint8_t* stg_base = smem + STAGES * stage_bytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stg_base + EPI_BYTES);
  uint64_t* empty_bar = full_bar + MAX_STAGES;

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);   // warp-uniform for the compiler
  const int lane = threadIdx.x & 31;
  const int unit = blockIdx.x, n_units = gridDim.x;
  pdl_trigger();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (has_res) tma_prefetch_desc(&tmR);
    if (has_aux) tma_prefetch_desc(&tmX);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  __syncthreads();
  const int kc_per_tap = (K + BK - 1) / BK;
  const int n_iters = ntaps * kc_per_tap;
  pdl_wait();

  if (warp < 4) {
    // ===================== TMA producer warpgroup =====================
    setmaxnreg_dec<PP_PRODUCER_REGS>();
    if (warp == 0 && lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int tile = unit; tile < total_tiles; tile += n_units) {
        const TileInfo t = decode_tile<BN>(tile, tiles_m, tiles_n);
        for (int i = 0; i < n_iters; i += KCH) {
          const int nch = min(KCH, n_iters - i);
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_expect_tx(&full_bar[s], nch * Cfg::STAGE_BYTES);
          load_operand_stage<BN, MODE>(smem + s * stage_bytes, &tmA, &tmB, &full_bar[s], t, i, nch, kc_per_tap, K, N, ntaps, tap_w, tap_sign,
                                       epi.mn3d);
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
        // epilogue inputs, one ring stage per 64 columns: residual box, then aux box (rows and columns outside [M, N] arrive as zeros)
        for (int j = 0; n_in && j < BN / 64; ++j) {
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_expect_tx(&full_bar[s], n_in * IN_BOX_BYTES);
          uint8_t* dst = smem + s * stage_bytes;
          if (has_res) tma_load_2d(dst, &tmR, &full_bar[s], t.n0 + j * 64, t.m0);
          if (has_aux) tma_load_2d(dst + (has_res ? IN_BOX_BYTES : 0), &tmX, &full_bar[s], t.n0 + j * 64, t.m0);
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroups: rows 64 wg .. 64 wg + 63 of every tile =====================
  setmaxnreg_inc<PP_CONSUMER_REGS>();
  const int wg = (warp >> 2) - 1;
  const int wq = warp & 3;                  // rows 16 wq .. 16 wq + 15 of the warpgroup's 64
  const uint32_t smem0 = smem_u32(smem);
  const uint64_t dseed = epi.drop_thresh ? drop_seed(epi.seed, epi.seed_off) : 0ull;   // after pdl_wait: the word is device data
  const EpiKind ek = epilogue_kind(epi, N);
  // epilogue: lane (er, eh) handles row er of the warp's 16, columns eh * 16 .. eh * 16 + 15 of each 32-column slice
  const int er = lane & 15, eh = lane >> 4;
  const int brow = wg * 64 + wq * 16 + er;  // this lane's tile row
  float* stg = reinterpret_cast<float*>(stg_base) + (warp - 4) * STG_WARP_FLOATS;
  float acc[BN / 2];
  int s = 0;
  uint32_t ph = 0;
  for (int tile = unit; tile < total_tiles; tile += n_units) {
    const TileInfo t = decode_tile<BN>(tile, tiles_m, tiles_n);
    mma_tile<BN, 0, MODE != 0>(acc, smem0, stage_bytes, KCH, STAGES, n_iters, wg, lane, s, ph, full_bar, empty_bar);
    const int orow = output_row(epi, t.m0 + brow, M);
#pragma unroll
    for (int j = 0; j < BN / 64; ++j) {
      // the residual and aux boxes of columns 64 j .. 64 j + 63, in ring stage s
      if (n_in) mbar_wait_unguarded(&full_bar[s], ph);
      const uint32_t res_box = smem0 + s * stage_bytes;
      const uint32_t aux_box = res_box + (has_res ? IN_BOX_BYTES : 0);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int sc = 2 * j + h;
        // fragment -> staging: this warp's 16 rows x 32 columns, then one row segment per lane
        __syncwarp();
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int f = sc * 4 + jj;
          float* p = stg + (lane >> 2) * STG_PITCH + jj * 8 + 2 * (lane & 3);
          *reinterpret_cast<float2*>(p) = make_float2(acc[4 * f], acc[4 * f + 1]);
          *reinterpret_cast<float2*>(p + 8 * STG_PITCH) = make_float2(acc[4 * f + 2], acc[4 * f + 3]);
        }
        __syncwarp();
        const int tc = sc * 32 + eh * 16;               // tile column of this lane's 16
        const int nb = t.n0 + tc;
        if (orow >= 0 && nb < N)
          epilogue_store16(epi, ek, dseed, smem_u32(stg + er * STG_PITCH + eh * 16), orow, nb, N, res_box, aux_box, brow, (tc & 63) >> 3);
      }
      if (n_in) {                               // this warp is done with the boxes: hand the stage back
        __syncwarp();
        mbar_arrive_if(&empty_bar[s], lane == 0);
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
    }
  }
}

static int g_sm_limit = 0;   // tuning hook: cap on the persistent grid (0 = every SM). A long-running co-resident kernel (an NCCL
                              // all-reduce overlapped with the backward pass) pins some SMs for its whole duration; with the static
                              // round-robin tile schedule the CTAs that cannot be placed run as a second wave. Capping the grid at
                              // the SM count minus the co-resident kernel's CTAs avoids the second wave.
static int sm_count_device() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}
static int sm_count() {
  const int n = sm_count_device();
  return (g_sm_limit > 0 && g_sm_limit < n) ? g_sm_limit : n;
}
// SMs the launch plan (tile width, K-split) is chosen for. In deterministic mode the split decides the summation order, so it
// depends on the problem shape and the device only, never on the grid cap; the grid itself may still be capped.
static int plan_sm_count() { return g_det.load(std::memory_order_relaxed) ? sm_count_device() : sm_count(); }

static long long* g_gemm_timeline = nullptr;
static int g_mn3d = 1;        // 1 (default) = MN-major operands through one 3-D TMA box per k-chunk (GemmEpi::mn3d); cb_debug_gemm_mn3d


// Shared-memory plan of one launch: the epilogue staging (TN / NN: 16 x 32 fp32 per consumer warp; WGRAD: none), n_in
// epilogue-input buffers of in_bytes (the residual / aux boxes of one tile), then as many 64-deep operand chunks as fit, grouped
// KCH per stage. Every stage costs one full / empty barrier round trip whatever its size, so deep stages are preferred to many
// shallow ones, except that a K loop longer than the ring keeps at least three stages. Ring depth cap:
//   WGRAD (one tile at a time): the K loop plus one stage.
//   TN / NN (ping-pong): both consumers' current tiles plus one stage, so that the producer has the next tile's first stage
//   in flight while the two tiles in hand are multiplied and the other consumer's epilogue runs. For the one-chunk 1x1 convs
//   that is three stages.
// Epilogue inputs (residual / aux boxes of one tile, in_bytes): two dedicated buffers, one per consumer, let a tile's inputs
// load under the other consumer's epilogue; they are taken when the ring beside them still holds a whole tile's K loop (the
// short K loops of the HBM-bound 1x1 convs). A K loop of at most 4 chunks that cannot have both gets one buffer. A longer K loop
// keeps the ring it has without inputs and lands its inputs in the ring stage after its operands (n_in = 0; needs in_bytes <=
// one stage): they load under the end of its main loop, and the buffer does not cost the compute-bound main loop ring depth.
struct SmemPlan {
  int epi_bytes, kch, stages, chunk_bytes, n_in;
};
static SmemPlan plan_ring(int bn, bool staging, int kiters, int force_kch, int in_bytes, int n_in) {
  SmemPlan p;
  const int limit = SMEM_LIMIT;
  p.chunk_bytes = BM * BK * 2 + bn * BK * 2;
  p.epi_bytes = staging ? EPI_BYTES : 0;
  p.n_in = n_in;
  const int chunks_fit = (limit - 1024 - GemmCfg<64>::BAR_BYTES - p.epi_bytes - n_in * in_bytes) / p.chunk_bytes;
  // K loop longer than the ring: the ring cycles within a tile, and the stage count, not the stage size, sets how far the
  // producer runs ahead. A stage depth is only taken if it leaves at least three stages (TN / NN 64-wide: four stages of two
  // instead of two of four; WGRAD 128 x 256: four one-chunk stages instead of two of two). H100, 128 x 64 TN / NN tiles, 9-tap
  // convs: two stages of four chunks ran 1.4-1.8 x slower than four stages of two.
  const int min_stages = kiters > chunks_fit ? 3 : 2;
  p.kch = 1;
  if (force_kch > 0) p.kch = force_kch;
  else if (kiters >= 4 && chunks_fit >= 4 * min_stages) p.kch = 4;
  else if (kiters >= 2 && chunks_fit >= 2 * min_stages) p.kch = 2;
  if (p.kch > kiters) p.kch = kiters;
  if (p.kch > 1 && chunks_fit / p.kch < 2) p.kch = 1;
  p.stages = chunks_fit / p.kch;
  if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
  const int stage_iters = ceil_div(kiters, p.kch);
  const int cap = staging ? 2 * stage_iters + 1 : (stage_iters + 1 > 2 ? stage_iters + 1 : 2);
  if (p.stages > cap) p.stages = cap;
  return p;
}
// TN / NN 128 x 256 (gemm_coop_kernel): the ring alone, four one-chunk stages of 48 KB; epilogue inputs pass through it.
static SmemPlan plan_smem(int bn, bool staging, int kiters, int force_kch = 0, int in_bytes = 0) {
  if (staging && bn == 256) return plan_ring(bn, staging, kiters, force_kch, 0, 0);
  const SmemPlan none = plan_ring(bn, staging, kiters, force_kch, 0, 0);
  if (in_bytes == 0) return none;
  const SmemPlan two = plan_ring(bn, staging, kiters, force_kch, in_bytes, 2);
  if (two.stages >= 2 && two.stages * two.kch >= kiters) return two;
  if (kiters > 4 && none.stages >= 2 && none.kch * none.chunk_bytes >= in_bytes) return none;
  return plan_ring(bn, staging, kiters, force_kch, in_bytes, 1);
}
// bytes of one tile's residual / aux boxes (TN / NN)
static int epi_in_bytes(const cb_gemm_desc& d, int bn) {
  return d.mode == CB_GEMM_WGRAD ? 0 : ((d.residual != nullptr) + (d.aux != nullptr)) * (bn / 64) * IN_BOX_BYTES;
}

// K-splits a launch asked for `want` splits of kc k-chunks runs: every split non-empty
static int real_splits(int kc, int want) {
  const int sp = want < 1 ? 1 : (want > kc ? kc : want);
  return ceil_div(kc, ceil_div(kc, sp));
}

// Deterministic weight gradients with a K-split: out[m, c] += ws[0][m, c] + ws[1][m, c] + ... + ws[S-1][m, c], added one plane
// at a time into a register copy of out (so the order is the split order whatever the grid), 4 columns per thread.
struct SplitReduceJob {
  float* out;
  const float* ws;            // [S][M][W]
  int64_t out_ld;
  int M, W, S;                // W = ntaps * N, a multiple of 8
};
struct SplitReduce {
  int njobs;
  SplitReduceJob j[8];
};
__global__ void __launch_bounds__(256) wgrad_split_reduce_kernel(const __grid_constant__ SplitReduce r) {
  pdl_wait();
  pdl_trigger();
  const SplitReduceJob& J = r.j[blockIdx.y];
  const int w4 = J.W / 4;
  const int64_t total = static_cast<int64_t>(J.M) * w4, plane = static_cast<int64_t>(J.M) * J.W;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * 256 + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * 256) {
    const int64_t m = i / w4;
    const int c = static_cast<int>(i - m * w4) * 4;
    float4* o = reinterpret_cast<float4*>(J.out + m * J.out_ld + c);
    float4 v = *o;
    const float* p = J.ws + m * J.W + c;
    for (int s = 0; s < J.S; ++s) {
      const float4 a = *reinterpret_cast<const float4*>(p + s * plane);
      v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
    }
    *o = v;
  }
}
static int launch_split_reduce(const SplitReduce& r, cudaStream_t stream, const char* what) {
  int64_t most = 0;
  for (int i = 0; i < r.njobs; ++i) most = std::max(most, static_cast<int64_t>(r.j[i].M) * (r.j[i].W / 4));
  const int gx = static_cast<int>(std::min<int64_t>(1024, (most + 255) / 256));
  launch_k(wgrad_split_reduce_kernel, dim3(gx, r.njobs), 256, 0, stream, r);
  return check_launch(what);
}

// MODE 0 / 2 (TN / NN): gemm_pingpong_kernel for BN = 64 / 128, gemm_coop_kernel for BN = 256. One CTA per SM.
template <int BN, int MODE>
static int launch_gemm(const cb_gemm_desc& d, const GemmEpi& epi_in, cudaStream_t stream) {
  GemmEpi epi = epi_in;
  using Cfg = GemmCfg<BN>;
  constexpr bool wide = BN == 256;
  static bool attr_set = false;
  const void* kern = wide ? reinterpret_cast<const void*>(gemm_coop_kernel<MODE>) : reinterpret_cast<const void*>(gemm_pingpong_kernel<wide ? 128 : BN, MODE>);
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(smem=%d): %s", SMEM_LIMIT, cudaGetErrorString(e));
      return CB_ERR_CUDA;
    }
    attr_set = true;
  }
  // Tensor maps are copied out of the cache into this frame (and from here into the kernel's parameter space)
  alignas(64) CUtensorMap ta, tb, tr, tx;
  bool mn3d = false;
  const int tiles_m = ceil_div(d.m, BM), tiles_n = ceil_div(d.n, BN);
  const int total = tiles_m * tiles_n;
  const int kiters = ceil_div(d.k, BK) * d.ntaps;
  bool ok = get_tmap_2d(&ta, d.a, d.k, d.a_rows, d.a_ld, BK, BM);
  if (MODE == 0) {
    ok = ok && get_tmap_2d(&tb, d.b, static_cast<uint64_t>(d.k) * d.ntaps, d.b_rows, d.b_ld, BK, BN);
  } else {
    mn3d = g_mn3d && d.n % 64 == 0 &&
           get_tmap_3d_mn(&tb, d.b, static_cast<uint64_t>(d.n) * d.ntaps, d.b_rows, d.b_ld, BK, BN / 64);
    // not asked for, or the driver refused the 3-D view: the 2-D boxes always work
    if (!mn3d) ok = ok && get_tmap_2d(&tb, d.b, static_cast<uint64_t>(d.n) * d.ntaps, d.b_rows, d.b_ld, 64, BK);
  }
  // epilogue inputs: residual / aux [M, N] at the tile's A rows, 128 x 64 boxes; unused map slots carry a copy of ta
  tr = ta;
  tx = ta;
  if (d.residual) ok = ok && get_tmap_2d(&tr, d.residual, d.n, d.m, d.res_ld, 64, BM);
  if (d.aux) ok = ok && get_tmap_2d(&tx, d.aux, d.n, d.m, d.aux_ld, 64, BM);
  if (!ok) return CB_ERR_CUDA;
  epi.mn3d = mn3d ? 1 : 0;
  const int units = sm_count();
  const int grid = total < units ? total : units;
  const int in_bytes = epi_in_bytes(d, BN);
  const SmemPlan sp = plan_smem(BN, true, kiters, (d.reserved >> 8) & 15, in_bytes);
  const int kch = sp.kch, stages = sp.stages;
  if (stages < 2) {
    set_error("cb_gemm: not enough shared memory for a 2-stage pipeline (BN=%d, epilogue %d B + inputs %d B)", BN, sp.epi_bytes,
              in_bytes);
    return CB_ERR_INVALID;
  }
  const int smem_bytes = stages * kch * Cfg::STAGE_BYTES + sp.n_in * in_bytes + sp.epi_bytes + Cfg::BAR_BYTES + 1024;
  if constexpr (wide)
    launch_gemm_k(gemm_coop_kernel<MODE>, grid, PP_THREADS, smem_bytes, stream, ta, tb, tr, tx, d.m, d.n, d.k, d.ntaps, d.tap_w, d.tap_sign,
                  tiles_m, tiles_n, total, stages, kch, epi);
  else
    launch_gemm_k(gemm_pingpong_kernel<BN, MODE>, grid, PP_THREADS, smem_bytes, stream, ta, tb, tr, tx, d.m, d.n, d.k, d.ntaps, d.tap_w,
                  d.tap_sign, tiles_m, tiles_n, total, stages, kch, sp.n_in, epi);
  return check_launch("cb_gemm");
}

// ------------------------------------------------------------------------------------------------
// Launch configuration: an analytic model picks the tile width (and the wgrad K-split). A persistent CTA's main loop costs about
// (k-iterations x stage bytes) / (operand ingest rate) plus a barrier round trip per stage, and the launch is done when the
// busiest SM is; a per-tile epilogue term is added. In the TN / NN ping-pong kernel a tile's epilogue overlaps the next tile's
// main loop and the other consumer's epilogue: a tile costs max(main loop, (main loop + epilogue) / 2), plus the last
// epilogue's exposed half.
// ------------------------------------------------------------------------------------------------
struct LaunchCfg {
  int bn, splits;
};

static LaunchCfg choose_config(const cb_gemm_desc& d, int units) {
  const int kc = ceil_div(d.k, BK);
  const bool wgrad = d.mode == CB_GEMM_WGRAD;
  if (!wgrad && (d.reserved & CB_GEMM_FORCE_WIDE)) return {256, 1};
  // TN / NN: a ping-pong consumer owning a 128 x 256 tile would need 256 fp32 accumulators per thread, more than its 232
  // registers, so an explicit block_n = 256 runs on 128-wide tiles; the 128 x 256 tile of gemm_coop_kernel is only ever the
  // model's pick (block_n = 0) or forced through reserved
  const int block_n = (!wgrad && d.block_n == 256) ? 128 : d.block_n;
  const bool wide_ok = !wgrad && d.block_n == 0 && !(d.reserved & CB_GEMM_NO_WIDE);
  static const int cand[3] = {64, 128, 256};
  LaunchCfg best = {64, 1};
  double best_cost = 1e30;
  for (int c = 0; c < 3; ++c) {
    const int bn = cand[c];
    if (block_n && bn != block_n) continue;
    if (!wgrad && bn == 256 && !wide_ok) continue;
    if (bn > 64 && d.n <= bn / 2) continue;               // mostly padding
    const int64_t base = static_cast<int64_t>(ceil_div(d.m, BM)) * ceil_div(d.n, bn) * (wgrad ? d.ntaps : 1);
    const int max_split = wgrad ? (d.split_k > 0 ? d.split_k : (kc < 32 ? kc : 32)) : 1;
    for (int sp = (wgrad && d.split_k > 0) ? d.split_k : 1; sp <= max_split; ++sp) {
      const int ips = ceil_div(wgrad ? kc : kc * d.ntaps, sp);
      const int real_sp = wgrad ? ceil_div(kc, ips) : 1;
      const int64_t tiles = base * real_sp;
      const double rounds = static_cast<double>((tiles + units - 1) / units);
      // the ring left beside the epilogue-input buffers of this tile width
      const SmemPlan pl = plan_smem(bn, !wgrad, ips, (d.reserved >> 8) & 15, epi_in_bytes(d, bn));
      if (pl.stages < 2) continue;
      // a ring of 2 chunks cannot cover the TMA round trip of a long K loop
      const double shallow = (pl.stages * pl.kch < 3 && ips > 2) ? 3.0 : 1.0;
      // per stage: ~450-cycle barrier round trip + bytes at ~60 B/clk; per tile: epilogue
      const double stage_cost = 450.0 + pl.kch * pl.chunk_bytes / 60.0;
      const double main_loop = ceil_div(ips, pl.kch) * stage_cost * shallow;
      double cost;
      if (wgrad) {
        cost = rounds * (main_loop + bn * 24.0) + 2500.0;
      } else if (bn == 256) {
        // one tile at a time: its epilogue, on all eight consumer warps, is not overlapped by another tile's main loop; a second
        // output (the gelu' stash) about doubles it. Fitted on an H100 to the TN / NN launches of the training step, each timed
        // on 128 x 256 tiles and on the model's pick of 128 x 64 / 128 x 128 (tools/profile_gemm_launches.py --ab): no pick
        // slower than the other tile
        cost = rounds * (main_loop + bn * 20.0 * (d.out2 ? 2.0 : 1.0)) + 2500.0;
      } else {
        const double epi = bn * 30.0;
        const double per_tile = main_loop > 0.5 * (main_loop + epi) ? main_loop : 0.5 * (main_loop + epi);
        cost = rounds * per_tile + 0.5 * epi + 2500.0;
      }
      // the 128 x 256 tile must beat the best ping-pong width by 5 %: within that the model cannot tell them apart
      if ((bn == 256 && !wgrad ? cost / 0.95 : cost) < best_cost) {
        best_cost = bn == 256 && !wgrad ? cost / 0.95 : cost;
        best = {bn, real_sp};
      }
    }
  }
  return best;
}

// ------------------------------------------------------------------------------------------------
// Weight gradients: ONE persistent launch walks the tiles of a group of independent dW = dY^T X problems. cb_gemm launches a
// single weight gradient as a group of one; cb_gemm_wgrad_group groups several (the four Linear layers of a BertLayer, the
// three / four convs of a bottleneck block). The problems of a group share the reduction length (tokens / pixels), so their
// tiles cost the same and the static round-robin schedule stays balanced; what the group buys is one prologue + one tail
// instead of four, tiles of all problems filling the SMs together, and - because four problems together have enough tiles -
// no K-split, i.e. half the fp32 red.global traffic of the single launches. The problem descriptors (tensor maps included)
// travel in the kernel's parameter space.
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
// DET: problem i's split planes (fp32 [splits][M][ntaps * N]), nullptr when it has one split. A trailing kernel parameter of its
// own, so that the parameters of the default instantiation keep their offsets.
struct WgradWorkspace {
  float* p[WG_MAX_PROBLEMS];
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

// DET: a problem with split planes in ws writes every tile's scaled partial into plane `split` with plain stores; the planes are
// added into out afterwards in split order (deterministic mode with a K-split).
template <int BN, bool DET = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    wgrad_group_kernel(const __grid_constant__ WgradGroup g, int STAGES, int KCH, const __grid_constant__ WgradWorkspace ws) {
  using Cfg = GemmCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const int stage_bytes = KCH * Cfg::STAGE_BYTES;           // a stage holds KCH consecutive 64-deep k-chunks (one barrier round trip)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * stage_bytes);
  uint64_t* empty_bar = full_bar + MAX_STAGES;
  // warp-uniform for the compiler: with a plain threadIdx.x >> 5 ptxas takes the consumer path for divergent and serialises
  // every wgmma behind the warpgroup arrive it inserts (advisory C7520), which leaves one m64nBNk16 in flight per warpgroup
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
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
    if (DET && ws.p[t.pi] != nullptr)
      wgrad_epilogue<BN, true>(acc, ws.p[t.pi] + static_cast<int64_t>(t.it_begin / P.iters_per_split) * P.M * P.ntaps * P.N +
                                        static_cast<int64_t>(t.tap) * P.N,
                               static_cast<int64_t>(P.ntaps) * P.N, P.scale, P.M, P.N, t.m0 + wrow + (lane >> 2), t.n0 * BN, lane);
    else
      wgrad_epilogue<BN>(acc, P.out + static_cast<int64_t>(t.tap) * P.N, P.out_ld, P.scale, P.M, P.N, t.m0 + wrow + (lane >> 2), t.n0 * BN, lane);
  }
}

// The n problems of descs (n = 1 for cb_gemm) with `splits` K-splits each in one launch. The ring stage depth follows
// descs[0].reserved bits 8-11 when set. ws (DET): the split planes of every problem with more than one split, one problem's after
// the previous ones'; a second launch adds them into out in split order.
template <int BN, bool DET>
static int launch_wgrad_group(const cb_gemm_desc* descs, int n, int splits, float* ws, cudaStream_t stream, const char* what) {
  using Cfg = GemmCfg<BN>;
  static bool attr_set = false;
  auto kern = wgrad_group_kernel<BN, DET>;
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
  SplitReduce red;
  red.njobs = 0;
  WgradWorkspace wsp;
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
    const int sp = real_splits(kc, splits);
    P.iters_per_split = ceil_div(kc, sp);
    wsp.p[i] = nullptr;
    if (DET && sp > 1) {
      wsp.p[i] = ws;
      red.j[red.njobs++] = {static_cast<float*>(d.out), ws, d.out_ld, d.m, d.ntaps * d.n, sp};
      ws += static_cast<int64_t>(sp) * d.m * d.ntaps * d.n;
    }
    P.tiles_m = ceil_div(d.m, BM);
    P.tiles_n = ceil_div(d.n, BN);
    P.tile_begin = total;
    total += P.tiles_m * P.tiles_n * d.ntaps * sp;
    if (P.iters_per_split > max_iters) max_iters = P.iters_per_split;
  }
  g.total_tiles = total;
  const SmemPlan sp = plan_smem(BN, false, max_iters, (descs[0].reserved >> 8) & 15);
  if (sp.stages < 2) {
    set_error("%s: not enough shared memory for a 2-stage pipeline (BN=%d)", what, BN);
    return CB_ERR_INVALID;
  }
  const int smem_bytes = sp.stages * sp.kch * Cfg::STAGE_BYTES + Cfg::BAR_BYTES + 1024;
  const int units = sm_count();
  launch_gemm_k(kern, total < units ? total : units, GEMM_THREADS, smem_bytes, stream, g, sp.stages, sp.kch, wsp);
  const int rc = check_launch(what);
  if (rc != CB_OK || red.njobs == 0) return rc;
  return launch_split_reduce(red, stream, what);
}

// Tile width and K-split of a grouped launch (groupable = false: the problems run as separate cb_gemm launches).
struct GroupPlan {
  bool groupable;
  int bn, split;
};
static GroupPlan group_plan(const cb_gemm_desc* descs, int n, int sms) {
  GroupPlan gp = {n >= 2 && n <= WG_MAX_PROBLEMS, 64, 1};
  // one schedule for all: reduction lengths within 2 x of each other, otherwise the round-robin tiles are unbalanced
  for (int i = 0; i < n; ++i)
    if (descs[i].k * 2 < descs[0].k || descs[0].k * 2 < descs[i].k) gp.groupable = false;
  if (!gp.groupable) return gp;
  // tile width: the widest that does not mostly pad, unless descs[0].block_n sets it; K-split: descs[0].split_k, or the one with
  // the least time per CTA
  int min_n = descs[0].n;
  for (int i = 1; i < n; ++i) min_n = descs[i].n < min_n ? descs[i].n : min_n;
  gp.bn = descs[0].block_n ? descs[0].block_n : (min_n >= 192 ? 256 : (min_n >= 96 ? 128 : 64));
  int64_t base = 0;
  int kc_min = 1 << 30, kc_max = 0;
  for (int i = 0; i < n; ++i) {
    base += static_cast<int64_t>(ceil_div(descs[i].m, BM)) * ceil_div(descs[i].n, gp.bn) * descs[i].ntaps;
    const int kc = ceil_div(descs[i].k, BK);
    kc_min = kc < kc_min ? kc : kc_min;
    kc_max = kc > kc_max ? kc : kc_max;
  }
  double best_cost = 1e30;
  for (int sp = 1; sp <= 8 && sp <= kc_min; ++sp) {
    const double waves = static_cast<double>((base * sp + sms - 1) / sms);
    // per wave: the tile's k-chunks, then its red.add epilogue, which takes about as long as 8 chunks of the main loop. Fitted
    // on an H100 to the BertLayer group (2624 tokens, 41 chunks; 128 x 256 tiles, 216 per split), 1 / 2 / 3 splits: 76 / 95 / 90 us
    const double cost = waves * (ceil_div(kc_max, sp) + 8.0);
    if (cost < best_cost) { best_cost = cost; gp.split = sp; }
  }
  if (descs[0].split_k > 0) gp.split = descs[0].split_k;
  return gp;
}

// workspace of one deterministic weight gradient run with `splits` K-splits (none for one split)
static int64_t wgrad_ws_bytes(const cb_gemm_desc& d, int splits) {
  return splits > 1 ? static_cast<int64_t>(splits) * d.m * d.ntaps * d.n * 4 : 0;
}
static int64_t group_ws_bytes(const cb_gemm_desc* descs, int n) {
  const GroupPlan gp = group_plan(descs, n, sm_count_device());
  int64_t bytes = 0;
  for (int i = 0; i < n; ++i) {
    const int64_t b = gp.groupable ? wgrad_ws_bytes(descs[i], real_splits(ceil_div(descs[i].k, BK), gp.split))
                                   : wgrad_ws_bytes(descs[i], choose_config(descs[i], sm_count_device()).splits);
    bytes = gp.groupable ? bytes + b : std::max(bytes, b);     // separate launches run one after another: one workspace for all
  }
  return bytes;
}

// What every weight-gradient descriptor must satisfy, for cb_gemm and for each problem of cb_gemm_wgrad_group.
static int check_wgrad_desc(const cb_gemm_desc& d, const char* who) {
  CB_REQUIRE(d.mode == CB_GEMM_WGRAD && d.out_fp32 == 1, "%s: not an fp32 WGRAD descriptor", who);
  CB_REQUIRE(d.a && d.b && d.out && d.m > 0 && d.n > 0 && d.k > 0, "%s: null operand / empty shape", who);
  CB_REQUIRE(d.m % 8 == 0 && d.n % 8 == 0, "%s: m, n must be multiples of 8 (got %d, %d)", who, d.m, d.n);
  CB_REQUIRE(d.out_ld % 4 == 0, "%s: out_ld must be a multiple of 4", who);
  CB_REQUIRE((reinterpret_cast<uintptr_t>(d.out) & 15) == 0, "%s: out must be 16-byte aligned", who);
  CB_REQUIRE((reinterpret_cast<uintptr_t>(d.a) & 15) == 0 && (reinterpret_cast<uintptr_t>(d.b) & 15) == 0,
             "%s: a and b must be 16-byte aligned (TMA)", who);
  CB_REQUIRE(d.ntaps == 1 || d.ntaps == 9, "%s: ntaps must be 1 or 9 (got %d)", who, d.ntaps);
  return CB_OK;
}

// Every weight-gradient launch, of one problem (what = "cb_gemm") or a group (what = "cb_gemm_wgrad_group"): tile width bn,
// `splits` K-splits per problem. In deterministic mode the split planes need descs[0].workspace (see launch_wgrad_group).
static int launch_wgrad(const cb_gemm_desc* descs, int n, int bn, int splits, cudaStream_t stream, const char* what) {
  int64_t need = 0;
  if (g_det.load(std::memory_order_relaxed))
    for (int i = 0; i < n; ++i) need += wgrad_ws_bytes(descs[i], real_splits(ceil_div(descs[i].k, BK), splits));
  const cb_gemm_desc& d0 = descs[0];
  CB_REQUIRE(need == 0 || (d0.workspace != nullptr && d0.workspace_bytes >= need && (reinterpret_cast<uintptr_t>(d0.workspace) & 15) == 0),
             "%s: deterministic mode needs a 16-byte aligned workspace of %lld bytes in descs[0] (%s_workspace_bytes), got %lld", what,
             static_cast<long long>(need), what, static_cast<long long>(d0.workspace ? d0.workspace_bytes : 0));
  float* ws = static_cast<float*>(d0.workspace);
  switch (bn) {
    case 64: return need ? launch_wgrad_group<64, true>(descs, n, splits, ws, stream, what)
                         : launch_wgrad_group<64, false>(descs, n, splits, ws, stream, what);
    case 128: return need ? launch_wgrad_group<128, true>(descs, n, splits, ws, stream, what)
                          : launch_wgrad_group<128, false>(descs, n, splits, ws, stream, what);
    case 256: return need ? launch_wgrad_group<256, true>(descs, n, splits, ws, stream, what)
                          : launch_wgrad_group<256, false>(descs, n, splits, ws, stream, what);
    default: set_error("%s: block_n must be 0, 64, 128 or 256 (got %d)", what, bn); return CB_ERR_INVALID;
  }
}

}  // namespace cb

/* bring-up / tuning hook (not part of the public header): device buffer of >= 32 x grid int64 receiving clock64() stamps of every CTA */
extern "C" void cb_debug_gemm_timeline(void* device_buf) { cb::g_gemm_timeline = static_cast<long long*>(device_buf); }
extern "C" void cb_debug_gemm_mn3d(int on) { cb::g_mn3d = on ? 1 : 0; }
// Weight gradients used to have a two-CTAs-per-SM instantiation (128 x 64 tiles) selected through this hook. With the wgmma of a
// stage pipelined, it was slower than one CTA per SM on every weight-gradient shape of the step, and it is gone; the hook stays so
// that callers that set it keep working.
extern "C" void cb_debug_gemm_occ2(int, double) {}
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
  // [0, 1] as nn.Dropout; p = 1 drops every element (make_drop)
  CB_REQUIRE(d.dropout_p >= 0.0f && d.dropout_p <= 1.0f, "cb_gemm: dropout_p %g outside [0, 1]", d.dropout_p);

  GemmEpi epi;
  epi.scale = d.scale;
  epi.shift = d.shift;
  epi.residual = static_cast<const __nv_bfloat16*>(d.residual);
  epi.aux = static_cast<const __nv_bfloat16*>(d.aux);
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

  if (d.mode == CB_GEMM_TN || d.mode == CB_GEMM_NN) {
    const bool nn = d.mode == CB_GEMM_NN;
    CB_REQUIRE(d.n % 8 == 0, "cb_gemm(TN): n must be a multiple of 8 (got %d)", d.n);
    CB_REQUIRE(d.k % 8 == 0, "cb_gemm(TN): k must be a multiple of 8 (got %d)", d.k);
    CB_REQUIRE(d.out_ld % 8 == 0, "cb_gemm(TN): out_ld must be a multiple of 8");
    CB_REQUIRE(!d.residual || d.res_ld % 8 == 0, "cb_gemm(TN): res_ld must be a multiple of 8");
    CB_REQUIRE(!d.aux || d.aux_ld % 8 == 0, "cb_gemm(TN): aux_ld must be a multiple of 8");
    CB_REQUIRE((reinterpret_cast<uintptr_t>(d.residual) & 15) == 0, "cb_gemm(TN): residual must be 16-byte aligned");
    CB_REQUIRE((reinterpret_cast<uintptr_t>(d.aux) & 15) == 0, "cb_gemm(TN): aux must be 16-byte aligned");
    // TMA reads A and B from 16-byte aligned bases; the epilogue writes out and out2 as 16-byte vectors
    CB_REQUIRE((reinterpret_cast<uintptr_t>(d.a) & 15) == 0, "cb_gemm(TN): a must be 16-byte aligned");
    CB_REQUIRE((reinterpret_cast<uintptr_t>(d.b) & 15) == 0, "cb_gemm(TN): b must be 16-byte aligned");
    CB_REQUIRE((reinterpret_cast<uintptr_t>(d.out) & 15) == 0, "cb_gemm(TN): out must be 16-byte aligned");
    CB_REQUIRE((reinterpret_cast<uintptr_t>(d.out2) & 15) == 0, "cb_gemm(TN): out2 must be 16-byte aligned");
    CB_REQUIRE(!d.out2 || d.out2_ld % 8 == 0, "cb_gemm(TN): out2_ld must be a multiple of 8");
    CB_REQUIRE(!(d.out2 && d.out_fp32), "cb_gemm(TN): out2 requires a bf16 primary output");
    CB_REQUIRE(d.rowmap == CB_ROWMAP_NONE || (d.map_h > 0 && d.map_w > 0), "cb_gemm: rowmap needs map_h/map_w");
    CB_REQUIRE(d.ntaps == 1 || d.tap_w > 2, "cb_gemm: tap modes need tap_w (padded row pitch in pixels)");
    CB_REQUIRE(d.block_n == 0 || d.block_n == 64 || d.block_n == 128 || d.block_n == 256, "cb_gemm: block_n must be 0, 64, 128 or 256 (got %d)",
               d.block_n);
    const LaunchCfg lc = choose_config(d, sm_count());
    switch (lc.bn) {
      case 64: return nn ? launch_gemm<64, 2>(d, epi, stream) : launch_gemm<64, 0>(d, epi, stream);
      case 128: return nn ? launch_gemm<128, 2>(d, epi, stream) : launch_gemm<128, 0>(d, epi, stream);
      case 256: return nn ? launch_gemm<256, 2>(d, epi, stream) : launch_gemm<256, 0>(d, epi, stream);
      default: CB_REQUIRE(false, "cb_gemm: no tile width for block_n %d", d.block_n);
    }
  } else {
    const int rc = check_wgrad_desc(d, "cb_gemm(WGRAD)");
    if (rc != CB_OK) return rc;
    const LaunchCfg lc = choose_config(d, plan_sm_count());
    return launch_wgrad(&d, 1, lc.bn, lc.splits, stream, "cb_gemm");
  }
  return CB_ERR_INVALID;
}

/* Several independent weight-gradient problems (CB_GEMM_WGRAD descriptors with the same reduction length) in ONE persistent launch. */
extern "C" int cb_gemm_wgrad_group(const cb_gemm_desc* descs, int n, void* stream_v) {
  using namespace cb;
  CB_REQUIRE(descs != nullptr && n >= 1, "cb_gemm_wgrad_group: no problems");
  for (int i = 0; i < n; ++i) {
    char who[48];
    snprintf(who, sizeof(who), "cb_gemm_wgrad_group: problem %d", i);
    const int rc = check_wgrad_desc(descs[i], who);
    if (rc != CB_OK) return rc;
  }
  const GroupPlan gp = group_plan(descs, n, plan_sm_count());
  if (!gp.groupable) {      // a single problem, too many, or very different reduction lengths: the ordinary launches
    for (int i = 0; i < n; ++i) {
      cb_gemm_desc d = descs[i];
      d.workspace = descs[0].workspace;       // stream-ordered launches: one workspace serves them all
      d.workspace_bytes = descs[0].workspace_bytes;
      const int rc = cb_gemm(&d, stream_v);
      if (rc != CB_OK) return rc;
    }
    return CB_OK;
  }
  return launch_wgrad(descs, n, gp.bn, gp.split, static_cast<cudaStream_t>(stream_v), "cb_gemm_wgrad_group");
}

/* The launch plan cb_gemm_wgrad_group runs the problems with: tile width and K-split per problem, or 0 and 0 when they are not
   grouped (each then runs as its own cb_gemm). A single weight gradient with block_n / split_k set to these runs each output
   element's sum in the group's order. */
extern "C" int cb_gemm_wgrad_group_plan(const cb_gemm_desc* descs, int n, int* bn, int* split) {
  using namespace cb;
  CB_REQUIRE(descs != nullptr && n >= 1 && bn != nullptr && split != nullptr, "cb_gemm_wgrad_group_plan: bad arguments");
  const GroupPlan gp = group_plan(descs, n, plan_sm_count());
  *bn = gp.groupable ? gp.bn : 0;
  *split = gp.groupable ? real_splits(ceil_div(descs[0].k, BK), gp.split) : 0;
  return CB_OK;
}

extern "C" int cb_gemm_tile_width(const cb_gemm_desc* d) {
  using namespace cb;
  if (d == nullptr || d->m <= 0 || d->n <= 0 || d->k <= 0) return 0;
  if (d->mode != CB_GEMM_WGRAD) return choose_config(*d, sm_count()).bn;
  return choose_config(*d, plan_sm_count()).bn;
}

extern "C" int64_t cb_gemm_workspace_bytes(const cb_gemm_desc* d) {
  using namespace cb;
  if (d == nullptr || d->mode != CB_GEMM_WGRAD || d->m <= 0 || d->n <= 0 || d->k <= 0) return 0;
  return wgrad_ws_bytes(*d, choose_config(*d, sm_count_device()).splits);
}

extern "C" int64_t cb_gemm_wgrad_group_workspace_bytes(const cb_gemm_desc* descs, int n) {
  using namespace cb;
  if (descs == nullptr || n < 1) return 0;
  for (int i = 0; i < n; ++i)
    if (descs[i].mode != CB_GEMM_WGRAD || descs[i].m <= 0 || descs[i].n <= 0 || descs[i].k <= 0) return 0;
  return group_ws_bytes(descs, n);
}
