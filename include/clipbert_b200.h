/*
 * clipbert_b200.h — C ABI of libclipbert_sm90.so, the H100 (sm_90a) kernels behind the ClipBERT
 * forward/backward hot path.
 *
 * The reference (jayleicn/ClipBERT) has no FFI: its hot path is a stack of torch.nn modules whose
 * arithmetic runs in third-party CUDA libraries (cuDNN, cuBLAS, apex). Each entry point below
 * replaces the library kernels reached from one reference call site (cited as file:line relative to
 * the reference root). Conventions:
 *   - every pointer is a device pointer into caller-owned memory; the library never allocates
 *     device memory, never synchronises, and enqueues all work on the `stream` argument
 *     (a cudaStream_t passed as void*), so every call is CUDA-graph capturable;
 *   - activations / packed weights are bf16 (uint16 storage), statistics / gradients are fp32,
 *     token ids are int64; accumulation is always fp32;
 *   - return 0 on success, a negative cb_status on failure; cb_last_error() gives a thread-local
 *     message. Nothing throws across the ABI. Shape / alignment violations are errors, not UB.
 */
#ifndef CLIPBERT_B200_H_
#define CLIPBERT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum cb_status {
  CB_OK = 0,
  CB_ERR_INVALID = -1, /* bad shape / alignment / null pointer */
  CB_ERR_CUDA = -2,    /* CUDA runtime or driver error */
  CB_ERR_UNSUPPORTED = -3
} cb_status;

const char* cb_last_error(void);
/* library version and the SM architecture it was compiled for (90 = sm_90a) */
int cb_version(void);
int cb_sm_arch(void);
/* number of kernels this library has launched since load (process-wide, all threads). */
int64_t cb_launch_count(void);
/* Programmatic dependent launch between this library's kernels (default OFF; env CB_PDL=1 or cb_set_pdl(1) enables):
 * each kernel's prologue overlaps the previous kernel's tail; every kernel issues griddepcontrol.wait before its first
 * global access, so results are identical to plain stream order. It can cancel the gain of running the wgrad GEMMs on a
 * second stream: early-launched dependent GEMM CTAs hold their ~200 KB of shared memory while they wait and keep the other
 * stream off those SMs.
 * enable = 2: every kernel EXCEPT the persistent GEMMs (an LN / attention / column-sum CTA waiting early holds a few KB).
 * Returns the previous setting. Replaces nothing in the reference (its ~400 launches per clip are plain stream-
 * ordered cuDNN/cuBLAS/ATen kernels, SURVEY.md section 8 a1). */
int cb_set_pdl(int enable);

/* Deterministic mode (default OFF; the Python package mirrors torch.are_deterministic_algorithms_enabled() into it). While it is
 * on, every accumulation of the library runs in a fixed order, so a training step gives the same bits on every run on the same
 * device model and build, whatever the grid cap (cb_debug_gemm_sm_limit), PDL setting, stream placement or co-running work:
 *   - CB_GEMM_WGRAD (cb_gemm, cb_gemm_wgrad_group): the K-split is chosen from the problem shape and the device's SM count only.
 *     With one split every output element gets one red.add (order-free). With S > 1 splits, split s writes its scaled partial
 *     tile with plain stores to plane s of the caller's workspace (fp32 [S][m][ntaps * n]) and a second launch adds the planes
 *     to out in split order 0..S-1: out + (p_0 + p_1 + ... + p_{S-1}) evaluated as ((out + p_0) + p_1) + ... . The workspace is
 *     cb_gemm_desc.workspace / workspace_bytes (cb_gemm_workspace_bytes; for a group descs[0]'s,
 *     cb_gemm_wgrad_group_workspace_bytes); a call without enough returns CB_ERR_INVALID.
 *   - the entry points that add into fp32 gradients / scalars with atomics (cb_layernorm_bwd with dgamma / dbeta / dbias_drop,
 *     cb_embed_text_bwd, cb_embed_visual_bwd, cb_colsum, cb_sumsq, cb_clip_lse_loss, cb_clip_pool_ce_loss) return
 *     CB_ERR_INVALID; their _det variants below, which take a caller-owned scratch, are used instead. A _det variant sums in
 *     its stated order whether or not the mode is on.
 * Returns the previous setting. */
int cb_set_deterministic(int enable);

/* Dropout stream position in DEVICE memory. The reference draws a fresh mask at every nn.Dropout call
 * (src/modeling/transformers.py:170,222,295,375; modeling.py:57,552). Here a mask is a pure function of
 * (seed, element index) and every mask-drawing entry point takes the seed BY VALUE, so a captured CUDA graph would
 * replay the same masks. cb_dropout_offset_bind(word) makes every launch issued AFTERWARDS (process-wide, until the
 * next bind; NULL unbinds) read the 64-bit `word` on the device when it RUNS and use  seed + word * odd_constant
 * instead of seed: the forward and the backward of one step bind the same word and regenerate the same masks, the
 * next replay sees an advanced word and draws new ones. cb_dropout_offset_advance enqueues a one-thread kernel:
 * ++*counter; if (snapshot) *snapshot = *counter - a step advances the model's counter once and binds the per-step
 * snapshot, so a later step (or a second forward before this one's backward) cannot change the masks of this one.
 *
 * The mask (pinned by tests/dropout_ref.py and tests/test_gpu_dropout.py):
 *   seed'   = seed + word * 0xD1342543DE82EF95 (mod 2^64) while a word is bound, else seed
 *   keep(e) = 16-bit lane (e & 3) of splitmix64(seed', e >> 2) >= thresh, thresh = round(p * 65536) clamped to [1, 65535]
 *             for 0 < p < 1; y = x / (1 - p) where kept, 0 elsewhere. p <= 0: no dropout. p >= 1: thresh = 65536 and a
 *             multiplier of 0, so every element is dropped (as nn.Dropout(p=1)).
 *   element index e of each consumer:
 *     cb_dropout                   i, the flat index into x
 *     cb_gemm epilogue (TN, NN)    out_row * n + col: n is the descriptor's column count (not out_ld), out_row the row
 *                                  after the row map
 *     cb_layernorm_bwd             row * 768 + col (dx_drop, dbias_drop)
 *     cb_embed_text_* / _visual_*  (seq * l + pos) * 768 + col: text rows at pos = t, visual cell j at pos = lt + j
 *     cb_attention_fwd / _bwd / _probs  ((seq * heads + h) * l + i) * l + j for probability P[i, j] of head h */
int cb_dropout_offset_bind(const uint64_t* device_word);
int cb_dropout_offset_advance(uint64_t* counter, uint64_t* snapshot, void* stream);

/* ------------------------------------------------------------------------------------------
 * Tensor-core contraction (wgmma, TMA operand staging, register accumulators).
 *
 * One descriptor covers every dense contraction on the path:
 *   nn.Linear            src/modeling/transformers.py:218-220,292,357,372,467  modeling.py:534-539
 *   d2 Conv2d 1x1 / 3x3  src/modeling/grid_feat.py:95 (detectron2 ResNet), :43-48 (grid_encoder)
 *   and their autograd dgrad / wgrad.
 *
 * mode CB_GEMM_TN : out[M,N] = epi( sum_t A[m + shift_t, 0:K] . B[n, t*K : (t+1)*K] )
 *     A: bf16 [a_rows, K]  (row stride a_ld)   B: bf16 [N, ntaps*K] (row stride b_ld)
 *     ntaps = 1 for Linear / 1x1 conv. ntaps = 9 is a 3x3 pad-1 conv over a zero-bordered
 *     ("padded") NHWC activation whose rows are flat pixels p = (img*(H+2) + y)*(W+2) + x;
 *     shift_t = tap_sign * ((t/3 - 1)*(W+2) + (t%3 - 1)). tap_sign = -1 gives the dgrad conv.
 *     ntaps = 4 ("row taps", TN only): shift_t = tap_sign * t * tap_w - the space-to-depth stem (cb_stem_s2d).
 * mode CB_GEMM_NN : as TN but B is stored [K, ntaps*N] row-major (the forward weight [out=K, in=N]
 *     read "MN-major"): out[m, n] = epi( sum_t sum_k A[m + shift_t, k] * B[k, t*N + n] ). This is
 *     the dgrad of Linear / conv straight from the forward weight layout (no transposed copy).
 * mode CB_GEMM_WGRAD : out[m, t*N + n] += rowscale[m] * sum_p A[p, m] * B[p + shift_t, n]
 *     A: bf16 [P, M] (dY), B: bf16 [P, N] (X); both operands are read "MN-major" straight from
 *     the activation layout; fp32 red.global.add accumulation. Persistent CTAs walk the 128 x block_n tiles of out (per
 *     tap), each tile over the whole of P or, with a K-split, over one of split_k consecutive ranges of P.
 *
 * Epilogue (TN), applied in this order on the fp32 accumulator v of element (m, n):
 *     v = v * scale[n] + shift[n]        (FrozenBN affine / bias; either may be NULL)
 *     v = dropout(v)                     (if dropout_p > 0; counter RNG keyed by seed + out index)
 *     v += residual[m, n]                (bf16, optional)
 *     if out2: out2[row, n] = v          (bf16 pre-activation stash, optional; gelu'(v) for CB_ACT_GELU_STASH_GRAD)
 *     v = act(v)                         (none / relu / gelu(erf) / tanh)
 *     v *= auxfn(aux[m, n])              (backward masks: relu' , gelu', tanh' ; optional)
 *     out[row(m), n] = v                 (bf16 or fp32)
 * row(m) re-maps between compact NHWC pixel rows and zero-bordered rows (cb_rowmap).
 * Rounding: the products of bf16 A and B are accumulated in fp32 on the tensor cores; every epilogue step above is one fp32
 * operation (gelu / gelu' use fast_erf, |error| <= 1.5e-7; tanh is tanh.approx.f32, relative error 2^-10.987); the result is
 * rounded once to bf16 (nearest even) unless out_fp32, and out2 once from its fp32 value. fp32 results below 2^-126 flush to
 * zero.
 * NaN / inf: a NaN or inf reaches out like any other value (a NaN in row m of A makes row m NaN; an overflowing accumulator
 * is +-inf). relu passes NaN and +inf and writes +0 for -inf and for a pre-activation of -0 or +0, so a NaN from an
 * overflowing bf16 conv reaches the loss. CB_AUX_RELU_MASK is a select, v = (aux > 0) ? v : 0, with aux > 0 meaning a
 * positive normal bf16 or +inf: a NaN, zero or subnormal aux gives 0 even for a NaN / inf v (the (act > 0) rule of every ReLU
 * backward below). Nothing is promised about gelu / gelu' of +-inf.
 * Alignment (checked, CB_ERR_INVALID and nothing launched otherwise): a, b, out, out2, residual, aux 16-byte aligned (TMA
 * reads the operands and epilogue inputs; out / out2 take 16-byte stores); n, k, out_ld, out2_ld, res_ld, aux_ld multiples
 * of 8. WGRAD: a, b, out 16-byte aligned, m, n multiples of 8, out_ld a multiple of 4.
 * ntaps = 9 with k % 64 != 0 is supported: the last 64-deep chunk of a tap reads the next tap's first columns of B, and they
 * meet the zero fill of A past column k, so the result is exact for finite B (an inf / NaN there would turn 0 * inf into NaN).
 * ------------------------------------------------------------------------------------------ */
enum { CB_GEMM_TN = 0, CB_GEMM_WGRAD = 1, CB_GEMM_NN = 2 };
enum {
  CB_ACT_NONE = 0, CB_ACT_RELU = 1, CB_ACT_GELU = 2, CB_ACT_TANH = 3,
  CB_ACT_GELU_STASH_GRAD = 4 /* out = gelu(v) and, instead of the pre-activation, out2 = gelu'(v) (bf16): the erf and the
                                exp(-v^2/2) are shared, and the backward of BertIntermediate (transformers.py:363-366)
                                becomes CB_AUX_MUL - one multiply - instead of re-evaluating erf + exp per element      */
};
enum {
  CB_AUX_NONE = 0,
  CB_AUX_RELU_MASK = 1, /* v = (aux > 0) ? v : 0       aux = forward output of the ReLU       */
  CB_AUX_GELU_GRAD = 2, /* v *= gelu'(aux)             aux = forward pre-activation            */
  CB_AUX_TANH_GRAD = 3, /* v *= 1 - aux^2              aux = forward tanh output               */
  CB_AUX_MUL = 4        /* v *= aux                    aux = stashed derivative (CB_ACT_GELU_STASH_GRAD) */
};
enum {
  CB_ROWMAP_NONE = 0,
  CB_ROWMAP_PAD = 1,  /* m indexes compact [img,H,W] pixels, output row is the padded pixel      */
  CB_ROWMAP_UNPAD = 2 /* m indexes padded [img,H+2,W+2] pixels, border rows are dropped          */
};

typedef struct cb_gemm_desc {
  int32_t mode;
  int32_t m, n, k; /* TN: rows, cols, per-tap K.  WGRAD: out rows (=A cols), out cols per tap, P */
  const void* a;
  int64_t a_rows, a_ld;
  const void* b;
  int64_t b_rows, b_ld;
  int32_t ntaps, tap_w, tap_sign; /* tap_w = W + 2 (padded row pitch in pixels) */
  int32_t split_k;                /* WGRAD only; 0 = let the library choose, else the number of K splits */
  /* epilogue */
  const float* scale;
  const float* shift;
  const void* residual; /* residual / aux: bf16 [m, n] at the A row m (TN / NN), base 16-byte aligned, ld a multiple of 8 */
  int64_t res_ld;
  const void* aux;
  int64_t aux_ld;
  int32_t aux_mode;
  int32_t act;
  void* out;
  int64_t out_ld;
  int32_t out_fp32;
  void* out2;
  int64_t out2_ld;
  int32_t rowmap, map_h, map_w; /* spatial size (unpadded) for cb_rowmap */
  float dropout_p;
  uint64_t dropout_seed;
  int32_t block_n;  /* 0 = let the library choose (64 / 128 / 256). An explicit block_n for TN / NN picks the ping-pong kernel's
                       128 x 64 or 128 x 128 tiles: there a 128 x 256 tile would need 256 fp32 accumulators per thread of
                       the warpgroup that owns it, more than its 232 registers, so an explicit 256 runs on 128-wide tiles.
                       TN / NN 128 x 256 tiles (both consumer warpgroups on one tile) are chosen by the library only, or
                       forced through reserved */
  int32_t reserved; /* tuning / test knobs: bits 8-11 k-chunks per pipeline stage (0 = automatic; for cb_gemm_wgrad_group,
                       descs[0]'s apply to the whole group); CB_GEMM_FORCE_WIDE / CB_GEMM_NO_WIDE (TN / NN, for tests and A/B
                       runs); other bits ignored */
  void* workspace;  /* deterministic mode, CB_GEMM_WGRAD: fp32 split planes, 16-byte aligned (NULL / ignored otherwise) */
  int64_t workspace_bytes;
} cb_gemm_desc;

/* cb_gemm_desc.reserved bits, TN / NN: run on 128 x 256 tiles whatever block_n says / never on 128 x 256 tiles */
#define CB_GEMM_FORCE_WIDE (1 << 12)
#define CB_GEMM_NO_WIDE (1 << 13)

int cb_gemm(const cb_gemm_desc* desc, void* stream);
/* tile width cb_gemm runs desc with (64, 128 or 256; for TN / NN 256 is the 128 x 256 tile of both consumer warpgroups), or 0
 * for an empty shape; launches nothing */
int cb_gemm_tile_width(const cb_gemm_desc* desc);
/* bytes of workspace a CB_GEMM_WGRAD descriptor needs in deterministic mode (0: one K-split, or not a weight gradient) */
int64_t cb_gemm_workspace_bytes(const cb_gemm_desc* desc);
/* the plan cb_gemm_wgrad_group runs n CB_GEMM_WGRAD problems with: *bn = tile width and *split = K-splits per problem, or 0 and 0
 * when they run as separate cb_gemm launches. A single weight gradient with block_n = *bn and split_k = *split sums every output
 * element in the group's order (ClipBertBaseModel's split layers, modeling.py); launches nothing */
int cb_gemm_wgrad_group_plan(const cb_gemm_desc* descs, int n, int* bn, int* split);
/* n independent CB_GEMM_WGRAD problems in ONE persistent launch: the weight gradients of the four Linear layers of a BertLayer
 * (autograd of transformers.py:238-301,363-381) or of the convs of one bottleneck block. The problems should share their
 * reduction length k (tokens / pixels); 1 <= n <= 8. One prologue and tail instead of n, no K-split when the group fills the SMs.
 * Falls back to n cb_gemm launches for n == 1, n > 8 or very different k. descs[0].block_n / split_k, when non-zero, set the tile
 * width / K-split of the whole group. Other epilogue fields than scale / out are ignored. */
int cb_gemm_wgrad_group(const cb_gemm_desc* descs, int n, void* stream);
/* the same for a group; the group reads its whole workspace from descs[0] (the problems' split planes one after another) */
int64_t cb_gemm_wgrad_group_workspace_bytes(const cb_gemm_desc* descs, int n);

/* ------------------------------------------------------------------------------------------
 * LayerNorm over rows of a bf16 [m, 768] matrix (fp32 statistics, warp-shuffle reductions).
 * Replaces apex FusedLayerNorm (src/modeling/transformers.py:32,165,293,373; modeling.py:12,58).
 * The residual add / dropout that precede it in BertSelfOutput / BertOutput
 * (transformers.py:297-301, 377-381) are fused into the producing cb_gemm epilogue.
 *   fwd : y = (x - mean) * rstd * gamma + beta ; stats[m] = (mean, rstd)
 *   bwd : dx (bf16) ; dx_drop = dx * dropout_mask(seed, element) (bf16, optional: the gradient
 *         entering the dense layer that fed this LN through dropout) ; dgamma / dbeta / dbias_drop
 *         (fp32, atomically accumulated; dbias_drop = column sums of dx_drop = that dense's bias grad)
 * ------------------------------------------------------------------------------------------ */
int cb_layernorm_fwd(const void* x, const float* gamma, const float* beta, void* y, float* stats, int m, int hidden,
                     float eps, void* stream);
int cb_layernorm_bwd(const void* dy, const void* x, const float* stats, const float* gamma, void* dx, void* dx_drop,
                     float* dgamma, float* dbeta, float* dbias_drop, int m, int hidden, float dropout_p,
                     uint64_t dropout_seed, void* stream);
/* Deterministic: the same kernel with B = min(ceil(m / 4), 264) blocks; block b stores its column sums (its four warps added in
 * warp order) to scratch row b of each output, and dgamma[c] += ((row_0[c] + row_1[c]) + ...) + row_{B-1}[c], blocks in order. */
int64_t cb_layernorm_bwd_scratch_bytes(int m);
int cb_layernorm_bwd_det(const void* dy, const void* x, const float* stats, const float* gamma, void* dx, void* dx_drop,
                         float* dgamma, float* dbeta, float* dbias_drop, int m, int hidden, float dropout_p,
                         uint64_t dropout_seed, float* scratch, int64_t scratch_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Embeddings. out is the bf16 [nseq * l, 768] encoder input; text rows go to positions [0, lt),
 * visual rows to [lt, l) of every sequence, i.e. the torch.cat([text; visual]) of
 * src/modeling/modeling.py:219-223 is a write offset, not a copy.
 *   text   : BertEmbeddings.forward (transformers.py:172-199): LN(word[id] + pos[t] + type[0]), dropout
 *   visual : VisualInputEmbedding.forward (modeling.py:62-101): mean over frames, + row/col position
 *            (modeling.py:124-153), + type[0], LN, dropout; the row gather of repeat_tensor_rows
 *            (src/datasets/data_utils.py:344-357) is fused: sequence s reads video seq2vid[s]
 *            (or s / n_ex when seq2vid is NULL). Tables / LN parameters are fp32.
 *   bwd    : scatter-adds into the fp32 table gradients; the visual backward also reduces over the
 *            sequences of a video and the frame mean, producing dgrid (bf16 [nvid, t, gh*gw, 768]).
 * ------------------------------------------------------------------------------------------ */
int cb_embed_text_fwd(const int64_t* ids, const float* word, const float* pos, const float* type0, const float* gamma,
                      const float* beta, void* out, float* stats, int nseq, int lt, int l, int vocab, int hidden,
                      float eps, float dropout_p, uint64_t seed, void* stream);
int cb_embed_text_bwd(const void* dh, const int64_t* ids, const float* word, const float* pos, const float* type0,
                      const float* gamma, const float* stats, float* dword, float* dpos, float* dtype0, float* dgamma,
                      float* dbeta, int nseq, int lt, int l, int vocab, int hidden, float dropout_p, uint64_t seed,
                      void* stream);
int cb_embed_visual_fwd(const void* grid, const int32_t* seq2vid, int n_ex, const float* rowemb, const float* colemb,
                        const float* type0, const float* gamma, const float* beta, void* out, float* stats, int nseq,
                        int t, int gh, int gw, int lt, int l, int hidden, float eps, float dropout_p, uint64_t seed,
                        void* stream);
int cb_embed_visual_bwd(const void* dh, const void* grid, const int32_t* seq2vid, const int32_t* vid_start, int n_ex,
                        const float* rowemb, const float* colemb, const float* type0, const float* gamma,
                        const float* stats, float* dv_tmp, void* dgrid, float* drow, float* dcol, float* dtype0,
                        float* dgamma, float* dbeta, int nseq, int nvid, int t, int gh, int gw, int lt, int l, int hidden,
                        float dropout_p, uint64_t seed, void* stream);
/* Deterministic backwards. The blocks of the kernels above (P = min(max(ceil(nseq / 8), 1), 32) per text position / grid cell)
 * store their parameter partials to scratch instead of adding them; each output is then the sum of its blocks' rows in block
 * order (cell, then x): dgamma, dbeta and d type[0] over every block, d pos[t] over the blocks of position t, d row[r] over the
 * cells of grid row r in column order, d col[c] over the cells of grid column c in row order. The text backward also stores
 * every row's fp32 word gradient; each table row word[id] then receives the sum of the rows carrying id, in row order
 * (b * lt + t), added once. Scratch: cb_embed_*_bwd_scratch_bytes. */
int64_t cb_embed_text_bwd_scratch_bytes(int nseq, int lt);
int cb_embed_text_bwd_det(const void* dh, const int64_t* ids, const float* word, const float* pos, const float* type0,
                          const float* gamma, const float* stats, float* dword, float* dpos, float* dtype0, float* dgamma,
                          float* dbeta, int nseq, int lt, int l, int vocab, int hidden, float dropout_p, uint64_t seed,
                          float* scratch, int64_t scratch_bytes, void* stream);
/* BertEmbeddings from word vectors (transformers.py:172-199: inputs_embeds = word_embeddings(input_ids), then + position +
 * token type, LayerNorm, dropout), for a hook on word_embeddings that sees or replaces word[ids]. vec: fp32 rows, row
 * r = b * lt + t at vec + r * vec_ld (vec_ld >= 768, a multiple of 4; 16-byte aligned); otherwise as cb_embed_text_fwd / _bwd /
 * _bwd_det, the same stats, dropout masks and parameter-gradient order. The backward writes dvec[r] (fp32, contiguous
 * [nseq * lt, 768], one writer per element) instead of adding into a word table; cb_embed_word_scatter adds such rows into the
 * table: every table row word[id] receives the sum of the rows carrying id, in row order, added once (one writer per table row,
 * the same bits in both modes). Scratch of _det: cb_embed_text_bwd_vectors_scratch_bytes. */
int cb_embed_text_fwd_vectors(const float* vec, int64_t vec_ld, const float* pos, const float* type0, const float* gamma,
                              const float* beta, void* out, float* stats, int nseq, int lt, int l, int hidden, float eps,
                              float dropout_p, uint64_t seed, void* stream);
int cb_embed_text_bwd_vectors(const void* dh, const float* vec, int64_t vec_ld, const float* pos, const float* type0,
                              const float* gamma, const float* stats, float* dvec, float* dpos, float* dtype0, float* dgamma,
                              float* dbeta, int nseq, int lt, int l, int hidden, float dropout_p, uint64_t seed, void* stream);
int64_t cb_embed_text_bwd_vectors_scratch_bytes(int nseq, int lt);
int cb_embed_text_bwd_vectors_det(const void* dh, const float* vec, int64_t vec_ld, const float* pos, const float* type0,
                                  const float* gamma, const float* stats, float* dvec, float* dpos, float* dtype0, float* dgamma,
                                  float* dbeta, int nseq, int lt, int l, int hidden, float dropout_p, uint64_t seed, float* scratch,
                                  int64_t scratch_bytes, void* stream);
int cb_embed_word_scatter(const int64_t* ids, const float* dvec, float* dword, int rows, int vocab, int hidden, void* stream);
int64_t cb_embed_visual_bwd_scratch_bytes(int nseq, int gh, int gw);
int cb_embed_visual_bwd_det(const void* dh, const void* grid, const int32_t* seq2vid, const int32_t* vid_start, int n_ex,
                            const float* rowemb, const float* colemb, const float* type0, const float* gamma,
                            const float* stats, float* dv_tmp, void* dgrid, float* drow, float* dcol, float* dtype0,
                            float* dgamma, float* dbeta, int nseq, int nvid, int t, int gh, int gw, int lt, int l, int hidden,
                            float dropout_p, uint64_t seed, float* scratch, int64_t scratch_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Fused self-attention, BertSelfAttention.forward (transformers.py:230-286):
 *   S = Q K^T / 8 + (1 - mask) * -10000 ; P = softmax(S) ; dropout(P) ; ctx = P V ; heads merged.
 * qkv: bf16 [nseq*l, 3*heads*64] (Q | K | V as produced by the fused N=2304 projection);
 * text_mask: int64 [nseq, lt] (visual tokens are always attendable, modeling.py:217-220);
 * ctx: bf16 [nseq*l, heads*64]; lse: fp32 [nseq, heads, l] log-sum-exp saved for the backward (fwd: may be NULL).
 * Arguments (checked on the host, nothing is launched otherwise): 0 <= lt <= l, 0 < nseq, heads <= 65535 (grid limits);
 * row pitches multiples of 8 with ld_qkv, ld_dqkv >= 3*heads*64 and ld_ctx >= heads*64 (ld_ctx is also dctx's pitch);
 * qkv, ctx, dctx and dqkv 16-byte aligned (read and written as 16-byte vectors).
 * The backward recomputes P tile by tile from Q, K and the SAVED lse, takes D_i = dO_i . ctx_i from the SAVED ctx, and
 * regenerates the dropout mask: dS = P (r dO V^T - D), dV = (P r)^T dO, dQ = dS K / 8, dK = dS^T Q / 8 (r: multipliers).
 * Rounding (fp32 arithmetic and accumulation everywhere else):
 *   tensor-core forward: x_ij = exp(S_ij - m_i) r_ij is rounded to bf16 before the P V product, m_i the running row maximum
 *     (the whole row when l <= 64, 64-key tiles 0..t on the longer path); the products are rescaled as m_i grows and divided
 *     by the unrounded (undropped) row sum;
 *   tensor-core backward: P r and dS are rounded to bf16 before the dV / dK / dQ products;
 *   CUDA-core kernels (cb_debug_attention_general): P and dS stay fp32. Every length runs on tensor
 * cores (mma.sync): l <= 64 in one CTA per (sequence, head); longer sequences in two kernels, one per 64-key tile
 * (dK, dV) and one per 64-query tile (dQ). Each output row is written by one CTA: no atomics, no workspace, results
 * bit-identical from run to run. cb_debug_attention_general(1) selects the CUDA-core kernels instead, for every length.
 * ------------------------------------------------------------------------------------------ */
int cb_attention_fwd(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, void* ctx, int64_t ld_ctx, float* lse,
                     int nseq, int l, int lt, int heads, int head_dim, float dropout_p, uint64_t seed, void* stream);
int cb_attention_bwd(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, const void* ctx, const void* dctx,
                     int64_t ld_ctx, const float* lse, void* dqkv, int64_t ld_dqkv, int nseq, int l, int lt, int heads,
                     int head_dim, float dropout_p, uint64_t seed, void* stream);
/* The attention probabilities themselves, for output_attentions (transformers.py:257-285: the attention_probs returned at
 * :284, after the dropout of :271): probs fp32 [nseq, heads, l, l], contiguous, 16-byte aligned;
 *   P[s, h, i, j] = exp(Q_i . K_j / 8 + madd_j - lse[s, h, i]) x dropout multiplier
 * with madd_j = -10000 for a text key whose mask entry is 0, else 0, and lse what cb_attention_fwd wrote for the same qkv,
 * mask and l (every forward kernel writes the same convention: max_j + log sum_j exp(S_ij - max_j) over the masked scores).
 * The mask is the forward's (same seed, same bound device word, element index above), so with dropout_p = 0 each row sums
 * to 1 and with dropout it is exactly the P the forward multiplied V by. Tensor cores (mma.sync), one CTA per (64-query
 * tile, head, sequence); rows and columns beyond l are never written. */
int cb_attention_probs(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, const float* lse, float* probs, int nseq,
                       int l, int lt, int heads, int head_dim, float dropout_p, uint64_t seed, void* stream);
/* Backward through the returned probabilities A = P r (r: the dropout multipliers, 0 or 1 / (1 - p)): with G = dloss / dA,
 * dprobs fp32 [nseq, heads, l, l], contiguous, 16-byte aligned at its base (a row starts at any 4-byte alignment),
 *   g_ij = r_ij G_ij ;  D_i = sum_j P_ij g_ij (= sum_j A_ij G_ij) ;  dS_ij = P_ij (g_ij - D_i)
 *   dQ_i += sum_j dS_ij K_j / 8 ;  dK_j += sum_i dS_ij Q_i / 8          (dV unchanged)
 * ADDED to the Q and K column blocks of dqkv (what cb_attention_bwd wrote: dS is linear in the upstream gradient, so the
 * two contributions sum); the V block, the pitch padding and everything outside the window are not touched. P is rebuilt
 * from qkv, the mask and lse as cb_attention_probs forms it (same seed, same bound device word); the returned tensor is never
 * read. drow: caller-owned fp32 scratch of nseq * heads * l floats (D). Arguments and alignment (qkv, dqkv, dprobs) are
 * checked as for cb_attention_bwd, nothing is launched otherwise.
 * Rounding: P, g, D and dS in fp32, dS rounded to bf16 before the dQ / dK products (mma.sync, fp32 accumulation), and each
 * dQ / dK element read, added to in fp32 and rounded to bf16 once. Two kernels, one per 64-query tile (D, then dQ) and one
 * per 64-key tile (dK); every element has one writer: no atomics, bit-identical from run to run. */
int cb_attention_probs_bwd(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, const float* lse, const float* dprobs,
                           float* drow, void* dqkv, int64_t ld_dqkv, int nseq, int l, int lt, int heads, int head_dim,
                           float dropout_p, uint64_t seed, void* stream);
/* cb_attention_probs_bwd with dQ and dK WRITTEN to the Q and K column blocks (dQ_i = sum_j dS_ij K_j / 8, dK_j = sum_i dS_ij
 * Q_i / 8, each rounded to bf16 once) instead of added: for a dqkv whose Q and K blocks hold nothing yet, the backward split at a
 * differentiable attention map (ClipBertBaseModel.layerwise_autograd), where G is the map's full gradient. Nothing is read from
 * dqkv; the V block, the pitch padding and everything outside the window are not touched. Same arguments, checks, rounding and
 * kernels (their store instantiations). */
int cb_attention_probs_bwd_store(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, const float* lse,
                                 const float* dprobs, float* drow, void* dqkv, int64_t ld_dqkv, int nseq, int l, int lt,
                                 int heads, int head_dim, float dropout_p, uint64_t seed, void* stream);
/* The value gradient of the attention backward alone, for the same split: with dO = dctx [nseq * l, >= heads * 64] bf16 (row
 * pitch ld_ctx) and P rebuilt from qkv, the mask and lse as cb_attention_probs forms it (same seed, same bound device word,
 * dropout multipliers r),
 *   dV_j = sum_i P_ij r_ij dO_i       per (sequence, head), every j < l
 * WRITTEN to the V column block of dqkv (bf16, rounded once); the Q and K blocks, the pitch padding and everything outside the
 * window are not touched. P r is rounded to bf16 before the product, as cb_attention_bwd does. Tensor cores (mma.sync), one CTA
 * per (64-key tile, head, sequence), one writer per element: no atomics, bit-identical from run to run. Arguments are checked as
 * for cb_attention_bwd (pitches multiples of 8 holding Q | K | V and heads x 64; qkv, dctx, dqkv 16-byte aligned); nothing is
 * launched otherwise. */
int cb_attention_bwd_dv(const void* qkv, int64_t ld_qkv, const int64_t* text_mask, const float* lse, const void* dctx,
                        int64_t ld_ctx, void* dqkv, int64_t ld_dqkv, int nseq, int l, int lt, int heads, int head_dim,
                        float dropout_p, uint64_t seed, void* stream);
/* The gradient the returned probabilities A receive from the context product ctx = A V (transformers.py:271-277), for
 * retain_grad() on the attentions: dctx [nseq * l, >= heads * 64] bf16 with row pitch ld_ctx (d loss / d context), V the third
 * column block of qkv;
 *   dprobs[s, h, i, j] = (accumulate ? dprobs[s, h, i, j] : 0) + sum_d dctx[s l + i, h 64 + d] V[s l + j, h 64 + d]
 * for every i, j < l: padded text keys, padded query rows and dropped positions get their value too (A is post-dropout, so
 * there is no dropout factor; no mask, lse or seed is read). dprobs fp32 [nseq, heads, l, l], contiguous, 16-byte aligned at
 * its base (a row starts at any 4-byte alignment); rows and columns beyond l are never written. Tensor cores (mma.sync, bf16
 * in, fp32 accumulation), one CTA per (64-query tile, head, sequence); accumulate = 1 reads each element and adds in fp32,
 * once. Every element has one writer: no atomics, bit-identical from run to run. Arguments are checked as for
 * cb_attention_probs (accumulate 0 or 1; pitches multiples of 8 holding Q | K | V and heads x 64; qkv, dctx, dprobs 16-byte
 * aligned); nothing is launched otherwise. */
int cb_attention_dprobs(const void* qkv, int64_t ld_qkv, const void* dctx, int64_t ld_ctx, float* dprobs, int accumulate,
                        int nseq, int l, int heads, int head_dim, void* stream);

/* ------------------------------------------------------------------------------------------
 * Small helpers on the transformer side.
 *   cb_colsum     out[n] += sum_m x[m, n]            bias gradients of nn.Linear (autograd of F.linear)
 *   cb_dropout    y = dropout(x)                     nn.Dropout before the classifier (modeling.py:552)
 *   cb_pad_cast   fp32 [rows, c] -> bf16 [rows, cpad] zero padded (d logits -> padded head gradient)
 *   cb_cast_scale fp32 -> bf16 operand packing, optional per-row scale (FrozenBN scale folded into the
 *                 conv weight: w'[o, :] = w[o, :] * gamma[o] * rsqrt(var[o] + 1e-5), d2 FrozenBatchNorm2d)
 * The packed value is the fp32 product rounded to nearest even (as w * s followed by .to(bfloat16)), except that the library
 * is built with flush-to-zero: a product below 2^-126 in magnitude packs as a zero of its sign (also cb_cast_scale_segments
 * and the packed copy of cb_adamw_step).
 * ------------------------------------------------------------------------------------------ */
int cb_colsum(const void* x, int64_t ld, float* out, int m, int n, void* stream);
/* deterministic: slab s of 128 rows stores its column sums (rows added in the kernel's order) to scratch row s, then
 * out[c] += ((slab_0[c] + slab_1[c]) + ...), slabs in order */
int64_t cb_colsum_scratch_bytes(int m, int n);
int cb_colsum_det(const void* x, int64_t ld, float* out, int m, int n, float* scratch, int64_t scratch_bytes, void* stream);
int cb_dropout(const void* x, void* y, int64_t n, float p, uint64_t seed, void* stream);
/* dx = dy * gelu'(u): backward of BertPredictionHeadTransform's activation (transformers.py:486-495). erf is fast_erf
 * (Abramowitz-Stegun 7.1.26, |error| <= 1.5e-7): within 1 bf16 ulp of the exact result plus |dy| * (0.75e-7 + 4 * 2^-24),
 * the floor that dominates the left tail where gelu' ~ 1e-6. u = +-inf gives NaN, as ATen's gelu backward (inf * pdf = inf * 0). */
int cb_gelu_bwd(const void* dy, const void* u, void* dx, int64_t n, void* stream);
int cb_pad_cast(const float* in, int64_t in_ld, void* out, int rows, int c, int cpad, void* stream);
int cb_cast_scale(const float* in, const float* rowscale, int64_t row_len, void* out, int64_t n, void* stream);
/* bf16 -> fp32: the averaged gradients come back from the bf16 wire format of the data-parallel exchange (the reference
 * all-reduces its gradients in fp16 under amp O2, src/tasks/run_video_retrieval.py:299-309,432); n elements, 16-byte aligned */
int cb_cast_bf16_f32(const void* in, float* out, int64_t n, void* stream);
/* the same for every conv of the backbone in one launch: segments is a device int64 [nseg][4] table
 * (element offset, element count, row length, offset into `scales` or -1); offsets are 64-element aligned */
int cb_cast_scale_segments(const float* master, void* packed, const int64_t* segments, int nseg, const float* scales, void* stream);

/* ------------------------------------------------------------------------------------------
 * CNN-side data movement (NHWC bf16, 8 channels per 128-bit access). Call sites replaced:
 * GridFeatBackbone.forward (src/modeling/grid_feat.py:89-105) -> detectron2 BasicStem /
 * BottleneckBlock (stride-in-1x1) / grid_encoder MaxPool2d+ReLU (grid_feat.py:43-48).
 *   cb_stem_im2col          7x7/s2/p3 patch gather of the NCHW RGB input into bf16 [n*ho*wo, kp] rows,
 *                           K = (r, s, c) with c in BGR order (the x[:, [2,1,0]] flip of grid_feat.py:92-94
 *                           is folded in); in_dtype 1 = uint8 frames with the ImageNorm mean subtraction
 *                           (src/datasets/data_utils.py:256-276) fused. The stem GEMM follows.
 *   cb_stem_s2d             the stem WITHOUT a patch matrix: space-to-depth(2) of the zero-padded BGR frame,
 *                           S[n, Y, X, (dy*2+dx)*4 + c] (c = 3 is a zero lane), Y < ho+3, X < wo+3. The 7x7/s2/p3 conv
 *                           (kernel zero-extended to 8x8) is then cb_gemm with ntaps = 4, k = 64, tap_w = wo+3 over
 *                           the matrix whose row m is the 64 contiguous bf16 starting at S pixel m: ld = 16 makes the
 *                           rows overlap (a_ld = 16 < k; 54 MB per 128 frames instead of 488 MB of patches), ld = 64
 *                           stores every 4-pixel window explicitly. Output rows follow the same (ho+3) x (wo+3) grid.
 *   cb_maxpool3x3s2         BasicStem max_pool2d(3, 2, 1); _strided reads an input whose pixel rows / images are
 *                           row_pitch / img_pitch pixels apart (the (ho+3) x (wo+3) grid of the s2d stem)
 *   cb_maxpool3x3s2_bwd     the gradient with respect to the frames (grid_feat.py:92-95 -> BasicStem.forward, backward): the
 *                           pool's backward fused with the stem's ReLU', dx[n*h*w, c] (compact, the gradient at the stem conv's
 *                           pre-ReLU output) from dy[n*ho*wo, c] and x, the pool input (the post-ReLU stem output; _strided: on
 *                           the pitches of cb_maxpool3x3s2_strided). Gather form: each element sums, in fp32 and window order, the
 *                           gradients of the <= 4 windows whose forward arg-max it is (first maximum, last NaN), rounds once and
 *                           keeps it where x > 0. One writer per element, no zero fill.
 *   cb_stem_dgrad           then the 7x7/s2/p3 transposed convolution to the frames: dx fp32 NCHW [n, 3, h, w] in RGB order (the
 *                           BGR flip undone) = sum_{k,r,s} dc1[n, (y+3-r)/2, (x+3-s)/2, k] * w[k, (r*7+s)*3 + c], dc1 bf16 compact
 *                           [n*ho*wo, 64], w the stem operand of the forward (bf16 [64, w_ld], FrozenBN scale and ImageNorm's
 *                           1 / std folded in), so dx is the gradient with respect to the frames the stem gather read (raw frames
 *                           included: the mean subtraction has unit derivative). mma.sync m16n8k16, fp32 accumulation in a fixed
 *                           order, one writer per element: the same bits on every run.
 *   cb_subsample2           input of a stride-2 1x1 conv (res3/4/5 block 0 conv1 + shortcut)
 *   cb_unsubsample2_mask    its backward fused with the ReLU mask of the producing block; act = NULL: the mask-free scatter
 *                           (dx = dsub at even pixels, +0 elsewhere), for a gradient whose mask the producing block applies
 *                           itself (cb_nhwc_intake)
 *   cb_maxpool2x2_relu_fwd  grid_encoder MaxPool2d(2,2) + ReLU (7x7 -> 3x3 at 224 px, 14x14 -> 7x7 at 448)
 *   cb_maxpool2x2_relu_bwd  its backward, written into the zero-bordered layout read by the 3x3 dgrad/wgrad
 *   cb_relu_mask            dx = dy * (act > 0)
 * The pools follow F.max_pool2d (max_pool2d_with_indices): a value replaces the running maximum when it is larger or NaN, so a
 * NaN in a window propagates (a NaN / inf from an overflowing bf16 conv reaches the loss as in the reference), equal maxima keep
 * the first in window order (the sign of a zero maximum is ATen's), and the 2x2 backward sends the gradient to that arg-max
 * (first maximum; last NaN). Two differences are pinned: the 2x2 forward writes +0 where the window maximum is -0 (ATen's ReLU
 * keeps -0), and ReLU' is (act > 0) in every ReLU backward of the library (the 2x2 backward on the window maximum,
 * cb_unsubsample2_mask, cb_relu_mask and CB_AUX_RELU_MASK alike), so a NaN activation gets gradient 0 where ATen's
 * threshold_backward passes it on. The forward already carries the NaN into the loss; one rule keeps the three paths equal.
 * ------------------------------------------------------------------------------------------ */
/* Frame resize + pad of the data pipeline (src/datasets/data_utils.py:202-234 ImageResize: F.interpolate(bilinear,
 * align_corners=False) to new_h x new_w, longer side = max_size; :136-160 ImagePad: zeros at the bottom / right up to
 * max_size x max_size; src/datasets/dataset_base.py:191-195). x: `planes` = n * c planes of h x w (in_dtype 0 fp32, 1 uint8),
 * y: fp32 [planes, max_size, max_size]. */
int cb_resize_pad(const void* x, int in_dtype, float* y, int planes, int h, int w, int new_h, int new_w, int max_size, void* stream);
/* dy: fp32 [planes, max_size, max_size] (the gradient of cb_resize_pad's output); dx: fp32 [planes, h, w]. Adjoint of
 * cb_resize_pad with the same (h, w, new_h, new_w, max_size): the pad region (rows >= new_h or columns >= new_w) contributes
 * nothing. Overwrites dx (every element written once) unless accumulate = 1, which adds into it in fp32. Gather form with the
 * forward's own taps and weights: each dx element sums its outputs' contributions in a fixed order (output row, then column),
 * so the bits are the same on every run; no atomics, no alignment requirement. */
int cb_resize_pad_bwd(const float* dy, float* dx, int planes, int h, int w, int new_h, int new_w, int max_size, int accumulate,
                      void* stream);
int cb_stem_im2col(const void* x, int in_dtype, void* out, int n, int h, int w, int kp, float mean_r, float mean_g,
                   float mean_b, void* stream);
int cb_stem_s2d(const void* x, int in_dtype, void* out, int n, int h, int w, int ld, float mean_r, float mean_g, float mean_b,
                void* stream);
int cb_maxpool3x3s2(const void* x, void* y, int n, int h, int w, int c, void* stream);
int cb_maxpool3x3s2_strided(const void* x, void* y, int n, int h, int w, int c, int64_t row_pitch, int64_t img_pitch, void* stream);
int cb_maxpool3x3s2_bwd(const void* dy, const void* x, void* dx, int n, int h, int w, int c, void* stream);
int cb_maxpool3x3s2_bwd_strided(const void* dy, const void* x, void* dx, int n, int h, int w, int c, int64_t row_pitch,
                                int64_t img_pitch, void* stream);
int cb_stem_dgrad(const void* dc1, const void* w, int w_ld, float* dx, int n, int h, int w_img, void* stream);
int cb_subsample2(const void* x, void* y, int n, int h, int w, int c, void* stream);
int cb_unsubsample2_mask(const void* dsub, const void* act, void* dx, int n, int h, int w, int c, void* stream);
int cb_maxpool2x2_relu_fwd(const void* x, void* y, int n, int h, int w, int c, void* stream);
int cb_maxpool2x2_relu_bwd(const void* dy, const void* x, void* dx_pad, int n, int h, int w, int c, void* stream);
int cb_relu_mask(const void* dy, const void* act, void* dx, int64_t n, void* stream);
/* A strided 4-D tensor into the engine's NHWC bf16 layout: out[pixel (n, y, x), ch] = bf16(x[n, ch, y, x]), element (n, ch, y, x)
 * of x at element offset n*sn + ch*sc + y*sh + x*sw (any non-negative strides: channels-last, contiguous NCHW, permuted, sliced
 * or expanded views); in_dtype 0 = fp32, 2 = bf16, 3 = fp16. out is compact [n*h*w, c] (out_bordered = 0) or the interior of a
 * zero-bordered [n, h+2, w+2, c] (out_bordered = 1: border rows are never written). act != NULL: out = (act > 0) ? bf16(x) : +0,
 * with act bf16 NHWC [n, h, w, c] in the same two layouts (act_bordered): the ReLU' of the block whose output gradient x is,
 * applied where it enters the block's backward (GridFeatBackbone's module path; a NaN passes where act > 0). One rounding,
 * one writer per element, no atomics: the same bits on every run. c % 8 == 0; out and act 16-byte aligned. Channels-last x
 * (sc = 1, 16-byte aligned 8-channel groups) takes 16-byte loads, contiguous NCHW planes a shared-memory transpose, anything
 * else a generic gather. Bound by HBM: x and act read once, out written once. */
int cb_nhwc_intake(const void* x, int in_dtype, int64_t sn, int64_t sc, int64_t sh, int64_t sw, int n, int c, int h, int w, const void* act,
                   int act_bordered, void* out, int out_bordered, void* stream);

/* ------------------------------------------------------------------------------------------
 * Clip-level score aggregation + loss of the training loops, pool_method "lse"
 * (src/tasks/run_video_retrieval.py:404-422, src/tasks/run_video_qa.py:484-501), forward AND backward in one launch:
 *   loss[0]  = mean_b ( logsumexp_{k,c} z[k,b,c] - logsumexp_k z[k,b,y_b] )          z = logits, fp32 [n_clips, nseq, ncls]
 *   dlogits  = grad_scale * d loss / d z   (fp32, same shape; NULL = forward only)   y = labels, int64 [nseq]
 * Replaces torch.stack + permute + two torch.logsumexp + torch.gather + mean and their autograd nodes (~45 ATen launches).
 * ------------------------------------------------------------------------------------------ */
int cb_clip_lse_loss(const float* logits, const int64_t* labels, float* loss, float* dlogits, int n_clips, int nseq, int ncls,
                     float grad_scale, void* stream);
/* pool_method "mean" (pool = 1) / "max" (pool = 2) of the same loops (run_video_retrieval.py:405-408, run_video_qa.py:485-488):
 * logits.mean(0) / logits.max(0)[0] followed by F.cross_entropy(reduction="none").mean(); same tensors as cb_clip_lse_loss.
 * For max, among clips with exactly equal logits the FIRST receives the gradient. Both clip losses clamp a label outside
 * [0, ncls) to 0 or ncls - 1 instead of raising as torch.gather / F.cross_entropy would. */
int cb_clip_pool_ce_loss(const float* logits, const int64_t* labels, float* loss, float* dlogits, int n_clips, int nseq, int ncls, int pool,
                         float grad_scale, void* stream);
/* deterministic: block b (256 examples) stores its share of the mean to scratch[b], then loss[0] = the ordered sum of the
 * ceil(nseq / 256) shares (thread t adds shares t, t + 256, ...; warps by xor butterfly; warp sums in warp order) */
int64_t cb_clip_loss_scratch_bytes(int nseq);
int cb_clip_lse_loss_det(const float* logits, const int64_t* labels, float* loss, float* dlogits, int n_clips, int nseq, int ncls,
                         float grad_scale, float* scratch, int64_t scratch_bytes, void* stream);
int cb_clip_pool_ce_loss_det(const float* logits, const int64_t* labels, float* loss, float* dlogits, int n_clips, int nseq, int ncls,
                             int pool, float grad_scale, float* scratch, int64_t scratch_bytes, void* stream);
/* F.cross_entropy(logits, labels, reduction="none") over `rows` rows of `ncls` fp32 logits (row pitch ld), labels int64 with
 * ignore_index (-100: loss 0, no gradient): the masked-LM loss over the vocabulary (src/modeling/modeling.py:286-299), the
 * ITM / multiple-choice / retrieval CE (:560-580, :430-436). fwd: loss[rows], lse[rows] (stash). bwd: dlogits[r, c] =
 * grad_loss[r] * (softmax(z)[c] - [c == y]) with row pitch dld. One block per row, one pass over the row each. A label outside
 * [0, ncls) is treated as ignore_index (loss 0, no gradient) instead of raising. -inf logits contribute exp(-inf) = 0. */
int cb_cross_entropy_fwd(const float* logits, int64_t ld, const int64_t* labels, float* loss, float* lse, int64_t rows, int ncls,
                         int64_t ignore_index, void* stream);
int cb_cross_entropy_bwd(const float* logits, int64_t ld, const int64_t* labels, const float* lse, const float* grad_loss, float* dlogits,
                         int64_t dld, int64_t rows, int ncls, int64_t ignore_index, void* stream);

/* ------------------------------------------------------------------------------------------
 * Data-parallel gradient exchange through the NVSwitch, replacing hvd.DistributedOptimizer.synchronize()
 * (src/tasks/run_video_retrieval.py:299-301,432) for a flat fp32 buffer that every rank has mapped at the same MULTICAST
 * address (symmetric memory): rank r reduces the r-th 1/world slice in the switch (multimem.ld_reduce.add), scales it
 * (1/world = average) and stores it into every rank's copy (multimem.st). n: elements (multiple of 4); max_ctas: CTAs this
 * launch may use (0 = 64; 128 threads each, small enough to share an SM with a GEMM CTA). The caller places a cross-rank barrier before (all gradients written) and after (all slices stored).
 * ------------------------------------------------------------------------------------------ */
int cb_nvls_allreduce_f32(void* multicast_ptr, int64_t n, int rank, int world, float scale, int max_ctas, void* stream);

/* ------------------------------------------------------------------------------------------
 * Fused optimizer step over the flat fp32 parameter buffers (SURVEY.md section 8 f2).
 *   cb_sumsq       out[0] += sum(x^2)  - the norm half of torch.nn.utils.clip_grad_norm_ as called at
 *                  src/tasks/run_video_retrieval.py:477-480 (one call per flat gradient buffer, caller zeroes out); with a
 *                  chunk table only the table's elements are summed (alignment padding between parameters and the
 *                  zero-padded classifier rows belong to no parameter), else x[0, n)
 *   cb_adamw_step  AdamW of src/optimization/adamw.py:40-103 (eps added to sqrt(v), bias-corrected step size,
 *                  decoupled decay p -= lr*wd*p AFTER the Adam update) on every element named by the chunk table,
 *                  with the clip coefficient min(1, max_norm / (sqrt(*grad_sumsq) + 1e-6)) applied to the gradient
 *                  on the fly (grad_sumsq NULL or max_norm <= 0: no clipping), optional zeroing of the gradient
 *                  (optimizer.zero_grad(), :486) and emission of the bf16 tensor-core operand copy (the apex amp O2
 *                  master->model copy, :307-309) with the FrozenBN scale folded in for conv weights.
 * chunks: int64 [nchunks][8] device = offset, numel (<= 65536), group, row_len, scale_off (-1 none), flags (bit 0: emit
 *         packed), elem0 (index of the chunk's first element inside its parameter), 0
 * hyper : fp32 [ngroups][8] device = lr, step_size (lr * sqrt(1-b2^t) / (1-b1^t) when correct_bias), weight_decay,
 *         beta1, beta2, eps, 0, 0  - refreshed by the caller each step, so the launch itself is graph-capturable.
 * ------------------------------------------------------------------------------------------ */
int cb_sumsq(const float* x, int64_t n, const int64_t* chunks, int nchunks, float* out, void* stream);
/* deterministic: block b (one per chunk-table row, else min(ceil(n / 1024), 1056) grid-stride blocks) stores its sum to
 * scratch[b], then out[0] += the ordered sum of the partials (as cb_clip_lse_loss_det) */
int64_t cb_sumsq_scratch_bytes(int64_t n, const int64_t* chunks, int nchunks);
int cb_sumsq_det(const float* x, int64_t n, const int64_t* chunks, int nchunks, float* out, float* scratch, int64_t scratch_bytes,
                 void* stream);
int cb_adamw_step(float* master, float* grad, float* exp_avg, float* exp_avg_sq, void* packed_bf16, const int64_t* chunks,
                  int nchunks, const float* hyper, const float* scales, const float* grad_sumsq, float max_norm, int zero_grad,
                  void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CLIPBERT_B200_H_ */
