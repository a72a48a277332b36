"""cb_gemm (TN, NN, WGRAD) and cb_gemm_wgrad_group, element by element, against a float64 restatement, on every kernel path.

Every case is built from its descriptor and forces its path: block_n, the k-chunks per stage (cb_gemm_desc.reserved bits 8-11),
the MN-major 3-D box (ops.set_mn3d) and the grid cap (ops.set_sm_limit, which puts many tiles on each persistent CTA at small
M). reserved always carries SINGLE, so no tuning table takes part. The epilogue kind (EK_* in csrc/gemm.cu) and the
epilogue-input placement (plan_smem: two dedicated buffers, one buffer, or the ring stage after the operands) are restated
below in Python; each case names the ones it expects and asserts them, and its test ID names them.

Reference. float64 from the exact bf16 / fp32 inputs the kernel read (TN / NN):
  acc[m, n] = sum_t sum_k A[m + shift_t, k] B_t[k, n]  (rows outside [0, a_rows) read as zero: TMA's fill)
  v = acc * scale[n] + shift[n] ; v *= r (dropout multiplier of output row * N + column) ; v += residual[m, n] ;
  out2 = v (or gelu'(v) for GELU_STASH_GRAD) ; v = act(v) ; v *= auxfn(aux[m, n]) ; out[row(m), n] = v
and next to it the terms T = sum_t |A| @ |B_t| (every |a b| the accumulator adds). WGRAD: out[m, t N + n] = out0 +
scale[m] sum_p A[p, m] B[p + shift_t, n], with T the same sum of |a b|.

Bounds, per element (U = 2^-24), carried through the epilogue as an absolute error e next to the value v:
  accumulation  e = 3 n U T, n = K ntaps: wgmma's fp32 accumulation aligns the addends of a k-block to the largest and
                truncates (Fasi, Higham, Mikaitis, Pranesh 2021), at most 2^-23 (k + 1) of the largest addend per block,
                below 3 n U sum|terms| (the argument of tests/test_gpu_attention_elementwise.py).
  each fp32 step (scale, shift, dropout multiply, residual add, aux multiply)  e' = |c| e + U |v'| for a multiply by the
                exact c, e' = e + U |v'| for an add of an exact value.
  relu          Lipschitz 1, exact: e' = e (0 where the select gives 0 exactly).
  gelu          fast_erf (Abramowitz-Stegun 7.1.26, 1.5e-7 absolute, plus its fp32 evaluation with rcp.approx and
                __expf: E_ERF = 1.5e-7 + 16 U): e' = 1.13 e + 0.5 |v| E_ERF + 4 U |gelu(v)| (|gelu'| <= 1.13).
  gelu'         (stash and CB_AUX_GELU_GRAD) Lipschitz |gelu''| <= 0.8 on the input error; 0.5 E_ERF from the cdf;
                |v| pdf(v) (6 + 5 v^2 / 2) U from __expf(-v^2/2) (2 + 1.17|x| ulp) and the rounding of v^2; 3 U |gelu'|.
  tanh          the library is built with --use_fast_math, so tanhf is tanh.approx.f32 (MUFU.TANH): relative error
                2^-10.987 (PTX ISA): e' = e + 2^-10.9 |tanh(v)|.
  1 - aux^2     U (aux^2 + |1 - aux^2|).
  final         bf16: 1 ulp_bf16(ref) + e (the fp32 value within e of ref, rounded once; its ulp may be one binade above
                ref's); fp32: e. Both + 2^-126 (the library flushes subnormal fp32 results to zero).
  WGRAD         |s| T U (3 P + 1) + (S + 1) U (|out0| + |s| T): the accumulation over P, the row scale, and one fp32
                addition per K-split (red.add or the deterministic plane sum) onto the initial value.

NaN / inf rules (include/clipbert_b200.h): a NaN in one row of A / one column of B gives NaN exactly in that row / column;
ReLU passes NaN and +inf, gives +0 for -inf and for a -0 pre-activation; CB_AUX_RELU_MASK is a select on (aux > 0) with
aux > 0 meaning a positive normal bf16 or +inf, so a NaN, zero or subnormal aux gives 0 on every epilogue kind, even for a
NaN / inf incoming value. Nothing is pinned about gelu of +-inf and no case feeds one.

K tail with ntaps = 9: the last k-chunk of a tap spans past K into the next tap's columns of B (TN: B is one [N, 9K] map),
but A's map ends at K, so those columns meet A's zero fill: the result is exact for finite B, and cb_gemm accepts it. The
K = 72 and K = 200 cases with ntaps = 9 check this.

Around the data: out and out2 are Guarded (sentinel guard bands and pitch columns; an element still holding the sentinel
was never written); under PAD the zero border must stay zero bits. A, B, residual, aux, scale and shift sit in NaN: 64 rows
before and after each window, and the pitch columns, so a read past a_rows / b_rows / K / N poisons the output. The border
rows of a padded activation are zero, as the contract requires. Each TN / NN case runs twice and must give the same bits;
deterministic WGRAD too. Every case prints "RATIO <path> <case>-<output> <max err / bound>".

The CPU runs the same cases (those small enough) through tests/ops_emulator.py and self-tests the reference: it equals
float64 autograd on small cases, and each deliberate fault below, computed in float64 and rounded once, is rejected.
"""
import contextlib
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dropout_ref as D
import ops_emulator as E
from elementwise import BF16, F32, F64, U, Guarded, _INT, _SENT, _record, check_bound, rne_bf16, ulp_bf16
from util import TOL_BF16_OP, relerr

SINGLE = 2                  # cb_gemm_desc.reserved bit 1: launch exactly this descriptor (no tuning-table lookup)
PAD_ROWS = 64               # NaN rows before and after each input window
TN, WGRAD, NN = 0, 1, 2
ACT = {"none": 0, "relu": 1, "gelu": 2, "tanh": 3, "stash": 4}
AUXM = {"none": 0, "mask": 1, "gelu": 2, "tanh": 3, "mul": 4}
NONE, PAD, UNPAD = 0, 1, 2
E_ERF = 1.5e-7 + 16 * U
TANH_REL = 2.0 ** -10.9
FTZ = 2.0 ** -126
FMAX = float(torch.finfo(F32).max)

# ------------------------------------------------------------------------------------------------ csrc/gemm.cu restated
SMEM_LIMIT, BM, BK, MAX_STAGES, BAR_BYTES = 232448, 128, 64, 8, 256
EPI_BYTES = 8 * 16 * 36 * 4         # fp32 staging: 8 consumer warps x 16 rows x STG_PITCH 36
IN_BOX = 128 * 64 * 2               # one epilogue-input box


def _cdiv(a, b):
    return -(-a // b)


def _tdiv(a, b):
    """C integer division (truncates toward zero)."""
    return int(a / b)


def plan_ring(bn, staging, kiters, force_kch, in_bytes, n_in):
    chunk = BM * BK * 2 + bn * BK * 2
    fit = _tdiv(SMEM_LIMIT - 1024 - BAR_BYTES - (EPI_BYTES if staging else 0) - n_in * in_bytes, chunk)
    min_stages = 3 if kiters > fit else 2
    kch = 1
    if force_kch > 0:
        kch = force_kch
    elif kiters >= 4 and fit >= 4 * min_stages:
        kch = 4
    elif kiters >= 2 and fit >= 2 * min_stages:
        kch = 2
    kch = min(kch, kiters)
    if kch > 1 and _tdiv(fit, kch) < 2:
        kch = 1
    stages = min(_tdiv(fit, kch), MAX_STAGES)
    si = _cdiv(kiters, kch)
    stages = min(stages, 2 * si + 1 if staging else max(si + 1, 2))
    return dict(kch=kch, stages=stages, n_in=n_in, chunk=chunk)


def plan_smem(bn, staging, kiters, force_kch=0, in_bytes=0):
    none = plan_ring(bn, staging, kiters, force_kch, 0, 0)
    if in_bytes == 0:
        return none
    two = plan_ring(bn, staging, kiters, force_kch, in_bytes, 2)
    if two["stages"] >= 2 and two["stages"] * two["kch"] >= kiters:
        return two
    if kiters > 4 and none["stages"] >= 2 and none["kch"] * none["chunk"] >= in_bytes:
        return none
    return plan_ring(bn, staging, kiters, force_kch, in_bytes, 1)


def tile_width(c):
    """choose_config for an explicit block_n: 256 runs as 128 on TN / NN; a width whose tile would be mostly padding
    (N <= BN / 2), or that leaves no 2-stage ring, is skipped, and the launch falls back to 64."""
    wgrad = c.mode == WGRAD
    bn = 128 if (not wgrad and c.bn == 256) else c.bn
    if bn > 64 and c.N <= bn // 2:
        return 64
    kc = _cdiv(c.K, BK)
    ips = _cdiv(kc, c.splits()) if wgrad else kc * c.ntaps
    if plan_smem(bn, not wgrad, ips, c.kch, c.in_bytes(bn))["stages"] < 2:
        return 64
    return bn


def placement(c):
    bn = tile_width(c)
    if not c.in_bytes(bn):
        return "noinputs"
    return {2: "twobuf", 1: "onebuf", 0: "ring"}[plan_smem(bn, True, _cdiv(c.K, BK) * c.ntaps, c.kch, c.in_bytes(bn))["n_in"]]


def kind(c):
    """The epilogue kind gemm_pingpong_kernel selects for the launch."""
    has_res, has_aux, has_shift, o2, drop = c.res, c.aux != "none", c.shift, c.out2, c.p > 0
    act, am = ACT[c.act], AUXM[c.aux]
    if c.N % 16 == 0 and not c.scale:
        if not drop and not o2 and not has_aux and act in (0, 1):
            return "SHIFT_ACT"
        if not drop and not o2 and not has_shift and has_aux and am == 1 and act == 0:
            return "RELU_MASK"
        if drop and not o2 and not has_aux and act == 0:
            return "DROP_RES"
        if not drop and o2 and not has_aux and not has_res and act == 4:
            return "GELU_STASH"
        if not drop and not o2 and not has_shift and has_aux and am == 4 and act == 0:
            return "AUX_MUL"
    return "GENERIC_GUARD" if c.N % 16 else "GENERIC"


# ------------------------------------------------------------------------------------------------ cases
class Case:
    """One TN / NN launch. img = (NB, H, W) for the tap and row-map modes: ntaps = 9 and UNPAD read a zero-bordered
    activation of NB (H + 2)(W + 2) rows; PAD writes one."""

    def __init__(self, mode, M, N, K, bn=64, kch=0, ntaps=1, sign=1, tap_w=0, rowmap=NONE, img=None, scale=False,
                 shift=False, res=False, aux="none", act="none", out2=False, fp32=False, p=0.0, word=False, sm=0, mn3d=1,
                 pitch=0, nan=None, expect=None):
        self.mode, self.N, self.K, self.bn, self.kch, self.ntaps, self.sign = mode, N, K, bn, kch, ntaps, sign
        self.rowmap, self.img, self.scale, self.shift, self.res, self.aux, self.act = rowmap, img, scale, shift, res, aux, act
        self.out2, self.fp32, self.p, self.word, self.sm, self.mn3d, self.pitch, self.nan = out2, fp32, p, word, sm, mn3d, pitch, nan
        self.padded = ntaps == 9 or rowmap == UNPAD
        if img is not None:
            NB, H, W = img
            M = NB * H * W if rowmap == PAD else NB * (H + 2) * (W + 2)
            tap_w = W + 2 if ntaps == 9 else tap_w
        self.M, self.tap_w = M, tap_w
        self.expect = expect

    def splits(self):
        return 1

    def in_bytes(self, bn):
        return (int(self.res) + int(self.aux != "none")) * (bn // 64) * IN_BOX

    @property
    def path(self):
        return "%s%d" % ("tn" if self.mode == TN else "nn", tile_width(self))

    @property
    def id(self):
        s = "%s-M%d-N%d-K%d-bn%d-%s-%s" % ("tn" if self.mode == TN else "nn", self.M, self.N, self.K, self.bn, kind(self), placement(self))
        s += "-kch%d" % self.kch if self.kch else "-kchauto"
        if self.ntaps > 1:
            s += "-taps%d%s" % (self.ntaps, "+" if self.sign > 0 else "-")
        s += {NONE: "", PAD: "-pad", UNPAD: "-unpad"}[self.rowmap]
        for flag, name in ((self.scale, "scale"), (self.shift, "shift"), (self.res, "res"), (self.out2, "out2"), (self.fp32, "f32")):
            if flag:
                s += "-" + name
        if self.aux != "none":
            s += "-aux" + self.aux
        if self.act != "none":
            s += "-" + self.act
        if self.p:
            s += "-p%g" % self.p + ("-word" if self.word else "")
        if self.sm:
            s += "-sm%d" % self.sm
        if self.mode == NN and not self.mn3d:
            s += "-mn2d"
        if self.pitch:
            s += "-pitch"
        if self.nan:
            s += "-" + self.nan
        return s


def _c(*a, **k):
    return Case(*a, **k)


CASES = [
    # tile widths, one tile (consumer 1 idle), 256 running as 128, N <= BN / 2 falling back to 64
    _c(TN, 1, 64, 64, bn=64, shift=True, act="relu", sm=1, expect=("SHIFT_ACT", "noinputs")),
    _c(TN, 127, 128, 72, bn=128, expect=("SHIFT_ACT", "noinputs")),
    _c(TN, 128, 256, 200, bn=256, shift=True, res=True, act="relu", pitch=16, expect=("SHIFT_ACT", "twobuf")),
    _c(TN, 129, 48, 64, bn=128, res=True, expect=("SHIFT_ACT", "twobuf")),
    _c(NN, 129, 128, 8, bn=64, fp32=True, expect=("SHIFT_ACT", "noinputs")),
    _c(NN, 300, 256, 72, bn=256, shift=True, act="relu", expect=("SHIFT_ACT", "noinputs")),
    # NN with the 3-D box on and off, and an N where it falls back to 2-D boxes
    _c(NN, 1000, 192, 256, bn=64, res=True, aux="mask", sm=2, expect=("RELU_MASK", "twobuf")),
    _c(NN, 1000, 192, 256, bn=64, res=True, aux="mask", sm=2, mn3d=0, expect=("RELU_MASK", "twobuf")),
    _c(NN, 1000, 256, 200, bn=128, aux="mask", expect=("RELU_MASK", "twobuf")),
    _c(NN, 333, 136, 72, bn=128, aux="mask", expect=("GENERIC_GUARD", "twobuf")),
    # k-chunks per stage forced to 1 / 2 / 4 and automatic, on a K loop longer than four chunks (inputs in the ring)
    _c(TN, 700, 256, 512, bn=128, kch=1, res=True, expect=("SHIFT_ACT", "ring")),
    _c(TN, 700, 256, 512, bn=128, kch=2, res=True, expect=("SHIFT_ACT", "ring")),
    _c(TN, 700, 256, 512, bn=128, kch=4, res=True, expect=("SHIFT_ACT", "ring")),
    _c(TN, 700, 256, 512, bn=128, res=True, expect=("SHIFT_ACT", "ring")),
    _c(NN, 700, 128, 3072, bn=64, res=True, aux="mask", sm=3, expect=("RELU_MASK", "ring")),
    _c(TN, 260, 768, 3072, bn=128, shift=True, res=True, p=0.1, expect=("DROP_RES", "ring")),
    # one epilogue-input buffer (residual + aux of a 128-wide tile beside a 4-chunk K loop), and two
    _c(NN, 900, 256, 256, bn=128, res=True, aux="mask", expect=("RELU_MASK", "onebuf")),
    _c(NN, 900, 256, 256, bn=128, res=True, aux="mul", kch=2, expect=("AUX_MUL", "onebuf")),
    _c(TN, 3000, 128, 64, bn=64, res=True, aux="mask", sm=3, expect=("RELU_MASK", "twobuf")),
    # many tiles per CTA at small M: 5 tiles on 1 / 2 / 3 CTAs (odd and even counts per consumer, ring and buffer phase wraps)
    _c(TN, 640, 64, 64, bn=64, shift=True, res=True, act="relu", sm=1, expect=("SHIFT_ACT", "twobuf")),
    _c(TN, 640, 64, 64, bn=64, shift=True, res=True, act="relu", sm=2, expect=("SHIFT_ACT", "twobuf")),
    _c(TN, 640, 64, 64, bn=64, shift=True, res=True, act="relu", sm=3, expect=("SHIFT_ACT", "twobuf")),
    _c(NN, 1100, 128, 128, bn=64, res=True, aux="mask", sm=1, expect=("RELU_MASK", "twobuf")),
    _c(NN, 1100, 128, 576, bn=128, res=True, sm=2, expect=("SHIFT_ACT", "ring")),
    # epilogue kinds
    _c(TN, 500, 768, 64, bn=128, shift=True, res=True, p=0.1, sm=2, expect=("DROP_RES", "twobuf")),
    _c(TN, 500, 256, 128, bn=64, shift=True, act="stash", out2=True, sm=2, expect=("GELU_STASH", "noinputs")),
    _c(NN, 500, 256, 128, bn=128, aux="mul", expect=("AUX_MUL", "twobuf")),
    _c(NN, 500, 256, 128, bn=64, res=True, aux="mul", pitch=8, expect=("AUX_MUL", "twobuf")),
    # the generic kind, field by field (N % 16 == 0), and with GUARD (N % 16 == 8)
    _c(TN, 300, 256, 192, bn=64, scale=True, expect=("GENERIC", "noinputs")),
    _c(TN, 300, 256, 192, bn=128, scale=True, shift=True, res=True, out2=True, act="relu", expect=("GENERIC", "twobuf")),
    _c(TN, 300, 256, 192, bn=64, shift=True, act="gelu", expect=("GENERIC", "noinputs")),
    _c(TN, 300, 256, 192, bn=64, shift=True, act="tanh", expect=("GENERIC", "noinputs")),
    _c(TN, 300, 256, 192, bn=64, shift=True, res=True, act="stash", out2=True, expect=("GENERIC", "twobuf")),
    _c(TN, 300, 256, 192, bn=64, shift=True, p=0.1, res=True, out2=True, act="relu", expect=("GENERIC", "twobuf")),
    _c(NN, 300, 256, 192, bn=64, res=True, aux="gelu", expect=("GENERIC", "twobuf")),
    _c(NN, 300, 256, 192, bn=128, res=True, aux="tanh", expect=("GENERIC", "onebuf")),
    _c(NN, 300, 256, 192, bn=64, shift=True, aux="mask", expect=("GENERIC", "twobuf")),
    _c(TN, 300, 256, 192, bn=64, scale=True, shift=True, fp32=True, expect=("GENERIC", "noinputs")),
    _c(TN, 300, 256, 192, bn=64, p=1.0, expect=("DROP_RES", "noinputs")),
    _c(TN, 129, 8, 64, bn=64, shift=True, act="relu", expect=("GENERIC_GUARD", "noinputs")),
    _c(TN, 129, 24, 72, bn=64, scale=True, shift=True, res=True, out2=True, act="gelu", expect=("GENERIC_GUARD", "twobuf")),
    _c(TN, 333, 136, 200, bn=128, scale=True, shift=True, fp32=True, act="tanh", expect=("GENERIC_GUARD", "noinputs")),
    _c(NN, 1000, 392, 64, bn=128, res=True, aux="mask", sm=3, expect=("GENERIC_GUARD", "twobuf")),
    _c(NN, 1000, 392, 64, bn=64, aux="gelu", p=0.1, expect=("GENERIC_GUARD", "twobuf")),
    _c(TN, 1000, 392, 64, bn=64, shift=True, act="stash", out2=True, sm=2, expect=("GENERIC_GUARD", "noinputs")),
    # taps: 3x3 forward (+1) and dgrad (-1) on TN and NN, K % 64 != 0 tails, row taps
    _c(TN, 0, 64, 64, bn=64, ntaps=9, sign=1, img=(2, 5, 6), rowmap=UNPAD, shift=True, act="relu", expect=("SHIFT_ACT", "noinputs")),
    _c(TN, 0, 128, 72, bn=128, ntaps=9, sign=1, img=(2, 7, 7), rowmap=UNPAD, res=True, sm=2, expect=("SHIFT_ACT", "ring")),
    _c(TN, 0, 136, 200, bn=64, ntaps=9, sign=-1, img=(1, 6, 9), expect=("GENERIC_GUARD", "noinputs")),
    _c(NN, 0, 64, 72, bn=64, ntaps=9, sign=-1, img=(2, 7, 7), rowmap=UNPAD, aux="mask", res=True, expect=("RELU_MASK", "ring")),
    _c(NN, 0, 128, 200, bn=128, ntaps=9, sign=1, img=(1, 5, 6), p=0.1, shift=True, res=True, rowmap=UNPAD, expect=("DROP_RES", "ring")),
    _c(NN, 0, 192, 64, bn=64, ntaps=9, sign=-1, img=(2, 5, 6), mn3d=0, expect=("SHIFT_ACT", "noinputs")),
    _c(TN, 600, 64, 64, bn=64, ntaps=4, sign=1, tap_w=9, shift=True, act="relu", expect=("SHIFT_ACT", "noinputs")),
    _c(TN, 600, 128, 64, bn=128, ntaps=4, sign=-1, tap_w=13, res=True, sm=2, expect=("SHIFT_ACT", "twobuf")),
    # row maps: PAD keeps the zero border; dropout keyed by the mapped row; UNPAD reads residual / aux in padded-row space
    _c(TN, 0, 256, 64, bn=128, img=(3, 5, 6), rowmap=PAD, shift=True, res=True, act="relu", sm=2, expect=("SHIFT_ACT", "twobuf")),
    _c(TN, 0, 64, 64, bn=64, img=(3, 5, 6), rowmap=PAD, res=True, aux="mask", pitch=8, expect=("RELU_MASK", "twobuf")),
    _c(TN, 0, 128, 128, bn=64, img=(2, 6, 7), rowmap=PAD, shift=True, p=0.1, res=True, expect=("DROP_RES", "twobuf")),
    _c(TN, 0, 136, 64, bn=64, img=(2, 6, 7), rowmap=PAD, shift=True, p=0.1, word=True, expect=("GENERIC_GUARD", "noinputs")),
    _c(TN, 0, 128, 64, bn=64, img=(2, 6, 7), rowmap=UNPAD, p=0.1, word=True, res=True, expect=("DROP_RES", "twobuf")),
    _c(NN, 0, 64, 128, bn=64, img=(3, 5, 6), rowmap=UNPAD, res=True, aux="mask", expect=("RELU_MASK", "twobuf")),
    _c(NN, 0, 64, 128, bn=64, img=(3, 5, 6), rowmap=UNPAD, aux="gelu", p=1.0, expect=("GENERIC", "twobuf")),
    # NaN / inf
    _c(TN, 300, 256, 64, bn=64, shift=True, act="relu", nan="nan_a_row", expect=("SHIFT_ACT", "noinputs")),
    _c(TN, 300, 136, 64, bn=64, shift=True, act="relu", nan="nan_a_row", expect=("GENERIC_GUARD", "noinputs")),
    _c(NN, 300, 256, 64, bn=128, shift=True, act="relu", out2=True, nan="nan_b_col", expect=("GENERIC", "noinputs")),
    _c(TN, 300, 256, 64, bn=64, shift=True, res=True, act="relu", nan="inf", expect=("SHIFT_ACT", "twobuf")),
    _c(TN, 300, 256, 64, bn=64, scale=True, act="relu", nan="inf", expect=("GENERIC", "noinputs")),
    _c(TN, 300, 256, 64, bn=64, act="relu", nan="neg_zero", expect=("SHIFT_ACT", "noinputs")),
    _c(NN, 300, 256, 64, bn=64, aux="mask", nan="nan_a_row", expect=("RELU_MASK", "twobuf")),
    _c(NN, 300, 256, 64, bn=64, res=True, aux="mask", nan="inf", expect=("RELU_MASK", "twobuf")),
    _c(NN, 300, 256, 64, bn=64, act="relu", aux="mask", nan="nan_a_row", expect=("GENERIC", "twobuf")),
    _c(NN, 300, 136, 64, bn=64, aux="mask", nan="inf", expect=("GENERIC_GUARD", "twobuf")),
]
NAN_CASES = [c for c in CASES if c.nan]


class WCase:
    """One weight gradient (or, with group, a cb_gemm_wgrad_group of problems)."""
    mode = WGRAD
    kch = 0
    ntaps = 1

    def __init__(self, M, N, P, bn=64, split=1, ntaps=1, img=None, scale=True, det=False, mn3d=1, sm=0, pitch=8):
        self.M, self.N, self.bn, self.split, self.ntaps, self.scale, self.det, self.mn3d, self.sm = M, N, bn, split, ntaps, scale, det, mn3d, sm
        self.pitch, self.img = pitch, img
        if ntaps == 9:
            NB, H, W = img
            P = NB * (H + 2) * (W + 2)
            self.tap_w = W + 2
        else:
            self.tap_w = 0
        self.K = P

    def splits(self):
        return self.split

    def real_splits(self):
        kc = _cdiv(self.K, BK)
        sp = max(1, min(self.split, kc))
        return _cdiv(kc, _cdiv(kc, sp))

    def in_bytes(self, bn):
        return 0

    @property
    def id(self):
        s = "wgrad-M%d-N%d-P%d-bn%d-split%d" % (self.M, self.N, self.K, self.bn, self.split)
        if self.real_splits() != self.split:
            s += "(%d)" % self.real_splits()
        if self.ntaps == 9:
            s += "-taps9"
        s += "-scale" if self.scale else "-noscale"
        if self.det:
            s += "-det"
        if not self.mn3d:
            s += "-mn2d"
        if self.sm:
            s += "-sm%d" % self.sm
        return s


WCASES = [
    WCase(128, 128, 256, bn=64),
    WCase(200, 136, 1000, bn=128, split=2),
    WCase(256, 256, 448, bn=256, split=3),
    WCase(64, 512, 448, bn=256, split=5, scale=False),
    WCase(384, 192, 960, bn=64, split=4, det=True),
    WCase(384, 192, 960, bn=128, split=3, det=True, mn3d=0),
    WCase(136, 64, 1000, bn=64, split=1, det=True, sm=2),
    WCase(128, 64, 0, bn=64, split=2, ntaps=9, img=(2, 5, 6)),
    WCase(200, 72, 0, bn=128, split=1, ntaps=9, img=(1, 7, 7), scale=False),
    WCase(64, 128, 0, bn=256, split=3, ntaps=9, img=(2, 6, 7), det=True),
    WCase(256, 256, 1100, bn=128, split=2, sm=3),
]
# groups: (name, problems, expected to run as one group launch)
GROUPS = [
    ("n2", [WCase(256, 128, 500), WCase(136, 64, 500, ntaps=1)], True),
    ("n4-taps", [WCase(128, 128, 0, ntaps=9, img=(2, 5, 6)), WCase(64, 256, 0, ntaps=1, img=None), WCase(200, 72, 0, ntaps=9, img=(2, 5, 6)),
                 WCase(72, 64, 150)], True),
    ("n8", [WCase(64 + 8 * i, 64 + 16 * (i % 3), 400 + 20 * i) for i in range(8)], True),
    ("n1", [WCase(200, 136, 700)], False),
    ("n9", [WCase(64, 64, 300) for _ in range(9)], False),
    ("k-apart", [WCase(128, 64, 200), WCase(64, 128, 900)], False),
]
for _name, _probs, _grp in GROUPS:
    for _w in _probs:
        if _w.ntaps == 1 and _name == "n4-taps" and _w.K == 0:
            _w.K = 2 * 7 * 8                            # the padded pixel count of the taps problems
GROUPS_DET = [("n3-taps-split2-det", [WCase(128, 128, 0, split=2, ntaps=9, img=(2, 5, 6)), WCase(64, 256, 112),
                                      WCase(200, 72, 0, ntaps=9, img=(2, 5, 6))], True)]


# ------------------------------------------------------------------------------------------------ inputs
class _Window:
    """A [rows, cols] input (bf16) with row pitch cols + pitch inside NaN: PAD_ROWS rows before and after, and the pitch
    columns."""

    def __init__(self, x, dev, pitch=8, dtype=BF16):
        rows, cols = x.shape
        ld = cols + pitch
        self.buf = torch.full(((rows + 2 * PAD_ROWS) * ld,), float("nan"), dtype=dtype, device=dev)
        self.t = self.buf[PAD_ROWS * ld:(PAD_ROWS + rows) * ld].view(rows, ld)[:, :cols]
        self.t.copy_(x)
        self.ld = ld


def _vec(x, dev):
    """fp32 vector in NaN: 8 before (keeps 16-byte alignment), 16 after."""
    buf = torch.full((x.numel() + 24,), float("nan"), dtype=F32, device=dev)
    buf[8:8 + x.numel()] = x
    return buf[8:8 + x.numel()]


def _border_zero(x, img):
    NB, H, W = img
    v = x.view(NB, H + 2, W + 2, -1)
    v[:, 0], v[:, -1], v[:, :, 0], v[:, :, -1] = 0, 0, 0, 0
    return x


_AUX_SPECIAL = [0x7FC0, 0xFFC0, 0x0000, 0x8000, 0x0001, 0x8001, 0x007F, 0x0080, 0x7F80, 0xFF80, 0x7F7F]


def _inputs(c, seed):
    g = torch.Generator().manual_seed(seed)
    M, N, K, nt = c.M, c.N, c.K, c.ntaps
    a_rows = M
    A = torch.randn(a_rows, K, generator=g, dtype=F64)
    if c.padded:
        _border_zero(A, c.img)
    B = torch.randn(N, nt * K, generator=g, dtype=F64) * 0.1 if c.mode == TN else torch.randn(K, nt * N, generator=g, dtype=F64) * 0.1
    ins = dict(A=A.to(BF16), B=B.to(BF16))
    if c.scale:
        ins["scale"] = (torch.rand(N, generator=g, dtype=F64) + 0.5).float()
    if c.shift:
        ins["shift"] = torch.randn(N, generator=g, dtype=F64).float()
    if c.res:
        ins["res"] = torch.randn(M, N, generator=g, dtype=F64).to(BF16)
    if c.aux != "none":
        x = torch.randn(M, N, generator=g, dtype=F64)
        if c.aux == "tanh":
            x = torch.tanh(x)
        x = x.to(BF16)
        if c.aux == "mask":           # NaN, signed zeros, subnormals, the smallest normal, infinities: one per row, rotating
            bits = x.view(torch.int16)
            for i in range(0, M, 3):
                bits[i, (7 * i) % N] = np.int16(np.uint16(_AUX_SPECIAL[(i // 3) % len(_AUX_SPECIAL)]).view(np.int16))
        ins["aux"] = x
    r0, c0 = min(7, M - 1), min(5, N - 1)
    if c.nan == "nan_a_row":
        ins["A"][r0, 3 % K] = float("nan")
    elif c.nan == "nan_b_col":
        if c.mode == TN:
            ins["B"][c0, 2] = float("nan")
        else:
            ins["B"][2, c0] = float("nan")
    elif c.nan == "inf":             # row r0 of A = 2^100 everywhere, column c0 of B = +2^100, column c0 + 1 = -2^100
        ins["A"][r0] = 2.0 ** 100
        if c.mode == TN:
            ins["B"][c0, :K], ins["B"][c0 + 1, :K] = 2.0 ** 100, -2.0 ** 100
        else:
            ins["B"][:, c0], ins["B"][:, c0 + 1] = 2.0 ** 100, -2.0 ** 100
    elif c.nan == "neg_zero":       # row r0 of A = -0 and column c0 of B positive: a -0 pre-activation at (r0, c0)
        ins["A"][r0] = -0.0
        if c.mode == TN:
            ins["B"][c0] = ins["B"][c0].abs()
        else:
            ins["B"][:, c0] = ins["B"][:, c0].abs()
    return ins


def _tap_shift(c, t):
    if c.ntaps == 9:
        return c.sign * ((t // 3 - 1) * c.tap_w + (t % 3 - 1))
    return c.sign * t * c.tap_w if c.ntaps > 1 else 0


def _shifted(A, shift, m):
    """[m, cols]: row i = A[i + shift], zero outside A (TMA's fill)."""
    out = torch.zeros(m, A.shape[1], dtype=A.dtype, device=A.device)
    lo, hi = max(0, -shift), min(m, A.shape[0] - shift)
    if hi > lo:
        out[lo:hi] = A[lo + shift:hi + shift]
    return out


def out_rows(c):
    """destination row of each GEMM row (-1: dropped) and the number of output rows (cb_rowmap)."""
    i = torch.arange(c.M)
    if c.rowmap == NONE:
        return i, c.M
    NB, H, W = c.img
    if c.rowmap == PAD:
        img, r = i // (H * W), i % (H * W)
        return (img * (H + 2) + r // W + 1) * (W + 2) + r % W + 1, NB * (H + 2) * (W + 2)
    img, r = i // ((H + 2) * (W + 2)), i % ((H + 2) * (W + 2))
    y, x = r // (W + 2), r % (W + 2)
    ok = (y >= 1) & (y <= H) & (x >= 1) & (x <= W)
    return torch.where(ok, (img * H + y - 1) * W + x - 1, torch.full_like(i, -1)), NB * H * W


def _gelu(v):
    return 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))


def _pdf(v):
    return torch.exp(-0.5 * v * v) / math.sqrt(2.0 * math.pi)


def _gelu_grad(v):
    return 0.5 * (1.0 + torch.erf(v / math.sqrt(2.0))) + v * _pdf(v)


def _gelu_grad_err(v):
    return 0.5 * E_ERF + v.abs() * _pdf(v) * (6.0 + 2.5 * v * v) * U + 3.0 * U * _gelu_grad(v).abs()


def relu_pos(x_bf16):
    """CB_AUX_RELU_MASK's (aux > 0): a positive normal bf16 or +inf."""
    b = x_bf16.view(torch.int16).to(torch.int64) & 0xFFFF
    return (b >= 0x0080) & (b <= 0x7F80)


def accumulate(c, A, B):
    """acc [M, N] and terms T [M, N], float64, from the bf16 operands (any device)."""
    A64, B64 = A.double(), B.double()
    acc = torch.zeros(c.M, c.N, dtype=F64, device=A.device)
    T = torch.zeros_like(acc)
    for t in range(c.ntaps):
        At = _shifted(A64, _tap_shift(c, t), c.M)
        Bt = B64[:, t * c.K:(t + 1) * c.K].t() if c.mode == TN else B64[:, t * c.N:(t + 1) * c.N]
        acc += At @ Bt
        T += At.abs() @ Bt.abs()
    return acc, T


def reference(c, ins, mult, acc_T=None):
    """(out, bound) and (out2, bound) or None, float64 [M, N] in GEMM-row order (see the module docstring)."""
    acc, T = accumulate(c, ins["A"], ins["B"]) if acc_T is None else acc_T
    dev = acc.device
    v = torch.where(acc.abs() > FMAX, acc.sign() * math.inf, acc)         # the fp32 accumulator overflows to +-inf
    e = 3.0 * c.K * c.ntaps * U * T
    zero = torch.zeros_like(v)
    if c.scale:
        s = ins["scale"].double().to(dev)
        v = v * s
        e = e * s + U * v.abs()
    if c.shift:
        v = v + ins["shift"].double().to(dev)
        e = e + U * v.abs()
    if mult is not None:
        r = mult.double().to(dev)
        v = torch.where(r == 0, zero, v * r)
        e = torch.where(r == 0, zero, e * r + U * v.abs())
    if c.res:
        v = v + ins["res"].double().to(dev)
        e = e + U * v.abs()
    o2 = None
    if c.act == "stash":
        g = _gelu_grad(v)
        o2 = (g, ulp_bf16(g) + 0.8 * e + _gelu_grad_err(v))
    elif c.out2:
        o2 = (v, ulp_bf16(v) + e)
    if c.act == "relu":
        neg = v <= 0
        v = torch.where(neg, zero, v)
        e = torch.where(v.isinf() | (neg & ~(e < math.inf)), zero, e)
    elif c.act in ("gelu", "stash"):
        y = _gelu(v)
        e = 1.13 * e + 0.5 * v.abs() * E_ERF + 4.0 * U * y.abs()
        v = y
    elif c.act == "tanh":
        v = torch.tanh(v)
        e = e + TANH_REL * v.abs()
    if c.aux != "none":
        x = ins["aux"]
        xd = x.double().to(dev)
        if c.aux == "mask":
            pos = relu_pos(x).to(dev)
            v, e = torch.where(pos, v, zero), torch.where(pos, e, zero)
        else:
            if c.aux == "gelu":
                gx, ex = _gelu_grad(xd), _gelu_grad_err(xd)
            elif c.aux == "tanh":
                gx = 1.0 - xd * xd
                ex = U * (xd * xd + gx.abs())
            else:
                gx, ex = xd, torch.zeros_like(xd)
            w = v * gx
            e = e * gx.abs() + v.abs() * ex + U * w.abs()
            v = w
    bound = e + FTZ + (0.0 if c.fp32 else ulp_bf16(v))
    if o2 is not None:
        o2 = (o2[0], o2[1] + FTZ)
    return (v, bound), o2


def _mult(c, seed, word):
    if not c.p:
        return None
    dst, _ = out_rows(c)
    return torch.from_numpy(D.multipliers(D.effective_seed(seed, word), D.gemm_index(dst.clamp(min=0).numpy(), c.N), c.p))


# ------------------------------------------------------------------------------------------------ running a case
class Backend:
    def __init__(self, name):
        self.emulated = name == "emulator"
        self.dev = torch.device("cpu") if self.emulated else torch.device("cuda:0")

    def gemm(self, **kw):
        if self.emulated:
            E.gemm(**kw)
        else:
            from clipbert_b200 import ops
            ops.gemm(**kw)


@contextlib.contextmanager
def _knobs(be, sm=0, mn3d=1, word=None):
    """Grid cap, 3-D box switch and bound dropout word for one case; restores the defaults."""
    mod = E
    if not be.emulated:
        from clipbert_b200 import ops as mod
        mod.set_sm_limit(sm)
        mod.set_mn3d(mn3d)
    w = None if word is None else torch.tensor([word], dtype=torch.int64, device=be.dev)
    mod.dropout_offset_bind(w)
    try:
        yield
    finally:
        mod.dropout_offset_bind(None)
        if not be.emulated:
            mod.set_sm_limit(0)
            mod.set_mn3d(1)


def _bits(t):
    return t.detach().cpu().contiguous().view(_INT[t.dtype]).clone()


def _run(be, c, ins, seed):
    dev = be.dev
    Aw = _Window(ins["A"], dev)
    Bw = _Window(ins["B"], dev)
    dst, n_dst = out_rows(c)
    odt = F32 if c.fp32 else BF16
    out = Guarded((n_dst, c.N), odt, dev, ld=c.N + c.pitch)
    out2 = Guarded((n_dst, c.N), BF16, dev, ld=c.N + c.pitch) if (c.out2 or c.act == "stash") else None
    if c.rowmap == PAD:               # the zero border of a padded output: must stay zero bits
        border = torch.ones(n_dst, dtype=torch.bool)
        border[dst] = False
        for o in (out, out2):
            if o is not None:
                o.t[border.to(dev)] = 0
    kw = dict(mode=c.mode, m=c.M, n=c.N, k=c.K, a=Aw.t, a_rows=c.M, a_ld=Aw.ld, b=Bw.t, b_rows=ins["B"].shape[0], b_ld=Bw.ld,
              ntaps=c.ntaps, tap_w=c.tap_w, tap_sign=c.sign, act=ACT[c.act], out=out.t, out_ld=out.t.stride(0) if out.t.dim() == 2 else c.N,
              out_fp32=int(c.fp32), rowmap=c.rowmap, dropout_p=c.p, dropout_seed=seed, block_n=c.bn, reserved=SINGLE | (c.kch << 8))
    if c.img is not None:
        kw.update(map_h=c.img[1], map_w=c.img[2])
    keep = [Aw, Bw]
    for name, field in (("scale", "scale"), ("shift", "shift")):
        if name in ins:
            kw[field] = _vec(ins[name].to(dev), dev)
            keep.append(kw[field])
    if c.res:
        w = _Window(ins["res"], dev, pitch=8 + c.pitch)
        kw.update(residual=w.t, res_ld=w.ld)
        keep.append(w)
    if c.aux != "none":
        w = _Window(ins["aux"], dev)
        kw.update(aux=w.t, aux_ld=w.ld, aux_mode=AUXM[c.aux])
        keep.append(w)
    if out2 is not None:
        kw.update(out2=out2.t, out2_ld=out2.t.stride(0))
    be.gemm(**kw)
    if not be.emulated:
        torch.cuda.synchronize()
    return out, out2


def _check_padded_border(c, o, what):
    if c.rowmap != PAD or o is None:
        return
    dst, n_dst = out_rows(c)
    border = torch.ones(n_dst, dtype=torch.bool)
    border[dst] = False
    assert bool((_bits(o.t)[border] == 0).all()), "%s %s: the zero border of the padded output was written" % (c.id, what)


def _compare(c, out, out2, refs):
    (ref, bound), o2 = refs
    dst, _ = out_rows(c)
    keep = dst >= 0
    ratios = {"out": check_bound("%s out" % c.id, out.t.cpu()[dst[keep]], ref.cpu()[keep], bound.cpu()[keep])}
    if o2 is not None:
        ratios["out2"] = check_bound("%s out2" % c.id, out2.t.cpu()[dst[keep]], o2[0].cpu()[keep], o2[1].cpu()[keep])
    return ratios


def _gemm_case(be, c):
    seed = 17 + c.M + 3 * c.N + c.K
    word = 0x5EED + c.M if c.word else None
    assert (kind(c), placement(c)) == c.expect, "%s: expected %s, the launch selects %s" % (c.id, c.expect, (kind(c), placement(c)))
    ins = _inputs(c, seed)
    with _knobs(be, c.sm, c.mn3d, word):
        out, out2 = _run(be, c, ins, seed)
        if not be.emulated:
            out_b, out2_b = _run(be, c, ins, seed)
    for o, name in ((out, "out"), (out2, "out2")):
        if o is not None:
            o.check("%s %s" % (c.id, name))
            _check_padded_border(c, o, name)
    if c.nan == "neg_zero":           # relu(+-0) is +0: every element of row r0 (a -0 pre-activation at column c0)
        r0 = min(7, c.M - 1)
        assert bool((_bits(out.t)[r0] == 0).all()), "%s: relu of a zero pre-activation is not +0: %s" % (c.id, _bits(out.t)[r0][:8].tolist())
    if not be.emulated:
        assert torch.equal(_bits(out.t), _bits(out_b.t)), "%s: out differs between two identical runs" % c.id
        if out2 is not None:
            assert torch.equal(_bits(out2.t), _bits(out2_b.t)), "%s: out2 differs between two identical runs" % c.id
    dev = be.dev
    ins_d = {k: v.to(dev) for k, v in ins.items()}
    refs = reference(c, ins_d, _mult(c, seed, word))
    ratios = _compare(c, out, out2, refs)
    for name, r in ratios.items():
        _record(c.path, "%s-%s" % (c.id, name), r)


_EMU_MAX = 4e7      # multiply-adds of the emulated cases (the CPU float64 reference and emulator)
EMU_CASES = [c for c in CASES if c.M * c.N * c.K * c.ntaps <= _EMU_MAX]


@pytest.mark.parametrize("be_name,case", [pytest.param("device", c, marks=pytest.mark.gpu, id="device-" + c.id) for c in CASES]
                         + [pytest.param("emulator", c, id="emulator-" + c.id) for c in EMU_CASES])
def test_gemm_elementwise(be_name, case):
    if be_name == "device" and not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    _gemm_case(Backend(be_name), case)


# ------------------------------------------------------------------------------------------------ WGRAD
def _w_inputs(w, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(w.K, w.M, generator=g, dtype=F64)
    B = torch.randn(w.K, w.N, generator=g, dtype=F64)
    if w.ntaps == 9:
        _border_zero(A, w.img)
        _border_zero(B, w.img)
    ins = dict(A=A.to(BF16), B=B.to(BF16), out0=torch.randn(w.M, w.ntaps * w.N, generator=g, dtype=F64).float())
    if w.scale:
        ins["scale"] = (torch.rand(w.M, generator=g, dtype=F64) + 0.5).float()
    return ins


def w_reference(w, ins, splits=None, drop_split=None):
    """out0 + scale[m] sum_p A[p, m] B[p + shift_t, n] and its bound; drop_split leaves that K-split's range out (a fault)."""
    A, B = ins["A"].double(), ins["B"].double()
    if drop_split is not None:
        kc = _cdiv(w.K, BK)
        ips = _cdiv(kc, w.real_splits())
        A = A.clone()
        A[drop_split * ips * BK:(drop_split + 1) * ips * BK] = 0
    acc, T = [], []
    for t in range(w.ntaps):
        sh = 0 if w.ntaps == 1 else (t // 3 - 1) * w.tap_w + (t % 3 - 1)
        Bt = _shifted(B, sh, w.K)
        acc.append(A.t() @ Bt)
        T.append(A.abs().t() @ Bt.abs())
    acc, T = torch.cat(acc, 1), torch.cat(T, 1)
    s = ins["scale"].double().to(acc.device)[:, None] if w.scale else torch.ones(w.M, 1, dtype=F64, device=acc.device)
    o0 = ins["out0"].double().to(acc.device)
    S = splits or w.real_splits()
    ref = o0 + s * acc
    bound = s * T * U * (3.0 * w.K + 1.0) + (S + 1.0) * U * (o0.abs() + s * T) + FTZ
    return ref, bound


def _w_launch(be, ws, ins_list, outs, group, raw_group=False):
    kws = []
    keep = []
    for w, ins, o in zip(ws, ins_list, outs):
        Aw, Bw = _Window(ins["A"], be.dev, pitch=w.pitch), _Window(ins["B"], be.dev, pitch=w.pitch)
        keep += [Aw, Bw]
        kw = dict(mode=WGRAD, m=w.M, n=w.N, k=w.K, a=Aw.t, a_rows=w.K, a_ld=Aw.ld, b=Bw.t, b_rows=w.K, b_ld=Bw.ld, ntaps=w.ntaps,
                  tap_w=w.tap_w, tap_sign=1, out=o.t, out_ld=o.t.stride(0), out_fp32=1, block_n=w.bn, split_k=w.split,
                  reserved=SINGLE)
        if w.scale:
            kw["scale"] = _vec(ins["scale"].to(be.dev), be.dev)
            keep.append(kw["scale"])
        kws.append(kw)
    if be.emulated:
        for kw in kws:                # the emulator's group is n cb_gemm launches
            E.gemm(**kw)
        return
    from clipbert_b200 import ops
    if raw_group:                     # cb_gemm_wgrad_group itself, also for n = 1 (ops.gemm_wgrad_group sends n = 1 to cb_gemm)
        if ops.deterministic():
            kws[0] = ops._with_workspace(kws[0], ops.gemm_wgrad_group_workspace_bytes(kws))
        ops._launch_gemm("cb_gemm_wgrad_group", kws)
    elif group:
        ops.gemm_wgrad_group(kws)
    else:
        ops.gemm(**kws[0])
    torch.cuda.synchronize()


@contextlib.contextmanager
def _deterministic(be, on):
    if not on or be.emulated:
        yield
        return
    from clipbert_b200 import ops
    torch.use_deterministic_algorithms(True)
    ops.deterministic()
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(False)
        ops.deterministic()


def _w_outs(be, ws, ins_list):
    return [Guarded((w.M, w.ntaps * w.N), F32, be.dev, ld=w.ntaps * w.N + 8, init=ins["out0"].to(be.dev)) for w, ins in zip(ws, ins_list)]


def _wgrad_case(be, tag, ws, group, det=False, expect_group=None):
    ins_list = [_w_inputs(w, 100 + i + w.M + w.N + w.K) for i, w in enumerate(ws)]
    sm = ws[0].sm
    with _knobs(be, sm, ws[0].mn3d), _deterministic(be, det):
        outs = _w_outs(be, ws, ins_list)
        _w_launch(be, ws, ins_list, outs, group, raw_group=group)
        if det and not be.emulated:
            outs_b = _w_outs(be, ws, ins_list)
            _w_launch(be, ws, ins_list, outs_b, group, raw_group=group)
    for i, (w, ins, o) in enumerate(zip(ws, ins_list, outs)):
        o.check("%s problem %d out" % (tag, i))
        if det and not be.emulated:
            assert torch.equal(_bits(o.t), _bits(outs_b[i].t)), "%s problem %d: deterministic mode is not bit-repeatable" % (tag, i)
        dev = be.dev
        ref, bound = w_reference(w, {k: v.to(dev) for k, v in ins.items()}, splits=8 if group else None)
        r = check_bound("%s problem %d" % (tag, i), o.t.cpu(), ref.cpu(), bound.cpu())
        _record("wgrad%d" % tile_width(w) if not group else "wgrad_group", "%s-p%d-out" % (tag, i), r)


W_EMU = [w for w in WCASES if w.M * w.N * w.K * w.ntaps <= _EMU_MAX]


@pytest.mark.parametrize("be_name,w", [pytest.param("device", w, marks=pytest.mark.gpu, id="device-" + w.id) for w in WCASES]
                         + [pytest.param("emulator", w, id="emulator-" + w.id) for w in W_EMU])
def test_wgrad_elementwise(be_name, w):
    if be_name == "device" and not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    _wgrad_case(Backend(be_name), w.id, [w], group=False, det=w.det)


def _group_plan(ws):
    """group_plan's groupable test: 2 <= n <= 8 and reduction lengths within 2x of the first."""
    n = len(ws)
    return 2 <= n <= 8 and all(not (w.K * 2 < ws[0].K or ws[0].K * 2 < w.K) for w in ws)


@pytest.mark.parametrize("be_name,name", [pytest.param("device", n, marks=pytest.mark.gpu, id="device-" + n) for n, _, _ in GROUPS + GROUPS_DET]
                         + [pytest.param("emulator", n, id="emulator-" + n) for n, _, _ in GROUPS])
def test_wgrad_group_elementwise(be_name, name):
    if be_name == "device" and not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ws, grouped = next((p, g) for n, p, g in GROUPS + GROUPS_DET if n == name)
    assert _group_plan(ws) == grouped, "%s: group_plan would %sgroup these problems" % (name, "not " if grouped else "")
    _wgrad_case(Backend(be_name), "group-" + name, ws, group=True, det=name.endswith("-det"))


def test_matrix_covers_every_path():
    """Every kernel path, epilogue kind and field, input placement, tap mode, row map and shape edge is in the matrix, and
    each case's expected kind / placement is the one the launch selects (asserted again when the case runs)."""
    for c in CASES:
        assert (kind(c), placement(c)) == c.expect, (c.id, kind(c), placement(c))
    assert {kind(c) for c in CASES} == {"SHIFT_ACT", "RELU_MASK", "DROP_RES", "GELU_STASH", "AUX_MUL", "GENERIC", "GENERIC_GUARD"}
    assert {placement(c) for c in CASES} == {"noinputs", "twobuf", "onebuf", "ring"}
    assert {(c.mode, c.bn) for c in CASES} >= {(m, b) for m in (TN, NN) for b in (64, 128, 256)}
    assert {c.kch for c in CASES} >= {0, 1, 2, 4} and {c.sm for c in CASES} >= {1, 2, 3}
    assert {c.mn3d for c in CASES if c.mode == NN and c.N % 64 == 0} == {0, 1} and any(c.mode == NN and c.N % 64 for c in CASES)
    assert {(c.mode, c.ntaps, c.sign) for c in CASES} >= {(TN, 9, 1), (TN, 9, -1), (NN, 9, 1), (NN, 9, -1), (TN, 4, 1)}
    assert {c.rowmap for c in CASES} == {NONE, PAD, UNPAD} and any(c.rowmap == UNPAD and (c.res or c.aux != "none") for c in CASES)
    assert {1, 127, 128, 129} <= {c.M for c in CASES} and {8, 24, 136, 392} <= {c.N for c in CASES}
    assert {8, 72, 200, 3072} <= {c.K for c in CASES} and any(c.N < c.bn // 2 for c in CASES)
    assert {c.act for c in CASES} == set(ACT) and {c.aux for c in CASES} == set(AUXM)
    assert {c.p for c in CASES} >= {0.1, 1.0} and any(c.word for c in CASES) and {c.rowmap for c in CASES if c.p} >= {PAD, UNPAD}
    assert any(c.fp32 for c in CASES) and any(c.out2 and c.act != "stash" for c in CASES)
    assert {w.bn for w in WCASES} == {64, 128, 256} and {w.split for w in WCASES} >= {1, 2, 3}
    assert any(w.real_splits() != w.split for w in WCASES) and {w.ntaps for w in WCASES} == {1, 9}
    assert {w.scale for w in WCASES} == {True, False} and any(w.det for w in WCASES)
    assert any(w.M % 128 for w in WCASES) and any(w.N % w.bn for w in WCASES) and any(w.K % 64 for w in WCASES)


# ------------------------------------------------------------------------------------------------ host checks
@pytest.mark.gpu
@pytest.mark.parametrize("field", ["a", "b", "out", "out2", "wgrad_a", "wgrad_b"])
def test_misaligned_base_is_rejected_without_launching(cuda, field):
    """cb_gemm refuses an A / B base TMA cannot read and an out / out2 base the epilogue's 16-byte stores cannot write; nothing
    is launched and the output is unchanged."""
    from clipbert_b200 import ops
    M, N, K = 256, 128, 64
    g = torch.Generator().manual_seed(3)

    def t(rows, cols, off=0):
        buf = (torch.randn(rows * cols + 8, generator=g)).to(cuda).to(BF16)
        return buf[off:off + rows * cols].view(rows, cols)

    A, B = t(M, K, 1 if field == "a" else 0), t(N, K, 1 if field == "b" else 0)
    C, C2 = t(M, N, 1 if field == "out" else 0), t(M, N, 1 if field == "out2" else 0)
    kw = dict(mode=TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=N, b_ld=K, act=ACT["stash"], out=C, out_ld=N, out2=C2, out2_ld=N,
              reserved=SINGLE)
    what = field
    if field.startswith("wgrad"):
        dY, X = t(K, M, 1 if field == "wgrad_a" else 0), t(K, N, 1 if field == "wgrad_b" else 0)
        C = torch.zeros(M, N, device=cuda)
        kw = dict(mode=WGRAD, m=M, n=N, k=K, a=dY, a_rows=K, a_ld=M, b=X, b_rows=K, b_ld=N, out=C, out_ld=N, out_fp32=1, reserved=SINGLE)
        what = "a and b"
    before = C.clone()
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match="%s must be 16-byte aligned" % what):
        ops.gemm(**kw)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0
    assert torch.equal(_bits(C), _bits(before))


# ------------------------------------------------------------------------------------------------ CPU self-tests
def _small(**kw):
    base = dict(mode=TN, M=300, N=136, K=200, bn=64)
    base.update(kw)
    return Case(base.pop("mode"), base.pop("M"), base.pop("N"), base.pop("K"), **base)


def _ref_ok(c, ins, got, mult=None, which="out"):
    (ref, bound), o2 = reference(c, ins, mult)
    if which == "out2":
        ref, bound = o2
    check_bound("fault", got, ref, bound)


def test_reference_accepts_itself_rounded_and_matches_autograd():
    """The reference rounded once passes its own bounds, and its unrounded value equals float64 torch / autograd: F.linear +
    shift + residual + gelu, gelu' from autograd, the 3x3 conv and its dgrad (F.conv2d / conv_transpose2d), the wgrad from
    autograd of conv2d."""
    c = _small(shift=True, res=True, act="stash", out2=True)
    ins = _inputs(c, 5)
    (ref, bound), o2 = reference(c, ins, None)
    check_bound("self", rne_bf16(ref), ref, bound)
    check_bound("self out2", rne_bf16(o2[0]), o2[0], o2[1])
    u = (F.linear(ins["A"].double(), ins["B"].double()) + ins["shift"].double() + ins["res"].double()).requires_grad_(True)
    with torch.enable_grad():
        y = F.gelu(u)
        (gu,) = torch.autograd.grad(y.sum(), u)
    assert torch.allclose(ref, y.detach(), rtol=1e-12, atol=1e-12) and torch.allclose(o2[0], gu, rtol=1e-12, atol=1e-12)
    # 3x3 forward (TN, +1) and dgrad (NN, -1) over a zero-bordered activation, interior rows
    NB, H, W = 2, 5, 6
    for mode, sign in ((TN, 1), (NN, -1)):
        c = Case(mode, 0, 64, 72, ntaps=9, sign=sign, img=(NB, H, W), rowmap=UNPAD)
        ins = _inputs(c, 6)
        (ref, _), _ = reference(c, ins, None)
        dst, _ = out_rows(c)
        x = ins["A"].double().view(NB, H + 2, W + 2, 72)[:, 1:-1, 1:-1].permute(0, 3, 1, 2)
        if mode == TN:
            wt = ins["B"].double().view(64, 3, 3, 72).permute(0, 3, 1, 2)
            want = F.conv2d(x, wt, padding=1)
        else:
            wt = ins["B"].double().view(72, 3, 3, 64).permute(0, 3, 1, 2)
            want = F.conv_transpose2d(x, wt, padding=1)
        assert torch.allclose(ref[dst >= 0], want.permute(0, 2, 3, 1).reshape(-1, 64), rtol=1e-12, atol=1e-10)
    w = WCase(64, 72, 0, ntaps=9, img=(NB, H, W), scale=False)
    ins = _w_inputs(w, 7)
    ref, bound = w_reference(w, ins)
    dy = ins["A"].double().view(NB, H + 2, W + 2, 64)[:, 1:-1, 1:-1].permute(0, 3, 1, 2)
    x = ins["B"].double().view(NB, H + 2, W + 2, 72)[:, 1:-1, 1:-1].permute(0, 3, 1, 2)
    wz = torch.zeros(64, 72, 3, 3, dtype=F64, requires_grad=True)
    with torch.enable_grad():
        F.conv2d(x, wz, padding=1).backward(dy)
    want = ins["out0"].double() + wz.grad.permute(0, 2, 3, 1).reshape(64, 9 * 72)
    assert torch.allclose(ref, want, rtol=1e-12, atol=1e-9)
    check_bound("self wgrad", ref.float(), ref, bound)


def test_fault_residual_of_one_warp_from_the_neighbouring_tile_is_rejected_but_passes_the_normwise_check():
    """Rows 16..31 of the last (partial) tile take their residual from the tile before: rejected element by element; with a
    shortcut small next to the product (as after a FrozenBN) on 16384 rows, the normwise TOL_BF16_OP check accepts it."""
    c = Case(TN, 16384 + 40, 256, 64, res=True)
    ins = _inputs(c, 8)
    ins["res"] = (ins["res"].double() * 0.05).to(BF16)
    bad = dict(ins)
    R = ins["res"].clone()
    m0 = (c.M // 128) * 128
    R[m0 + 16:m0 + 32] = ins["res"][m0 - 128 + 16:m0 - 128 + 32]
    bad["res"] = R
    (got, _), _ = reference(c, bad, None)
    with pytest.raises(AssertionError, match="out of bound"):
        _ref_ok(c, ins, rne_bf16(got))
    (ref, _), _ = reference(c, ins, None)
    assert relerr(rne_bf16(got), ref) < TOL_BF16_OP


def test_fault_last_8_of_k_dropped_is_rejected():
    c = _small()
    ins = _inputs(c, 9)
    bad = dict(ins, A=ins["A"].clone())
    bad["A"][:, -8:] = 0
    (got, _), _ = reference(c, bad, None)
    with pytest.raises(AssertionError, match="out of bound"):
        _ref_ok(c, ins, rne_bf16(got))


def test_fault_dropout_keyed_by_out_ld_is_rejected():
    c = _small(N=128, p=0.1, shift=True, res=True)
    ins = _inputs(c, 10)
    seed = 77
    good = _mult(c, seed, None)
    dst, _ = out_rows(c)
    bad = torch.from_numpy(D.multipliers(seed, D.gemm_index(dst.numpy(), c.N + 16), c.p))[:, :c.N]
    (got, _), _ = reference(c, ins, bad)
    with pytest.raises(AssertionError, match="out of bound"):
        _ref_ok(c, ins, rne_bf16(got), good)


def test_fault_one_tap_shifted_by_one_pixel_is_rejected():
    c = Case(TN, 0, 64, 64, ntaps=9, img=(2, 5, 6), rowmap=UNPAD)
    ins = _inputs(c, 11)
    acc, T = accumulate(c, ins["A"], ins["B"])
    t = 5
    A64, B64 = ins["A"].double(), ins["B"].double()
    Bt = B64[:, t * c.K:(t + 1) * c.K].t()
    acc_bad = acc - _shifted(A64, _tap_shift(c, t), c.M) @ Bt + _shifted(A64, _tap_shift(c, t) + 1, c.M) @ Bt
    (got, _), _ = reference(c, ins, None, acc_T=(acc_bad, T))
    dst, _ = out_rows(c)
    (ref, bound), _ = reference(c, ins, None)
    with pytest.raises(AssertionError, match="out of bound"):
        check_bound("fault", rne_bf16(got)[dst >= 0], ref[dst >= 0], bound[dst >= 0])


def test_fault_last_8_columns_unwritten_is_rejected():
    """N % 16 == 8: the last 8 columns still hold the output's sentinel."""
    c = _small(N=136)
    ins = _inputs(c, 12)
    (ref, _), _ = reference(c, ins, None)
    got = rne_bf16(ref)
    got.view(torch.int16)[:, -8:] = _SENT[BF16]
    with pytest.raises(AssertionError, match="never written"):
        _ref_ok(c, ins, got)


def test_fault_one_wgrad_split_missing_is_rejected():
    w = WCase(128, 64, 1000, split=3)
    ins = _w_inputs(w, 13)
    ref, bound = w_reference(w, ins)
    got, _ = w_reference(w, ins, drop_split=1)
    with pytest.raises(AssertionError, match="out of bound"):
        check_bound("fault", got.float(), ref, bound)


def test_fault_scale_applied_per_row_is_rejected():
    c = _small(N=128, scale=True, shift=True)
    ins = _inputs(c, 14)
    acc, T = accumulate(c, ins["A"], ins["B"])
    s_row = ins["scale"].double()[torch.arange(c.M) % c.N][:, None]
    bad = dict(ins)
    del bad["scale"]
    cb = _small(N=128, shift=True)
    (got, _), _ = reference(cb, bad, None, acc_T=(acc * s_row, T))
    with pytest.raises(AssertionError, match="out of bound"):
        _ref_ok(c, ins, rne_bf16(got))


def test_fault_out2_holding_gelu_instead_of_its_derivative_is_rejected():
    c = _small(N=128, shift=True, act="stash", out2=True)
    ins = _inputs(c, 15)
    (y, _), _ = reference(c, ins, None)
    with pytest.raises(AssertionError, match="out of bound"):
        _ref_ok(c, ins, rne_bf16(y), which="out2")


def test_fault_one_row_off_by_two_percent_is_rejected_but_passes_the_normwise_check():
    c = Case(TN, 60000, 256, 64)
    ins = _inputs(c, 16)
    (ref, bound), _ = reference(c, ins, None)
    got = ref.clone()
    got[4321] *= 1.02
    with pytest.raises(AssertionError, match="out of bound"):
        check_bound("fault", rne_bf16(got), ref, bound)
    assert relerr(rne_bf16(got), ref) < TOL_BF16_OP


def test_nan_rules_of_the_reference():
    """The rules the NaN / inf cases pin: relu(NaN) = NaN, relu(+inf) = +inf, relu(-inf) = relu(-0) = +0; a NaN, zero or
    subnormal aux masks (0) even a NaN / inf value; a NaN in one row of A / one column of B is NaN exactly there."""
    c = _small(N=128, act="relu")
    ins = _inputs(c, 17)
    ins["A"][3, 0] = float("nan")
    ins["B"][9, 1] = float("nan")
    (ref, _), _ = reference(c, ins, None)
    nan = torch.isnan(ref)
    assert bool(nan[3].all()) and bool(nan[:, 9].all()) and int(nan.sum()) == c.N + c.M - 1
    v = torch.tensor([float("nan"), math.inf, -math.inf, -0.0, 1.0], dtype=F64)
    r = torch.where(v <= 0, torch.zeros_like(v), v)
    assert torch.isnan(r[0]) and r[1] == math.inf and _bits(r[2:4].float()).eq(0).all() and r[4] == 1.0
    x = torch.tensor([0x7FC0, 0xFFC0, 0, 0x8000, 1, 0x7F, 0x80, 0x7F80, 0xFF80, 0x3F80], dtype=torch.int32).to(torch.int16).view(BF16)
    assert relu_pos(x).tolist() == [False, False, False, False, False, False, True, True, False, True]


def test_emulator_relu_and_mask_follow_the_header():
    """ops_emulator.gemm: ReLU passes NaN and gives +0 for -0; the mask is a select, so a NaN value under a masked aux is 0."""
    M, N, K = 2, 16, 8
    A = torch.zeros(M, K, dtype=BF16)
    A[0, 0] = float("nan")
    A[1, :] = -0.0
    B = torch.ones(N, K, dtype=BF16)
    out = torch.empty(M, N, dtype=BF16)
    E.gemm(mode=TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=N, b_ld=K, act=1, out=out, out_ld=N)
    assert bool(torch.isnan(out[0]).all()) and bool((_bits(out[1]) == 0).all())
    aux = torch.full((M, N), -1.0, dtype=BF16)
    aux[0, :4] = 1.0
    E.gemm(mode=TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=N, b_ld=K, aux=aux, aux_ld=N, aux_mode=1, out=out, out_ld=N)
    assert bool(torch.isnan(out[0, :4]).all()) and bool((out[0, 4:] == 0).all())
