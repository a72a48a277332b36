"""cb_attention_fwd / cb_attention_bwd, element by element, against a float64 restatement, on every kernel path.

Each case runs the forward and then the backward and compares ctx, lse and dqkv, every element, with float64 computed from
the same bf16 Q, K, V, dO, the int64 text mask and the fp32 dropout multipliers of tests/dropout_ref.py (r below):

  forward   S_ij = Q_i . K_j / 8 + madd_j   (madd_j = -10000 for a masked text key, else 0)
            lse_i = logsumexp_j S_ij ;  P = exp(S - lse) ;  Pd = P r ;  O = Pd V
  backward  from the kernel's OWN ctx (bf16) and lse (fp32), as the kernel reads them:
            P = exp(S - lse) ;  D_i = dO_i . ctx_i ;  dS = P (r dO V^T - D) ;  dV = Pd^T dO ;  dQ = dS K / 8 ;  dK = dS^T Q / 8

The reference replays each path's rounding points (include/clipbert_b200.h), which keeps the bounds tight:
  - tensor-core forward: x_ij = exp(S_ij - m_i^(t)) r_ij is rounded to bf16, m_i^(t) the running row maximum over the 64-key
    tiles 0..t (the whole row when L <= 64: one tile); the rounded values are rescaled by exp(m^(t) - m), summed against V
    and divided by the unrounded row sum l_i = sum_j exp(S_ij - m_i);
  - tensor-core backward: Pd and dS are rounded to bf16 before the dV / dK / dQ products;
  - CUDA-core kernels (cb_debug_attention_general) and the CPU emulator: no intermediate rounding.

Bounds, per element, never normwise (U = 2^-24; first order in the fp32 errors, each error stated in float64 next to the
reference as a product of absolute values):
  S      e_S = U (192 sum_d |Q_id K_jd| / 8 + 2 T_ij),  T_ij = sum_d |Q_id K_jd| / 8 + |madd_j|. The dot products of 64 exact
         bf16 products run on mma.sync, whose fp32 accumulation is not round-to-nearest: it aligns the addends of a k-block
         to the largest and truncates (Fasi, Higham, Mikaitis, Pranesh 2021), at most 2^-23 (k + 1) of the largest addend per
         16-product block, so below 3 n U sum|terms| = 192 U sum|terms| for n = 64. 2 T: the rounding of s / 8 + madd (and
         one more for the |madd| = 10000 part, which is what the error is made of when every key of a row is masked).
  m      the kernel's running row maximum m'^(t) over tiles 0..t is the fp32 S' of one key, and only keys with
         S_ij + e_S,ij >= m_i^(t) - e_S at the float64 argmax can be it: |dm^(t)| <= e_M^(t), the largest e_S of those
         candidates. A masked key (e_S holds 2 U 10000) is a candidate only when every key of tiles 0..t is masked.
  exp    __expf(x) carries 2 + 1.173 |x| ulp = (4 + 2.35 |x|) U (CUDA C Programming Guide), plus the rounding of the
         subtraction that forms x and of the multiplication by r: E(x) = (6 + 4 |x|) U.
  rescale rho_ij = U (6 (nt - 1 - t(j)) + 4 (m - m^(t(j)))): the __expf of each later rescale step (nt = ceil(L / 64) tiles).
         The rescale arguments m'^(t) - m'^(t+1) telescope: the maxima themselves cancel between x, the rescales and l.
  l      l' = e^-m' sum_j e^S'_ij (1 + E + rho): relative error lambda_i = sum_j P_ij (e_S + E + rho)_ij + U (L + 2 nt) up
         to the common factor e^-dm', which cancels in ctx and in lse (the terms, the fp32 sum of L of them).
  x      the kernel's fp32 x_ij = exp(S'_ij - m'^(t)) r_ij is off by the relative eps_ij = e_S + e_M^(t) + E(S - m^(t)).
         Tensor-core paths: x is rounded to bf16, replayed in the reference, and the kernel's x may lie on the other side of a
         bf16 rounding boundary: amb_ij = |rne_bf16(x + eps x) - rne_bf16(x - eps x)| (zero away from a boundary). Where it
         does not flip, the rounding snaps x back to the reference's value, so the shift e^-dm^(t) that would cancel against
         the rescales and l stays: e_M^(t) enters w below. Without intermediate rounding the maxima cancel (e_M = 0) and
         the ambiguity is the error itself, eps x.
  ctx    |got - ref| <= 1 ulp_bf16(ref) + sum_j amb_ij R_ij / l_i |V_jd| + 2 U sum_j W_ij w_ij |V_jd|, W = X R / l the
         weights the reference multiplies V by, w_ij = (e_M^(t(j)) + rho_ij + lambda_i) / U + 3 (L + nt) + 2: the snapped
         maximum, the rescales, the row sum, the P V accumulation on mma.sync (3 U per addend, as for S) and 1 / l_i.
  lse    m' + __logf(l') = log sum_j e^S'_ij (1 + ...): m' cancels, |got - ref| <= 2 (lambda_i + U |lse_i|) + 2^-21.41 +
         6 U ln L (__logf: 2^-21.41 absolute on [0.5, 2], else 3 ulp <= 6 U |log l|; U |lse|: the final addition).
  Pd, dS (backward) e_P = P (e_S + E(S - lse)); e_Pd = r e_P + U Pd; e_dP = 192 U sum_d |dO_id V_jd| (as S);
         e_D = 64 U sum_d |dO_id ctx_id| (64 exact products, round-to-nearest); g = r dP - D, e_g = r e_dP + e_D +
         U (r |dP| + |g|); e_dS = P e_g + e_P |g| + U |dS|; amb of Pd and dS as for x (absolute errors: dS cancels).
  dV, dK, dQ  1 ulp_bf16(ref) + sum amb |B| + 2 U 3 (L + 1) sum |A| |B|, with (A, B) = (Pd, dO), (dS, Q / 8), (dS, K / 8):
         the L-long product on mma.sync (3 U per addend) and its scaling.
  The factor 2 on the first-order terms covers what the first-order expansion drops (products of the relative errors above,
  all far below 2^-8 here). 1 ulp: the final rounding of an fp32 value within the other terms of ref (0.5 ulp of the fp32
  value, which may be one binade above ref).

Guards and edges: ctx, lse and dqkv are Guarded (sentinel guard bands and pitch padding, unchanged afterwards; an element
still holding the sentinel was never written). The inputs sit in NaN: qkv / ctx / dctx pitch columns and 64 rows before and
after each window, so a read outside a kernel's window poisons its output. Each case runs twice and must give the same bits
(one CTA writes each output element, no atomics), and the forward without lse must give the same ctx bits. Every case prints
"RATIO <path> <case> <max err / bound>" per output.

Paths (csrc/attention.cu, csrc/attention_tc.cu), selected by the cb_debug_attention_* switches and the length:
  tc48        attn_tc_fwd_kernel<3> / attn_tc_bwd_kernel<3>                    L <= 48 (rows48 on, the default)
  tc64        attn_tc_fwd_kernel<4> / attn_tc_bwd_kernel<4>                    48 < L <= 64, or L <= 48 with rows48 off
  flash_pipe  attn_tc_fwd_flash_kernel<true> / attn_tc_bwd_kv_kernel + _q_kernel   L > 64 (the default)
  flash_sync  attn_tc_fwd_flash_kernel<false> / the same backward              L > 64 with flash_pipe off
  cuda_core   attn_fwd_kernel / attn_bwd_kv_kernel + attn_bwd_q_kernel         cb_debug_attention_general(1), any L
The CPU runs the packed cases through tests/ops_emulator.py under the CUDA-core (fp32 P) convention, and self-tests the
reference and the bounds: the float64 result of each deliberate fault (six kernel mistakes, and 2 % ctx / 0.003 lse row
errors in sequences with masked keys), rounded to bf16, must be rejected.
"""
import contextlib
import ctypes
import math

import numpy as np
import pytest
import torch

import dropout_ref as D
import ops_emulator as E
from elementwise import BF16, F32, F64, U, Guarded, _INT, _record, check_bound, rne_bf16, ulp_bf16
from util import TOL_BF16_OP, relerr

HD = 64
NSEQ = 3
PAD_ROWS = 64                       # NaN rows before and after each input window

# ------------------------------------------------------------------------------------------------ paths
# path -> (switch settings, lengths it covers)
PATHS = {
    "tc48": (dict(rows48=1), lambda L: L <= 48),
    "tc64": (dict(rows48=0), lambda L: L <= 64),
    "flash_pipe": (dict(flash_pipe=1), lambda L: L > 64),
    "flash_sync": (dict(flash_pipe=0), lambda L: L > 64),
    "cuda_core": (dict(general=1), lambda L: True),
}
ROUNDED = {"tc48": True, "tc64": True, "flash_pipe": True, "flash_sync": True, "cuda_core": False, "emulator": False}
LENGTHS = {
    "tc48": [1, 2, 9, 16, 17, 41, 47, 48],
    "tc64": [49, 63, 64, 9, 41],
    "flash_pipe": [65, 69, 80, 127, 128, 129, 149, 150, 169, 174, 193, 521],
    "flash_sync": [65, 69, 80, 127, 128, 129, 149, 150, 169, 174, 193, 521],
    "cuda_core": [1, 41, 64, 65, 129, 521],
}
# text length per L: the shapes of the earlier normwise tests (41/32, 150/100, 64/64, 9/0, 48/32, 49/32, 65/20, 69/20,
# 128/64, 149/100, 169/25, 174/30, 521/512, 80/0), lt = L where every key is text, lt = L - 9 (one 3x3 frame) elsewhere
LT = {1: 1, 2: 2, 9: 0, 16: 16, 17: 8, 41: 32, 47: 38, 48: 32, 49: 32, 63: 63, 64: 64, 65: 20, 69: 20, 80: 0, 127: 118,
      128: 64, 129: 129, 149: 100, 150: 100, 169: 25, 174: 30, 193: 193, 521: 512}


class Case:
    def __init__(self, path, L, p=0.0, heads=None, values="randn", pitched=False, word=False):
        heads = heads or (4 if L > 512 else 12)             # 521 tokens: 4 heads keep the float64 reference at a few seconds
        self.path, self.L, self.lt, self.p, self.heads, self.values = path, L, LT[L], p, heads, values
        self.pitched, self.word = pitched, word
        if path in PATHS:
            assert PATHS[path][1](L), "%s does not run at L = %d" % (path, L)

    @property
    def id(self):
        s = "%s-L%d-lt%d-p%g" % (self.path, self.L, self.lt, self.p)
        s += "-H%d" % self.heads
        if self.values != "randn":
            s += "-" + self.values
        if self.pitched:
            s += "-pitched"
        if self.word:
            s += "-word"
        return s


def _cases():
    out = []
    for path, lengths in LENGTHS.items():
        for n, L in enumerate(lengths):
            out.append(Case(path, L, p=0.1 if n % 2 else 0.0, values="peaked" if n % 3 == 2 else "randn"))
        L1, Llong = lengths[len(lengths) // 2], lengths[-2]
        out.append(Case(path, L1, p=1.0))
        out.append(Case(path, L1, p=0.1, word=True))
        out.append(Case(path, Llong, p=0.1, pitched=True))
        # heads 1 and 16 at L = 41 (one tile) and at L = 169 (three tiles: the multi-tile kernels index heads per tile)
        for Lh in [L for L in (41, 169) if PATHS[path][1](L)]:
            for h in (1, 16):
                out.append(Case(path, Lh, p=0.1 if h == 16 else 0.0, heads=h))
    return out


CASES = _cases()
# the emulator has no paths: each distinct packed problem once
_EMU = {}
for _c in CASES:
    if not _c.pitched and not _c.word and _c.path in ("tc48", "tc64", "flash_pipe", "cuda_core"):
        _EMU.setdefault((_c.L, _c.p, _c.heads, _c.values), Case("emulator", _c.L, _c.p, _c.heads, _c.values))
EMU_CASES = list(_EMU.values())


@contextlib.contextmanager
def _path(path):
    """Sets the path's cb_debug_attention_* switches; restores the defaults (general 0, flash 1, rows48 1, flash_pipe 1)."""
    from clipbert_b200 import _lib, ops
    sw = PATHS[path][0]
    try:
        _lib.lib().cb_debug_attention_general(ctypes.c_int(sw.get("general", 0)))
        ops.set_attention_rows48(sw.get("rows48", 1))
        ops.set_attention_flash_pipe(sw.get("flash_pipe", 1))
        ops.set_attention_flash(1)
        yield
    finally:
        _lib.lib().cb_debug_attention_general(ctypes.c_int(0))
        ops.set_attention_rows48(1)
        ops.set_attention_flash_pipe(1)
        ops.set_attention_flash(1)


# ------------------------------------------------------------------------------------------------ inputs
def _mask(L, lt):
    """int64 [NSEQ, lt] ([NSEQ, 1] of ones when lt = 0: never read). Sequence 0: masked tail keys (and, for lt >= 128 with
    L > 128, the second 64-key tile masked: the running maximum stays while a whole tile contributes nothing); sequence 1: the
    first 64-key tile entirely masked when lt >= 64 and L > 128 (the running maximum jumps by ~10000 at tile 1), else one
    masked key; sequence 2: every text key masked when lt = L (every key of every row masked), else all live."""
    if lt == 0:
        return torch.ones(NSEQ, 1, dtype=torch.int64)
    m = torch.ones(NSEQ, lt, dtype=torch.int64)
    if lt >= 2:
        m[0, lt - max(1, lt // 3):] = 0
        m[1, lt // 2] = 0
    if L > 128 and lt >= 128:
        m[0, 64:128] = 0
    if L > 128 and lt >= 64:
        m[1, :64] = 0
    if lt == L:
        m[2] = 0
    return m


def _inputs(case):
    g = torch.Generator().manual_seed(1000 * case.L + case.heads + int(case.p * 10) + (7 if case.values == "peaked" else 0))
    n, L, hid = NSEQ, case.L, case.heads * HD
    qkv = torch.randn(n * L, 3 * hid, generator=g, dtype=F64)
    if case.values == "peaked":                 # saturated softmax: P near one-hot, dS cancels
        qkv[:, :2 * hid] *= 4
    dout = torch.randn(n * L, hid, generator=g, dtype=F64)
    return qkv.to(BF16), dout.to(BF16), _mask(L, case.lt)


def _madd(mask, L, lt):
    madd = torch.zeros(NSEQ, L, dtype=F64)
    if lt:
        madd[:, :lt] = (mask[:, :lt] == 0).double() * -10000.0
    return madd


def _mult(case, seed, word):
    if case.p == 0:
        return torch.ones(NSEQ, case.heads, case.L, case.L, dtype=F64)
    return torch.from_numpy(D.multipliers(D.effective_seed(seed, word), D.attention_index(NSEQ, case.heads, case.L), case.p)).double()


def _split(x, heads):
    """[NSEQ * L, k * heads * 64] -> k tensors [NSEQ, heads, L, 64] float64."""
    x = x.detach().cpu().double().contiguous()
    L = x.shape[0] // NSEQ
    return [t.reshape(NSEQ, L, heads, HD).permute(0, 2, 1, 3) for t in x.view(NSEQ, L, -1, heads * HD).unbind(2)]


def _merge(t):
    """[NSEQ, heads, L, 64] -> [NSEQ * L, heads * 64]."""
    n, h, L, d = t.shape
    return t.permute(0, 2, 1, 3).reshape(n * L, h * d)


# ------------------------------------------------------------------------------------------------ reference
def _amb(x, e):
    """|rne_bf16(x + e) - rne_bf16(x - e)|: the bf16 values an fp32 value within e of x can round to differ by this much."""
    return (rne_bf16(x + e).double() - rne_bf16(x - e).double()).abs()


def _inter(x, e, rounded):
    """An intermediate the kernel forms in fp32 (error <= e): the value the reference uses and the ambiguity it carries."""
    if rounded:
        return rne_bf16(x).double(), _amb(x, e)
    return x, e


def _scores(q, k, madd):
    qk_abs = q.abs() @ k.abs().transpose(-1, -2) / 8.0
    S = q @ k.transpose(-1, -2) / 8.0 + madd[:, None, None, :]
    T = qk_abs + madd.abs()[:, None, None, :]
    return S, U * (192.0 * qk_abs + 2.0 * T)


def _E(x):
    return U * (6.0 + 4.0 * x.abs())


def _max_error(S, eS, nt):
    """Bound on the error of the kernel's running row maximum m'^(t) over the keys of tiles 0..t, [.., L, nt]. m' is the fp32
    S' of some key j*; S'_j* >= S'_a >= m - e_S,a (a: the float64 argmax), so S_j* + e_S,j* >= m - e_S,a. Only such keys (the
    candidates) can be the kernel's maximum, and |m' - m| <= max over the candidates of e_S. A masked key (e_S carries
    2 U 10000) is a candidate only when every key up to that tile is masked."""
    L = S.shape[-1]
    out = []
    for t in range(nt):
        Sp, ep = S[..., :min(L, 64 * (t + 1))], eS[..., :min(L, 64 * (t + 1))]
        mx, arg = Sp.max(-1, keepdim=True)
        cand = Sp + ep >= mx - ep.gather(-1, arg)
        out.append(torch.where(cand, ep, torch.zeros_like(ep)).max(-1).values)
    return torch.stack(out, -1)


def forward_ref(q, k, v, madd, r, rounded):
    """ctx [NSEQ, H, L, 64], lse [NSEQ, H, L] and their bounds (see the module docstring)."""
    L = q.shape[2]
    nt = (L + 63) // 64
    S, eS = _scores(q, k, madd)
    pad = torch.full(S.shape[:-1] + (nt * 64 - L,), -math.inf, dtype=F64)
    tile_max = torch.cat([S, pad], -1).unflatten(-1, (nt, 64)).max(-1).values
    run = torch.cummax(tile_max, -1).values                                    # m^(t) [.., L, nt]
    t_of_j = torch.arange(L) // 64
    mt = run[..., t_of_j]                                                      # m^(t(j)) [.., L, L]
    m = run[..., -1:]                                                          # row maximum [.., L, 1]
    eMt = _max_error(S, eS, nt)[..., t_of_j] if rounded else torch.zeros_like(S)   # |dm^(t(j))|, where it does not cancel
    x = torch.exp(S - mt) * r
    X, ambX = _inter(x, x * (eS + eMt + _E(S - mt)), rounded)
    R = torch.exp(mt - m)
    Pu = torch.exp(S - m)
    l = Pu.sum(-1, keepdim=True)
    P = Pu / l
    rho = U * (6.0 * (nt - 1 - t_of_j).double() + 4.0 * (m - mt))
    lam = (P * (eS + _E(S - mt) + rho)).sum(-1, keepdim=True) + U * (L + 2 * nt)
    W = X * R / l
    O = W @ v
    w = (eMt + rho + lam) / U + 3.0 * (L + nt) + 2.0
    bound_O = ulp_bf16(O) + (ambX * R / l) @ v.abs() + 2.0 * U * ((W.abs() * w) @ v.abs())
    lse = (m + torch.log(l)).squeeze(-1)
    bound_lse = 2.0 * lam.squeeze(-1) + 2.0 * U * lse.abs() + 2.0 ** -21.41 + 6.0 * U * math.log(max(L, 2))
    return O, bound_O, lse, bound_lse


def backward_ref(q, k, v, madd, r, ctx, lse, dout, rounded):
    """dq, dk, dv [NSEQ, H, L, 64] and their bounds, from the kernel's ctx (bf16) and lse (fp32)."""
    L = q.shape[2]
    S, eS = _scores(q, k, madd)
    lse = lse.detach().cpu().double()[..., None]
    P = torch.exp(S - lse)
    eP = P * (eS + _E(S - lse))
    Pd = P * r
    dP = dout @ v.transpose(-1, -2)
    edP = 192.0 * U * (dout.abs() @ v.abs().transpose(-1, -2))
    Dv = (dout * ctx).sum(-1, keepdim=True)
    eD = 64.0 * U * (dout.abs() * ctx.abs()).sum(-1, keepdim=True)
    gg = r * dP - Dv
    eg = r * edP + eD + U * (r * dP.abs() + gg.abs())
    dS = P * gg
    edS = P * eg + eP * gg.abs() + U * dS.abs()
    PdX, ambPd = _inter(Pd, r * eP + U * Pd, rounded)
    dSX, ambdS = _inter(dS, edS, rounded)
    depth = 3.0 * (L + 1)
    out = []
    for A, amb, B, s in ((dSX, ambdS, k, 0.125), (dSX.transpose(-1, -2), ambdS.transpose(-1, -2), q, 0.125),
                         (PdX.transpose(-1, -2), ambPd.transpose(-1, -2), dout, 1.0)):
        ref = A @ B * s
        out.append((ref, ulp_bf16(ref) + (amb @ B.abs()) * s + 2.0 * U * depth * (A.abs() @ B.abs()) * s))
    return out


def _reference(case, qkv, dout, mask, r, ctx_got, lse_got, rounded):
    q, k, v = _split(qkv, case.heads)
    madd = _madd(mask, case.L, case.lt)
    O, bO, lse, blse = forward_ref(q, k, v, madd, r, rounded)
    (ctx_k,) = _split(ctx_got, case.heads)
    (do,) = _split(dout, case.heads)
    grads = backward_ref(q, k, v, madd, r, ctx_k, lse_got, do, rounded)
    return (O, bO), (lse, blse), grads


def _check_all(tag, case, ctx_got, lse_got, dqkv_got, refs):
    (O, bO), (lse, blse), grads = refs
    ratios = {"ctx": check_bound("%s ctx" % tag, ctx_got, _merge(O), _merge(bO)),
              "lse": check_bound("%s lse" % tag, lse_got, lse, blse)}
    dq, dk, dv = (t.detach().cpu().view(NSEQ * case.L, -1) for t in dqkv_got.cpu().contiguous().view(NSEQ * case.L, 3, -1).unbind(1))
    for name, got, (ref, b) in zip(("dq", "dk", "dv"), (dq, dk, dv), grads):
        ratios[name] = check_bound("%s %s" % (tag, name), got, _merge(ref), _merge(b))
    return ratios


# ------------------------------------------------------------------------------------------------ running a case
class _Window:
    """A [rows, cols] bf16 input with row pitch ld inside NaN: PAD_ROWS rows before and after, and the pitch columns."""

    def __init__(self, x, ld, dev):
        rows, cols = x.shape
        self.buf = torch.full(((rows + 2 * PAD_ROWS) * ld,), float("nan"), dtype=BF16, device=dev)
        self.t = self.buf[PAD_ROWS * ld:(PAD_ROWS + rows) * ld].view(rows, ld)[:, :cols]
        self.t.copy_(x)
        self.ld = ld


def _run(be, case, qkv, dout, mask, seed, with_lse=True):
    """One forward and one backward; returns the Guarded ctx, lse, dqkv."""
    n, L, hid = NSEQ, case.L, case.heads * HD
    dev = be.dev
    ld_qkv, ld_ctx, ld_dqkv = (3 * hid + 64, hid + 40, 3 * hid + 24) if case.pitched else (3 * hid, hid, 3 * hid)
    ctx = Guarded((n * L, hid), BF16, dev, ld=ld_ctx)
    lse = Guarded((n, case.heads, L), F32, dev)
    dqkv = Guarded((n * L, 3 * hid), BF16, dev, ld=ld_dqkv)
    mask_d = mask.to(dev)
    if be.emulated:
        assert not case.pitched
        E.attention_fwd(qkv, mask_d, ctx.t, lse.t if with_lse else None, n, L, case.lt, case.heads, case.p, seed)
        E.attention_bwd(qkv, mask_d, ctx.t, dout, lse.t, dqkv.t, n, L, case.lt, case.heads, case.p, seed)
        return ctx, lse, dqkv
    from clipbert_b200 import ops
    xin = _Window(qkv, ld_qkv, dev)
    din = _Window(dout, ld_ctx, dev)
    # the backward reads ctx through the same pitch as dctx: its padding columns are the Guarded sentinel, a NaN
    ops._call("cb_attention_fwd", ops._p(xin.t), ld_qkv, ops._p(mask_d), ops._p(ctx.t), ld_ctx, ops._p(lse.t) if with_lse else None,
              n, L, case.lt, case.heads, HD, case.p, seed, ops._s())
    if with_lse:
        ops._call("cb_attention_bwd", ops._p(xin.t), ld_qkv, ops._p(mask_d), ops._p(ctx.t), ops._p(din.t), ld_ctx, ops._p(lse.t),
                  ops._p(dqkv.t), ld_dqkv, n, L, case.lt, case.heads, HD, case.p, seed, ops._s())
    torch.cuda.synchronize()
    return ctx, lse, dqkv


class Backend:
    def __init__(self, name):
        self.name = name
        self.emulated = name == "emulator"
        self.dev = torch.device("cpu") if self.emulated else torch.device("cuda:0")


def _bits(t):
    return t.detach().cpu().contiguous().view(_INT[t.dtype]).clone()


@contextlib.contextmanager
def _bound_word(be, word):
    w = None if word is None else torch.tensor([word], dtype=torch.int64, device=be.dev)
    if be.emulated:
        mod = E
    else:
        from clipbert_b200 import ops as mod
    mod.dropout_offset_bind(w)
    try:
        yield
    finally:
        mod.dropout_offset_bind(None)


def _attention_case(be, case):
    seed = 4242 + case.L
    word = 0x1234567 + case.L if case.word else None
    qkv, dout, mask = _inputs(case)
    ctxmgr = contextlib.nullcontext() if be.emulated else _path(case.path)
    with ctxmgr, _bound_word(be, word):
        ctx, lse, dqkv = _run(be, case, qkv, dout, mask, seed)
        for t, name in ((ctx, "ctx"), (lse, "lse"), (dqkv, "dqkv")):
            t.check("%s %s" % (case.id, name))
        if not be.emulated:
            ctx2, lse2, dqkv2 = _run(be, case, qkv, dout, mask, seed)
            ctx3, _, _ = _run(be, case, qkv, dout, mask, seed, with_lse=False)
    if not be.emulated:
        for a, b, name in ((ctx, ctx2, "ctx"), (lse, lse2, "lse"), (dqkv, dqkv2, "dqkv")):
            assert torch.equal(_bits(a.t), _bits(b.t)), "%s: %s differs between two identical runs" % (case.id, name)
        assert torch.equal(_bits(ctx.t), _bits(ctx3.t)), "%s: ctx of the forward without lse differs" % case.id
        ctx3.check("%s ctx (no lse)" % case.id)
    if case.p >= 1:
        assert bool((ctx.t.cpu() == 0).all()) and bool((dqkv.t.cpu() == 0).all()), "%s: p = 1 must give zeros" % case.id
    r = _mult(case, seed, word)
    refs = _reference(case, qkv, dout, mask, r, ctx.t, lse.t, ROUNDED[case.path])
    ratios = _check_all(case.id, case, ctx.t, lse.t, dqkv.t, refs)
    for name, v in ratios.items():
        _record(case.path, "%s-%s" % (case.id, name), v)


@pytest.mark.parametrize("be_name,case", [pytest.param("device", c, marks=pytest.mark.gpu, id="device-" + c.id) for c in CASES]
                         + [pytest.param("emulator", c, id=c.id) for c in EMU_CASES])
def test_attention_elementwise(be_name, case):
    if be_name == "device" and not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    _attention_case(Backend(be_name), case)


def test_matrix_covers_every_path_and_the_earlier_shapes():
    """Each path runs at lengths it is selected for (asserted in Case), at both dropout rates, p = 1, a bound dropout word, a
    pitched call and heads 1 / 16; every (L, lt) of the earlier normwise tests is in the matrix."""
    for path in PATHS:
        mine = [c for c in CASES if c.path == path]
        assert {0.0, 0.1, 1.0} <= {c.p for c in mine} and any(c.word for c in mine) and any(c.pitched for c in mine)
        assert 12 in {c.heads for c in mine}
        assert {(L, h) for L in (41, 169) if PATHS[path][1](L) for h in (1, 16)} <= {(c.L, c.heads) for c in mine}
    have = {(c.L, c.lt) for c in CASES}
    earlier = [(41, 32), (150, 100), (64, 64), (9, 0), (48, 32), (49, 32), (65, 20), (69, 20), (128, 64), (149, 100), (169, 25),
               (174, 30), (521, 512), (80, 0)]
    assert set(earlier) <= have, set(earlier) - have
    for L in LENGTHS["tc48"]:
        assert L <= 48                                          # attn_tc_*_kernel<3>
    for L in LENGTHS["tc64"]:
        assert L <= 64 and (L > 48 or PATHS["tc64"][0]["rows48"] == 0)   # attn_tc_*_kernel<4>


# ------------------------------------------------------------------------------------------------ CPU self-tests
def _fault_setup(L=65, heads=2, p=0.1):
    case = Case("emulator", L, p=p, heads=heads)
    qkv, dout, mask = _inputs(case)
    seed = 99
    r = _mult(case, seed, None)
    q, k, v = _split(qkv, heads)
    (do,) = _split(dout, heads)
    madd = _madd(mask, L, case.lt)
    O, bO, lse, blse = forward_ref(q, k, v, madd, r, True)
    ctx = rne_bf16(_merge(O))                       # what a correct tensor-core forward returns, to within its bound
    lse32 = lse.float()
    (ctx_k,) = _split(ctx, heads)
    grads = backward_ref(q, k, v, madd, r, ctx_k, lse32, do, True)
    return dict(case=case, q=q, k=k, v=v, do=do, madd=madd, r=r, O=O, bO=bO, lse=lse, blse=blse, ctx=ctx, ctx_k=ctx_k,
                lse32=lse32, grads=grads, mask=mask, seed=seed)


def _fwd_ok(s, O):
    check_bound("fault ctx", rne_bf16(_merge(O)), _merge(s["O"]), _merge(s["bO"]))


def _bwd_ok(s, grads):
    for name, (got, _), (ref, b) in zip(("dq", "dk", "dv"), grads, s["grads"]):
        check_bound("fault " + name, rne_bf16(_merge(got)), _merge(ref), _merge(b))


def test_reference_accepts_itself_rounded_and_matches_autograd():
    """The reference rounded once to bf16 passes its own bounds; its unrounded (p = 0) form equals float64 autograd of
    softmax(Q K^T / 8 + madd) V."""
    s = _fault_setup(p=0.0)
    _fwd_ok(s, s["O"])
    _bwd_ok(s, s["grads"])
    q, k, v = (t.clone().requires_grad_(True) for t in (s["q"], s["k"], s["v"]))
    with torch.enable_grad():
        o = torch.softmax(q @ k.transpose(-1, -2) / 8.0 + s["madd"][:, None, None, :], -1) @ v
        o.backward(s["do"])
    O, _, lse, _ = forward_ref(s["q"], s["k"], s["v"], s["madd"], s["r"], False)
    assert torch.allclose(O, o.detach(), rtol=0, atol=1e-12)
    ex = backward_ref(s["q"], s["k"], s["v"], s["madd"], s["r"], o.detach(), lse, s["do"], False)
    for (got, _), want in zip(ex, (q.grad, k.grad, v.grad)):
        assert torch.allclose(got, want, rtol=0, atol=1e-10)


def test_fault_masked_key_treated_as_live_is_rejected():
    s = _fault_setup()
    madd = s["madd"].clone()
    j = int((madd[0] < 0).nonzero()[0])
    madd[0, j] = 0.0
    O = forward_ref(s["q"], s["k"], s["v"], madd, s["r"], True)[0]
    with pytest.raises(AssertionError, match="out of bound"):
        _fwd_ok(s, O)


def test_fault_dropout_index_shifted_by_one_key_is_rejected():
    s = _fault_setup()
    c = s["case"]
    idx = D.attention_index(NSEQ, c.heads, c.L) + np.uint64(1)
    r = torch.from_numpy(D.multipliers(D.effective_seed(s["seed"]), idx, c.p)).double()
    O = forward_ref(s["q"], s["k"], s["v"], s["madd"], r, True)[0]
    with pytest.raises(AssertionError, match="out of bound"):
        _fwd_ok(s, O)


def test_fault_last_key_of_L65_omitted_is_rejected():
    s = _fault_setup(L=65)
    madd = s["madd"].clone()
    madd[:, 64] = -1e9                               # exp(-1e9) = 0: key 64 contributes nothing
    O = forward_ref(s["q"], s["k"], s["v"], madd, s["r"], True)[0]
    with pytest.raises(AssertionError, match="out of bound"):
        _fwd_ok(s, O)


def test_fault_lse_of_one_row_off_by_a_hundredth_is_rejected_but_passes_the_normwise_check():
    """lse + 0.01 in one (sequence, head, row) scales that row's backward P by 1 %: the per-element check rejects it, the
    normwise relerr < 2 TOL_BF16_OP the earlier attention tests used accepts it."""
    s = _fault_setup()
    lse = s["lse32"].clone()
    lse[1, 0, 7] += 0.01
    grads = backward_ref(s["q"], s["k"], s["v"], s["madd"], s["r"], s["ctx_k"], lse, s["do"], True)
    with pytest.raises(AssertionError, match="out of bound"):
        _bwd_ok(s, grads)
    got = torch.cat([_merge(g) for g, _ in grads], 1)
    ref = torch.cat([_merge(g) for g, _ in s["grads"]], 1)
    assert relerr(rne_bf16(got), ref) < 2 * TOL_BF16_OP


@pytest.mark.parametrize("L", [65, 169])
def test_row_faults_in_sequences_with_masked_keys_are_rejected(L):
    """In the sequences that have masked keys (as every padded caption does), a ctx row scaled by 2 % and an lse off by 0.003
    are rejected: a masked key's error (2 U 10000 in S) does not widen the bounds of rows that have live keys."""
    s = _fault_setup(L=L)
    for b in (0, 1):
        assert bool((s["madd"][b] < 0).any()) and bool((s["madd"][b] == 0).any())
        O = s["O"].clone()
        O[b, 0, L - 1] *= 1.02
        with pytest.raises(AssertionError, match="out of bound"):
            _fwd_ok(s, O)
        lse = s["lse"].float()
        lse[b, 0, L - 1] += 0.003
        with pytest.raises(AssertionError, match="out of bound"):
            check_bound("fault lse", lse, s["lse"], s["blse"])
        check_bound("lse", s["lse"].float(), s["lse"], s["blse"])


def test_fault_backward_without_the_inverse_keep_probability_is_rejected():
    s = _fault_setup()
    grads = backward_ref(s["q"], s["k"], s["v"], s["madd"], (s["r"] > 0).double(), s["ctx_k"], s["lse32"], s["do"], True)
    with pytest.raises(AssertionError, match="out of bound"):
        _bwd_ok(s, grads)


def test_fault_one_heads_dk_without_the_eighth_is_rejected():
    s = _fault_setup()
    grads = [(g.clone(), b) for g, b in s["grads"]]
    grads[1][0][:, 1] *= 8.0
    with pytest.raises(AssertionError, match="out of bound"):
        _bwd_ok(s, grads)


def test_emulated_backward_reads_the_saved_lse():
    """ops_emulator.attention_bwd follows the header: it rebuilds P from the lse it is given (and D from the ctx it is given),
    so a perturbed lse changes dqkv."""
    case = Case("emulator", 41, heads=2)
    qkv, dout, mask = _inputs(case)
    hid = case.heads * HD
    ctx = torch.empty(NSEQ * case.L, hid, dtype=BF16)
    lse = torch.empty(NSEQ, case.heads, case.L)
    E.attention_fwd(qkv, mask, ctx, lse, NSEQ, case.L, case.lt, case.heads, 0.0, 0)
    outs = []
    for l_in in (lse, lse + 0.05):
        d = torch.empty(NSEQ * case.L, 3 * hid, dtype=BF16)
        E.attention_bwd(qkv, mask, ctx, dout, l_in, d, NSEQ, case.L, case.lt, case.heads, 0.0, 0)
        outs.append(d)
    assert not torch.equal(outs[0], outs[1])
