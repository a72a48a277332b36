"""Element-by-element comparison helpers shared by the float64 kernel tests (test_gpu_memory_bound_kernels.py,
test_gpu_attention_elementwise.py) - TEST INFRASTRUCTURE ONLY.

  - Guarded: an output between guard bands (and pitch padding) of a sentinel NaN bit pattern no kernel produces;
  - rne_bf16 / ulp_bf16: float64 -> bf16 with one rounding, and the bf16 ulp of a float64 value;
  - check_bitexact / check_bound / check_bf16 / check_sum: per-element checks that also reject an element still holding the
    sentinel (never written) and a NaN / infinity the reference does not have;
  - _record: the "RATIO <kernel> <case> <max err / bound>" line each case prints (pytest -s shows them).
"""
import numpy as np
import torch

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24                      # unit roundoff of fp32
G = 64                              # guard elements on each side of an output (keeps 16-byte alignment for bf16 and fp32)
_INT = {BF16: torch.int16, F32: torch.int32}
_SENT = {BF16: 0x7FA5, F32: 0x7FC05A5A}     # NaN bit patterns no kernel produces


def _record(kernel, case, ratio):
    print("RATIO %s %s %.3g" % (kernel, case, ratio))


# ------------------------------------------------------------------------------------------------ guard bands
class Guarded:
    """A [rows, cols] (or flat) output with row pitch ld inside a buffer of G sentinel elements before and after it; the
    pitch padding is sentinel too. ``t`` is the view handed to the kernel."""

    def __init__(self, shape, dtype, dev, ld=None, init=None):
        shape = tuple(shape)
        cols = shape[-1]
        rows = int(np.prod(shape[:-1])) if len(shape) > 1 else 1
        ld = cols if ld is None else ld
        n = rows * ld
        self.dtype = dtype
        self.buf = torch.empty(2 * G + n, dtype=dtype, device=dev)
        self.buf.view(_INT[dtype]).fill_(_SENT[dtype])
        body = self.buf[G:G + n].view(rows, ld)[:, :cols]
        self.t = body.view(shape) if ld == cols else body
        self.inside = torch.zeros(2 * G + n, dtype=torch.bool)
        self.inside[G:G + n].view(rows, ld)[:, :cols] = True
        if init is not None:
            self.t.copy_(init)

    def check(self, what):
        bits = self.buf.view(_INT[self.dtype]).cpu().long() & (0xFFFF if self.dtype == BF16 else 0xFFFFFFFF)
        bad = (~self.inside) & (bits != _SENT[self.dtype])
        if bad.any():
            i = int(bad.nonzero()[0])
            raise AssertionError("%s: %d guard / padding elements written, first at buffer offset %d (output spans %d..%d): 0x%x"
                                 % (what, int(bad.sum()), i, G, self.buf.numel() - G, int(bits[i])))


# ------------------------------------------------------------------------------------------------ comparison helper
def rne_bf16(x64):
    """float64 -> bf16 with ONE rounding to nearest even (torch's own conversion goes through fp32 and rounds twice): round
    to odd at fp32 first, which keeps enough information for the second rounding to be correct."""
    a = x64.detach().cpu().to(F64).numpy()
    f = a.astype(np.float32)
    bits = f.view(np.uint32).copy()
    with np.errstate(invalid="ignore"):
        inexact = np.isfinite(a) & (f.astype(np.float64) != a)
        down = inexact & (np.abs(f.astype(np.float64)) > np.abs(a))
    bits[down] -= 1
    bits[inexact] |= 1
    b = ((bits.astype(np.uint64) + 0x7FFF + ((bits >> 16) & 1)) >> 16).astype(np.uint16)
    b[np.isnan(a)] = 0x7FC0
    return torch.from_numpy(b.view(np.int16)).view(BF16).reshape(x64.shape)


def ulp_bf16(x64):
    e = torch.floor(torch.log2(x64.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def _locate(kernel, what, bad, got, ref, bound=None):
    i = tuple(int(v) for v in bad.nonzero()[0])
    msg = "%s: %d of %d elements %s; first at %s: got %r ref %r" % (kernel, int(bad.sum()), bad.numel(), what, i, float(got[i]),
                                                                  float(ref[i]))
    if bound is not None:
        msg += " |err| %.3g bound %.3g" % (abs(float(got[i]) - float(ref[i])), float(bound[i]))
    raise AssertionError(msg)


def _reject_unwritten(kernel, g):
    """The guard sentinel is a NaN pattern and a fresh Guarded body holds it: an element still holding it was never written
    (and would otherwise pass wherever the reference is NaN)."""
    if g.dtype in _SENT:
        left = (g.view(_INT[g.dtype]).long() & (0xFFFF if g.dtype == BF16 else 0xFFFFFFFF)) == _SENT[g.dtype]
        if left.any():
            _locate(kernel, "never written (still the sentinel)", left, g.double(), g.double())


def check_bitexact(kernel, got, ref64):
    """got (bf16 / fp32) must equal ref64 rounded once to got's type; both NaN counts as equal."""
    g = got.detach().cpu()
    _reject_unwritten(kernel, g)
    want = rne_bf16(ref64) if g.dtype == BF16 else ref64.detach().cpu().to(g.dtype)
    it = _INT[g.dtype]
    bad = (g.view(it) != want.view(it)) & ~(torch.isnan(g) & torch.isnan(want))
    if bad.any():
        _locate(kernel, "not bit-exact", bad, g.double(), ref64.detach().cpu().double())
    return 0.0


def check_bound(kernel, got, ref64, bound):
    """|got - ref| <= bound element by element; a NaN / infinity must be matched exactly. Returns max err / bound."""
    _reject_unwritten(kernel, got.detach().cpu())
    g = got.detach().cpu().double()
    r = ref64.detach().cpu().double().expand_as(g)
    bound = bound.detach().cpu().double().expand_as(g)
    finite = torch.isfinite(r)
    same_nonfinite = (g == r) | (torch.isnan(g) & torch.isnan(r))
    bad_nf = ~finite & ~same_nonfinite
    if bad_nf.any():
        _locate(kernel, "wrong where the reference is not finite", bad_nf, g, r)
    err = torch.where(finite, (g - r).abs(), torch.zeros_like(r))
    bad = finite & ~(err <= bound)          # also catches a NaN / inf where the reference is finite
    if bad.any():
        _locate(kernel, "out of bound", bad, g, r, bound)
    ratio = torch.where(bound > 0, err / bound, torch.zeros_like(err))
    return float(ratio[finite].max()) if finite.any() else 0.0


def check_bf16(kernel, got, ref64, k, terms=None, c=0.0, a=None):
    """bf16 output: k * ulp_bf16(ref) + c * U * terms (fp32 arithmetic before the rounding) + a (documented approximation)."""
    r = ref64.detach().cpu().double()
    bound = k * ulp_bf16(r)
    if terms is not None:
        bound = bound + c * U * terms.detach().cpu().double()
    if a is not None:
        bound = bound + a
    return check_bound(kernel, got, r, bound)


def check_sum(kernel, got, ref64, terms, c):
    """fp32 result of a reduction / fp32 arithmetic: c * 2^-24 * sum|terms|."""
    return check_bound(kernel, got, ref64, c * U * terms.detach().cpu().double())
