"""Element-by-element checks of the memory-bound entry points of include/clipbert_b200.h (casts, GELU backward, pools,
column sums, LayerNorm, losses, optimizer step) against float64 references computed from the same bf16 / fp32 inputs the
kernel read, at the shapes and values where such kernels go wrong: ragged blocks, tails, pitches, row-scale boundaries inside
a vector, ties, signed zeros, NaN and infinities.

Bounds, per element (never normwise):
  - outputs with one rounding (casts, pools, pad / subsample / mask copies): bit-exact to the float64 result rounded once,
    to nearest even, to the output type (NaN matches NaN whatever its payload);
  - other bf16 outputs: |got - ref| <= k * ulp_bf16(ref) + c * 2^-24 * sum|terms| + a, where the middle term is the fp32
    arithmetic before the final rounding and a is an absolute floor used only where the kernel documents an approximation
    (fast_erf in cb_gelu_bwd);
  - fp32 reductions and fp32 results: |got - ref| <= c * 2^-24 * sum|terms|, c about the reduction depth, sum|terms| computed
    in float64 next to the reference (a bound relative to the result would be meaningless under cancellation).
Every output lives between guard bands (and pitch padding where the ABI has a pitch) filled with a sentinel bit pattern that
must be unchanged afterwards; accumulating outputs start from random values, so "+=" is checked and not "=". Each case prints
its largest err / bound ratio ("RATIO <kernel> <case> <ratio>"; pytest -s shows them).

Each test runs on the H100 ("device", marked gpu; "device_det" for the _det variants of the accumulating entry points) and on
the CPU through tests/ops_emulator.py ("emulator"), so the helper, references, guard bands and bounds run on every change."""
import contextlib
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dropout_ref as D
import ops_emulator as E
from elementwise import BF16, F32, F64, G, U, Guarded, _record, check_bf16, check_bitexact, check_sum, rne_bf16


# ------------------------------------------------------------------------------------------------ backends
class Backend:
    def __init__(self, name, dev, ops, sumsq, adamw_step, det=False):
        self.name, self.dev, self.ops, self.sumsq, self.adamw_step, self.det = name, dev, ops, sumsq, adamw_step, det

    @property
    def emulated(self):
        return self.name == "emulator"

    @contextlib.contextmanager
    def run(self):
        """Launches inside run the _det variants on "device_det" (the wrappers follow torch's deterministic flag)."""
        prev = torch.are_deterministic_algorithms_enabled()
        if self.det:
            torch.use_deterministic_algorithms(True)
        try:
            yield
        finally:
            if self.det:
                torch.use_deterministic_algorithms(prev)
        if not self.emulated:
            torch.cuda.synchronize()


def _make_backend(name):
    if name == "emulator":
        return Backend(name, torch.device("cpu"), E, E.opt_sumsq, E.opt_adamw_step)
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import clipbert_b200  # noqa: F401
    from clipbert_b200 import ops, optim
    return Backend(name, torch.device("cuda:0"), ops, optim.sumsq, optim.adamw_step, det=(name == "device_det"))


@pytest.fixture(params=[pytest.param("device", marks=pytest.mark.gpu), "emulator"])
def be(request):
    return _make_backend(request.param)


@pytest.fixture(params=[pytest.param("device", marks=pytest.mark.gpu), pytest.param("device_det", marks=pytest.mark.gpu), "emulator"])
def be_acc(request):
    """For the entry points that accumulate: atomics, the ordered _det variant, and the emulator."""
    return _make_backend(request.param)


# ------------------------------------------------------------------------------------------------ the helper itself (CPU)
def _bf16_sample(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, generator=g, dtype=F64) * 3).to(BF16)


def test_helper_accepts_a_correctly_rounded_result():
    g = torch.Generator().manual_seed(1)
    ref = torch.randn(4096, generator=g, dtype=F64)
    ref[:4] = torch.tensor([1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 1.0 + 2.0 ** -8 + 2.0 ** -40, -0.0], dtype=F64)   # ties, a near-tie
    got = rne_bf16(ref)
    assert got.view(torch.int16)[:4].tolist() == [0x3F80, 0x3F82, 0x3F81, -0x8000]
    check_bitexact("helper", got, ref)
    assert check_bf16("helper", got, ref, k=1) <= 0.5 + 1e-12


def test_helper_rejects_an_element_two_ulp_off():
    ref = _bf16_sample(1000).double()
    got = rne_bf16(ref).clone()
    got.view(torch.int16)[417] += 2
    with pytest.raises(AssertionError, match=r"first at \(417,\)"):
        check_bitexact("helper", got, ref)
    with pytest.raises(AssertionError, match="out of bound"):
        check_bf16("helper", got, ref, k=1)


def test_helper_rejects_nan_against_finite_and_finite_against_nan():
    ref = _bf16_sample(64).double()
    got = rne_bf16(ref).clone()
    got[5] = float("nan")
    with pytest.raises(AssertionError):
        check_bitexact("helper", got, ref)
    with pytest.raises(AssertionError, match="out of bound"):
        check_bf16("helper", got, ref, k=1)
    ref2 = ref.clone()
    ref2[9] = float("nan")
    with pytest.raises(AssertionError):
        check_bitexact("helper", rne_bf16(ref), ref2)
    with pytest.raises(AssertionError, match="not finite"):
        check_sum("helper", ref.float(), ref2, ref.abs(), 4)


def test_helper_rejects_an_element_left_at_the_sentinel():
    out = Guarded((16,), BF16, torch.device("cpu"))
    ref = torch.full((16,), float("nan"), dtype=F64)
    out.t[:15] = float("nan")                   # element 15 keeps the sentinel NaN pattern: never written
    with pytest.raises(AssertionError, match="never written"):
        check_bitexact("helper", out.t, ref)
    with pytest.raises(AssertionError, match="never written"):
        check_bf16("helper", out.t, ref, k=1)


def test_helper_rejects_a_touched_guard_element():
    for dtype in (BF16, F32):
        out = Guarded((3, 5), dtype, torch.device("cpu"), ld=8)
        out.t.zero_()
        out.check("helper")
        out.buf[G + 5].zero_()                  # pitch padding of row 0
        with pytest.raises(AssertionError, match="guard"):
            out.check("helper")
        out = Guarded((7,), dtype, torch.device("cpu"))
        out.buf[G + 7].zero_()                  # first element after the output
        with pytest.raises(AssertionError, match="guard"):
            out.check("helper")


# ------------------------------------------------------------------------------------------------ values
def _special_f32(n, seed):
    """fp32 values that stress a bf16 rounding: exact ties, near-ties, subnormals, overflow, signed zeros, NaN, inf."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(n, generator=g) * torch.pow(2.0, torch.randint(-20, 20, (n,), generator=g).float())
    bits = v.view(torch.int32)
    k = torch.arange(n)
    bits[k % 7 == 1] = (bits[k % 7 == 1] & ~0xFFFF) | 0x8000            # exact ties
    bits[k % 7 == 2] = (bits[k % 7 == 2] & ~0xFFFF) | 0x7FFF            # just below a tie
    bits[k % 7 == 3] = (bits[k % 7 == 3] & ~0xFFFF) | 0x8001            # just above a tie
    special = torch.tensor([0.0, -0.0, float("inf"), -float("inf"), float("nan"), 3.4e38, -3.39e38, 1e-40, -1e-41, 1.2e-38])
    v[: len(special)] = special[:n]
    return v


def _bf16_all(lo, hi):
    """Every finite bf16 value in [lo, hi]."""
    b = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(BF16)
    f = b.float()
    return b[torch.isfinite(f) & (f >= lo) & (f <= hi)]


# ------------------------------------------------------------------------------------------------ casts
@pytest.mark.parametrize("n", [8, 13, 1003, 4096 + 5], ids=lambda n: "n%d" % n)
def test_cast_bf16_f32(be, n):
    """cb_cast_bf16_f32: exact widening, including the scalar tail (n % 8 != 0)."""
    x = _special_f32(n, n).to(BF16).to(be.dev)
    out = Guarded((n,), F32, be.dev)
    with be.run():
        be.ops.cast_bf16_f32(x, out.t)
    out.check("cast_bf16_f32")
    _record("cast_bf16_f32", "n%d" % n, check_bitexact("cast_bf16_f32", out.t, x.cpu().double()))


@pytest.mark.parametrize("rows,c,in_ld,cpad", [(5, 13, 20, 16), (3, 3129, 3136, 3136), (2, 2, 9, 8)],
                         ids=["c13-ld20-pad16", "c3129-ld3136", "c2-ld9-pad8"])
def test_pad_cast(be, rows, c, in_ld, cpad):
    """cb_pad_cast: fp32 [rows, c] with row pitch in_ld > c -> bf16 [rows, cpad], zero padded; one rounding."""
    src = Guarded((rows, c), F32, be.dev, ld=in_ld, init=_special_f32(rows * c, c).view(rows, c))
    out = Guarded((rows, cpad), BF16, be.dev)
    with be.run():
        be.ops.pad_cast(src.t, out.t)
    out.check("pad_cast")
    ref = torch.zeros(rows, cpad, dtype=F64)
    ref[:, :c] = src.t.cpu().double()
    _record("pad_cast", "c%d" % c, check_bitexact("pad_cast", out.t, ref))


def _scaled_ref(src, scales_per_elem, ftz):
    """The packed operand is RNE_bf16 of the fp32 product (as torch's w * s followed by .to(bfloat16)). ftz: the library is
    built with flush-to-zero, so a product below 2^-126 in magnitude packs as a zero of its sign (pinned in the header)."""
    prod = (src.cpu().float() * scales_per_elem.cpu().float()).double()
    return torch.where(prod.abs() < 2.0 ** -126, prod * 0.0, prod) if ftz else prod


@pytest.mark.parametrize("row_len,rows", [(147, 3), (9 * 64, 2), (3, 21), (1, 9)], ids=["row147", "row576", "row3", "row1"])
def test_cast_scale(be, row_len, rows):
    """cb_cast_scale with a per-row scale whose rows are not a multiple of 4 long: the scale changes inside a float4."""
    n = row_len * rows
    g = torch.Generator().manual_seed(row_len)
    src = torch.randn(n, generator=g).to(be.dev)
    scale = (torch.rand(rows, generator=g) + 0.5).to(be.dev)
    out = Guarded((n,), BF16, be.dev)
    with be.run():
        be.ops.cast_scale(src, out.t, scale, row_len)
    out.check("cast_scale")
    per = scale.cpu()[torch.arange(n) // row_len]
    _record("cast_scale", "row%d" % row_len, check_bitexact("cast_scale", out.t, _scaled_ref(src, per, not be.emulated)))


def test_cast_scale_segments_leaves_the_gaps_untouched(be):
    """cb_cast_scale_segments: several 64-aligned segments, row lengths 147 / 576 / 3, some without a scale, gaps between them."""
    segs = [(0, 441, 147, 0), (512, 1152, 576, 3), (1728, 63, 3, 5), (1856, 100, 10, -1), (2048, 5, 5, -1)]
    n = 2112
    g = torch.Generator().manual_seed(7)
    master = _special_f32(n, 7)
    master[torch.isnan(master) | torch.isinf(master)] = 1.0
    master = master.to(be.dev)
    scales = (torch.rand(40, generator=g) + 0.5).to(be.dev)
    old = _bf16_sample(n, 8)
    out = Guarded((n,), BF16, be.dev, init=old)
    table = torch.tensor(segs, dtype=torch.int64, device=be.dev)
    with be.run():
        be.ops.cast_scale_segments(master, out.t, table, scales)
    out.check("cast_scale_segments")
    ref = old.double().clone()
    covered = torch.zeros(n, dtype=torch.bool)
    for off, cnt, row_len, soff in segs:
        per = torch.ones(cnt) if soff < 0 else scales.cpu()[soff + torch.arange(cnt) // row_len]
        ref[off:off + cnt] = _scaled_ref(master[off:off + cnt], per, not be.emulated)
        covered[off:off + cnt] = True
    got = out.t.cpu()
    assert torch.equal(got[~covered].view(torch.int16), old[~covered].view(torch.int16)), "an element between segments was written"
    _record("cast_scale_segments", "5seg", check_bitexact("cast_scale_segments", got, ref))


# ------------------------------------------------------------------------------------------------ GELU backward
# cdf = (1 + erf(u / sqrt 2)) / 2 in fp32 cancels in the left tail (erf ~ -1), where gelu' ~ 1e-6: an absolute error of a few
# 2^-24 from the fp32 evaluation, plus, on the device, the 1.5e-7 of fast_erf (Abramowitz-Stegun 7.1.26, csrc/common.cuh)
GELU_FP32_FLOOR = 0.5 * 8 * U
GELU_FAST_ERF_FLOOR = 0.5 * 1.5e-7


def _gelu_grad64(u):
    """ATen's gelu backward formula in float64 (NaN at +-inf, as ATen: inf * pdf(inf) = inf * 0)."""
    return 0.5 * (1.0 + torch.erf(u / math.sqrt(2.0))) + u * torch.exp(-0.5 * u * u) / math.sqrt(2.0 * math.pi)


@pytest.mark.parametrize("case", ["every_bf16_in_pm12", "n8_inf_nan_zero"])
def test_gelu_bwd(be, case):
    """cb_gelu_bwd: dx = dy * gelu'(u) over every finite bf16 u in [-12, 12] and +-inf; k = 1 ulp plus the absolute floor
    |dy| * (GELU_FP32_FLOOR + GELU_FAST_ERF_FLOOR on the device), which dominates the left tail."""
    if case == "n8_inf_nan_zero":
        u = torch.tensor([float("inf"), -float("inf"), 0.0, -0.0, float("nan"), -12.0, 12.0, -3.0]).to(BF16)
    else:
        u = torch.cat([_bf16_all(-12.0, 12.0), torch.tensor([float("inf"), -float("inf")]).to(BF16)])
        u = torch.cat([u, torch.zeros((-u.numel()) % 8, dtype=BF16)])
    dy = _bf16_sample(u.numel(), 3)
    out = Guarded((u.numel(),), BF16, be.dev)
    with be.run():
        be.ops.gelu_bwd(dy.to(be.dev), u.to(be.dev), out.t)
    out.check("gelu_bwd")
    ref = dy.double() * _gelu_grad64(u.double())
    a = dy.double().abs() * (GELU_FP32_FLOOR + (0.0 if be.emulated else GELU_FAST_ERF_FLOOR))
    _record("gelu_bwd", case, check_bf16("gelu_bwd", out.t, ref, k=1, a=a))


# ------------------------------------------------------------------------------------------------ CNN data movement
def _pool_values(kind, n, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "random":
        v = torch.randn(n, generator=g)
    elif kind == "ties_and_signed_zeros":        # few distinct values: many exact ties, +0 / -0 maxima
        v = torch.tensor([0.0, -0.0, 1.0, -1.0, 0.5])[torch.randint(0, 5, (n,), generator=g)]
    else:                                        # "nan_and_inf"
        v = torch.randn(n, generator=g)
        r = torch.randint(0, 40, (n,), generator=g)
        v[r == 0] = float("nan")
        v[r == 1] = float("inf")
        v[r == 2] = -float("inf")
    return v.to(BF16)


POOL_VALUES = ["random", "ties_and_signed_zeros", "nan_and_inf"]


@pytest.mark.parametrize("values", POOL_VALUES)
@pytest.mark.parametrize("n,h,w,c,strided", [(1, 112, 112, 64, False), (1, 224, 224, 64, True), (1, 384, 384, 64, True), (2, 1, 1, 8, False),
                                             (1, 2, 2, 16, True), (2, 37, 53, 24, False), (1, 9, 9, 8, True)],
                         ids=["stem224", "stem448_strided", "stem768_strided", "1x1", "2x2_strided", "37x53", "c8_strided"])
def test_maxpool3x3s2(be, n, h, w, c, strided, values):
    """cb_maxpool3x3s2 / _strided: F.max_pool2d(3, 2, 1) semantics, bit-exact: NaN propagates, first maximum of equal ones
    (so the sign of a zero maximum is ATen's)."""
    rp, ip = (w + 3, (h + 3) * (w + 3)) if strided else (w, h * w)
    x = _pool_values(values, n * ip * c, h * w + c)
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    out = Guarded((n * ho * wo * c,), BF16, be.dev)
    with be.run():
        if strided:
            be.ops.maxpool3x3s2(x.to(be.dev), out.t, n, h, w, c, rp, ip)
        else:
            be.ops.maxpool3x3s2(x.to(be.dev), out.t, n, h, w, c)
    out.check("maxpool3x3s2")
    xv = torch.as_strided(x.double(), (n, h, w, c), (ip * c, rp * c, c, 1))
    ref = F.max_pool2d(xv.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1).reshape(-1)
    _record("maxpool3x3s2", "%dx%d-%s" % (h, w, values), check_bitexact("maxpool3x3s2", out.t, ref))


@pytest.mark.parametrize("values", POOL_VALUES)
@pytest.mark.parametrize("hw,c", [(14, 16), (24, 8), (7, 16), (3, 8), (2, 24)], ids=["14", "24", "7", "3", "2"])
def test_maxpool2x2_relu_fwd_bwd(be, hw, c, values):
    """cb_maxpool2x2_relu_fwd / _bwd against F.max_pool2d(2, 2) + ReLU and the pool's autograd: NaN propagates forward and
    the gradient goes to ATen's arg-max (first maximum; last NaN). Pinned, as the header states: the forward writes +0 for a
    window whose maximum is -0 (ATen's ReLU keeps -0), and ReLU' is (max > 0), so a NaN maximum gets no gradient."""
    n = 2
    x = _pool_values(values, n * hw * hw * c, hw * c)
    dy = _bf16_sample(n * (hw // 2) ** 2 * c, hw)
    y = Guarded((n * (hw // 2) ** 2 * c,), BF16, be.dev)
    dx = Guarded((n * (hw + 2) ** 2 * c,), BF16, be.dev)
    with be.run():
        be.ops.maxpool2x2_relu_fwd(x.to(be.dev), y.t, n, hw, hw, c)
        be.ops.maxpool2x2_relu_bwd(dy.to(be.dev), x.to(be.dev), dx.t, n, hw, hw, c)
    y.check("maxpool2x2_relu_fwd")
    dx.check("maxpool2x2_relu_bwd")
    xv = x.double().view(n, hw, hw, c).permute(0, 3, 1, 2).clone().requires_grad_(True)
    with torch.enable_grad():
        pooled = F.max_pool2d(xv, 2, 2)
        up = dy.double().view(n, hw // 2, hw // 2, c).permute(0, 3, 1, 2)
        pooled.backward(torch.where(pooled.detach() > 0, up, torch.zeros_like(up)))
    ref_y = torch.relu(pooled.detach()).permute(0, 2, 3, 1).reshape(-1) + 0.0      # + 0.0: -0 -> +0 (pinned above)
    ref_dx = torch.zeros(n, hw + 2, hw + 2, c, dtype=F64)
    ref_dx[:, 1:-1, 1:-1] = xv.grad.permute(0, 2, 3, 1)
    _record("maxpool2x2_relu_fwd", "%d-%s" % (hw, values), check_bitexact("maxpool2x2_relu_fwd", y.t, ref_y))
    _record("maxpool2x2_relu_bwd", "%d-%s" % (hw, values), check_bitexact("maxpool2x2_relu_bwd", dx.t, ref_dx.reshape(-1)))


@pytest.mark.parametrize("n,h,w,c", [(1, 7, 9, 16), (2, 13, 13, 8), (1, 1, 3, 8), (1, 56, 56, 24)], ids=["7x9", "13x13", "1x3", "56x56"])
def test_subsample2_and_unsubsample2_mask(be, n, h, w, c):
    """cb_subsample2 / cb_unsubsample2_mask at odd sizes, and cb_relu_mask on the same activations; the masks are (act > 0)
    as the header states (a NaN or -0 activation masks; a masked element is +0)."""
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    x = _pool_values("nan_and_inf", n * h * w * c, h * w)
    act = _pool_values("ties_and_signed_zeros", n * h * w * c, c)
    act[::11] = float("nan")
    dsub = _bf16_sample(n * ho * wo * c, w)
    dy = _bf16_sample(n * h * w * c, h)
    y = Guarded((n * ho * wo * c,), BF16, be.dev)
    dx = Guarded((n * h * w * c,), BF16, be.dev)
    dr = Guarded((n * h * w * c,), BF16, be.dev)
    with be.run():
        be.ops.subsample2(x.to(be.dev), y.t, n, h, w, c)
        be.ops.unsubsample2_mask(dsub.to(be.dev), act.to(be.dev), dx.t, n, h, w, c)
        be.ops.relu_mask(dy.to(be.dev), act.to(be.dev), dr.t)
    y.check("subsample2")
    dx.check("unsubsample2_mask")
    dr.check("relu_mask")
    keep = act.double() > 0
    check_bitexact("relu_mask", dr.t, torch.where(keep, dy.double(), torch.zeros(dy.shape, dtype=F64)))
    check_bitexact("subsample2", y.t, x.double().view(n, h, w, c)[:, ::2, ::2].reshape(-1))
    full = torch.zeros(n, h, w, c, dtype=F64)
    full[:, ::2, ::2] = dsub.double().view(n, ho, wo, c)
    ref = torch.where(act.double().view(n, h, w, c) > 0, full, torch.zeros_like(full))
    _record("unsubsample2_mask", "%dx%d" % (h, w), check_bitexact("unsubsample2_mask", dx.t, ref.reshape(-1)))


# ------------------------------------------------------------------------------------------------ column sums
COLSUM_CASES = [(m, 264, None) for m in (1, 127, 128, 129, 5000)] + [(129, n, None) for n in (8, 2304, 3080)] + [(5000, 3080, 3096), (127, 8, 24)]


@pytest.mark.parametrize("m,n,ld", COLSUM_CASES, ids=["m%d-n%d%s" % (m, n, "" if ld is None else "-ld%d" % ld) for m, n, ld in COLSUM_CASES])
def test_colsum(be_acc, m, n, ld):
    """cb_colsum / _det: out[c] += sum_m x[m, c] with ragged 128-row slabs and partial 256-column blocks; out starts random."""
    be = be_acc
    g = torch.Generator().manual_seed(m * n)
    x = (torch.randn(m, n, generator=g) * 4).to(BF16)
    xin = Guarded((m, n), BF16, be.dev, ld=ld or n, init=x)
    pre = torch.randn(n, generator=g)
    out = Guarded((n,), F32, be.dev, init=pre)
    with be.run():
        be.ops.colsum(xin.t, out.t, m, n, ld)
    out.check("colsum")
    x64 = x.double()
    c = 16 + 8 + math.ceil(m / 128) + 2
    _record("colsum", "m%d-n%d" % (m, n), check_sum("colsum", out.t, pre.double() + x64.sum(0), pre.double().abs() + x64.abs().sum(0), c))


# ------------------------------------------------------------------------------------------------ LayerNorm
HID = 768
LN_ROWS = [1, 3, 4, 5, 1055, 1056, 1057, 3001]


def _ln_input(m, kind, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "random":
        x = torch.randn(m, HID, generator=g)
    elif kind == "offset40":                    # after a residual add: mean ~ 40, unit spread
        x = 40.0 + torch.randn(m, HID, generator=g)
    else:                                       # "constant": variance 0, only eps remains
        x = torch.randn(m, 1, generator=g).expand(m, HID)
    return x.to(BF16)


LN_CASES = [(m, "random", 1e-12) for m in LN_ROWS] + [(1057, "offset40", 1e-12), (5, "offset40", 1e-5), (1056, "constant", 1e-12),
                                                     (3, "constant", 1e-5)]


@pytest.mark.parametrize("m,kind,eps", LN_CASES, ids=["m%d-%s-eps%g" % c for c in LN_CASES])
def test_layernorm_fwd(be, m, kind, eps):
    """cb_layernorm_fwd: y within 1 ulp of bf16 plus the fp32 arithmetic of (x - mean) * rstd * gamma + beta; stats against
    the float64 mean / rstd."""
    g = torch.Generator().manual_seed(m + 7)
    x = _ln_input(m, kind, m)
    gamma = (torch.rand(HID, generator=g) + 0.5).to(be.dev)
    beta = (torch.randn(HID, generator=g) * 0.1).to(be.dev)
    y = Guarded((m, HID), BF16, be.dev)
    stats = Guarded((m, 2), F32, be.dev)
    with be.run():
        be.ops.layernorm_fwd(x.to(be.dev), gamma, beta, y.t, stats.t, eps)
    y.check("layernorm_fwd y")
    stats.check("layernorm_fwd stats")
    x64, g64, b64 = x.double(), gamma.cpu().double(), beta.cpu().double()
    mean = x64.mean(1)
    var = ((x64 - mean[:, None]) ** 2).mean(1)
    rstd = 1.0 / torch.sqrt(var + eps)
    ref = (x64 - mean[:, None]) * rstd[:, None] * g64 + b64
    terms = (x64.abs() + mean.abs()[:, None]) * rstd[:, None] * g64.abs() + b64.abs()
    ry = check_bf16("layernorm_fwd", y.t, ref, k=1, terms=terms, c=32)
    rm = check_sum("layernorm_fwd mean", stats.t[:, 0], mean, x64.abs().mean(1), 32)
    rel = torch.where(var > 0, 1.0 + mean.abs() * rstd, torch.ones_like(var))
    rr = check_sum("layernorm_fwd rstd", stats.t[:, 1], rstd, rstd * rel, 32)
    _record("layernorm_fwd", "m%d-%s" % (m, kind), max(ry, rm, rr))


LN_BWD_CASES = [(m, 0.0, False) for m in LN_ROWS] + [(1057, 0.1, True), (5, 0.1, True), (3001, 0.1, False)]


@pytest.mark.parametrize("m,p,with_drop", LN_BWD_CASES, ids=["m%d-p%g%s" % (m, p, "-dx_drop" if d else "") for m, p, d in LN_BWD_CASES])
def test_layernorm_bwd(be_acc, m, p, with_drop):
    """cb_layernorm_bwd / _det: dx (and dx_drop with the mask of tests/dropout_ref.py) per element; dgamma / dbeta / dbias_drop
    added into pre-filled gradients, against float64 sums with the reduction depth of the ragged / grid-stride block plan."""
    be = be_acc
    g = torch.Generator().manual_seed(m + 11)
    x = _ln_input(m, "random" if m != 1057 else "offset40", m)
    x64 = x.double()
    mean = x64.mean(1)
    rstd = 1.0 / torch.sqrt(((x64 - mean[:, None]) ** 2).mean(1) + 1e-12)
    stats32 = torch.stack([mean, rstd], 1).float()
    dy = (torch.randn(m, HID, generator=g)).to(BF16)
    gamma = (torch.rand(HID, generator=g) + 0.5)
    pre = [torch.randn(HID, generator=g) for _ in range(3)]
    dx = Guarded((m, HID), BF16, be.dev)
    dxd = Guarded((m, HID), BF16, be.dev) if with_drop else None
    dgam, dbet, dbias = (Guarded((HID,), F32, be.dev, init=t) for t in pre)
    seed = 1234 + m
    with be.run():
        be.ops.layernorm_bwd(dy.to(be.dev), x.to(be.dev), stats32.to(be.dev), gamma.to(be.dev), dx.t, None if dxd is None else dxd.t,
                             dgam.t, dbet.t, dbias.t, p, seed)
    for t, name in ((dx, "dx"), (dxd, "dx_drop"), (dgam, "dgamma"), (dbet, "dbeta"), (dbias, "dbias_drop")):
        if t is not None:
            t.check("layernorm_bwd " + name)
    mu, rs = stats32[:, 0].double()[:, None], stats32[:, 1].double()[:, None]
    xhat = (x64 - mu) * rs
    gy = dy.double() * gamma.double()
    a1, a2 = gy.mean(1, keepdim=True), (gy * xhat).mean(1, keepdim=True)
    ref = rs * (gy - a1 - xhat * a2)
    xh_terms = (x64.abs() + mu.abs()) * rs
    terms = rs * (gy.abs() + gy.abs().mean(1, keepdim=True) + xh_terms * (gy.abs() * xh_terms).mean(1, keepdim=True))
    ratios = [check_bf16("layernorm_bwd dx", dx.t, ref, k=1, terms=terms, c=32)]
    drop_src = dx.t
    if with_drop:
        mult = torch.from_numpy(D.multipliers(D.effective_seed(seed), D.layernorm_index(m), p)).double()
        ratios.append(check_bf16("layernorm_bwd dx_drop", dxd.t, ref * mult, k=1, terms=terms * mult, c=32))
        drop_src = dxd.t
    blocks = min(math.ceil(m / 4), 264)
    c = math.ceil(m / blocks) + 4 + blocks + 8
    dy64 = dy.double()
    ratios.append(check_sum("layernorm_bwd dgamma", dgam.t, pre[0].double() + (dy64 * xhat).sum(0),
                            pre[0].double().abs() + (dy64.abs() * xh_terms).sum(0), c + 8))
    ratios.append(check_sum("layernorm_bwd dbeta", dbet.t, pre[1].double() + dy64.sum(0), pre[1].double().abs() + dy64.abs().sum(0), c))
    d64 = drop_src.cpu().double()       # dbias_drop: the column sums of the bf16 tensor the dense's dgrad reads
    ratios.append(check_sum("layernorm_bwd dbias_drop", dbias.t, pre[2].double() + d64.sum(0), pre[2].double().abs() + d64.abs().sum(0), c))
    _record("layernorm_bwd", "m%d-p%g" % (m, p), max(ratios))


# ------------------------------------------------------------------------------------------------ cross entropy
CE_CASES = [(ncls, "normal") for ncls in (1, 2, 5, 255, 256, 257, 3129, 30522)] + [
    (3129, "offset+1e4"), (257, "offset-1e4"), (30522, "neginf_lanes"), (300, "neginf_lanes"), (257, "neginf_lanes"),
    (256, "neginf_lanes"), (5, "neginf_lanes"), (2, "neginf_lanes")]


def _ce_logits(rows, ncls, kind, seed):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(rows, ncls, generator=g) * 3
    if kind == "offset+1e4":
        z += 1e4
    elif kind == "offset-1e4":
        z -= 1e4
    elif kind == "neginf_lanes":
        # -inf as the FIRST logit some threads of the 256-thread block see (lanes 0, 1, 31, 255, shifted by the row); when
        # ncls > 256 + lane the same thread reads a finite logit afterwards, the case whose online update once produced NaN
        for r in range(rows):
            for c in (0, 1, 31, 255, 256 + 7, 2 * 256 + 31):
                if c < ncls - 1:
                    z[r, (c + r) % (ncls - 1)] = -float("inf")
        z[:, ncls - 1] = 1.0
    return z


@pytest.mark.parametrize("ncls,kind", CE_CASES, ids=["ncls%d-%s" % c for c in CE_CASES])
def test_cross_entropy(be, ncls, kind):
    """cb_cross_entropy_fwd / _bwd with row pitches ld, dld > ncls, ignore_index rows and out-of-range labels (pinned: loss 0
    and no gradient, instead of raising as F.cross_entropy does). __expf / __logf: the bound carries their documented error."""
    rows = 6
    z = _ce_logits(rows, ncls, kind, ncls)
    y = torch.randint(0, ncls, (rows,), generator=torch.Generator().manual_seed(1))
    if kind == "neginf_lanes":
        y[:] = ncls - 1
    y[1] = -100
    y[4] = ncls + 3 if rows > 4 else y[4]
    zin = Guarded((rows, ncls), F32, be.dev, ld=ncls + 8, init=z)
    loss, lse = Guarded((rows,), F32, be.dev), Guarded((rows,), F32, be.dev)
    gl = torch.rand(rows, generator=torch.Generator().manual_seed(2)) + 0.5
    dz = Guarded((rows, ncls), F32, be.dev, ld=ncls + 3)
    yd = y.to(be.dev)
    with be.run():
        be.ops.cross_entropy_fwd(zin.t, yd, loss.t, lse.t)
    lse_got = lse.t.cpu().clone()
    with be.run():
        be.ops.cross_entropy_bwd(zin.t, yd, lse.t, gl.to(be.dev), dz.t)
    for t, name in ((zin, "logits"), (loss, "loss"), (lse, "lse"), (dz, "dlogits")):
        t.check("cross_entropy " + name)
    z64 = z.double()
    m = z64.max(1).values
    ref_lse = torch.logsumexp(z64, 1)
    ok = (y >= 0) & (y < ncls)
    zy = torch.where(ok, z64[torch.arange(rows), y.clamp(0, ncls - 1)], torch.zeros(rows, dtype=F64))
    ref_loss = torch.where(ok, ref_lse - zy, torch.zeros(rows, dtype=F64))
    depth = 16 + math.ceil(ncls / 256)
    lse_terms = m.abs() + 1.0 + math.log(ncls)
    r1 = check_sum("cross_entropy lse", lse_got, ref_lse, lse_terms, depth)
    r2 = check_sum("cross_entropy loss", loss.t, ref_loss, torch.where(ok, lse_terms + zy.abs(), torch.zeros(rows, dtype=F64)), depth)
    # backward from the lse it read: __expf(x) carries 2 + 1.173 |x| ulp (CUDA programming guide)
    p = torch.exp(z64 - lse_got.double()[:, None])
    onehot = torch.zeros_like(p)
    onehot[ok, y[ok]] = 1.0
    g64 = (gl.double() * ok.double())[:, None]
    ref_d = g64 * (p - onehot)
    x = (z64 - lse_got.double()[:, None]).abs()
    terms = g64 * (torch.where(p > 0, p * (4 + 1.2 * x), torch.zeros_like(p)) + onehot)
    r3 = check_sum("cross_entropy dlogits", dz.t, ref_d, terms, 2)
    _record("cross_entropy", "ncls%d-%s" % (ncls, kind), max(r1, r2, r3))


# ------------------------------------------------------------------------------------------------ clip losses
CLIP_CASES = [(1, 1), (255, 2), (256, 16), (257, 2), (600, 16), (600, 1)]


@pytest.mark.parametrize("pool", ["lse", "mean", "max"])
@pytest.mark.parametrize("nseq,n_clips", CLIP_CASES, ids=["nseq%d-clips%d" % c for c in CLIP_CASES])
def test_clip_losses(be_acc, nseq, n_clips, pool):
    """cb_clip_lse_loss / cb_clip_pool_ce_loss (mean, max) and their _det variants, grad_scale 0.75, exact ties across clips
    for max (pinned: the FIRST maximal clip receives the gradient), labels out of range (pinned: clamped to [0, ncls))."""
    be = be_acc
    ncls = 5
    g = torch.Generator().manual_seed(nseq * 31 + n_clips)
    z = torch.randn(n_clips, nseq, ncls, generator=g) * 2
    if n_clips > 1:
        z[1, ::3] = z[0, ::3]                   # exact ties between clip 0 and clip 1
    y = torch.randint(0, ncls, (nseq,), generator=g)
    y[::7] = -1
    y[3::7] = ncls + 2
    gs = 0.75
    loss = Guarded((1,), F32, be.dev)
    dz = Guarded((n_clips, nseq, ncls), F32, be.dev)
    zd, yd = z.to(be.dev), y.to(be.dev)
    with be.run():
        if pool == "lse":
            be.ops.clip_lse_loss(zd, yd, loss.t, dz.t, n_clips, nseq, ncls, gs)
        else:
            be.ops.clip_pool_ce_loss(zd, yd, loss.t, dz.t, n_clips, nseq, ncls, 1 if pool == "mean" else 2, gs)
    loss.check("clip loss")
    dz.check("clip dlogits")
    yc = y.clamp(0, ncls - 1)
    z64 = z.double()
    b = torch.arange(nseq)
    if pool == "lse":
        lg = z64.permute(1, 0, 2)                                        # [nseq, clips, ncls]
        lse_all = torch.logsumexp(lg.reshape(nseq, -1), 1)
        zy = lg[b, :, yc]                                                # [nseq, clips]
        lse_y = torch.logsumexp(zy, 1)
        per = lse_all - lse_y
        d = torch.exp(lg - lse_all[:, None, None])
        d[b, :, yc] -= torch.exp(zy - lse_y[:, None])
        ref_d = (d * gs / nseq).permute(1, 0, 2)
        terms_l = lse_all.abs() + lse_y.abs() + 1
        t = torch.exp(lg - lse_all[:, None, None]) * (1 + lse_all.abs()[:, None, None])
        t[b, :, yc] += torch.exp(zy - lse_y[:, None]) * (1 + lse_y.abs()[:, None])
        terms_d = t.permute(1, 0, 2) * gs / nseq
        cd = 8 + 2 * n_clips * ncls
    else:
        if pool == "mean":
            pooled = z64.mean(0)
            arg = None
        else:
            arg = torch.zeros(nseq, ncls, dtype=torch.long)
            best = z64[0].clone()
            for k in range(1, n_clips):                                  # first maximum wins
                take = z64[k] > best
                best = torch.where(take, z64[k], best)
                arg = torch.where(take, torch.full_like(arg, k), arg)
            pooled = best
        lse = torch.logsumexp(pooled, 1)
        per = lse - pooled[b, yc]
        gp = torch.exp(pooled - lse[:, None])
        gp[b, yc] -= 1.0
        gp = gp * gs / nseq
        if pool == "mean":
            ref_d = (gp / n_clips)[None].expand(n_clips, nseq, ncls)
        else:
            ref_d = torch.zeros(n_clips, nseq, ncls, dtype=F64)
            ref_d.scatter_(0, arg[None], gp[None])
        terms_l = lse.abs() + pooled[b, yc].abs() + pooled.abs().max(1).values * n_clips + 1
        terms_d = ((torch.exp(pooled - lse[:, None]) + 1) * (1 + lse.abs()[:, None]) * gs / nseq)[None].expand(n_clips, nseq, ncls)
        cd = 8 + 2 * n_clips + 2 * ncls
    ref_loss = per.mean()
    cl = 8 + 2 * n_clips * ncls + math.ceil(math.log2(nseq + 1)) + math.ceil(nseq / 256) + 8
    r1 = check_sum("clip loss", loss.t, ref_loss.reshape(1), (terms_l.sum() / nseq).reshape(1), cl)
    r2 = check_sum("clip dlogits", dz.t, ref_d, terms_d, cd)
    _record("clip_%s_loss" % pool, "nseq%d-clips%d" % (nseq, n_clips), max(r1, r2))


# ------------------------------------------------------------------------------------------------ optimizer
# chunk table rows: offset, numel, group, row_len, scale_off, flags (bit 0: emit packed), elem0. Gaps between chunks are the
# alignment padding of the flat buffers: no buffer may change there.
_CHUNKS = [
    (0, 441, 0, 147, 0, 1, 0),              # 3 rows of 147, scalar tail of 1
    (448, 1152, 1, 576, 3, 1, 290),         # row boundary at i = 286: a float4 group (284..287) straddles two row scales
    (1664, 63, 0, 3, 10, 1, 7),             # row length 3: every float4 spans two or three rows; tail of 3
    (1792, 1000, 1, 0, -1, 1, 0),           # no scale, emitted
    (2816, 500, 0, 0, -1, 0, 0),            # not emitted: packed stays untouched
]
_NFLAT = 3392
_LR = 1e-3


def adamw_restated(p, g, m, v, coef, lr, step_size, wd, b1, b2, eps):
    """One AdamW step of src/optimization/adamw.py:40-103 in float64 with the clip coefficient applied to the gradient;
    returns (p, m, v) and the sum|terms| bounds of the fp32 evaluation of each."""
    g = g * coef
    m_new = m * b1 + (1.0 - b1) * g
    v_new = v * b2 + (1.0 - b2) * g * g
    denom = v_new.sqrt() + eps
    upd = step_size * (m_new / denom)
    p1 = p - upd
    p_new = p1 - lr * wd * p1 if wd > 0 else p1
    tm = (m * b1).abs() + ((1.0 - b1) * g).abs() * 4
    tv = (v * b2).abs() + ((1.0 - b2) * g * g).abs() * 4
    tp = p.abs() + step_size * (tm + m_new.abs() * 4) / denom + lr * wd * p1.abs()
    return (p_new, m_new, v_new), (tp, tm, tv)


def test_adamw_restatement_matches_the_oracle():
    """The float64 restatement above against oracle/adamw_ref.py (itself pinned to the reference's AdamW class)."""
    from oracle import adamw_ref
    g = torch.Generator().manual_seed(3)
    p, gr = torch.randn(50, generator=g, dtype=F64), torch.randn(50, generator=g, dtype=F64)
    m, v = torch.randn(50, generator=g, dtype=F64) * 0.1, torch.rand(50, generator=g, dtype=F64) * 0.1
    for step, wd, correct in ((1, 0.01, True), (3, 0.0, True), (2, 0.01, False)):
        ss = _LR * math.sqrt(1 - 0.999 ** step) / (1 - 0.9 ** step) if correct else _LR
        (p1, m1, v1), _ = adamw_restated(p, gr, m, v, 1.0, _LR, ss, wd, 0.9, 0.999, 1e-6)
        p2, m2, v2 = adamw_ref.adamw_step(p, gr, m, v, step, _LR, (0.9, 0.999), 1e-6, wd, correct)
        assert torch.allclose(p1, p2, rtol=0, atol=1e-15) and torch.equal(m1, m2) and torch.equal(v1, v2)


def _chunk_mask():
    inside = torch.zeros(_NFLAT, dtype=torch.bool)
    for off, n, *_ in _CHUNKS:
        inside[off:off + n] = True
    return inside


def test_sumsq_over_a_chunk_table(be_acc):
    """cb_sumsq / _det with a chunk table: only the table's elements enter; out starts random."""
    be = be_acc
    g = torch.Generator().manual_seed(9)
    x = torch.randn(_NFLAT, generator=g) * 3
    x[~_chunk_mask()] = 1e30            # padding must not enter the norm
    pre = torch.rand(1, generator=g) * 10
    out = Guarded((1,), F32, be.dev, init=pre)
    table = torch.tensor([list(c) + [0] for c in _CHUNKS], dtype=torch.int64)
    with be.run():
        be.sumsq(x.to(be.dev), table.to(be.dev), len(_CHUNKS), out.t)
    out.check("sumsq")
    x64 = x.double()[_chunk_mask()]
    ref = pre.double() + (x64 ** 2).sum()
    c = math.ceil(1152 / 1024) + 16 + len(_CHUNKS) + 4
    _record("sumsq", "5chunks", check_sum("sumsq", out.t, ref, pre.double() + (x64 ** 2).sum(), c))


@pytest.mark.parametrize("zero_grad", [False, True], ids=["keep_grad", "zero_grad"])
@pytest.mark.parametrize("clip", ["off", "on", "at_max_norm"])
def test_adamw_step_three_steps(be, clip, zero_grad):
    """cb_adamw_step driven by a hand-built chunk table for three steps: master / exp_avg / exp_avg_sq against the float64
    restatement from the kernel's previous state; the packed bf16 copy bit-exact to RNE(bf16(fp32(p_new * scale))) of the
    kernel's own master; grad zeroed or kept; every element outside the chunks untouched in all five buffers."""
    g = torch.Generator().manual_seed(21)
    sent = torch.full((_NFLAT,), 7.0)
    master = torch.where(_chunk_mask(), torch.randn(_NFLAT, generator=g), sent)
    m = torch.where(_chunk_mask(), torch.zeros(_NFLAT), sent)
    v = m.clone()
    grad = sent.clone()
    packed_old = _bf16_sample(_NFLAT, 22)
    bufs = [Guarded((_NFLAT,), F32, be.dev, init=t) for t in (master, grad, m, v)]
    packed = Guarded((_NFLAT,), BF16, be.dev, init=packed_old)
    scales = (torch.rand(64, generator=g) + 0.5)
    table = torch.tensor([list(c) + [0] for c in _CHUNKS], dtype=torch.int64).to(be.dev)
    inside = _chunk_mask()
    ratio = 0.0
    for step in (1, 2, 3):
        gnew = torch.randn(_NFLAT, generator=g) * 0.5
        gt = bufs[1].t.cpu()
        gt[inside] = gnew[inside]
        bufs[1].t.copy_(gt)
        before = [b.t.cpu().double() for b in bufs]
        gsq = (gt.double()[inside] ** 2).sum().float()
        norm = math.sqrt(float(gsq))
        max_norm = {"off": 0.0, "on": 0.5 * norm, "at_max_norm": norm}[clip]
        # group 0: bias-corrected step size, weight decay; group 1: bias correction folded out, no weight decay
        hyper = torch.tensor([[_LR, _LR * math.sqrt(1 - 0.999 ** step) / (1 - 0.9 ** step), 0.01, 0.9, 0.999, 1e-6, 0, 0],
                              [_LR, _LR, 0.0, 0.9, 0.999, 1e-6, 0, 0]], dtype=F32)
        with be.run():
            be.adamw_step(bufs[0].t, bufs[1].t, bufs[2].t, bufs[3].t, packed.t, table, len(_CHUNKS), hyper.to(be.dev),
                          scales.to(be.dev), None if clip == "off" else gsq.reshape(1).to(be.dev), max_norm, zero_grad)
        for b, name in zip(bufs + [packed], ("master", "grad", "exp_avg", "exp_avg_sq", "packed")):
            b.check("adamw_step " + name)
        after = [b.t.cpu() for b in bufs]
        for name, b0, b1 in zip(("master", "grad", "exp_avg", "exp_avg_sq"), before, after):
            assert torch.equal(b1[~inside].double(), b0[~inside]), "adamw_step wrote %s outside the chunks" % name
        pk = packed.t.cpu()
        coef = 1.0 if clip == "off" else min(1.0, max_norm / (math.sqrt(float(gsq)) + 1e-6))
        for off, n, grp, row_len, soff, flags, elem0 in _CHUNKS:
            sl = slice(off, off + n)
            h = [float(t) for t in hyper[grp][:6]]
            (p_ref, m_ref, v_ref), (tp, tm, tv) = adamw_restated(before[0][sl], before[1][sl], before[2][sl], before[3][sl], coef,
                                                                h[0], h[1], h[2], h[3], h[4], h[5])
            ratio = max(ratio, check_sum("adamw_step master", after[0][sl], p_ref, tp, 12),
                        check_sum("adamw_step exp_avg", after[2][sl], m_ref, tm, 4),
                        check_sum("adamw_step exp_avg_sq", after[3][sl], v_ref, tv, 4))
            assert torch.equal(after[1][sl], torch.zeros(n) if zero_grad else before[1][sl].float()), "adamw_step grad"
            if flags & 1:
                per = torch.ones(n) if soff < 0 else scales[soff + (elem0 + torch.arange(n)) // row_len]
                check_bitexact("adamw_step packed", pk[sl], _scaled_ref(after[0][sl], per, not be.emulated))
            else:
                assert torch.equal(pk[sl].view(torch.int16), packed_old[sl].view(torch.int16)), "adamw_step emitted an unflagged chunk"
        assert torch.equal(pk[~inside].view(torch.int16), packed_old[~inside].view(torch.int16)), "packed written outside the chunks"
    _record("adamw_step", "clip_%s-%s" % (clip, "zero" if zero_grad else "keep"), ratio)


# ------------------------------------------------------------------------------------------------ embeddings
def _per_pos(nseq):
    """Blocks per text position / grid cell of the embedding backwards (embed_bwd_per_pos): 1 at nseq <= 8, 32 from 249 on."""
    return max(1, min(math.ceil(nseq / 8), 32))


def _ln_rows(v, gamma, beta, src_terms, eps=1e-12):
    """float64 LayerNorm of the rows of v, the fp32 stats the kernel would store, and sum|terms| of y (src_terms: |addends| of v)."""
    mean = v.mean(1)
    rstd = 1.0 / torch.sqrt(((v - mean[:, None]) ** 2).mean(1) + eps)
    y = (v - mean[:, None]) * rstd[:, None] * gamma + beta
    terms = (src_terms + mean.abs()[:, None]) * rstd[:, None] * gamma.abs() + beta.abs()
    return y, mean, rstd, terms


def _ln_rows_bwd(dy, v, src_terms, stats32, gamma):
    """d v of the LayerNorm from the fp32 stats the kernel reads; sum|terms| of each element and of each row's x-hat."""
    mu, rs = stats32[:, 0].double()[:, None], stats32[:, 1].double()[:, None]
    xhat = (v - mu) * rs
    gy = dy * gamma
    d = rs * (gy - gy.mean(1, keepdim=True) - xhat * (gy * xhat).mean(1, keepdim=True))
    xt = (src_terms + mu.abs()) * rs
    terms = rs * (gy.abs() + gy.abs().mean(1, keepdim=True) + xt * (gy.abs() * xt).mean(1, keepdim=True))
    return d, xhat, xt, terms


def _check_table(kernel, got, pre, sums, abs_sums, elem_terms, depth):
    """fp32 table gradient: pre + sums, with depth * 2^-24 * (|pre| + sum|d|) for the additions and 32 * 2^-24 * sum|terms| for
    the rows being added."""
    return check_sum(kernel, got, pre.double() + sums, depth * (pre.double().abs() + abs_sums) + 32 * elem_terms, 1)


TEXT_CASES = [(1, 40, 0.0), (7, 40, 0.0), (7, 1, 0.0), (64, 40, 0.1), (320, 40, 0.0)]


@pytest.mark.parametrize("nseq,lt,p", TEXT_CASES, ids=["nseq%d-lt%d-p%g" % c for c in TEXT_CASES])
def test_embed_text(be_acc, nseq, lt, p):
    """cb_embed_text_fwd / _bwd / _bwd_det: per_pos 1 -> 32 (several rows per warp), ids 0 and vocab - 1, one id repeated in every
    sequence; the forward leaves the visual rows [lt, l) of out untouched; table gradients start random."""
    be = be_acc
    vocab, l, npos = 1000, lt + 9, lt + 3
    g = torch.Generator().manual_seed(nseq * 100 + lt)
    ids = torch.randint(0, vocab, (nseq, lt), generator=g)
    ids[0, 0], ids[-1, -1] = 0, vocab - 1
    ids[:, lt // 2] = 7                          # one word in every sequence: its table row gathers nseq rows
    word, pos, typ = torch.randn(vocab, HID, generator=g), torch.randn(npos, HID, generator=g), torch.randn(2, HID, generator=g)
    gamma, beta = torch.rand(HID, generator=g) + 0.5, torch.randn(HID, generator=g) * 0.1
    old = _bf16_sample(nseq * l * HID, 5).view(nseq * l, HID)
    out = Guarded((nseq * l, HID), BF16, be.dev, init=old)
    stats = Guarded((nseq * lt, 2), F32, be.dev)
    d = {k: t.to(be.dev) for k, t in dict(ids=ids, word=word, pos=pos, typ=typ, gamma=gamma, beta=beta).items()}
    seed = 99 + nseq
    with be.run():
        be.ops.embed_text_fwd(d["ids"], d["word"], d["pos"], d["typ"], d["gamma"], d["beta"], out.t, stats.t, nseq, lt, l, 1e-12, p, seed)
    out.check("embed_text_fwd out")
    stats.check("embed_text_fwd stats")
    got = out.t.cpu().view(nseq, l, HID)
    assert torch.equal(got[:, lt:].view(torch.int16), old.view(nseq, l, HID)[:, lt:].view(torch.int16)), "text launch wrote visual rows"
    w64, p64, t64 = word.double()[ids.reshape(-1)], pos.double()[:lt].repeat(nseq, 1), typ.double()[0]
    v = w64 + p64 + t64
    src = w64.abs() + p64.abs() + t64.abs()
    y, mean, rstd, terms = _ln_rows(v, gamma.double(), beta.double(), src)
    mult = torch.ones(nseq * lt, HID, dtype=F64) if not p else torch.from_numpy(
        D.multipliers(D.effective_seed(seed), D.embedding_index(nseq, l, range(lt)), p)).double().reshape(nseq * lt, HID)
    r = [check_bf16("embed_text_fwd out", got[:, :lt].reshape(-1, HID), y * mult, k=1, terms=terms * mult, c=32),
         check_sum("embed_text_fwd mean", stats.t[:, 0], mean, src.mean(1), 32),
         check_sum("embed_text_fwd rstd", stats.t[:, 1], rstd, rstd * (1.0 + mean.abs() * rstd), 32)]

    stats32 = torch.stack([mean, rstd], 1).float()
    dh = _bf16_sample(nseq * l * HID, 6).view(nseq * l, HID)
    pre = dict(word=torch.randn(vocab, HID, generator=g), pos=torch.randn(npos, HID, generator=g), typ=torch.randn(2, HID, generator=g),
               gamma=torch.randn(HID, generator=g), beta=torch.randn(HID, generator=g))
    gd = {k: Guarded(t.shape, F32, be.dev, init=t) for k, t in pre.items()}
    with be.run():
        be.ops.embed_text_bwd(dh.to(be.dev), d["ids"], d["word"], d["pos"], d["typ"], d["gamma"], stats32.to(be.dev), gd["word"].t,
                              gd["pos"].t, gd["typ"].t, gd["gamma"].t, gd["beta"].t, nseq, lt, l, p, seed)
    for k, t in gd.items():
        t.check("embed_text_bwd d" + k)
    dy = dh.double().view(nseq, l, HID)[:, :lt].reshape(-1, HID) * mult
    dv, xhat, xt, tdv = _ln_rows_bwd(dy, v, src, stats32, gamma.double())
    P = _per_pos(nseq)
    rows_per_block = math.ceil(nseq / P) + 4
    flat = ids.reshape(-1)
    cnt = torch.bincount(flat, minlength=vocab).double()[:, None]
    z = lambda n: torch.zeros(n, HID, dtype=F64)  # noqa: E731
    r.append(_check_table("embed_text_bwd dword", gd["word"].t, pre["word"], z(vocab).index_add_(0, flat, dv),
                          z(vocab).index_add_(0, flat, dv.abs()), z(vocab).index_add_(0, flat, tdv), cnt + 8))
    dpos = z(npos)
    dpos[:lt] = dv.view(nseq, lt, HID).sum(0)
    apos, tpos = z(npos), z(npos)
    apos[:lt], tpos[:lt] = dv.abs().view(nseq, lt, HID).sum(0), tdv.view(nseq, lt, HID).sum(0)
    r.append(_check_table("embed_text_bwd dpos", gd["pos"].t, pre["pos"], dpos, apos, tpos, rows_per_block + P + 8))
    all_depth = rows_per_block + P * lt + 8
    dt, at, tt = z(2), z(2), z(2)
    dt[0], at[0], tt[0] = dv.sum(0), dv.abs().sum(0), tdv.sum(0)
    r.append(_check_table("embed_text_bwd dtype0", gd["typ"].t, pre["typ"], dt, at, tt, all_depth))
    r.append(check_sum("embed_text_bwd dgamma", gd["gamma"].t, pre["gamma"].double() + (dy * xhat).sum(0),
                       all_depth * (pre["gamma"].double().abs() + (dy.abs() * xt).sum(0)), 1))
    r.append(check_sum("embed_text_bwd dbeta", gd["beta"].t, pre["beta"].double() + dy.sum(0),
                       all_depth * (pre["beta"].double().abs() + dy.abs().sum(0)), 1))
    _record("embed_text", "nseq%d-lt%d" % (nseq, lt), max(r))


VISUAL_CASES = [(1, 1, 3, 3, None, 0.0), (7, 2, 7, 7, [3, 1, 3], 0.1), (64, 4, 12, 12, "uniform16", 0.0), (320, 1, 3, 3, [1, 40, 7, 100, 2, 170], 0.0)]


@pytest.mark.parametrize("nseq,T,gh,gw,layout,p", VISUAL_CASES,
                         ids=["nseq%d-T%d-%dx%d-%s" % (n, T, a, b, "ragged" if isinstance(lay, list) else "uniform") for n, T, a, b, lay, _ in VISUAL_CASES])
def test_embed_visual(be_acc, nseq, T, gh, gw, layout, p):
    """cb_embed_visual_fwd / _bwd / _bwd_det: 1, 2 and 4 frames, 3x3 / 7x7 / 12x12 grids, uniform (n_ex) and ragged
    (seq2vid / vid_start) sequence-to-video maps; the forward leaves the text rows [0, lt) untouched; dgrid is the frame mean's
    gradient of each video's summed rows; table gradients start random."""
    be = be_acc
    lt, Lv = 5, gh * gw
    l = lt + Lv
    if isinstance(layout, list):
        counts, n_ex = layout, 0
    else:
        n_ex = 1 if layout is None else 16
        counts = [n_ex] * (nseq // n_ex)
    nvid = len(counts)
    vid = torch.repeat_interleave(torch.arange(nvid), torch.tensor(counts))
    vid_start = torch.tensor([0] + list(np.cumsum(counts)), dtype=torch.int32)
    g = torch.Generator().manual_seed(nseq * 10 + T)
    grid = (torch.randn(nvid, T, Lv, HID, generator=g)).to(BF16)
    row, col, typ = torch.randn(gh + 2, HID, generator=g), torch.randn(gw + 2, HID, generator=g), torch.randn(2, HID, generator=g)
    gamma, beta = torch.rand(HID, generator=g) + 0.5, torch.randn(HID, generator=g) * 0.1
    s2v = None if n_ex else vid.to(torch.int32).to(be.dev)
    vs = None if n_ex else vid_start.to(be.dev)
    old = _bf16_sample(nseq * l * HID, 15).view(nseq * l, HID)
    out = Guarded((nseq * l, HID), BF16, be.dev, init=old)
    stats = Guarded((nseq * Lv, 2), F32, be.dev)
    d = {k: t.to(be.dev) for k, t in dict(grid=grid, row=row, col=col, typ=typ, gamma=gamma, beta=beta).items()}
    seed = 77 + nseq
    with be.run():
        be.ops.embed_visual_fwd(d["grid"], s2v, n_ex, d["row"], d["col"], d["typ"], d["gamma"], d["beta"], out.t, stats.t, nseq, T, gh, gw,
                                lt, l, 1e-12, p, seed)
    out.check("embed_visual_fwd out")
    stats.check("embed_visual_fwd stats")
    got = out.t.cpu().view(nseq, l, HID)
    assert torch.equal(got[:, :lt].view(torch.int16), old.view(nseq, l, HID)[:, :lt].view(torch.int16)), "visual launch wrote text rows"
    j = torch.arange(Lv)
    g64 = grid.double()
    gm = g64.mean(1)[vid].reshape(nseq * Lv, HID)
    ga = g64.abs().mean(1)[vid].reshape(nseq * Lv, HID)
    r64, c64, t64 = row.double()[j // gw].repeat(nseq, 1), col.double()[j % gw].repeat(nseq, 1), typ.double()[0]
    v = gm + r64 + c64 + t64
    src = ga + r64.abs() + c64.abs() + t64.abs()
    y, mean, rstd, terms = _ln_rows(v, gamma.double(), beta.double(), src)
    mult = torch.ones(nseq * Lv, HID, dtype=F64) if not p else torch.from_numpy(
        D.multipliers(D.effective_seed(seed), D.embedding_index(nseq, l, range(lt, l)), p)).double().reshape(nseq * Lv, HID)
    r = [check_bf16("embed_visual_fwd out", got[:, lt:].reshape(-1, HID), y * mult, k=1, terms=terms * mult, c=32),
         check_sum("embed_visual_fwd mean", stats.t[:, 0], mean, src.mean(1), 32),
         check_sum("embed_visual_fwd rstd", stats.t[:, 1], rstd, rstd * (1.0 + mean.abs() * rstd), 32)]

    stats32 = torch.stack([mean, rstd], 1).float()
    dh = _bf16_sample(nseq * l * HID, 16).view(nseq * l, HID)
    pre = dict(row=torch.randn(gh + 2, HID, generator=g), col=torch.randn(gw + 2, HID, generator=g), typ=torch.randn(2, HID, generator=g),
               gamma=torch.randn(HID, generator=g), beta=torch.randn(HID, generator=g))
    gd = {k: Guarded(t.shape, F32, be.dev, init=t) for k, t in pre.items()}
    dv_tmp = Guarded((nseq * Lv, HID), F32, be.dev)
    dgrid = Guarded((nvid * T * Lv, HID), BF16, be.dev)
    with be.run():
        be.ops.embed_visual_bwd(dh.to(be.dev), d["grid"], s2v, vs, n_ex, d["row"], d["col"], d["typ"], d["gamma"], stats32.to(be.dev),
                                dv_tmp.t, dgrid.t, gd["row"].t, gd["col"].t, gd["typ"].t, gd["gamma"].t, gd["beta"].t, nseq, nvid, T,
                                gh, gw, lt, l, p, seed)
    for k, t in gd.items():
        t.check("embed_visual_bwd d" + k)
    dv_tmp.check("embed_visual_bwd dv_tmp")
    dgrid.check("embed_visual_bwd dgrid")
    dy = dh.double().view(nseq, l, HID)[:, lt:].reshape(-1, HID) * mult
    dv, xhat, xt, tdv = _ln_rows_bwd(dy, v, src, stats32, gamma.double())
    r.append(check_sum("embed_visual_bwd dv_tmp", dv_tmp.t, dv, tdv, 32))
    z = lambda *s: torch.zeros(*s, dtype=F64)  # noqa: E731
    per_vid = [z(nvid, Lv, HID).index_add_(0, vid, t.view(nseq, Lv, HID)) for t in (dv, dv.abs(), tdv)]
    cnt = torch.tensor(counts, dtype=F64)[:, None, None]
    ref_dg = (per_vid[0] / T)[:, None].expand(nvid, T, Lv, HID).reshape(-1, HID)
    t_dg = (((cnt + 2) * per_vid[1] + 32 * per_vid[2]) / T)[:, None].expand(nvid, T, Lv, HID).reshape(-1, HID)
    r.append(check_bf16("embed_visual_bwd dgrid", dgrid.t, ref_dg, k=1, terms=t_dg, c=1))
    P = _per_pos(nseq)
    rows_per_block = math.ceil(nseq / P) + 4
    cell = [t.view(nseq, Lv, HID).sum(0) for t in (dv, dv.abs(), tdv)]
    for name, idx, n_tab, per in (("row", j // gw, gh + 2, gw), ("col", j % gw, gw + 2, gh)):
        sums = [z(n_tab, HID).index_add_(0, idx, c_) for c_ in cell]
        r.append(_check_table("embed_visual_bwd d" + name, gd[name].t, pre[name], sums[0], sums[1], sums[2], rows_per_block + P * per + 8))
    all_depth = rows_per_block + P * Lv + 8
    dt, at, tt = z(2, HID), z(2, HID), z(2, HID)
    dt[0], at[0], tt[0] = dv.sum(0), dv.abs().sum(0), tdv.sum(0)
    r.append(_check_table("embed_visual_bwd dtype0", gd["typ"].t, pre["typ"], dt, at, tt, all_depth))
    r.append(check_sum("embed_visual_bwd dgamma", gd["gamma"].t, pre["gamma"].double() + (dy * xhat).sum(0),
                       all_depth * (pre["gamma"].double().abs() + (dy.abs() * xt).sum(0)), 1))
    r.append(check_sum("embed_visual_bwd dbeta", gd["beta"].t, pre["beta"].double() + dy.sum(0),
                       all_depth * (pre["beta"].double().abs() + dy.abs().sum(0)), 1))
    _record("embed_visual", "nseq%d-T%d-%dx%d" % (nseq, T, gh, gw), max(r))


# ------------------------------------------------------------------------------------------------ frame resize + pad
RESIZE_CASES = [(3, 1, 600, 1, 32, 32, torch.uint8), (3, 600, 1, 32, 1, 32, F32), (2, 3, 5, 19, 32, 32, F32),
                (3, 360, 640, 252, 448, 448, torch.uint8)]


@pytest.mark.parametrize("planes,h,w,nh,nw,S,dtype", RESIZE_CASES,
                         ids=["1x600-to-1x32-u8", "600x1-to-32x1-f32", "3x5-upscale-to-19x32-f32", "360x640-to-252x448-u8"])
def test_resize_pad(be, planes, h, w, nh, nw, S, dtype):
    """cb_resize_pad against float64 F.interpolate(bilinear, align_corners=False) + zero padding: extreme aspect ratios, a large
    upscale, max_size 32. The fp32 source coordinates carry a few 2^-24 * (h + w) of error into the interpolation weights,
    hence the bound; the padding must be exactly zero."""
    g = torch.Generator().manual_seed(h * w)
    x = torch.randint(0, 256, (planes, h, w), generator=g).to(dtype) if dtype == torch.uint8 else torch.randn(planes, h, w, generator=g) * 50
    y = Guarded((planes, S, S), F32, be.dev)
    with be.run():
        be.ops.resize_pad(x.to(be.dev), y.t, nh, nw)
    y.check("resize_pad")
    ref = torch.zeros(planes, S, S, dtype=F64)
    ref[:, :nh, :nw] = F.interpolate(x.double()[:, None], size=(nh, nw), mode="bilinear", align_corners=False)[:, 0]
    terms = torch.zeros(planes, S, S, dtype=F64)
    terms[:, :nh, :nw] = float(x.double().abs().max()) * (8 + 8 * (h + w))
    _record("resize_pad", "%dx%d-to-%dx%d" % (h, w, nh, nw), check_sum("resize_pad", y.t, ref, terms, 1))
