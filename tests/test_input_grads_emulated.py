"""Frame gradients on CPU: cb_maxpool3x3s2_bwd and cb_stem_dgrad restated in torch below, the float64 references and bounds of
tests/test_gpu_input_grads.py checked against deliberately wrong results, the entry points' argument checks, and the module and
end-to-end cases of that file that fit a CPU replayed with the C-ABI calls answered by tests/ops_emulator.py plus these two
restatements."""
import contextlib
import ctypes

import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input

import ops_emulator as E
import test_gpu_input_grads as IG
from elementwise import BF16, F64, check_bound

CPU = torch.device("cpu")


# ------------------------------------------------------------------------------------------------ restatements
def maxpool3x3s2_bwd(dy, x, dx, n, h, w, c, row_pitch=None, img_pitch=None):
    """The header's cb_maxpool3x3s2_bwd[_strided]: the gradients of the windows whose arg-max (F.max_pool2d's: first maximum,
    last NaN) is the element, summed, kept where x > 0."""
    row_pitch = w if row_pitch is None else row_pitch
    img_pitch = h * w if img_pitch is None else img_pitch
    xv = torch.as_strided(x, (n, h, w, c), (img_pitch * c, row_pitch * c, c, 1), x.storage_offset())
    v, _ = IG.pool_bwd_ref(dy.view(n, (h - 1) // 2 + 1, (w - 1) // 2 + 1, c), xv)
    dx.view(-1).copy_(v.reshape(-1))


def stem_dgrad(dc1, w, dx, n, h, wimg):
    """The header's cb_stem_dgrad: the 7x7/s2/p3 input gradient of the BGR frames from dc1 and the stem operand, in RGB order."""
    v, _ = IG.stem_dgrad_ref(dc1, w, n, h, wimg)
    dx.copy_(v)


@contextlib.contextmanager
def emulated_ops():
    from clipbert_b200 import ops
    with E.emulated_ops() as calls:
        saved = {k: getattr(ops, k) for k in ("maxpool3x3s2_bwd", "stem_dgrad")}

        def counted(name, fn):
            calls[name] = 0

            def f(*a, **k):
                calls[name] += 1
                return fn(*a, **k)
            return f
        ops.maxpool3x3s2_bwd = counted("maxpool3x3s2_bwd", maxpool3x3s2_bwd)
        ops.stem_dgrad = counted("stem_dgrad", stem_dgrad)
        try:
            yield calls
        finally:
            for k, f in saved.items():
                setattr(ops, k, f)


# ------------------------------------------------------------------------------------------------ references and faults
def _pool_case(size=97, n=2, nan=False):
    h = IG._conv_out(size)
    dy, x = IG.pool_inputs(n, h, h, seed=size)
    if not nan:
        x = torch.where(torch.isnan(x), torch.zeros_like(x), x)
    ref, bound = IG.pool_bwd_ref(dy, x)
    return dy, x, ref, bound


def _pool_windows(dy, x, last_max=False, relu=True):
    """A gather-form restatement with a selectable tie rule (no NaN in x): the window's first or last maximum gets its gradient."""
    x64 = x.double().permute(0, 3, 1, 2)
    n, c, h, w = x64.shape
    cols = F.unfold(F.pad(x64, (1, 1, 1, 1), value=float("-inf")), 3, stride=2).view(n, c, 9, -1)
    k = 8 - cols.flip(2).argmax(2) if last_max else cols.argmax(2)          # window-local (r, s) of the winner
    wo = (w - 1) // 2 + 1
    oy, ox = torch.arange(k.shape[-1]) // wo, torch.arange(k.shape[-1]) % wo
    iy, ix = 2 * oy - 1 + k // 3, 2 * ox - 1 + k % 3
    out = torch.zeros(n, c, h * w, dtype=F64).scatter_add_(2, iy * w + ix, dy.double().permute(0, 3, 1, 2).flatten(2)).view(n, c, h, w)
    if relu:
        out = torch.where(x64 > 0, out, torch.zeros_like(out))
    return out.permute(0, 2, 3, 1).to(BF16)


def test_pool_reference_accepts_the_restatements():
    """The first-maximum gather restatement and the emulator's restatement pass the bound (NaN, ties, -0, zero windows)."""
    dy, x, ref, bound = _pool_case()
    check_bound("pool first-max", _pool_windows(dy, x), ref, bound)
    dy, x, ref, bound = _pool_case(nan=True)
    n, h = x.shape[0], x.shape[1]
    out = torch.empty(n * h * h, 64, dtype=BF16)
    maxpool3x3s2_bwd(dy, x, out, n, h, h, 64)
    check_bound("pool emulated", out.view(x.shape), ref, bound)
    assert bool((bound == 0).any()) and bool((bound > 0).any())


def test_fault_last_maximum_tie_rule_is_rejected():
    dy, x, ref, bound = _pool_case()
    with pytest.raises(AssertionError, match="out of bound"):
        check_bound("fault", _pool_windows(dy, x, last_max=True), ref, bound)


def test_fault_missing_relu_derivative_is_rejected():
    dy, x, ref, bound = _pool_case()
    with pytest.raises(AssertionError, match="out of bound"):
        check_bound("fault", _pool_windows(dy, x, relu=False), ref, bound)


def _stem_operand(std):
    with E.emulated_ops():
        return IG.stem_operand(CPU, IG.PIXEL_STD if std else None)


def _stem_case(size=97, n=1, std=True):
    w = _stem_operand(std)
    ho = IG._conv_out(size)
    dc1 = IG.dc1_input(n, ho, ho, seed=size)
    ref, bound = IG.stem_dgrad_ref(dc1, w, n, size, size)
    return dc1, w, ref, bound


def test_stem_reference_accepts_the_restatement_and_matches_autograd():
    """The restatement rounded to fp32 passes; the reference is float64 autograd of <conv2d(x_bgr, w, 2, 3), dc1> w.r.t. RGB x."""
    dc1, w, ref, bound = _stem_case()
    out = torch.empty(1, 3, 97, 97)
    stem_dgrad(dc1, w, out, 1, 97, 97)
    check_bound("stem emulated", out, ref, bound)
    x = torch.zeros(1, 3, 97, 97, dtype=F64, requires_grad=True)
    with torch.enable_grad():
        y = F.conv2d(x[:, [2, 1, 0]], IG.stem_weight64(w), stride=2, padding=3)
        (y * dc1.double().view(1, 49, 49, 64).permute(0, 3, 1, 2)).sum().backward()
    assert torch.allclose(x.grad, ref, rtol=1e-12, atol=1e-12)


def test_fault_bgr_not_undone_is_rejected():
    dc1, w, ref, bound = _stem_case()
    with pytest.raises(AssertionError, match="out of bound"):
        check_bound("fault", ref[:, [2, 1, 0]].float(), ref, bound)


def test_fault_missing_std_fold_is_rejected():
    dc1, w, ref, bound = _stem_case(std=True)
    bad, _ = IG.stem_dgrad_ref(dc1, _stem_operand(False), 1, 97, 97)
    with pytest.raises(AssertionError, match="out of bound"):
        check_bound("fault", bad.float(), ref, bound)


def test_fault_stride_phase_off_by_one_is_rejected():
    """Each output column takes the taps of the next one (x + 1: the other stride phase)."""
    dc1, w, ref, bound = _stem_case(std=False)
    bad = torch.zeros_like(ref)
    bad[..., :-1] = ref[..., 1:]
    with pytest.raises(AssertionError, match="out of bound"):
        check_bound("fault", bad.float(), ref, bound)
    ok = conv2d_input((1, 3, 97, 97), IG.stem_weight64(w), dc1.double().view(1, 49, 49, 64).permute(0, 3, 1, 2), stride=2, padding=3)
    check_bound("phase", ok[:, [2, 1, 0]].float(), ref, bound)


# ------------------------------------------------------------------------------------------------ argument checks
def _status(name, *args):
    from clipbert_b200 import _lib as L, ops
    n0 = ops.launch_count()
    rc = ops._fn(name)(*args)
    assert rc != 0 and name.replace("_strided", "") in L.lib().cb_last_error().decode()
    assert ops.launch_count() == n0


def test_maxpool3x3s2_bwd_rejects_bad_arguments():
    _status("cb_maxpool3x3s2_bwd", 16, 16, 16, 2, 8, 8, 12, None)                 # c not a multiple of 8


def test_maxpool3x3s2_bwd_strided_rejects_bad_arguments():
    _status("cb_maxpool3x3s2_bwd_strided", 16, 16, 16, 2, 8, 8, 64, 7, 64, None)   # row pitch below the width


def test_stem_dgrad_rejects_bad_arguments():
    _status("cb_stem_dgrad", 16, 16, 100, ctypes.c_void_p(16), 1, 32, 32, None)     # w_ld below the 147 taps


# ------------------------------------------------------------------------------------------------ module and end-to-end replays
EMU_MODULE_CASES = [IG.ModuleCase(1, 2, 64), IG.ModuleCase(1, 1, 66, "im2col", 1, "raw"), IG.ModuleCase(1, 2, 64, "s2d16", 3, "bf16")]


@pytest.fixture(scope="module")
def cnn_sd():
    from oracle import synth
    return synth.cnn_state_dict(42)


@pytest.mark.parametrize("case", EMU_MODULE_CASES, ids=[c.id for c in EMU_MODULE_CASES])
def test_backbone_frame_gradient_matches_oracle_on_emulated_ops(cnn_sd, case):
    with emulated_ops() as calls:
        IG.run_module_against_oracle(CPU, case, cnn_sd)
    assert calls["maxpool3x3s2_bwd"] == 1 and calls["stem_dgrad"] == 1


def test_parameter_gradients_unchanged_on_emulated_ops(cnn_sd):
    with emulated_ops():
        IG.run_parameter_gradients_unchanged(CPU, cnn_sd, size=64)


@pytest.fixture(scope="module")
def full_sd():
    from oracle import synth
    return synth.full_state_dict(42)


@pytest.mark.parametrize("path,frozen", [("forward", "all"), ("forward_clips", "cnn"), ("encode_clips", "all")])
def test_clipbert_frame_gradient_matches_oracle_on_emulated_ops(full_sd, path, frozen):
    with emulated_ops() as calls:
        IG.run_e2e_against_oracle(CPU, full_sd, path, frozen, size=64, frames=1, videos=1)
    assert calls["stem_dgrad"] == 1
