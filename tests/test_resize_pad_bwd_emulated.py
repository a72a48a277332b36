"""Gradients through the input stage on the CPU: input_stage.resize_pad as an autograd op on the emulated entry points
(tests/ops_emulator.py, plus cb_resize_pad_bwd restated below as F.interpolate's own backward) against float64 autograd, an
end-to-end replay from decoded frames, and the references and bounds of tests/test_gpu_resize_pad_bwd.py checked against
deliberately wrong adjoints: an edge clamp dropped, the pad region leaking gradient, the x and y weights swapped and a
half-pixel offset."""
import contextlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import ops_emulator as E
import test_gpu_resize_pad_bwd as RB
import test_input_grads_emulated as IGE
from elementwise import F32, check_bound

CPU = torch.device("cpu")


# ------------------------------------------------------------------------------------------------ restatement
def resize_pad_bwd(dy, dx, new_h, new_w, accumulate=False):
    """The header's cb_resize_pad_bwd: the adjoint of the emulator's resize_pad (F.interpolate's own backward); the pad region
    of dy contributes nothing."""
    h, w, s = dx.shape[-2], dx.shape[-1], dy.shape[-1]
    x = torch.zeros(dx.numel() // (h * w), 1, h, w, dtype=F32, requires_grad=True)
    with torch.enable_grad():
        r = F.interpolate(x, size=(new_h, new_w), mode="bilinear", align_corners=False)
        (g,) = torch.autograd.grad(r, x, dy.reshape(-1, 1, s, s)[:, :, :new_h, :new_w].float())
    if accumulate:
        dx.add_(g.view(dx.shape))
    else:
        dx.copy_(g.view(dx.shape))


@contextlib.contextmanager
def emulated_input_stage(ops_context=E.emulated_ops):
    """The emulated ops with the restatement above counted in calls["resize_pad_bwd"], and input_stage's device check lifted
    (as the emulator does for modeling / grid_feat)."""
    from clipbert_b200 import input_stage, ops
    with ops_context() as calls:
        saved = input_stage._require_cuda, ops.resize_pad_bwd
        calls["resize_pad_bwd"] = 0

        def counted(*a, **k):
            calls["resize_pad_bwd"] += 1
            return resize_pad_bwd(*a, **k)
        ops.resize_pad_bwd = counted
        input_stage._require_cuda = lambda t: None
        try:
            yield calls
        finally:
            input_stage._require_cuda, ops.resize_pad_bwd = saved


def _fits(c):
    from clipbert_b200.input_stage import get_resize_size
    return (c.nh, c.nw) == get_resize_size(c.h, c.w, c.s) and c.h * c.w <= 1500 * 1500


OP_CASES = [c for c in RB.KERNEL_CASES if _fits(c)] + [RB._fit(2, 1, 17, 41, "1xN"), RB._fit(2, 37, 53, 47, "odd-S"),
                                                       RB._fit(1, 1, 1, 9, "1x1")]


@pytest.mark.parametrize("case", OP_CASES, ids=[c.id for c in OP_CASES])
def test_autograd_op_on_emulated_ops_matches_float64_autograd(case):
    from clipbert_b200 import input_stage
    g = torch.Generator().manual_seed(case.w)
    x = (torch.rand(1, case.planes, case.h, case.w, generator=g) * 255).requires_grad_(True)
    dy = torch.randn(1, case.planes, case.s, case.s, generator=g)
    with emulated_input_stage() as calls:
        out = input_stage.resize_pad(x, case.s)
        (dx,) = torch.autograd.grad(out, x, dy)
        with torch.no_grad():
            input_stage.resize_pad(x, case.s)
        input_stage.resize_pad(x.detach(), case.s)
    assert calls["resize_pad"] == 3 and calls["resize_pad_bwd"] == 1
    assert dx.shape == x.shape and dx.dtype == F32
    ref, bound = RB.interp_ref(dy[0], case.h, case.w, case.nh, case.nw)
    check_bound("emulated resize_pad backward " + case.id, dx[0], ref, bound)


def test_emulated_entry_point_accumulates():
    case = RB.Case(2, 13, 17, 117, 40, 128, "up9-x2.4")
    dy = RB._dy(case, 1)
    dx0 = torch.randn(case.planes, case.h, case.w)
    dx = dx0.clone()
    resize_pad_bwd(dy, dx, case.nh, case.nw, accumulate=True)
    ref, bound = RB.interp_ref(dy, case.h, case.w, case.nh, case.nw)
    check_bound("emulated accumulate", dx, ref + dx0.double(), bound + 2.0 ** -24 * (ref.abs() + dx0.double().abs()))


# ------------------------------------------------------------------------------------------------ references and faults
FAULT_CASE = RB.Case(2, 13, 17, 117, 40, 128, "up9-x2.4")        # upscales: both edge rules matter; sh != sw; a pad region


def adjoint(dy, case, clamp=True, merge=True, half_pixel=True, swap=False, leak=False):
    """R^T dy from the float64 tap matrices, with the planted faults, rounded to fp32 like the kernel's output."""
    sy, sx = np.float32(case.h) / np.float32(case.nh), np.float32(case.w) / np.float32(case.nw)
    if swap:
        sy, sx = sx, sy
    e = 1 if leak else 0            # one pad row and column take part, with the taps their index would have
    kw = dict(clamp=clamp, merge=merge, half_pixel=half_pixel)
    my, mx = RB.taps64(case.nh + e, case.h, scale=sy, **kw), RB.taps64(case.nw + e, case.w, scale=sx, **kw)
    return (my.t() @ dy.double()[:, :case.nh + e, :case.nw + e] @ mx).float()


def test_references_accept_the_exact_adjoint_and_agree():
    dy = RB._dy(FAULT_CASE, 2)
    ref, bound = RB.adjoint_ref(dy, FAULT_CASE.h, FAULT_CASE.w, FAULT_CASE.nh, FAULT_CASE.nw)
    check_bound("exact adjoint", adjoint(dy, FAULT_CASE), ref, bound)
    g, gb = RB.interp_ref(dy, FAULT_CASE.h, FAULT_CASE.w, FAULT_CASE.nh, FAULT_CASE.nw)
    check_bound("exact adjoint vs F.interpolate", adjoint(dy, FAULT_CASE), g, gb)
    # the matrices of the fp32 taps and of float64 F.interpolate differ only by the taps' rounding
    assert float((ref - g).abs().max()) < 1e-3 * float(g.abs().max())


@pytest.mark.parametrize("fault", [dict(clamp=False), dict(merge=False), dict(leak=True), dict(swap=True), dict(half_pixel=False)],
                         ids=["top-left-clamp-dropped", "bottom-right-merge-dropped", "pad-region-leaks", "x-y-swapped",
                              "half-pixel-offset"])
def test_planted_fault_fails_the_bound(fault):
    dy = RB._dy(FAULT_CASE, 2)
    bad = adjoint(dy, FAULT_CASE, **fault)
    ref, bound = RB.adjoint_ref(dy, FAULT_CASE.h, FAULT_CASE.w, FAULT_CASE.nh, FAULT_CASE.nw)
    with pytest.raises(AssertionError, match="out of bound"):
        check_bound("fault", bad, ref, bound)
    g, gb = RB.interp_ref(dy, FAULT_CASE.h, FAULT_CASE.w, FAULT_CASE.nh, FAULT_CASE.nw)
    with pytest.raises(AssertionError, match="out of bound"):
        check_bound("fault", bad, g, gb)


# ------------------------------------------------------------------------------------------------ end to end
@pytest.fixture(scope="module")
def full_sd():
    from oracle import synth
    return synth.full_state_dict(42)


@pytest.mark.parametrize("path,frozen", [("forward", "all"), ("encode_clips", "all")])
def test_decoded_frame_gradient_matches_oracle_on_emulated_ops(full_sd, path, frozen):
    with emulated_input_stage(IGE.emulated_ops) as calls:
        RB.run_e2e(CPU, full_sd, path, frozen, h=40, w=50, size=64, frames=1, videos=1)
    assert calls["resize_pad"] == 1 and calls["resize_pad_bwd"] == 1 and calls["stem_dgrad"] == 1
