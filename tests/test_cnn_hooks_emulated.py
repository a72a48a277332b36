"""GridFeatBackbone's module path (hooks on the CNN's modules) on a CPU: the model-level runners of tests/test_gpu_cnn_hooks.py
replayed with the C-ABI calls answered by tests/ops_emulator.py, plus restatements of the two new entry points kept here
(cb_nhwc_intake, and cb_unsubsample2_mask with act = NULL), so the shared emulator is unchanged. Planted faults in those
restatements must make the checks fail."""
import contextlib

import pytest
import torch

import ops_emulator as E
import test_gpu_cnn_hooks as H
import test_input_grads_emulated as IGE

CPU = torch.device("cpu")
SIZE = 64


def unsubsample2_mask(dsub, act, dx, n, h, w, c):
    if act is not None:
        return E.unsubsample2_mask(dsub, act, dx, n, h, w, c)
    H.unsubsample2_ref(dsub, act, dx, n, h, w, c)


@contextlib.contextmanager
def emulated_ops(intake=H.intake_ref, unsub=unsubsample2_mask):
    from clipbert_b200 import ops
    with IGE.emulated_ops() as calls:
        saved = {k: getattr(ops, k) for k in ("nhwc_intake", "unsubsample2_mask")}
        calls["nhwc_intake"] = 0

        def counted(*a, **k):
            calls["nhwc_intake"] += 1
            return intake(*a, **k)
        ops.nhwc_intake, ops.unsubsample2_mask = counted, unsub
        try:
            yield calls
        finally:
            for k, f in saved.items():
                setattr(ops, k, f)


@pytest.fixture(scope="module")
def cnn_sd():
    from oracle import synth
    return synth.cnn_state_dict(42)


# ------------------------------------------------------------------------------------------------ the restatement itself
@pytest.mark.parametrize("layout", H.INTAKE_LAYOUTS)
@pytest.mark.parametrize("bordered", [False, True], ids=["compact", "bordered"])
def test_intake_reference_accepts_itself(layout, bordered):
    H.run_intake_case(CPU, layout, torch.float32, bordered, True, impl=H.intake_ref)


def _fault_border(x, out, act=None, out_bordered=False, act_bordered=False):
    H.intake_ref(x, out, act, out_bordered, act_bordered)
    if out_bordered:
        out.view(x.shape[0], x.shape[2] + 2, x.shape[3] + 2, -1)[:, 0] = 1.0


def _fault_no_mask(x, out, act=None, out_bordered=False, act_bordered=False):
    H.intake_ref(x, out, None, out_bordered, act_bordered)


def _fault_mask_twice(x, out, act=None, out_bordered=False, act_bordered=False):
    """The mask applied twice, the second time against the wrong (compact-vs-bordered) rows."""
    H.intake_ref(x, out, act, out_bordered, act_bordered)
    if act is not None:
        n, c, h, w = x.shape
        a = act.view(-1)[: n * h * w * c].view(n, h, w, c).permute(0, 3, 1, 2)
        H.intake_ref(torch.where(a > 0, x, torch.zeros_like(x)), out, act, out_bordered, act_bordered)


@pytest.mark.parametrize("fault", [_fault_border, _fault_no_mask, _fault_mask_twice])
def test_intake_check_rejects_faults(fault):
    with pytest.raises(AssertionError):
        H.run_intake_case(CPU, "channels_last", torch.float32, True, True, impl=fault)


# ------------------------------------------------------------------------------------------------ module path replays
def test_hook_outputs_and_gradients_match_oracle(cnn_sd):
    with emulated_ops() as calls:
        H.run_against_oracle(CPU, cnn_sd, SIZE, 2, True)
    assert calls["nhwc_intake"] == 16          # one masked intake per block on the module path


@pytest.mark.parametrize("freeze_at,frames_grad", [(2, True), (3, False)])
def test_observe_only_hooks_leave_gradients_bit_identical(cnn_sd, freeze_at, frames_grad):
    with emulated_ops():
        H.run_observe_only_bits(CPU, cnn_sd, SIZE, freeze_at, frames_grad, runs=1)


def test_requires_grad_rule(cnn_sd):
    for freeze_at in (1, 2, 3):
        for frames_grad in (False, True):
            m = H.backbone(CPU, cnn_sd, freeze_at)
            store, handles = H.observe(m)
            with emulated_ops():
                m(H.frames(CPU, SIZE, n_frms=1).requires_grad_(frames_grad))
            for name in H.SITES:
                assert store["rg"][name] == H.required(name, freeze_at, frames_grad), (freeze_at, frames_grad, name)


def test_outputs_are_engine_activations(cnn_sd):
    with emulated_ops():
        H.run_outputs_are_engine_activations(CPU, cnn_sd, SIZE)


def test_interventions_match_oracle(cnn_sd):
    with emulated_ops():
        H.run_interventions(CPU, cnn_sd, SIZE)


def test_semantics(cnn_sd):
    with emulated_ops():
        H.run_semantics(CPU, cnn_sd, SIZE)


def test_refusals(cnn_sd):
    with emulated_ops():
        H.run_refusals(CPU, cnn_sd)


def test_no_hooks_no_module_path(cnn_sd):
    """Without a hook the default path runs: no intake, no mask-free scatter."""
    m = H.backbone(CPU, cnn_sd)
    with emulated_ops() as calls:
        m(H.frames(CPU, SIZE, n_frms=1).requires_grad_(True)).float().sum().backward()
    assert calls["nhwc_intake"] == 0


# ------------------------------------------------------------------------------------------------ planted faults
def _ignore_replacement(x, out, act=None, out_bordered=False, act_bordered=False):
    """A replaced output ignored: the intake of a forward replacement (no mask) writes nothing."""
    if act is not None:
        H.intake_ref(x, out, act, out_bordered, act_bordered)


def _ignore_hook_gradient(x, out, act=None, out_bordered=False, act_bordered=False):
    """A hook's gradient ignored: a masked intake of a rewritten gradient sees its zeroed channels restored to ones."""
    x = torch.where(x == 0, torch.ones_like(x), x) if act is not None else x
    H.intake_ref(x, out, act, out_bordered, act_bordered)


def _masked_unsubsample(dsub, act, dx, n, h, w, c):
    """The mask-free scatter masked anyway (by a pattern that is not the producing block's ReLU')."""
    if act is not None:
        return E.unsubsample2_mask(dsub, act, dx, n, h, w, c)
    H.unsubsample2_ref(dsub, None, dx, n, h, w, c)
    dx.view(n, h, w, c)[:, :, ::2] = 0


@pytest.mark.parametrize("runner,kw", [
    ("bits", dict(intake=_fault_no_mask)),
    ("bits", dict(intake=_fault_mask_twice)),
    ("bits", dict(unsub=_masked_unsubsample)),
    ("interventions", dict(intake=_ignore_replacement)),
    ("interventions", dict(intake=_ignore_hook_gradient)),
    ("interventions", dict(intake=_fault_border)),
], ids=["mask-missing", "mask-twice", "scatter-masked", "replacement-ignored", "hook-gradient-ignored", "border-written"])
def test_module_path_checks_reject_faults(cnn_sd, runner, kw):
    with emulated_ops(**kw), pytest.raises((AssertionError, RuntimeError)):
        if runner == "bits":
            H.run_observe_only_bits(CPU, cnn_sd, SIZE, 2, True, runs=1)
        else:
            H.run_interventions(CPU, cnn_sd, SIZE)
