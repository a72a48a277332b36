"""Deterministic mode on CPU: the real engines (modeling.py, optim.py) run a training step with the library's entry points answered
by tests/ops_emulator.py, plus the restatement below of the deterministic entry points. With torch's flag set, every accumulating
call of the step must reach a deterministic entry point with scratch of at least the size the library's own query gives (the
queries are host code and run without a GPU), and no atomic entry point may be reached; with the flag clear, the step issues the
same calls as before. torch fills every torch.empty with NaN under the flag, so the bit equality of the two runs also shows that
no step reads memory nothing wrote."""
import contextlib

import pytest
import torch

import ops_emulator as E
import test_gpu_deterministic as G

CPU = torch.device("cpu")
# wrapper -> (deterministic entry point, the emulator's restatement of what it computes)
DET = {"layernorm_bwd": "layernorm_bwd_det", "embed_text_bwd": "embed_text_bwd_det", "embed_visual_bwd": "embed_visual_bwd_det",
       "colsum": "colsum_det", "clip_lse_loss": "clip_lse_loss_det", "clip_pool_ce_loss": "clip_pool_ce_loss_det"}


def _need(ops, name, args):
    """Scratch bytes the library asks for (its host-side queries)."""
    if name == "layernorm_bwd_det":
        return ops.layernorm_bwd_scratch_bytes(args[1].shape[0])
    if name == "embed_text_bwd_det":
        return ops.embed_text_bwd_scratch_bytes(args[12], args[13])
    if name == "embed_visual_bwd_det":
        return ops.embed_visual_bwd_scratch_bytes(args[17], args[20], args[21])
    if name == "colsum_det":
        return ops.colsum_scratch_bytes(args[2], args[3])
    return ops.clip_loss_scratch_bytes(args[5])


@contextlib.contextmanager
def emulated_deterministic_ops():
    from clipbert_b200 import ops, optim
    real = {n: getattr(ops, n) for n in list(DET) + ["gemm", "gemm_wgrad_group"]}
    real_sumsq = optim.sumsq
    saved = {n: getattr(ops, n) for n in list(DET.values()) + ["sumsq_det", "_launch_gemm", "_call", "set_deterministic"]}
    with E.emulated_ops() as calls:
        for n, f in real.items():            # the product's dispatching wrappers, not the emulator's stand-ins
            setattr(ops, n, f)
        optim.sumsq = real_sumsq
        det_calls = {n: 0 for n in list(DET.values()) + ["sumsq_det", "gemm_all", "gemm_wgrad", "gemm_wgrad_split"]}

        def restated(name, body):
            def f(*args):
                scratch = args[-1]
                assert scratch.dtype == torch.float32 and scratch.numel() * 4 >= _need(ops, name, args), name
                det_calls[name] += 1
                body(*args[:-1])
            return f
        for plain, name in DET.items():
            body = getattr(E, plain)
            if plain in ("layernorm_bwd", "embed_text_bwd", "embed_visual_bwd", "colsum"):
                setattr(ops, name, restated(name, body))
            else:
                setattr(ops, name, restated(name, lambda *a, _b=body: _b(*a)))

        def sumsq_det(x, n, chunks, nchunks, out, scratch):
            assert scratch.numel() * 4 >= ops.sumsq_scratch_bytes(n, chunks, nchunks)
            det_calls["sumsq_det"] += 1
            E.opt_sumsq(x, chunks, nchunks, out)
        ops.sumsq_det = sumsq_det

        def launch_gemm(name, kws):
            det_calls["gemm_all"] += len(kws)
            if kws[0].get("mode", 0) == 1:
                need = ops.gemm_workspace_bytes(kws[0]) if name == "cb_gemm" else ops.gemm_wgrad_group_workspace_bytes(kws)
                ws = kws[0].get("workspace")
                assert need == 0 or (ws is not None and ws.numel() * 4 >= need and kws[0]["workspace_bytes"] >= need), (name, need)
                det_calls["gemm_wgrad"] += len(kws)
                det_calls["gemm_wgrad_split"] += need > 0
            for kw in kws:
                E.gemm(**{k: v for k, v in kw.items() if k not in ("workspace", "workspace_bytes")})
        ops._launch_gemm = launch_gemm

        def no_native(name, *a):
            raise AssertionError("%s reached the native library in an emulated deterministic step" % name)
        ops._call = no_native
        ops.set_deterministic = lambda on: False
        try:
            yield calls, det_calls
        finally:
            for n, f in saved.items():
                setattr(ops, n, f)
            ops._lib_deterministic = False


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)


def _step(weights):
    """transformer forward + backward (dropout 0.1) and the clipped optimizer step -> loss, gradients, parameters, moments"""
    from clipbert_b200.optim import FusedAdamW
    from test_gpu_optim import e2e_param_groups
    torch.manual_seed(0)
    model = G._retrieval_transformer(weights, CPU)
    opt = FusedAdamW([g for g in e2e_param_groups(model) if g["params"]], lr=5e-5, betas=(0.9, 0.98), model=model)
    loss, grad, dgrid = (t.clone() for t in G._transformer_step(model, CPU, gh=2, lt=9))
    norm = opt.clip_grad_norm(1.0).clone()
    opt.step()
    h = opt._plan[0]
    return [loss, grad, dgrid, norm, h["flat"].master.clone(), h["exp_avg"].clone(), h["exp_avg_sq"].clone()]


def test_flag_routes_every_accumulation_through_deterministic_entry_points(weights):
    with E.emulated_ops() as calls:
        plain = _step(weights)
        before = dict(calls)
    with G.deterministic():
        with emulated_deterministic_ops() as (calls, det_calls):
            det = _step(weights)
            after = dict(calls)
    # each accumulating call went to its deterministic entry point, with the scratch the library asks for
    for wrapper, name in DET.items():
        assert det_calls[name] == before[wrapper], (wrapper, det_calls[name], before[wrapper])
    assert det_calls["layernorm_bwd_det"] > 0 and det_calls["colsum_det"] > 0 and det_calls["embed_text_bwd_det"] == 1
    assert det_calls["sumsq_det"] >= 1 and det_calls["gemm_wgrad"] > 0
    # non-accumulating calls are unchanged
    assert det_calls["gemm_all"] == before["gemm"]
    for n in ("layernorm_fwd", "attention_fwd", "attention_bwd", "embed_text_fwd", "embed_visual_fwd", "pad_cast"):
        assert after[n] == before[n], n
    # the restated entry points compute what the plain ones do, and nothing read torch's NaN-filled uninitialised memory
    for a, b in zip(plain, det):
        assert torch.equal(a, b)
        assert bool(torch.isfinite(b).all())


def test_flag_clear_keeps_the_call_sequence():
    """With the flag clear the wrappers never consult the deterministic entry points (nothing from the library is reachable on
    CPU, so any such call would raise)."""
    from clipbert_b200 import ops
    assert not torch.are_deterministic_algorithms_enabled()
    recorded = []
    saved = ops._call, ops._s
    ops._call, ops._s = (lambda name, *a: recorded.append(name)), (lambda: None)
    try:
        x = torch.zeros(16, 8, dtype=torch.bfloat16)
        out = torch.zeros(8)
        ops.colsum(x, out, 16, 8)
        ops.layernorm_bwd(x, x, torch.zeros(16, 2), out, x, None, out, out, None, 0.0, 0)
        ops.clip_lse_loss(out, out, out, None, 1, 1, 8)
    finally:
        ops._call, ops._s = saved
    assert recorded == ["cb_colsum", "cb_layernorm_bwd", "cb_clip_lse_loss"]
