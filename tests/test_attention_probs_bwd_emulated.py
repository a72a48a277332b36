"""cb_attention_probs_bwd on CPU: the float64 reference and its per-element bound of tests/test_gpu_attention_probs_bwd.py
checked against autograd and against deliberately wrong results, and the module tests of that file replayed with the C-ABI
calls answered by tests/ops_emulator.py, ops.attention_probs by tests/test_base_model_emulated.py and ops.attention_probs_bwd by
the float64 restatement below."""
import contextlib
import math

import numpy as np
import pytest
import torch

import dropout_ref as D
import ops_emulator
import test_base_model_emulated as BE
import test_gpu_attention_elementwise as A
import test_gpu_attention_probs_bwd as PB
from elementwise import F64, check_bound, rne_bf16
from util import relerr

CPU = torch.device("cpu")


def attention_probs_bwd(qkv, text_mask, lse, dprobs, drow, dqkv, nseq, l, lt, heads, p, seed):
    """The header's cb_attention_probs_bwd in float64: P from the GIVEN lse, g = r G, D = sum P g (written to drow),
    dS = P (g - D); dQ += dS K / 8 and dK += dS^T Q / 8 added into dqkv's Q and K blocks, V untouched."""
    q, k, _, s = ops_emulator._attention_scores(qkv, text_mask, nseq, l, lt, heads)
    pr = torch.exp(s - lse.double()[..., None])
    mult = ops_emulator._drop_mult(p, seed, D.attention_index(nseq, heads, l))
    g = dprobs.double() if mult is None else dprobs.double() * mult.double()
    dv = (pr * g).sum(-1, keepdim=True)
    drow.view(nseq, heads, l).copy_(dv.squeeze(-1))
    ds = pr * (g - dv)
    scale = 1.0 / math.sqrt(q.shape[-1])
    blocks = dqkv.view(nseq, l, 3, -1)
    for j, grad in ((0, ds @ k * scale), (1, ds.transpose(-1, -2) @ q * scale)):
        blocks[:, :, j].copy_(blocks[:, :, j].double() + grad.permute(0, 2, 1, 3).reshape(nseq, l, -1))


@contextlib.contextmanager
def emulated_ops():
    from clipbert_b200 import ops
    with BE.emulated_ops() as calls:
        saved = ops.attention_probs_bwd
        calls["attention_probs_bwd"] = 0

        def counted(*a, **k):
            calls["attention_probs_bwd"] += 1
            return attention_probs_bwd(*a, **k)
        ops.attention_probs_bwd = counted
        try:
            yield calls
        finally:
            ops.attention_probs_bwd = saved


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)


# ------------------------------------------------------------------------------------------------ reference and bound
def _setup(L=65, heads=2, p=0.1, seed=99):
    n = A.NSEQ
    lt = L - 9
    g = torch.Generator().manual_seed(L)
    qkv = torch.randn(n * L, 3 * heads * 64, generator=g, dtype=F64).to(torch.bfloat16)
    mask = A._mask(L, lt)
    q, k, _ = A._split(qkv, heads)
    madd = A._madd(mask, L, lt)
    lse = torch.logsumexp(q @ k.transpose(-1, -2) / 8.0 + madd[:, None, None, :], -1).float()
    idx = D.attention_index(n, heads, L)
    r = torch.from_numpy(D.multipliers(D.effective_seed(seed), idx, p)).double()
    Gr = torch.randn(n, heads, L, L, generator=g, dtype=F64).float().double()
    dq0, dk0 = ((torch.randn(n, heads, L, 64, generator=g, dtype=F64) * 0.05).to(torch.bfloat16).double() for _ in range(2))
    ref = PB.probs_bwd_ref(q, k, madd, lse, r, Gr, dq0, dk0)
    return dict(q=q, k=k, madd=madd, lse=lse, r=r, G=Gr, dq0=dq0, dk0=dk0, ref=ref, idx=idx, seed=seed, p=p, L=L)


def _ok(s, grads):
    for name, (got, _), (ref, bound) in zip(("dq", "dk"), grads, s["ref"]):
        check_bound("fault " + name, rne_bf16(got), ref, bound)


def _faulty(s, **over):
    a = dict(s, **over)
    return PB.probs_bwd_ref(a["q"], a["k"], a["madd"], a["lse"], a["r"], a["G"], a["dq0"], a["dk0"])


def test_reference_accepts_itself_and_matches_autograd():
    """The reference rounded once to bf16 passes its own bound; without the bf16 rounding of dS its increment equals float64
    autograd of sum(A G) with A = softmax(Q K^T / 8 + madd) r."""
    s = _setup()
    _ok(s, s["ref"])
    q, k = (t.clone().requires_grad_(True) for t in (s["q"], s["k"]))
    with torch.enable_grad():
        a = torch.softmax(q @ k.transpose(-1, -2) / 8.0 + s["madd"][:, None, None, :], -1) * s["r"]
        (a * s["G"]).sum().backward()
    pr = torch.exp(s["q"] @ s["k"].transpose(-1, -2) / 8.0 + s["madd"][:, None, None, :] - s["lse"].double()[..., None])
    g = s["r"] * s["G"]
    ds = pr * (g - (pr * g).sum(-1, keepdim=True))
    # the float32 lse makes P differ from softmax by ~1e-7 relative
    assert torch.allclose(ds @ s["k"] / 8.0, q.grad, rtol=1e-5, atol=1e-6)
    assert torch.allclose(ds.transpose(-1, -2) @ s["q"] / 8.0, k.grad, rtol=1e-5, atol=1e-6)


def test_fault_missing_eighth_is_rejected():
    s = _setup()
    grads = [(old + (ref - old) * 8.0, b) for old, (ref, b) in zip((s["dq0"], s["dk0"]), s["ref"])]
    with pytest.raises(AssertionError, match="out of bound"):
        _ok(s, grads)


def test_fault_missing_row_term_D_is_rejected():
    s = _setup()
    pr = torch.exp(s["q"] @ s["k"].transpose(-1, -2) / 8.0 + s["madd"][:, None, None, :] - s["lse"].double()[..., None])
    ds = pr * (s["r"] * s["G"])                       # dS without - D
    grads = [(s["dq0"] + ds @ s["k"] / 8.0, None), (s["dk0"] + ds.transpose(-1, -2) @ s["q"] / 8.0, None)]
    with pytest.raises(AssertionError, match="out of bound"):
        _ok(s, grads)


def test_fault_dropout_index_shifted_by_one_key_is_rejected():
    s = _setup()
    r = torch.from_numpy(D.multipliers(D.effective_seed(s["seed"]), s["idx"] + np.uint64(1), s["p"])).double()
    with pytest.raises(AssertionError, match="out of bound"):
        _ok(s, _faulty(s, r=r))


def test_fault_last_key_of_L65_left_out_is_rejected():
    s = _setup(L=65)
    madd = s["madd"].clone()
    madd[:, 64] = -1e9                                # exp(-1e9) = 0: key 64 takes no part
    with pytest.raises(AssertionError, match="out of bound"):
        _ok(s, _faulty(s, madd=madd))


def test_emulated_restatement_agrees_with_the_reference():
    """ops.attention_probs_bwd as the CPU replays answer it: the increments of dQ / dK are the reference's up to the bf16
    rounding of dS the reference replays (the restatement keeps dS in float64), V is untouched."""
    s = _setup(L=41, heads=2)
    n, L, heads = A.NSEQ, 41, 2
    qkv = torch.cat([A._merge(s["q"]), A._merge(s["k"]), torch.randn(n * L, heads * 64, dtype=F64)], 1).to(torch.bfloat16)
    mask = A._mask(L, L - 9)
    dqkv = torch.cat([A._merge(s["dq0"]), A._merge(s["dk0"]), torch.ones(n * L, heads * 64, dtype=F64)], 1).to(torch.bfloat16)
    drow = torch.empty(n * heads * L)
    ops_emulator.dropout_offset_bind(None)
    attention_probs_bwd(qkv, mask, s["lse"], s["G"].float(), drow, dqkv, n, L, L - 9, heads, s["p"], s["seed"])
    hid = heads * 64
    for j, ((ref, _), old) in enumerate(zip(s["ref"], (s["dq0"], s["dk0"]))):
        got = dqkv[:, j * hid:(j + 1) * hid].double() - A._merge(old)
        assert relerr(got, A._merge(ref - old)) < 2.0 ** -7
    assert bool((dqkv[:, 2 * hid:] == 1).all())


# ------------------------------------------------------------------------------------------------ module replays
@pytest.mark.parametrize("with_outputs", [False, True])
def test_attention_loss_gradients_match_oracle_on_emulated_ops(weights, with_outputs):
    with emulated_ops() as calls:
        PB.run_attention_loss_gradients(CPU, weights, "cpu", with_outputs)
    assert calls["attention_probs_bwd"] == len(PB.ATTN_LAYERS) and calls["attention_bwd"] == 12


def test_gradient_at_dropped_positions_changes_nothing_on_emulated_ops(weights):
    with emulated_ops():
        PB.run_dropped_positions_do_not_matter(CPU, weights, "cpu")


def test_switch_semantics_on_emulated_ops(weights):
    with emulated_ops() as calls:
        PB.run_switch_semantics(CPU, weights, "cpu", launches=calls)
    assert calls["attention_probs_bwd"] == 0


def test_head_bert_attention_gradients_on_emulated_ops(weights):
    with emulated_ops() as calls:
        PB.run_head_bert_gradients_land_in_the_flat_buffer(CPU, weights, "cpu")
    assert calls["attention_probs_bwd"] == 1
