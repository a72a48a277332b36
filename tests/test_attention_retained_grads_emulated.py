"""cb_attention_dprobs and retain_grad() on ClipBertBaseModel's outputs, on CPU: the float64 reference and its per-element bound of
tests/test_gpu_attention_retained_grads.py checked against deliberately wrong results, and the module tests of that file
replayed with the C-ABI calls answered by tests/ops_emulator.py (plus the restatements of cb_attention_probs and
cb_attention_probs_bwd of the earlier emulated tests) and ops.attention_dprobs by the float64 restatement below."""
import contextlib

import pytest
import torch

import test_attention_probs_bwd_emulated as PBE
import test_gpu_attention_elementwise as A
import test_gpu_attention_retained_grads as RG
from elementwise import F64, check_bound

CPU = torch.device("cpu")


def attention_dprobs(qkv, dctx, dprobs, accumulate, nseq, l, heads):
    """The header's cb_attention_dprobs in float64: dprobs = (dprobs if accumulate else 0) + dO V^T per head, V the third column
    block of qkv, dO = dctx."""
    hd = dctx.shape[1] // heads
    v = qkv.view(nseq, l, 3, heads, hd)[:, :, 2].double().permute(0, 2, 1, 3)
    do = dctx.view(nseq, l, heads, hd).double().permute(0, 2, 1, 3)
    out = do @ v.transpose(-1, -2)
    if accumulate:
        out = out + dprobs.double()
    dprobs.copy_(out)


@contextlib.contextmanager
def emulated_ops():
    from clipbert_b200 import ops
    with PBE.emulated_ops() as calls:
        saved = ops.attention_dprobs
        calls["attention_dprobs"] = 0

        def counted(*a, **k):
            calls["attention_dprobs"] += 1
            return attention_dprobs(*a, **k)
        ops.attention_dprobs = counted
        try:
            yield calls
        finally:
            ops.attention_dprobs = saved


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)


# ------------------------------------------------------------------------------------------------ reference and bound
def _setup(L=65, heads=2, accumulate=1):
    case = RG.Case(L, heads, accumulate, False)
    qkv, dctx, old = RG.case_inputs(case)
    ref, bound = RG.case_reference(case, qkv, dctx, old)
    return dict(case=case, qkv=qkv, dctx=dctx, old=old, ref=ref, bound=bound)


def _ok(s, got64):
    check_bound("fault dprobs", got64.float(), s["ref"], s["bound"])


def test_reference_accepts_itself_and_matches_autograd():
    """The reference rounded to fp32 passes its own bound, and dO V^T is float64 autograd of sum(ctx * dO) with ctx = A V."""
    s = _setup()
    _ok(s, s["ref"])
    _, _, v = A._split(s["qkv"], 2)
    (do,) = A._split(s["dctx"], 2)
    a = torch.rand(A.NSEQ, 2, 65, 65, dtype=F64, requires_grad=True)
    with torch.enable_grad():
        ((a @ v) * do).sum().backward()
    assert torch.allclose(s["ref"] - s["old"].double(), a.grad, rtol=1e-12, atol=1e-12)


def test_fault_missing_last_key_tile_at_L65_is_rejected():
    s = _setup(L=65)
    bad = s["ref"].clone()
    bad[..., 64] = s["old"].double()[..., 64]        # key 64, the whole second key tile, never added
    with pytest.raises(AssertionError, match="out of bound"):
        _ok(s, bad)


def test_fault_V_taken_from_the_K_block_is_rejected():
    s = _setup(L=41)
    qkv = s["qkv"].clone()
    hid = 2 * 64
    k = torch.randn(qkv.shape[0], hid, generator=torch.Generator().manual_seed(5), dtype=F64).to(torch.bfloat16)
    qkv[:, hid:2 * hid] = k
    qkv_wrong = qkv.clone()
    qkv_wrong[:, 2 * hid:] = k                       # the V block read from K's columns
    bad, _ = RG.case_reference(s["case"], qkv_wrong, s["dctx"], s["old"])
    with pytest.raises(AssertionError, match="out of bound"):
        _ok(s, bad)


def test_fault_accumulate_ignored_is_rejected():
    s = _setup(L=41, accumulate=1)
    bad, _ = RG.case_reference(s["case"], s["qkv"], s["dctx"], None)
    with pytest.raises(AssertionError, match="out of bound"):
        _ok(s, bad)


@pytest.mark.parametrize("accumulate", [0, 1])
def test_emulated_restatement_agrees_with_the_reference(accumulate):
    """ops.attention_dprobs as the CPU replays answer it passes the kernel's bound (NaN Q and K blocks: only V is read)."""
    s = _setup(L=41, heads=2, accumulate=accumulate)
    out = torch.empty(A.NSEQ, 2, 41, 41) if s["old"] is None else s["old"].clone()
    attention_dprobs(s["qkv"], s["dctx"], out, accumulate, A.NSEQ, 41, 2)
    _ok(s, out.double())


# ------------------------------------------------------------------------------------------------ module replays
@pytest.mark.parametrize("direct", [False, True])
def test_retained_grads_match_oracle_on_emulated_ops(weights, direct):
    with emulated_ops() as calls:
        RG.run_retained_grads_against_oracle(CPU, weights, "cpu", direct)
    assert calls["attention_dprobs"] == 12 and calls["attention_bwd"] == 12


def test_retained_grads_of_a_heads_bert_on_emulated_ops(weights):
    with emulated_ops() as calls:
        RG.run_retained_grads_against_oracle(CPU, weights, "cpu", True, head=True)
    assert calls["attention_dprobs"] == 12


def test_gradient_at_dropped_positions_is_dO_Vt_on_emulated_ops(weights):
    with emulated_ops():
        RG.run_dropped_positions_get_dO_Vt(CPU, weights, "cpu")


def test_retain_grad_semantics_on_emulated_ops(weights):
    with emulated_ops() as calls:
        RG.run_semantics(CPU, weights, "cpu", launches=calls)


def test_a_non_contiguous_retained_grad_is_copied_then_accumulated():
    """A .grad that is not contiguous (set by hand, say) is copied into a fresh contiguous tensor that accumulates dO V^T."""
    from clipbert_b200 import modeling
    s = _setup(L=41, heads=2, accumulate=1)
    t = torch.zeros(A.NSEQ, 2, 41, 41)
    t.grad = s["old"].transpose(-1, -2).contiguous().transpose(-1, -2)
    assert not t.grad.is_contiguous()
    with emulated_ops() as calls:
        modeling._add_retained_attention_grad(t, s["qkv"], s["dctx"], A.NSEQ, 41, 2)
    assert calls["attention_dprobs"] == 1 and t.grad.is_contiguous()
    _ok(s, t.grad.double())
