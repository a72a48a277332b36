"""ClipBertBaseModel.layerwise_autograd on CPU: the float64 references and bounds of tests/test_gpu_layerwise_autograd.py checked
against themselves and against deliberately wrong results, and its module tests replayed with the C-ABI calls answered by
tests/ops_emulator.py, the attention-map restatements of the earlier emulated tests and the float64 restatements of the two
split kernels below. Planted faults in the node chain must fail the comparison with the oracle."""
import contextlib
import math

import numpy as np
import pytest
import torch

import dropout_ref as D
import ops_emulator
import test_attention_retained_grads_emulated as RGE
import test_gpu_attention_elementwise as A
import test_gpu_attention_probs_bwd as PB
import test_gpu_layerwise_autograd as LW
from elementwise import F64, check_bound

CPU = torch.device("cpu")


def attention_bwd_dv(qkv, text_mask, lse, dctx, dqkv, nseq, l, lt, heads, p, seed):
    """The header's cb_attention_bwd_dv in float64: P = exp(S - lse) from the GIVEN lse, dV = (P r)^T dO written to dqkv's V
    block; the Q and K blocks untouched."""
    _, _, _, s = ops_emulator._attention_scores(qkv, text_mask, nseq, l, lt, heads)
    pr = torch.exp(s - lse.double()[..., None])
    mult = ops_emulator._drop_mult(p, seed, D.attention_index(nseq, heads, l))
    if mult is not None:
        pr = pr * mult.double()
    dv = pr.transpose(-1, -2) @ ops_emulator._heads(dctx, nseq, l, heads)
    dqkv.view(nseq, l, 3, -1)[:, :, 2].copy_(dv.permute(0, 2, 1, 3).reshape(nseq, l, -1))


def attention_probs_bwd_store(qkv, text_mask, lse, dprobs, drow, dqkv, nseq, l, lt, heads, p, seed):
    """The header's cb_attention_probs_bwd_store in float64: P from the GIVEN lse, g = r G, D = sum P g (written to drow),
    dS = P (g - D); dQ = dS K / 8 and dK = dS^T Q / 8 written to dqkv's Q and K blocks (their old contents never read), V
    untouched."""
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
        blocks[:, :, j].copy_(grad.permute(0, 2, 1, 3).reshape(nseq, l, -1))


@contextlib.contextmanager
def emulated_ops():
    """The emulated ops of the retained-gradient replays, with ops.attention_bwd_dv and ops.attention_probs_bwd_store answered
    by the restatements above (and counted)."""
    from clipbert_b200 import ops
    with RGE.emulated_ops() as calls:
        saved = {n: getattr(ops, n) for n in ("attention_bwd_dv", "attention_probs_bwd_store")}

        def counted(name, fn):
            def f(*a, **k):
                calls[name] += 1
                return fn(*a, **k)
            return f
        for name, fn in (("attention_bwd_dv", attention_bwd_dv), ("attention_probs_bwd_store", attention_probs_bwd_store)):
            calls[name] = 0
            setattr(ops, name, counted(name, fn))
        try:
            yield calls
        finally:
            for name, fn in saved.items():
                setattr(ops, name, fn)


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)


# ------------------------------------------------------------------------------------------------ reference and bound
def _setup(L=65, heads=2, p=0.1):
    case = LW.Case(L, heads, p, False)
    qkv, dctx, dqkv0, mask, seed, word, r = LW.case_inputs(case)
    q, k, _ = A._split(qkv, heads)
    (do,) = A._split(dctx, heads)
    madd = A._madd(mask, L, case.lt)
    lse = torch.logsumexp(q @ k.transpose(-1, -2) / 8.0 + madd[:, None, None, :], -1).float()
    ref, bound = LW.dv_ref(q, k, madd, lse, r, do)
    return dict(case=case, qkv=qkv, dctx=dctx, mask=mask, seed=seed, word=word, r=r, q=q, k=k, do=do, madd=madd, lse=lse, ref=ref,
                bound=bound)


def _ok(s, got):
    check_bound("fault dv", got, s["ref"], s["bound"])


def test_dv_reference_accepts_itself_and_matches_autograd():
    """The reference rounded to bf16 passes its own bound; without the bf16 rounding of P r it is float64 autograd of
    sum(ctx dO) with ctx = (softmax(Q K^T / 8 + madd) r) V."""
    s = _setup()
    _ok(s, s["ref"].to(torch.bfloat16).double())
    v = torch.zeros_like(s["do"]).requires_grad_(True)
    with torch.enable_grad():
        a = torch.softmax(s["q"] @ s["k"].transpose(-1, -2) / 8.0 + s["madd"][:, None, None, :], -1) * s["r"]
        ((a @ v) * s["do"]).sum().backward()
    assert torch.allclose(v.grad, s["ref"], rtol=2e-2, atol=2e-2)


def test_fault_dv_dropout_index_shifted_by_one_key_is_rejected():
    s = _setup()
    idx = D.attention_index(A.NSEQ, 2, 65) + np.uint64(1)
    r = torch.from_numpy(D.multipliers(D.effective_seed(s["seed"], s["word"]), idx, 0.1)).double()
    bad, _ = LW.dv_ref(s["q"], s["k"], s["madd"], s["lse"], r, s["do"])
    with pytest.raises(AssertionError, match="out of bound"):
        _ok(s, bad)


def test_fault_dv_without_dropout_is_rejected():
    s = _setup()
    bad, _ = LW.dv_ref(s["q"], s["k"], s["madd"], s["lse"], torch.ones_like(s["r"]), s["do"])
    with pytest.raises(AssertionError, match="out of bound"):
        _ok(s, bad)


def test_fault_dv_last_key_tile_left_out_is_rejected():
    s = _setup(L=65)
    bad = s["ref"].clone()
    bad[..., 64, :] = 0                                 # key 64: the second key tile never written
    with pytest.raises(AssertionError, match="out of bound"):
        _ok(s, bad)


def test_fault_store_that_adds_to_garbage_is_rejected():
    """The store mode's bound: a dQ / dK added to what the block held instead of written fails."""
    s = PBE_setup()
    zero = torch.zeros_like(s["q"])
    (rq, bq), _ = PB.probs_bwd_ref(s["q"], s["k"], s["madd"], s["lse"], s["r"], s["G"], zero, zero)
    check_bound("store dq", rq.to(torch.bfloat16).double(), rq, bq)
    with pytest.raises(AssertionError, match="out of bound"):
        check_bound("store dq", (rq + s["dq0"]).to(torch.bfloat16).double(), rq, bq)


def PBE_setup():
    import test_attention_probs_bwd_emulated as PBE
    return PBE._setup(L=41, heads=2)


@pytest.mark.parametrize("which", ["dv", "store"])
def test_emulated_restatements_agree_with_the_references(which):
    """ops.attention_bwd_dv / attention_probs_bwd_store as the CPU replays answer them: the written block within the reference
    (up to the bf16 rounding of P r / dS the reference replays), the other blocks untouched."""
    s = _setup(L=41, heads=2, p=0.1)
    n, L, heads, hid = A.NSEQ, 41, 2, 128
    dqkv = torch.full((n * L, 3 * hid), 7.0, dtype=torch.bfloat16)
    ops_emulator.dropout_offset_bind(torch.tensor([s["word"]]))
    try:
        if which == "dv":
            attention_bwd_dv(s["qkv"], s["mask"], s["lse"], s["dctx"], dqkv, n, L, s["case"].lt, heads, 0.1, s["seed"])
            (got,) = A._split(dqkv[:, 2 * hid:], heads)
            assert float((got - s["ref"]).abs().max()) < 4e-2 * float(s["ref"].abs().max())
            assert bool((dqkv[:, :2 * hid] == 7).all())
        else:
            G = torch.randn(n, heads, L, L, dtype=F64).float()
            drow = torch.empty(n * heads * L)
            attention_probs_bwd_store(s["qkv"], s["mask"], s["lse"], G, drow, dqkv, n, L, s["case"].lt, heads, 0.1, s["seed"])
            zero = torch.zeros_like(s["q"])
            (rq, _), (rk, _) = PB.probs_bwd_ref(s["q"], s["k"], s["madd"], s["lse"], s["r"], G.double(), zero, zero, rounded=False)
            gq, gk, _ = A._split(dqkv, heads)
            for got, ref in ((gq, rq), (gk, rk)):
                assert float((got - ref).abs().max()) < 2e-2 * float(ref.abs().max())
            assert bool((dqkv[:, 2 * hid:] == 7).all())
    finally:
        ops_emulator.dropout_offset_bind(None)


# ------------------------------------------------------------------------------------------------ module replays
def test_layerwise_gradients_match_oracle_on_emulated_ops(weights):
    with emulated_ops() as calls:
        LW.run_against_oracle(CPU, weights, "cpu")
    assert calls["attention_bwd_dv"] > 0 and calls["attention_probs_bwd_store"] > 0 and calls["attention_bwd"] == 0


def test_semantics_on_emulated_ops(weights):
    with emulated_ops():
        LW.run_semantics(CPU, weights, "cpu")


def test_head_bert_on_emulated_ops(weights):
    with emulated_ops() as calls:
        LW.run_head_bert(CPU, weights, "cpu")
    assert calls["attention_probs_bwd_store"] == 6 and calls["attention_bwd_dv"] == 5     # A_5 .. A_0, C_4 .. C_0


def test_chefer_relevance_on_emulated_ops(weights):
    with emulated_ops():
        LW.run_chefer_hooks_equal_retain_grad(CPU, weights, "cpu")


def test_switch_on_gives_the_launches_and_bits_of_the_switch_off_on_emulated_ops(weights):
    with emulated_ops() as calls:
        LW.run_bits_switch_on_equals_off(CPU, weights, "cpu", launches=calls)


# ------------------------------------------------------------------------------------------------ planted faults
def _planted(weights, monkeypatch, name, fn):
    from clipbert_b200 import ops
    with emulated_ops():
        monkeypatch.setattr(ops, name, fn)
        with pytest.raises(AssertionError):
            LW.run_against_oracle(CPU, weights, "cpu")


def test_fault_dv_never_handed_over_fails_the_oracle(weights, monkeypatch):
    """C_k's dV left out of the V block (zeros): every gradient below the top layer is wrong."""
    def no_dv(qkv, text_mask, lse, dctx, dqkv, nseq, l, lt, heads, p, seed):
        dqkv.view(nseq, l, 3, -1)[:, :, 2].zero_()
    _planted(weights, monkeypatch, "attention_bwd_dv", no_dv)


def test_fault_map_gradient_without_the_context_term_fails_the_oracle(weights, monkeypatch):
    """C_k returning zero for the map (A_k then sees only the direct term and the hooks' view of it)."""
    def zero_dprobs(qkv, dctx, dprobs, accumulate, nseq, l, heads):
        if not accumulate:
            dprobs.zero_()
    _planted(weights, monkeypatch, "attention_dprobs", zero_dprobs)


def test_fault_store_mode_that_keeps_the_old_block_fails_the_oracle(weights, monkeypatch):
    """dQ / dK added to the garbage of a fresh dqkv instead of written."""
    import test_attention_probs_bwd_emulated as PBE

    def add_instead(*a):
        dqkv = a[5]
        dqkv.view(-1)[: dqkv.numel() // 2].fill_(0.5)
        PBE.attention_probs_bwd(*a)
    _planted(weights, monkeypatch, "attention_probs_bwd_store", add_instead)


def test_overlapped_exchange_is_refused(weights):
    with emulated_ops():
        model = LW._model(weights, CPU)
        model._engine._grad_ready_hook = lambda g: None
        grid, ids, mask, L, g = LW.RG._inputs("cpu", 1)
        with pytest.raises(RuntimeError, match="enable_overlapped_allreduce"):
            model(ids, grid, mask)
        with torch.no_grad():
            model(ids, grid, mask)                      # a pass that records no autograd is not the switch's business
