"""ClipBertBaseModel.layerwise_autograd: a bert(...) pass as a chain of autograd nodes (embeddings, one node per encoder layer -
two, A_k and C_k, when the maps are differentiable - and the pooler), so that tensor hooks, torch.autograd.grad and
backward(inputs=...) on the hidden states and attention maps follow torch's own semantics; and the two kernels of the split at a
map, cb_attention_bwd_dv and cb_attention_probs_bwd_store.

Kernels, element by element against float64 from the same bf16 Q / K / dO, the forward's own lse and the multipliers r of
tests/dropout_ref.py (U = 2^-24; S, e_S, E as in test_gpu_attention_elementwise.py):
  dV = (P r)^T dO        P = exp(S - lse), e_P = P (e_S + E(S - lse)); P r (one fp32 product, e = r e_P + U |P r|) is rounded to
                         bf16 before the product (replayed, with the ambiguity amb of a value within e of a rounding boundary);
                         |err| <= 1 ulp_bf16(ref) + 2 U |ref| + amb^T |dO| + 2 U 3 (L + 1) |P r|^T |dO|
  dQ, dK (store)         the bound of cb_attention_probs_bwd (test_gpu_attention_probs_bwd.py) with dQ0 = dK0 = 0
Each written block lies between guard bands and pitch padding of a NaN sentinel; the block a kernel must not touch holds values
that are checked bit for bit afterwards, and an element still holding the sentinel fails.

Module, against fp32 autograd through the oracle (attention dropout 0.1 on, its maps post-dropout through the oracle's drop hook
with the run's own masks): autograd.grad on the maps and hidden states, hook-observed gradients, and a hook that zeroes one head's
gradient (the parameter gradients and d visual_inputs then follow it, the oracle running the same hook).

The CPU half (tests/test_layerwise_autograd_emulated.py) checks that the bounds reject deliberately wrong results, and replays the
module tests below on tests/ops_emulator.py.
"""
import contextlib
import gc

import pytest
import torch

import dropout_ref as D
import test_gpu_attention_elementwise as A
import test_gpu_attention_probs_bwd as PB
import test_gpu_attention_retained_grads as RG
from elementwise import BF16, F32, F64, U, Guarded, _INT, _record, check_bound, ulp_bf16

pytestmark = pytest.mark.gpu

HD = 64
NSEQ = A.NSEQ
MAP_LAYERS = (0, 5, 11)


# ------------------------------------------------------------------------------------------------ kernel references
def dv_ref(q, k, madd, lse, r, do):
    """(dV, bound) [NSEQ, H, L, 64] float64 from the bf16 Q / K / dO, the kernel's lse and the multipliers r."""
    L = q.shape[2]
    S, eS = A._scores(q, k, madd)
    lse = lse.detach().cpu().double()[..., None]
    P = torch.exp(S - lse)
    eP = P * (eS + A._E(S - lse))
    Pr = P * r
    X, amb = A._inter(Pr, r * eP + U * Pr.abs(), True)
    Xt, ambt = X.transpose(-1, -2), amb.transpose(-1, -2)
    ref = Xt @ do
    bound = ulp_bf16(ref) + 2.0 * U * ref.abs() + ambt @ do.abs() + 2.0 * U * 3.0 * (L + 1) * (Xt.abs() @ do.abs())
    return ref, bound


class Case:
    def __init__(self, L, heads, p, pitched):
        self.L, self.heads, self.p, self.pitched = L, heads, p, pitched
        self.lt = L - 9 if L > 9 else L

    @property
    def id(self):
        return "L%d-H%d-p%g%s" % (self.L, self.heads, self.p, "-pitched" if self.pitched else "")


LENGTHS = [1, 2, 9, 17, 41, 48, 49, 64, 65, 69, 128, 149, 169, 521]


def _cases():
    out = [Case(L, (1, 3, 12)[n % 3] if L < 512 else 1, 0.1 if n % 2 else 0.0, n % 3 == 1) for n, L in enumerate(LENGTHS)]
    return out + [Case(41, 12, 0.1, True), Case(69, 12, 0.0, True), Case(65, 3, 0.1, False), Case(521, 3, 0.1, True)]


CASES = _cases()


def _bits(t):
    return t.detach().cpu().contiguous().view(_INT[t.dtype]).clone()


def case_inputs(case):
    """qkv, dctx, the block values dqkv holds before the call, the mask and the multipliers (seed / device word of the case)."""
    n, L, H = NSEQ, case.L, case.heads
    hid = H * HD
    g = torch.Generator().manual_seed(41 * L + H + int(10 * case.p))
    qkv = torch.randn(n * L, 3 * hid, generator=g, dtype=F64).to(BF16)
    dctx = torch.randn(n * L, hid, generator=g, dtype=F64).to(BF16)
    dqkv0 = (torch.randn(n * L, 3 * hid, generator=g, dtype=F64) * 0.05).to(BF16)
    seed, word = 555 + L, (0x3456 + L if case.p > 0 else None)
    r = torch.ones(n, H, L, L, dtype=F64) if case.p == 0 else \
        torch.from_numpy(D.multipliers(D.effective_seed(seed, word), D.attention_index(n, H, L), case.p)).double()
    return qkv, dctx, dqkv0, A._mask(L, case.lt), seed, word, r


def _forward_lse(ops, xin, ld_qkv, mask_d, case, seed, dev):
    n, L, H = NSEQ, case.L, case.heads
    ctx = torch.empty(n * L, H * HD, dtype=BF16, device=dev)
    lse = torch.empty(n, H, L, dtype=F32, device=dev)
    ops._call("cb_attention_fwd", ops._p(xin.t), ld_qkv, ops._p(mask_d), ops._p(ctx), H * HD, ops._p(lse), n, L, case.lt, H, HD,
              case.p, seed, ops._s())
    return lse


def _run_kernel_case(case, dev, which):
    """which = "dv" (cb_attention_bwd_dv) or "store" (cb_attention_probs_bwd_store); returns the checked dqkv."""
    from clipbert_b200 import ops
    n, L, H = NSEQ, case.L, case.heads
    hid = H * HD
    qkv, dctx, dqkv0, mask, seed, word, r = case_inputs(case)
    ld_qkv, ld_ctx, ld_dqkv = (3 * hid + 64, hid + 40, 3 * hid + 24) if case.pitched else (3 * hid, hid, 3 * hid)
    xin, din = A._Window(qkv, ld_qkv, dev), A._Window(dctx, ld_ctx, dev)
    mask_d = mask.to(dev)
    written = slice(2 * hid, 3 * hid) if which == "dv" else slice(0, 2 * hid)
    kept = [slice(0, 2 * hid)] if which == "dv" else [slice(2 * hid, 3 * hid)]
    g = torch.Generator().manual_seed(L + 7)
    G = torch.randn(n, H, L, L, generator=g, dtype=F64).float().double()
    w = None if word is None else torch.tensor([word], dtype=torch.int64, device=dev)     # bound: must outlive the launches
    ops.dropout_offset_bind(w)
    try:
        lse_t = _forward_lse(ops, xin, ld_qkv, mask_d, case, seed, dev)
        lse = PB._nan_window(lse_t, dev)
        dprobs = PB._nan_window(G.float(), dev)
        runs = []
        for _ in range(2):
            out = Guarded((n * L, 3 * hid), BF16, dev, ld=ld_dqkv)
            for s in kept:
                out.t[:, s].copy_(dqkv0[:, s].to(dev))
            if which == "dv":
                ops._call("cb_attention_bwd_dv", ops._p(xin.t), ld_qkv, ops._p(mask_d), ops._p(lse), ops._p(din.t), ld_ctx,
                          ops._p(out.t), ld_dqkv, n, L, case.lt, H, HD, case.p, seed, ops._s())
            else:
                drow = torch.full((n * H * L,), float("nan"), dtype=F32, device=dev)
                ops._call("cb_attention_probs_bwd_store", ops._p(xin.t), ld_qkv, ops._p(mask_d), ops._p(lse), ops._p(dprobs),
                          ops._p(drow), ops._p(out.t), ld_dqkv, n, L, case.lt, H, HD, case.p, seed, ops._s())
            torch.cuda.synchronize()
            runs.append(out)
    finally:
        ops.dropout_offset_bind(None)
    a, b = runs
    assert torch.equal(_bits(a.buf), _bits(b.buf)), "%s: two identical runs differ" % case.id
    a.check("%s %s dqkv" % (case.id, which))
    got = a.t.cpu()
    for s in kept:
        assert torch.equal(_bits(got[:, s]), _bits(dqkv0[:, s])), "%s: a block %s must not touch was written" % (case.id, which)
    q, k, _ = A._split(qkv, H)
    (do,) = A._split(dctx, H)
    madd = A._madd(mask, L, case.lt)
    if which == "dv":
        ref, bound = dv_ref(q, k, madd, lse_t, r, do)
        _record("bwd_dv", case.id, check_bound(case.id + " dv", got[:, written], A._merge(ref), A._merge(bound)))
    else:
        zero = torch.zeros_like(q)
        (rq, bq), (rk, bk) = PB.probs_bwd_ref(q, k, madd, lse_t, r, G, zero, zero)
        _record("probs_bwd_store", case.id + "-dq", check_bound(case.id + " dq", got[:, :hid], A._merge(rq), A._merge(bq)))
        _record("probs_bwd_store", case.id + "-dk", check_bound(case.id + " dk", got[:, hid:2 * hid], A._merge(rk), A._merge(bk)))
    return got


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_attention_bwd_dv_elementwise(cuda, case):
    _run_kernel_case(case, cuda, "dv")


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_attention_probs_bwd_store_elementwise(cuda, case):
    _run_kernel_case(case, cuda, "store")


def test_case_matrix_covers_lengths_heads_dropout_and_pitches():
    assert {c.L for c in CASES} == set(LENGTHS) and {c.heads for c in CASES} == {1, 3, 12}
    assert {c.p for c in CASES} == {0.0, 0.1} and {c.pitched for c in CASES} == {False, True}


def test_split_kernels_reject_bad_arguments(cuda):
    from clipbert_b200 import ops
    n, L, H = 2, 41, 3
    hid = H * HD
    qkv = torch.zeros(n * L * 3 * hid + 8, dtype=BF16, device=cuda)
    dctx = torch.zeros(n * L * hid + 8, dtype=BF16, device=cuda)
    mask = torch.ones(n, L - 9, dtype=torch.int64, device=cuda)
    lse = torch.zeros(n * H * L, device=cuda)
    dprobs = torch.zeros(n * H * L * L + 4, device=cuda)
    drow = torch.zeros(n * H * L, device=cuda)
    dqkv = torch.full((n * L * 3 * hid + 8,), 2.5, dtype=BF16, device=cuda)
    P = ops._p

    def dv(q=qkv, ld_q=3 * hid, d=dctx, ld_c=hid, dq=dqkv, ld_dq=3 * hid, nseq=n, lt=L - 9, heads=H, hd=64, ls=lse):
        ops._call("cb_attention_bwd_dv", P(q), ld_q, P(mask), P(ls), P(d), ld_c, P(dq), ld_dq, nseq, L, lt, heads, hd, 0.0, 1, ops._s())

    def store(q=qkv, ld_q=3 * hid, d=dprobs, dq=dqkv, ld_dq=3 * hid, nseq=n, lt=L - 9, heads=H, hd=64, dr=drow, **_):
        ops._call("cb_attention_probs_bwd_store", P(q), ld_q, P(mask), P(lse), P(d), P(dr), P(dq), ld_dq, nseq, L, lt, heads, hd, 0.0, 1,
                  ops._s())

    for call in (dv, store):
        for kw in (dict(lt=L + 1), dict(lt=-1), dict(heads=0), dict(nseq=0), dict(nseq=65536), dict(heads=65536), dict(dq=None)):
            with pytest.raises(RuntimeError, match="bad arguments"):
                call(**kw)
        for kw in (dict(ld_q=3 * hid - 8), dict(ld_dq=3 * hid - 8), dict(ld_q=3 * hid + 4)):
            with pytest.raises(RuntimeError, match="row pitches"):
                call(**kw)
        for kw in (dict(q=qkv[1:]), dict(dq=dqkv[1:])):
            with pytest.raises(RuntimeError, match="16-byte aligned"):
                call(**kw)
        with pytest.raises(RuntimeError, match="head_dim"):
            call(hd=32)
    for kw in (dict(ld_c=hid - 8), dict(ld_c=hid + 4)):
        with pytest.raises(RuntimeError, match="row pitches"):
            dv(**kw)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        dv(d=dctx[1:])
    with pytest.raises(RuntimeError, match="bad arguments"):
        dv(ls=None)
    with pytest.raises(RuntimeError, match="bad arguments"):
        store(dr=None)
    torch.cuda.synchronize()
    assert bool((dqkv == 2.5).all())                 # nothing was launched


# ------------------------------------------------------------------------------------------------ module
def _model(weights, dev, layerwise=True, head=False, p=0.1, **cfg):
    m = RG._model(weights, dev, head=head, attention_probs_dropout_prob=p, **cfg)
    m.layerwise_autograd = layerwise
    return m


def _masks_of_last_call(eng, nseq, L, p):
    """The attention dropout multipliers of the engine's last forward: its seed and the device word it bound."""
    seed = (eng._seed_base + eng._call_count * 1000003) & (2 ** 64 - 1)
    word = int(eng._drop_counter.reshape(-1)[0].item())
    idx = D.attention_index(nseq, 12, L)
    return {i: torch.from_numpy(D.multipliers(D.effective_seed(seed + 16 * (i + 1) + 1, word), idx, p)) for i in range(12)}


def _oracle(weights, ids, grid, mask, mult):
    """fp32 oracle pass with the given attention masks: (seq, pooled, layer inputs, post-dropout maps, state dict, grid leaf)."""
    from oracle import clipbert_ref as R
    rec = {}

    def drop(site, layer, x):
        if site == "attn_probs":
            x = x * mult[layer]
            rec[layer] = x
        return x
    sd = {k: (v.clone().requires_grad_(True) if k.startswith("transformer.bert.") else v) for k, v in weights.items()}
    gr = grid.clone().requires_grad_(True)
    seq_r, pooled_r, layers_r = R.clipbert_base_model(ids, gr, mask, sd, return_layers=True, drop=drop)
    return seq_r, pooled_r, list(layers_r), [rec[i] for i in range(12)], sd, gr


def _score(seq, pooled, hidden, attn, wp, W, dh):
    s = (pooled.float() * wp).sum() + (seq.float() * dh[12]).sum() * 0.5
    s = s + sum((attn[i] * W[i]).sum() for i in MAP_LAYERS)
    return s + (hidden[3].float() * dh[3]).sum()


def _directs(nseq, L, g, dev):
    wp = torch.randn(nseq, 768, generator=g).to(torch.bfloat16).float()
    W = {i: torch.randn(nseq, 12, L, L, generator=g) for i in MAP_LAYERS}
    dh = {k: (torch.randn(nseq, L, 768, generator=g) * 0.1).to(torch.bfloat16).float() for k in (3, 12)}
    return (wp, W, dh), (wp.to(dev), {i: w.to(dev) for i, w in W.items()}, {k: v.to(dev) for k, v in dh.items()})


def _record_hooks(tensors):
    seen = [None] * len(tensors)
    for n, t in enumerate(tensors):
        t.register_hook(lambda g, n=n: seen.__setitem__(n, g.detach().clone()))
    return seen


def _zero_head(layer, head):
    def hook(g):
        g = g.clone()
        g[:, head] = 0
        return g
    return hook


def run_against_oracle(dev, weights, size):
    """autograd.grad on all 12 maps and all 13 hidden states, then a backward with hooks on every map and hidden state, against
    the oracle doing the same; then a hook zeroing head 4 of attentions[5]: parameter gradients and d visual_inputs."""
    model = _model(weights, dev).train()
    eng = model._engine
    grid, ids, mask, L, g = RG._inputs(size, 131)
    nseq = ids.shape[0]
    (wp, W, dh), (wpd, Wd, dhd) = _directs(nseq, L, g, dev)
    gc = grid.clone().to(dev).requires_grad_(True)
    seq, pooled, hidden, attn = model(ids.to(dev), gc, mask.to(dev))
    assert seq is hidden[12] and all(a.requires_grad for a in attn)
    mult = _masks_of_last_call(eng, nseq, L, 0.1)
    seq_r, pooled_r, layers_r, rec, sd, gr = _oracle(weights, ids, grid, mask, mult)
    score = _score(seq, pooled, hidden, attn, wpd, Wd, dhd)
    score_r = _score(seq_r, pooled_r, layers_r, rec, wp, W, dh)
    for what, ours, theirs in (("attentions", attn, rec), ("hidden_states", hidden, layers_r)):
        got = torch.autograd.grad(score, list(ours), retain_graph=True)
        ref = torch.autograd.grad(score_r, list(theirs), retain_graph=True)
        for n, (a, b) in enumerate(zip(got, ref)):
            RG._close("autograd.grad %s[%d]" % (what, n), a, b)
    seen = _record_hooks(list(attn) + list(hidden))
    seen_r = _record_hooks(list(rec) + list(layers_r))
    score.backward(retain_graph=True)
    score_r.backward(retain_graph=True)
    for n, (a, b) in enumerate(zip(seen, seen_r)):
        RG._close("hook %d" % n, a, b)
    PB._compare_grads(model, sd, gc, gr)
    # a hook that zeroes one head's gradient: every gradient below layer 5 follows it
    model.zero_grad(set_to_none=False)
    gc.grad = None
    for t in list(sd.values()) + [gr]:
        if isinstance(t, torch.Tensor) and t.grad is not None:
            t.grad = None
    attn[5].register_hook(_zero_head(5, 4))
    rec[5].register_hook(_zero_head(5, 4))
    score.backward()
    score_r.backward()
    checked = PB._compare_grads(model, sd, gc, gr)
    assert checked >= 12 * 15
    assert float(model.encoder.layer[4].attention.self.query.weight.grad.abs().sum()) > 0


@pytest.mark.parametrize("size", ["224px", "448px", "512tok"])
def test_layerwise_gradients_against_oracle(cuda, weights, size):
    run_against_oracle(cuda, weights, size)


@contextlib.contextmanager
def _deterministic():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _flat_bits(model):
    return model._engine._flat.grad.detach().clone().view(torch.int32)


def run_semantics(dev, weights, size="224px"):
    """autograd.grad leaves the flat gradient buffer bit-identical; retain_graph gives a second backward equal to the first
    (hooks see the same bits, parameter gradients double); without it torch's own error; a second pass without the switch
    still runs one node. Deterministic mode, dropout on."""
    model = _model(weights, dev, hidden_dropout_prob=0.1).train()
    grid, ids, mask, L, g = RG._inputs(size, 133)
    nseq = ids.shape[0]
    _, (wpd, Wd, dhd) = _directs(nseq, L, g, dev)
    ids, mask, gdev = ids.to(dev), mask.to(dev), grid.to(dev)
    with _deterministic():
        seq, pooled, hidden, attn = model(ids, gdev.clone().requires_grad_(True), mask)
        _score(seq, pooled, hidden, attn, wpd, Wd, dhd).backward()         # a flat buffer that holds something
        before = _flat_bits(model)
        grads_before = [p.grad for p in model.parameters()]
        gc = gdev.clone().requires_grad_(True)
        seq, pooled, hidden, attn = model(ids, gc, mask)
        score = _score(seq, pooled, hidden, attn, wpd, Wd, dhd)
        ga = torch.autograd.grad(score, [attn[5]], retain_graph=True)[0]
        gh = torch.autograd.grad(score, [hidden[7]], retain_graph=True)[0]
        gboth = torch.autograd.grad(score, [attn[5], hidden[7]], retain_graph=True)
        assert torch.equal(gboth[0], ga) and torch.equal(gboth[1], gh)
        assert torch.equal(_flat_bits(model), before) and gc.grad is None
        assert all(a is b for a, b in zip(grads_before, [p.grad for p in model.parameters()]))
        score.backward(inputs=[hidden[2]], retain_graph=True)
        assert torch.equal(_flat_bits(model), before) and gc.grad is None and hidden[2].grad is not None
        # retain_graph: the second backward through the same pass gives the same gradients
        model.zero_grad(set_to_none=False)
        seen = _record_hooks([attn[5], hidden[7], hidden[0]])
        score.backward(retain_graph=True)
        once = [t.clone() for t in seen] + [model._engine._flat.grad.clone(), gc.grad.clone()]
        score.backward()
        twice = [t.clone() for t in seen] + [model._engine._flat.grad.clone(), gc.grad.clone()]
        for a, b in zip(once[:3], twice[:3]):
            assert torch.equal(a, b)
        assert torch.equal(twice[4], 2 * once[4])
        assert float((twice[3] - 2 * once[3]).abs().max()) <= 1e-6 * float(once[3].abs().max())
        with pytest.raises(RuntimeError, match="second time"):
            score.backward()
    assert float(ga.abs().sum()) > 0 and float(gh.float().abs().sum()) > 0


def test_semantics_autograd_grad_and_retain_graph(cuda, weights):
    run_semantics(cuda, weights)


def test_memory_returns_to_its_collected_baseline(cuda, weights):
    model = _model(weights, cuda).train()
    grid, ids, mask, L, g = RG._inputs("448px", 135)
    _, (wpd, Wd, dhd) = _directs(ids.shape[0], L, g, cuda)
    ids, mask, gdev = ids.to(cuda), mask.to(cuda), grid.to(cuda)

    def step(partial):
        gc = gdev.clone().requires_grad_(True)
        out = model(ids, gc, mask)
        score = _score(*out, wpd, Wd, dhd)
        if partial:
            torch.autograd.grad(score, [out[3][7]])
        else:
            score.backward()
        return torch.cuda.memory_allocated()

    step(False)
    gc.collect()            # the baseline without garbage an earlier test left in reference cycles (collected at any time later)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    for partial in (False, True, False):
        step(partial)
        torch.cuda.synchronize()
        assert torch.cuda.memory_allocated() == base, partial


def run_head_bert(dev, weights, size="224px"):
    """A head's bert with the switch on: the gradients land in the head's flat buffer; refused with the overlapped exchange."""
    bert = _model(weights, dev, head=True, p=0.0)
    head = bert._engine
    grid, ids, mask, L, g = RG._inputs(size, 137)
    W = torch.randn(ids.shape[0], 12, L, L, generator=g).to(dev)
    seq, pooled, hidden, attn = bert(ids.to(dev), grid.to(dev), mask.to(dev))
    seen = _record_hooks([attn[5]])
    (attn[5] * W).sum().backward()
    assert torch.equal(seen[0], W)
    flat = head._flat
    lo, hi = flat.grad.data_ptr(), flat.grad.data_ptr() + 4 * flat.grad.numel()
    for p in bert.parameters():
        assert p.grad is None or lo <= p.grad.data_ptr() < hi
    lay = bert.encoder.layer
    assert float(lay[5].attention.self.query.weight.grad.abs().sum()) > 0 and float(lay[6].attention.self.query.weight.grad.abs().sum()) == 0
    assert float(lay[5].attention.self.value.weight.grad.abs().sum()) == 0
    assert float(lay[4].attention.self.value.weight.grad.abs().sum()) > 0
    head._grad_ready_hook = lambda g: None
    try:
        with pytest.raises(RuntimeError, match="enable_overlapped_allreduce"):
            bert(ids.to(dev), grid.to(dev), mask.to(dev))
    finally:
        head._grad_ready_hook = None


def test_head_bert_gradients_land_in_the_flat_buffer(cuda, weights):
    run_head_bert(cuda, weights)


def chefer_relevance(attn, grads):
    """Chefer et al. (2021), rule 6: R = I + sum over layers of mean_heads((grad * A)^+) R, [nseq, L, L]."""
    nseq, _, L, _ = attn[0].shape
    R = torch.eye(L, dtype=torch.float32, device=attn[0].device).expand(nseq, L, L).clone()
    for a, gr in zip(attn, grads):
        cam = (gr * a.detach()).clamp(min=0).mean(1)
        R = R + torch.bmm(cam, R)
    return R


def run_chefer_hooks_equal_retain_grad(dev, weights, size="224px"):
    """The relevance from gradients saved by register_hook (switch on) equals the one from retain_grad() (switch off)."""
    grid, ids, mask, L, g = RG._inputs(size, 139)
    target = torch.randn(ids.shape[0], 768, generator=g).to(dev)
    rel = []
    for layerwise in (True, False):
        model = _model(weights, dev, layerwise=layerwise, p=0.0).eval()
        seq, pooled, hidden, attn = model(ids.to(dev), grid.to(dev), mask.to(dev))
        if layerwise:
            saved = _record_hooks(list(attn))
        else:
            for a in attn:
                a.retain_grad()
        (pooled.float() * target).sum().backward()
        grads = saved if layerwise else [a.grad for a in attn]
        rel.append(chefer_relevance(attn, grads))
    RG._close("Chefer relevance", rel[0], rel[1])


def test_chefer_relevance_from_hooks_equals_retain_grad(cuda, weights):
    run_chefer_hooks_equal_retain_grad(cuda, weights)


def run_bits_switch_on_equals_off(dev, weights, size="224px", launches=None):
    """Deterministic mode, differentiable_attentions off, dropout on: the switch on gives the launches and the parameter and
    visual_inputs gradient bits of the switch off. launches: the emulated-ops call counter on the CPU replay."""
    grid, ids, mask, L, g = RG._inputs(size, 141)
    _, (wpd, _, dhd) = _directs(ids.shape[0], L, g, dev)
    ids, mask = ids.to(dev), mask.to(dev)
    res = []
    with _deterministic():
        for on in (False, True):
            model = _model(weights, dev, layerwise=on, hidden_dropout_prob=0.1)
            model.differentiable_attentions = False
            model.train()
            gc = grid.clone().to(dev).requires_grad_(True)
            before = dict(launches) if launches is not None else None
            with PB._timing(dev) as ev:
                seq, pooled, hidden, attn = model(ids, gc, mask)
                loss = (pooled.float() * wpd).sum() + (seq.float() * dhd[12]).sum() + (hidden[3].float() * dhd[3]).sum()
                loss.backward()
                names = [e[0] for e in ev] if ev is not None else \
                    {k: v - before[k] for k, v in launches.items() if k != "dropout_offset_bind"}     # host state, not a launch
            res.append((names, PB._grad_bits(model, gc)))
    assert res[0][0] == res[1][0]
    for a, b in zip(res[0][1], res[1][1]):
        assert torch.equal(a, b)


def test_switch_on_gives_the_bits_of_the_switch_off(cuda, weights):
    run_bits_switch_on_equals_off(cuda, weights)


def _hooked_step(model, ids, gdev, mask, wpd, Wd, dhd):
    model.zero_grad(set_to_none=False)
    seq, pooled, hidden, attn = model(ids, gdev, mask)
    for i in range(12):
        attn[i].register_hook(_zero_head(i, i % 12))
    seen = _record_hooks([attn[2], hidden[6]])
    _score(seq, pooled, hidden, attn, wpd, Wd, dhd).backward()
    return seen


def test_three_runs_give_the_same_bits(cuda, weights):
    model = _model(weights, cuda, hidden_dropout_prob=0.1).train()
    eng = model._engine
    grid, ids, mask, L, g = RG._inputs("448px", 143)
    _, (wpd, Wd, dhd) = _directs(ids.shape[0], L, g, cuda)
    ids, mask, gdev = ids.to(cuda), mask.to(cuda), grid.to(cuda)
    with torch.no_grad():
        model(ids, gdev, mask)
    state = (eng._call_count, int(eng._drop_counter.item()))
    runs = []
    with _deterministic():
        for _ in range(3):
            PB._rewind(eng, state)
            seen = _hooked_step(model, ids, gdev, mask, wpd, Wd, dhd)
            runs.append([t.clone() for t in seen] + [p.grad.detach().clone() for p in model.parameters()])
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a, b)


def test_cuda_graph_replay_matches_eager(cuda, weights):
    """Hooks on every map (one head zeroed each) with dropout, captured once: a replay rewound to an eager step's position gives
    that step's bits."""
    model = _model(weights, cuda, hidden_dropout_prob=0.1).train()
    eng = model._engine
    grid, ids, mask, L, g = RG._inputs("224px", 145)
    _, (wpd, Wd, dhd) = _directs(ids.shape[0], L, g, cuda)
    ids, mask, gdev = ids.to(cuda), mask.to(cuda), grid.to(cuda).to(torch.bfloat16)
    params = list(model.parameters())
    with _deterministic():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                _hooked_step(model, ids, gdev, mask, wpd, Wd, dhd)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        calls0, w0 = eng._call_count, int(eng._drop_counter.item())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            captured = _hooked_step(model, ids, gdev, mask, wpd, Wd, dhd)
        eng._call_count = calls0
        eng._drop_counter.fill_(w0)
        seen = _hooked_step(model, ids, gdev, mask, wpd, Wd, dhd)
        torch.cuda.synchronize()
        eager = [t.clone() for t in seen] + [p.grad.detach().clone() for p in params]
        eng._drop_counter.fill_(w0)
        graph.replay()
        torch.cuda.synchronize()
        replay = [t.clone() for t in captured] + [p.grad.detach().clone() for p in params]
    assert float(eager[0].abs().sum()) > 0 and float(eager[2].abs().sum()) > 0
    for a, b in zip(eager, replay):
        assert torch.equal(a, b)


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)
