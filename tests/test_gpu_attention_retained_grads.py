"""retain_grad() on the outputs of ClipBertBaseModel.forward, and cb_attention_dprobs, the kernel behind the attention maps'.

After backward(), a retained output's .grad is what the reference's tensor would hold:
  attentions[l]      G_l + dO_l V_l^T per head (G_l: the loss's direct term on the map, dO_l: d loss / d context of layer l,
                     V_l: the layer's bf16 value block), at every (i, j) < L, dropped positions included;
  hidden_states[k]   the full gradient at the input of layer k (the engine's dx at that boundary, direct terms included);
  sequence_output    the same as hidden_states[12] (one tensor in the reference): the top gradient, pooler path included.

Kernel, element by element against float64 from the same bf16 dO and V (U = 2^-24):
  dprobs = old + dO V^T ;  |err| <= U |ref| (the fp32 add to the old value) + 3 (64 + 1) U sum_d |dO| |V| (the 64-long product on
  mma.sync with fp32 accumulation)
with the Q and K blocks of qkv and the pitch padding NaN (only V may be read) and NaN guard bands around dprobs.

The CPU half (tests/test_attention_retained_grads_emulated.py) checks that the bound rejects deliberately wrong results, and
replays the module tests below on tests/ops_emulator.py with a float64 restatement answering ops.attention_dprobs.
"""
import contextlib
import warnings

import pytest
import torch

import dropout_ref as D
import test_gpu_attention_elementwise as A
import test_gpu_attention_probs_bwd as PB
import test_gpu_base_model as G
from elementwise import BF16, F32, F64, U, Guarded, _INT, _record, check_bound
from util import TOL_GRAD, cosine, make_cfg, relerr

pytestmark = pytest.mark.gpu

HD = 64
NSEQ = A.NSEQ


# ------------------------------------------------------------------------------------------------ reference
def dprobs_ref(do, v, old):
    """(ref, bound) [NSEQ, H, L, L] float64 from dO, V [NSEQ, H, L, 64] (float64 of bf16) and the old values (None: not
    accumulated)."""
    ref = do @ v.transpose(-1, -2)
    if old is not None:
        ref = old + ref
    bound = U * ref.abs() + 3.0 * (HD + 1) * U * (do.abs() @ v.abs().transpose(-1, -2))
    return ref, bound


class Case:
    def __init__(self, L, heads, accumulate, pitched):
        self.L, self.heads, self.accumulate, self.pitched = L, heads, accumulate, pitched

    @property
    def id(self):
        return "L%d-H%d-acc%d%s" % (self.L, self.heads, self.accumulate, "-pitched" if self.pitched else "")


LENGTHS = [1, 2, 9, 17, 41, 48, 49, 64, 65, 69, 128, 149, 169, 521]


def _cases():
    out = []
    for n, L in enumerate(LENGTHS):
        out.append(Case(L, (1, 3, 12)[n % 3] if L < 512 else 3, n % 2, n % 3 == 1))
    out += [Case(41, 12, 1, True), Case(69, 12, 0, True), Case(169, 1, 1, False), Case(65, 3, 1, True), Case(521, 1, 0, True)]
    return out


CASES = _cases()


def _bits(t):
    return t.detach().cpu().contiguous().view(_INT[t.dtype]).clone()


def case_inputs(case, seed=0):
    """bf16 qkv [NSEQ * L, 3 hid] with NaN Q and K blocks (the kernel reads V only), dctx [NSEQ * L, hid], and the old fp32
    values of dprobs (None unless accumulating)."""
    n, L, hid = NSEQ, case.L, case.heads * HD
    g = torch.Generator().manual_seed(17 * L + case.heads + 1000 * case.accumulate + seed)
    qkv = torch.randn(n * L, 3 * hid, generator=g, dtype=F64)
    qkv[:, :2 * hid] = float("nan")
    dctx = torch.randn(n * L, hid, generator=g, dtype=F64)
    old = torch.randn(n, case.heads, L, L, generator=g).float() if case.accumulate else None
    return qkv.to(BF16), dctx.to(BF16), old


def case_reference(case, qkv, dctx, old):
    _, _, v = A._split(qkv, case.heads)
    (do,) = A._split(dctx, case.heads)
    return dprobs_ref(do, v, None if old is None else old.double())


def _run_case(case, dev):
    from clipbert_b200 import ops
    n, L, H = NSEQ, case.L, case.heads
    hid = H * HD
    qkv, dctx, old = case_inputs(case)
    ld_qkv, ld_ctx = (3 * hid + 64, hid + 40) if case.pitched else (3 * hid, hid)
    xin, din = A._Window(qkv, ld_qkv, dev), A._Window(dctx, ld_ctx, dev)
    runs = []
    for _ in range(2):
        out = Guarded((n, H, L, L), F32, dev, init=None if old is None else old.to(dev))
        ops._call("cb_attention_dprobs", ops._p(xin.t), ld_qkv, ops._p(din.t), ld_ctx, ops._p(out.t), case.accumulate, n, L, H, HD,
                  ops._s())
        torch.cuda.synchronize()
        runs.append(out)
    a, b = runs
    assert torch.equal(_bits(a.buf), _bits(b.buf)), "%s: two identical runs differ" % case.id
    a.check(case.id + " dprobs")
    ref, bound = case_reference(case, qkv, dctx, old)
    _record("dprobs", case.id, check_bound(case.id, a.t.cpu(), ref, bound))


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_attention_dprobs_elementwise(cuda, case):
    _run_case(case, cuda)


def test_case_matrix_covers_lengths_heads_modes_and_pitches():
    assert {c.L for c in CASES} == set(LENGTHS) and {c.heads for c in CASES} == {1, 3, 12}
    assert {c.accumulate for c in CASES} == {0, 1} and {c.pitched for c in CASES} == {False, True}


def test_attention_dprobs_rejects_bad_arguments(cuda):
    from clipbert_b200 import ops
    n, L, H = 2, 41, 3
    hid = H * HD
    qkv = torch.zeros(n * L * 3 * hid + 8, dtype=BF16, device=cuda)
    dctx = torch.zeros(n * L * hid + 8, dtype=BF16, device=cuda)
    dprobs = torch.full((n * H * L * L + 4,), 2.5, device=cuda)
    P = ops._p

    def call(q=qkv, ld_q=3 * hid, d=dctx, ld_c=hid, out=dprobs, acc=0, nseq=n, heads=H, hd=64):
        ops._call("cb_attention_dprobs", P(q), ld_q, P(d), ld_c, P(out), acc, nseq, L, heads, hd, ops._s())

    for kw in (dict(acc=2), dict(acc=-1), dict(heads=0), dict(nseq=0), dict(nseq=65536), dict(heads=65536), dict(out=None),
               dict(d=None)):
        with pytest.raises(RuntimeError, match="bad arguments"):
            call(**kw)
    for kw in (dict(ld_q=3 * hid - 8), dict(ld_c=hid - 8), dict(ld_q=3 * hid + 4), dict(ld_c=hid + 4)):
        with pytest.raises(RuntimeError, match="row pitches"):
            call(**kw)
    for kw in (dict(q=qkv[1:]), dict(d=dctx[1:]), dict(out=dprobs[1:])):
        with pytest.raises(RuntimeError, match="16-byte aligned"):
            call(**kw)
    with pytest.raises(RuntimeError, match="head_dim"):
        call(hd=32)
    torch.cuda.synchronize()
    assert bool((dprobs == 2.5).all())                # nothing was launched


# ------------------------------------------------------------------------------------------------ module
HIDDEN_DIRECT = (3, 12)


def _inputs(size, seed):
    """(grid, ids, mask, L, g) at 224 px (L = 41, padded captions), 448 px (L = 69), 512 tokens (L = 521); small on the CPU."""
    from oracle import synth
    nseq, lt, gh = {"224px": (3, 32, 3), "448px": (2, 20, 7), "512tok": (1, 512, 3), "cpu": (2, 12, 2)}[size]
    g = torch.Generator().manual_seed(seed)
    grid = (torch.randn(nseq, 2, gh, gh, 768, generator=g).abs()).to(torch.bfloat16).float()
    ids, mask = synth.synth_text(nseq, lt, seed=seed + 1)
    return grid, ids, mask, lt + gh * gh, g


def _model(weights, cuda, head=False, **cfg):
    """A differentiable-attention ClipBertBaseModel: standalone, or the bert of a retrieval head."""
    if not head:
        return PB._model(weights, cuda, **cfg)
    import clipbert_b200 as cb
    c = make_cfg(**dict(dict(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0), **cfg))
    c.output_hidden_states = c.output_attentions = True
    h = cb.ClipBertForVideoTextRetrieval(c)
    h.load_state_dict({k[len("transformer."):]: v for k, v in weights.items() if k.startswith("transformer.")})
    h = h.to(cuda)
    h.bert.differentiable_attentions = True
    return h.bert


def _retain_all(seq, hidden, attn):
    for t in (seq,) + tuple(hidden) + tuple(attn):
        t.retain_grad()


def _close(what, got, ref):
    assert got is not None, what
    e, c = relerr(got, ref), cosine(got, ref)
    assert e < TOL_GRAD and c > 0.999, (what, e, c)


def _compare_retained(seq, hidden, attn, rec, layers_r):
    for i in range(12):
        _close("attentions[%d]" % i, attn[i].grad, rec[i].grad)
    for k in range(13):
        _close("hidden_states[%d]" % k, hidden[k].grad, layers_r[k].grad)
    _close("sequence_output", seq.grad, layers_r[12].grad)


def run_retained_grads_against_oracle(cuda, weights, size, direct, head=False):
    """The score from pooled alone, or with direct terms on the maps of PB.ATTN_LAYERS, on hidden_states[3] / [12] and on
    sequence_output: every map, every hidden state and sequence_output retained, against fp32 autograd through the oracle
    with retain_grad() on its recorded maps and layer inputs."""
    from oracle import clipbert_ref as R
    model = _model(weights, cuda, head=head).train()      # dropout p = 0
    grid, ids, mask, L, g = _inputs(size, 111)
    nseq = ids.shape[0]
    wp = torch.randn(nseq, 768, generator=g).to(torch.bfloat16).float()
    W = {i: torch.randn(nseq, 12, L, L, generator=g) for i in PB.ATTN_LAYERS}
    dh = {k: (torch.randn(nseq, L, 768, generator=g) * 0.1).to(torch.bfloat16).float() for k in HIDDEN_DIRECT}
    dseq = (torch.randn(nseq, L, 768, generator=g) * 0.1).to(torch.bfloat16).float()
    sd = {k: (v.clone().requires_grad_(True) if k.startswith("transformer.bert.") else v) for k, v in weights.items()}
    rec, drop = G._oracle_probs()
    seq_r, pooled_r, layers_r = R.clipbert_base_model(ids, grid.clone().requires_grad_(True), mask, sd, return_layers=True, drop=drop)
    for t in list(rec.values()) + list(layers_r):
        t.retain_grad()
    loss_r = (pooled_r * wp).sum()
    if direct:
        loss_r = loss_r + sum((rec[i] * W[i]).sum() for i in PB.ATTN_LAYERS) + (seq_r * dseq).sum()
        loss_r = loss_r + sum((layers_r[k] * v).sum() for k, v in dh.items())
    loss_r.backward()
    seq, pooled, hidden, attn = model(ids.to(cuda), grid.to(cuda).requires_grad_(True), mask.to(cuda))
    _retain_all(seq, hidden, attn)
    loss = (pooled.float() * wp.to(cuda)).sum()
    if direct:
        loss = loss + sum((attn[i] * W[i].to(cuda)).sum() for i in PB.ATTN_LAYERS) + (seq.float() * dseq.to(cuda)).sum()
        loss = loss + sum((hidden[k].float() * v.to(cuda)).sum() for k, v in dh.items())
    loss.backward()
    _compare_retained(seq, hidden, attn, rec, layers_r)
    assert attn[0].grad.dtype == torch.float32 and hidden[0].grad.dtype == torch.bfloat16


@pytest.mark.parametrize("direct", [False, True])
@pytest.mark.parametrize("size", ["224px", "448px", "512tok"])
def test_retained_grads_against_oracle(cuda, weights, size, direct):
    run_retained_grads_against_oracle(cuda, weights, size, direct)


def test_retained_grads_of_a_heads_bert_against_oracle(cuda, weights):
    run_retained_grads_against_oracle(cuda, weights, "224px", True, head=True)


def run_dropped_positions_get_dO_Vt(cuda, weights, size="448px"):
    """Attention dropout 0.1: the maps are post-dropout, so at a dropped position the map is 0 but its gradient is dO V^T, not 0.
    Against the oracle driven by the kernel's own masks (tests/dropout_ref.py at the call's seed and device word)."""
    from oracle import clipbert_ref as R
    p = 0.1
    model = _model(weights, cuda, attention_probs_dropout_prob=p).train()
    eng = model._engine
    grid, ids, mask, L, g = _inputs(size, 113)
    nseq = ids.shape[0]
    wp = torch.randn(nseq, 768, generator=g).to(torch.bfloat16).float()
    seq, pooled, hidden, attn = model(ids.to(cuda), grid.to(cuda), mask.to(cuda))
    seed = (eng._seed_base + eng._call_count * 1000003) & (2 ** 64 - 1)
    word = int(eng._drop_counter.reshape(-1)[0].item())
    _retain_all(seq, hidden, attn)
    (pooled.float() * wp.to(cuda)).sum().backward()
    idx = D.attention_index(nseq, 12, L)
    mult = {i: torch.from_numpy(D.multipliers(D.effective_seed(seed + 16 * (i + 1) + 1, word), idx, p)) for i in range(12)}
    rec = {}

    def drop(site, layer, x):
        if site == "attn_probs":
            x = x * mult[layer]
            rec[layer] = x
        return x
    sd = {k: (v.clone().requires_grad_(True) if k.startswith("transformer.bert.") else v) for k, v in weights.items()}
    seq_r, pooled_r, layers_r = R.clipbert_base_model(ids, grid, mask, sd, return_layers=True, drop=drop)
    for t in list(rec.values()) + list(layers_r):
        t.retain_grad()
    (pooled_r * wp).sum().backward()
    _compare_retained(seq, hidden, attn, rec, layers_r)
    for i in range(12):
        dropped = mult[i] == 0
        assert bool(dropped.any()) and bool((attn[i].detach().cpu()[dropped] == 0).all())
        got, ref = attn[i].grad.cpu()[dropped], rec[i].grad[dropped]
        assert float(got.abs().sum()) > 0
        _close("attentions[%d] at dropped positions" % i, got, ref)


def test_gradient_at_dropped_positions_is_dO_Vt(cuda, weights):
    run_dropped_positions_get_dO_Vt(cuda, weights)


@contextlib.contextmanager
def _deterministic():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _grad_or_none(t):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                # .grad of a non-leaf that retains nothing: torch warns, returns None
        return t.grad


def run_semantics(cuda, weights, size="224px", launches=None):
    """Deterministic mode, dropout on, every run rewound to the same stream position. Nothing retained: no cb_attention_dprobs.
    Retained hidden states and sequence_output: the same launches, in order, and the same parameter and visual_inputs gradient
    bits. One retained map: exactly one cb_attention_dprobs more, the same gradient bits. The outputs not retained keep
    .grad None. With differentiable_attentions off, torch's own error for a tensor without grad.
    launches: the emulated-ops call counter on the CPU replay (the launch list there)."""
    model = _model(weights, cuda, attention_probs_dropout_prob=0.1, hidden_dropout_prob=0.1).train()
    eng = model._engine
    grid, ids, mask, L, g = _inputs(size, 115)
    ids, mask, gdev = ids.to(cuda), mask.to(cuda), grid.to(cuda)
    with torch.no_grad():
        model(ids, gdev, mask)                           # creates the dropout counter
    state = (eng._call_count, int(eng._drop_counter.reshape(-1)[0].item()))
    res = {}
    with _deterministic():
        for what in ("none", "hidden", "map"):
            with torch.no_grad():
                model(ids, gdev, mask)                   # the repack of the bf16 weights a backward leaves due is not timed
            PB._rewind(eng, state)
            model.zero_grad(set_to_none=False)
            gc = gdev.clone().requires_grad_(True)
            before = dict(launches) if launches is not None else None
            with PB._timing(cuda) as ev:
                seq, pooled, hidden, attn = model(ids, gc, mask)
                kept = {"none": (), "hidden": (hidden[3], hidden[12], seq), "map": (attn[5],)}[what]
                for t in kept:
                    t.retain_grad()
                (seq.float().sum() * 0.01 + pooled.float().sum()).backward()
                names = [e[0] for e in ev] if ev is not None else {k: v - before[k] for k, v in launches.items()}
            for t in (seq, pooled) + tuple(hidden) + tuple(attn):
                if not any(t is k for k in kept):
                    assert _grad_or_none(t) is None
            for t in kept:
                assert t.grad is not None
            res[what] = (names, PB._grad_bits(model, gc))
            if what == "map":
                assert float(attn[5].grad.abs().sum()) > 0
    if launches is None:
        assert "cb_attention_dprobs" not in res["none"][0] and res["hidden"][0] == res["none"][0]
        with_map = res["map"][0]
        assert with_map.count("cb_attention_dprobs") == 1
        assert [n for n in with_map if n != "cb_attention_dprobs"] == res["none"][0]
    else:
        assert res["none"][0]["attention_dprobs"] == 0 and res["hidden"][0] == res["none"][0]
        assert res["map"][0] == dict(res["none"][0], attention_dprobs=1)
    for what in ("hidden", "map"):
        for a, b in zip(res["none"][1], res[what][1]):
            assert torch.equal(a, b), what
    off = G._base(weights, cuda).train()
    attn_off = off(ids, gdev.clone().requires_grad_(True), mask)[3]
    with pytest.raises(RuntimeError, match="requires_grad"):
        attn_off[0].retain_grad()


def test_retain_grad_semantics_launches_and_bits(cuda, weights):
    run_semantics(cuda, weights)


def _retained_step(model, ids, gdev, mask, wp):
    model.zero_grad(set_to_none=False)
    seq, pooled, hidden, attn = model(ids, gdev, mask)
    kept = (attn[0], attn[5], attn[11], hidden[0], hidden[7], seq)
    for t in kept:
        t.retain_grad()
    (pooled.float() * wp).sum().add_((attn[5] * 0.5).sum()).backward()
    return kept


def test_cuda_graph_replay_matches_eager(cuda, weights):
    """Retained maps and hidden states with dropout, captured once: a replay rewound to an eager step's position gives that
    step's .grad bits (and parameter gradients)."""
    model = _model(weights, cuda, attention_probs_dropout_prob=0.1, hidden_dropout_prob=0.1).train()
    eng = model._engine
    grid, ids, mask, L, g = _inputs("224px", 117)
    ids, mask, gdev = ids.to(cuda), mask.to(cuda), grid.to(cuda).to(torch.bfloat16)
    wp = torch.randn(ids.shape[0], 768, generator=g).to(cuda)
    params = list(model.parameters())
    with _deterministic():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                _retained_step(model, ids, gdev, mask, wp)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        calls0, w0 = eng._call_count, int(eng._drop_counter.item())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            captured = _retained_step(model, ids, gdev, mask, wp)
        eng._call_count = calls0
        eng._drop_counter.fill_(w0)
        kept = _retained_step(model, ids, gdev, mask, wp)
        torch.cuda.synchronize()
        eager = [t.grad.detach().clone() for t in kept] + [p.grad.detach().clone() for p in params]
        eng._drop_counter.fill_(w0)
        graph.replay()
        torch.cuda.synchronize()
        replay = [t.grad.detach().clone() for t in captured] + [p.grad.detach().clone() for p in params]
    assert float(eager[0].abs().sum()) > 0 and float(eager[3].float().abs().sum()) > 0
    for a, b in zip(eager, replay):
        assert torch.equal(a, b)


def test_deterministic_mode_three_runs_give_the_same_bits(cuda, weights):
    model = _model(weights, cuda, attention_probs_dropout_prob=0.1, hidden_dropout_prob=0.1).train()
    eng = model._engine
    grid, ids, mask, L, g = _inputs("448px", 119)
    ids, mask, gdev = ids.to(cuda), mask.to(cuda), grid.to(cuda)
    wp = torch.randn(ids.shape[0], 768, generator=g).to(cuda)
    with torch.no_grad():
        model(ids, gdev, mask)
    state = (eng._call_count, int(eng._drop_counter.item()))
    runs = []
    with _deterministic():
        for _ in range(3):
            PB._rewind(eng, state)
            kept = _retained_step(model, ids, gdev, mask, wp)
            runs.append([t.grad.detach().clone() for t in kept] + [p.grad.detach().clone() for p in model.parameters()])
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a, b)


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)
