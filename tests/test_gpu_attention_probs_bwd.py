"""cb_attention_probs_bwd, the backward through the attention probabilities ClipBertBaseModel returns, and the module switch
ClipBertBaseModel.differentiable_attentions that uses it.

Kernel, element by element against float64 from the same bf16 Q / K, the forward's own lse (fp32) and the multipliers r of
tests/dropout_ref.py, with G = d loss / d A (A = P r) and dQ0 / dK0 the bf16 values dqkv held before the call:

  P = exp(S - lse) ;  g = r G ;  D_i = sum_j P_ij g_ij ;  dS = P (g - D) ;  dQ = dQ0 + dS K / 8 ;  dK = dK0 + dS^T Q / 8

Bounds, per element (U = 2^-24, first order; S, e_S, E and the bf16 ambiguity amb as in test_gpu_attention_elementwise.py):
  P, g   e_P = P (e_S + E(S - lse)) ;  e_g = U |g| (the product r G)
  D      e_D = sum_j (e_P |g| + P e_g) + (L + 2) U sum_j |P g|  (the products and an fp32 sum of L terms in any order)
  dS     e_dS = P (e_g + e_D + U |g - D|) + e_P |g - D| + U |dS| ;  dS is rounded to bf16 before the products (replayed, with
         the ambiguity amb of a value within e_dS of a bf16 rounding boundary)
  dQ, dK 1 ulp_bf16(ref) + 2 U |ref| + sum amb |B| / 8 + 2 U 3 (L + 1) sum |dS| |B| / 8: the L-long product on mma.sync, the
         fp32 add to the old value and the one rounding to bf16.

The CPU half (tests/test_attention_probs_bwd_emulated.py) checks that the bound rejects deliberately wrong results, and
replays the module tests below on tests/ops_emulator.py with a float64 restatement answering ops.attention_probs_bwd.
"""
import contextlib

import pytest
import torch

import dropout_ref as D
import test_gpu_attention_elementwise as A
import test_gpu_base_model as G
from elementwise import BF16, F32, F64, U, Guarded, _INT, _record, check_bound, ulp_bf16
from util import TOL_GRAD, cosine, relerr

pytestmark = pytest.mark.gpu

HD = 64
NSEQ = A.NSEQ
NAN_PAD = 64                # NaN floats before and after the dprobs / lse windows (keeps 16-byte alignment)


# ------------------------------------------------------------------------------------------------ reference
def probs_bwd_ref(q, k, madd, lse, r, Gr, dq0, dk0, rounded=True):
    """[(dQ, bound), (dK, bound)] as [NSEQ, H, L, 64] float64, from the bf16 Q / K, the kernel's lse, the multipliers r and the
    upstream gradient Gr (float64 of the fp32 values), added to dq0 / dk0. rounded: dS is rounded to bf16 before the products,
    as the tensor-core kernel does (False: the CPU emulator, which keeps it unrounded)."""
    L = q.shape[2]
    S, eS = A._scores(q, k, madd)
    lse = lse.detach().cpu().double()[..., None]
    P = torch.exp(S - lse)
    eP = P * (eS + A._E(S - lse))
    g = r * Gr
    eg = U * g.abs()
    Dv = (P * g).sum(-1, keepdim=True)
    eD = (eP * g.abs() + P * eg).sum(-1, keepdim=True) + (L + 2) * U * (P * g).abs().sum(-1, keepdim=True)
    gd = g - Dv
    dS = P * gd
    edS = P * (eg + eD + U * gd.abs()) + eP * gd.abs() + U * dS.abs()
    dSX, amb = A._inter(dS, edS, rounded)
    depth = 3.0 * (L + 1)
    out = []
    for Am, ambm, B, old in ((dSX, amb, k, dq0), (dSX.transpose(-1, -2), amb.transpose(-1, -2), q, dk0)):
        ref = old + Am @ B * 0.125
        bound = ulp_bf16(ref) + 2.0 * U * ref.abs() + (ambm @ B.abs()) * 0.125 + 2.0 * U * depth * (Am.abs() @ B.abs()) * 0.125
        out.append((ref, bound))
    return out


def _lt(mode, L):
    return {"lt0": 0, "ltL": L, "pad": L - 9 if L > 9 else L}[mode]


class Case:
    def __init__(self, L, lt_mode="pad", p=0.0, heads=None, pattern="randn", pitched=False):
        self.L, self.lt_mode, self.lt, self.p = L, lt_mode, _lt(lt_mode, L), p
        self.heads = heads or (2 if L > 512 else 3)
        self.pattern, self.pitched = pattern, pitched

    @property
    def id(self):
        s = "L%d-%s-p%g-H%d-%s" % (self.L, self.lt_mode, self.p, self.heads, self.pattern)
        return s + ("-pitched" if self.pitched else "")


LENGTHS = [1, 2, 9, 17, 41, 48, 49, 64, 65, 69, 128, 149, 169, 521]


def _cases():
    out = []
    modes = ("pad", "lt0", "ltL")
    for n, L in enumerate(LENGTHS):
        out.append(Case(L, modes[n % 3], p=0.1 if n % 2 else 0.0, pitched=n % 4 == 1))
    out += [Case(41, "pad", p=0.1), Case(169, "pad", p=0.0), Case(65, "ltL", p=0.1)]
    out += [Case(69, "pad", p=0.1, heads=12)]
    out += [Case(L, "pad", p=0.0, pattern="rowconst") for L in (41, 69)]
    out += [Case(L, "pad", p=0.1, pattern="rowconst") for L in (17,)]
    out += [Case(L, "pad", p=0.1, pattern="single") for L in (65, 149)]
    out += [Case(L, "pad", p=0.1, pattern="dropped", pitched=True) for L in (41, 169)]
    return out


CASES = _cases()


def _upstream(case, r, g):
    """G (float64, exactly representable in fp32) for the case's pattern."""
    shape = (NSEQ, case.heads, case.L, case.L)
    if case.pattern == "randn":
        Gr = torch.randn(shape, generator=g, dtype=F64)
    elif case.pattern == "rowconst":                  # dS = 0 at p = 0: dQ / dK stay within rounding of their input
        Gr = torch.randn(shape[:-1] + (1,), generator=g, dtype=F64).expand(shape).contiguous()
    elif case.pattern == "single":
        Gr = torch.zeros(shape, dtype=F64)
        Gr[NSEQ - 1, case.heads - 1, case.L - 1, case.L // 2] = 3.0
    else:                                             # "dropped": non-zero only where the forward dropped
        Gr = torch.randn(shape, generator=g, dtype=F64) * (r == 0).double()
    return Gr.float().double()


def _nan_window(x, dev):
    """A contiguous fp32 tensor with NAN_PAD NaN floats on either side (a read outside it shows)."""
    buf = torch.full((x.numel() + 2 * NAN_PAD,), float("nan"), dtype=F32, device=dev)
    t = buf[NAN_PAD:NAN_PAD + x.numel()].view(x.shape)
    t.copy_(x)
    return t


def _bits(t):
    return t.detach().cpu().contiguous().view(_INT[t.dtype]).clone()


def _run_case(case, dev):
    from clipbert_b200 import ops
    n, L, H = NSEQ, case.L, case.heads
    hid = H * HD
    seed = 777 + L
    word = 0x2345 + L if case.p > 0 else None
    g = torch.Generator().manual_seed(31 * L + H + int(10 * case.p))
    qkv = torch.randn(n * L, 3 * hid, generator=g, dtype=F64).to(BF16)
    mask = A._mask(L, case.lt)
    r = torch.ones(n, H, L, L, dtype=F64) if case.p == 0 else \
        torch.from_numpy(D.multipliers(D.effective_seed(seed, word), D.attention_index(n, H, L), case.p)).double()
    Gr = _upstream(case, r, g)
    dqkv0 = (torch.randn(n * L, 3 * hid, generator=g, dtype=F64) * 0.05).to(BF16)
    ld_qkv, ld_dqkv = (3 * hid + 64, 3 * hid + 24) if case.pitched else (3 * hid, 3 * hid)
    xin = A._Window(qkv, ld_qkv, dev)
    mask_d = mask.to(dev)
    w = None if word is None else torch.tensor([word], dtype=torch.int64, device=dev)
    ops.dropout_offset_bind(w)
    try:
        ctx = torch.empty(n * L, hid, dtype=BF16, device=dev)
        lse_t = torch.empty(n, H, L, dtype=F32, device=dev)
        ops._call("cb_attention_fwd", ops._p(xin.t), ld_qkv, ops._p(mask_d), ops._p(ctx), hid, ops._p(lse_t), n, L, case.lt, H, HD,
                  case.p, seed, ops._s())
        lse = _nan_window(lse_t, dev)
        dprobs = _nan_window(Gr.float(), dev)
        runs = []
        for _ in range(2):
            dqkv = Guarded((n * L, 3 * hid), BF16, dev, ld=ld_dqkv, init=dqkv0.to(dev))
            drow = torch.full((n * H * L,), float("nan"), dtype=F32, device=dev)
            ops._call("cb_attention_probs_bwd", ops._p(xin.t), ld_qkv, ops._p(mask_d), ops._p(lse), ops._p(dprobs), ops._p(drow),
                      ops._p(dqkv.t), ld_dqkv, n, L, case.lt, H, HD, case.p, seed, ops._s())
            torch.cuda.synchronize()
            runs.append(dqkv)
    finally:
        ops.dropout_offset_bind(None)
    a, b = runs
    assert torch.equal(_bits(a.buf), _bits(b.buf)), "%s: two identical runs differ" % case.id
    a.check(case.id + " dqkv")
    got = a.t.cpu()
    assert torch.equal(_bits(got[:, 2 * hid:]), _bits(dqkv0[:, 2 * hid:])), "%s: the V block was written" % case.id
    if case.pattern == "dropped":
        assert torch.equal(_bits(got), _bits(dqkv0)), "%s: G on dropped elements changed dqkv" % case.id
    q, k, _ = A._split(qkv, H)
    dq0, dk0, _ = A._split(dqkv0, H)
    madd = A._madd(mask, L, case.lt)
    (rq, bq), (rk, bk) = probs_bwd_ref(q, k, madd, lse_t, r, Gr, dq0, dk0)
    got_q, got_k = got[:, :hid], got[:, hid:2 * hid]
    _record("probs_bwd", case.id + "-dq", check_bound(case.id + " dq", got_q, A._merge(rq), A._merge(bq)))
    _record("probs_bwd", case.id + "-dk", check_bound(case.id + " dk", got_k, A._merge(rk), A._merge(bk)))
    if case.pattern == "rowconst" and case.p == 0:
        for got_x, old in ((got_q, dqkv0[:, :hid]), (got_k, dqkv0[:, hid:2 * hid])):
            assert bool(((got_x.double() - old.double()).abs() <= ulp_bf16(old.double())).all()), case.id
    return got


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_attention_probs_bwd_elementwise(cuda, case):
    _run_case(case, cuda)


def test_case_matrix_covers_the_lengths_masks_and_patterns():
    assert {c.L for c in CASES} == set(LENGTHS)
    assert {c.lt_mode for c in CASES} == {"pad", "lt0", "ltL"} and {c.p for c in CASES} == {0.0, 0.1}
    assert {c.pattern for c in CASES} == {"randn", "rowconst", "single", "dropped"}
    assert any(c.heads == 12 for c in CASES) and any(c.pitched for c in CASES)


def test_attention_probs_bwd_rejects_bad_arguments(cuda):
    from clipbert_b200 import ops
    n, L = 2, 41
    hid = G.HEADS * 64
    qkv, mask, lt = G._qkv_case(L, False, 3, n, cuda)
    lse = torch.zeros(n, G.HEADS, L, device=cuda)
    dprobs = torch.zeros(n * G.HEADS * L * L + 4, device=cuda)
    drow = torch.zeros(n * G.HEADS * L, device=cuda)
    dqkv = torch.zeros(n * L * 3 * hid + 8, dtype=BF16, device=cuda)
    P = ops._p

    def call(q=qkv, ld_q=3 * hid, d=dprobs, dq=dqkv, ld_dq=3 * hid, nseq=n, lt_=lt, heads=G.HEADS, hd=64, dr=drow):
        ops._call("cb_attention_probs_bwd", P(q), ld_q, P(mask), P(lse), P(d), P(dr), P(dq), ld_dq, nseq, L, lt_, heads, hd, 0.0, 1,
                  ops._s())

    before = dqkv.clone()
    for kw in (dict(lt_=L + 1), dict(lt_=-1), dict(heads=0), dict(nseq=65536), dict(heads=65536), dict(dr=None)):
        with pytest.raises(RuntimeError, match="bad arguments"):
            call(**kw)
    for kw in (dict(ld_q=3 * hid - 8), dict(ld_dq=3 * hid - 8), dict(ld_q=3 * hid + 4)):
        with pytest.raises(RuntimeError, match="row pitches"):
            call(**kw)
    for kw in (dict(q=qkv.view(-1)[1:]), dict(dq=dqkv[1:]), dict(d=dprobs[1:])):
        with pytest.raises(RuntimeError, match="16-byte aligned"):
            call(**kw)
    with pytest.raises(RuntimeError, match="head_dim"):
        call(hd=32)
    torch.cuda.synchronize()
    assert torch.equal(dqkv, before)                  # nothing was launched


# ------------------------------------------------------------------------------------------------ module
ATTN_LAYERS = (0, 5, 11)


def _module_case(size):
    """(nseq, lt, gh) of the module cases: 224 px (L = 41, padded captions), 448 px (L = 69); small on the CPU replay."""
    return {"224px": (3, 32, 3), "448px": (2, 20, 7), "cpu": (2, 12, 2)}[size]


def _inputs(size, seed):
    from oracle import synth
    nseq, lt, gh = _module_case(size)
    g = torch.Generator().manual_seed(seed)
    grid = (torch.randn(nseq, 2, gh, gh, 768, generator=g).abs()).to(torch.bfloat16).float()
    ids, mask = synth.synth_text(nseq, lt, seed=seed + 1)
    L = lt + gh * gh
    W = {i: torch.randn(nseq, 12, L, L, generator=g) for i in ATTN_LAYERS}
    return grid, ids, mask, L, W, g


def _model(weights, cuda, **cfg):
    m = G._base(weights, cuda, **cfg)
    m.differentiable_attentions = True
    return m


def _compare_grads(model, sd, gc, gr):
    assert gc.grad is not None and relerr(gc.grad, gr.grad) < TOL_GRAD and cosine(gc.grad, gr.grad) > 0.999, relerr(gc.grad, gr.grad)
    bad, checked = [], 0
    for name, p in model.named_parameters():
        ref = sd["transformer.bert." + name].grad
        if ref is None or float(ref.abs().sum()) == 0.0:
            assert p.grad is None or float(p.grad.abs().sum()) == 0.0, name
            continue
        if name.endswith("attention.self.key.bias"):      # mathematically zero: rounding noise on both sides
            continue
        e, c = relerr(p.grad, ref), cosine(p.grad, ref)
        checked += 1
        if not (e < TOL_GRAD and c > 0.999):
            bad.append((name, e, c))
    assert not bad, bad[:10]
    return checked


def run_attention_loss_gradients(cuda, weights, size, with_outputs):
    """A loss on the attentions of layers 0, 5 and 11 (alone, or with d sequence, d pooled and d hidden-state terms) into every
    transformer parameter and visual_inputs, against fp32 autograd through the oracle, whose drop hook hands out each layer's
    probabilities as autograd tensors."""
    from oracle import clipbert_ref as R
    model = _model(weights, cuda).train()                 # dropout p = 0 (see G._base)
    grid, ids, mask, L, W, g = _inputs(size, 91)
    nseq = ids.shape[0]
    dseq, dpool = torch.randn(nseq, L, 768, generator=g) * 0.1, torch.randn(nseq, 768, generator=g)
    dh = {3: torch.randn(nseq, L, 768, generator=g) * 0.1, 12: torch.randn(nseq, L, 768, generator=g) * 0.1}
    dseq, dpool = dseq.to(torch.bfloat16).float(), dpool.to(torch.bfloat16).float()
    dh = {k: v.to(torch.bfloat16).float() for k, v in dh.items()}
    sd = {k: (v.clone().requires_grad_(True) if k.startswith("transformer.bert.") else v) for k, v in weights.items()}
    gr = grid.clone().requires_grad_(True)
    rec, drop = G._oracle_probs()
    seq_r, pooled_r, layers_r = R.clipbert_base_model(ids, gr, mask, sd, return_layers=True, drop=drop)
    loss_r = sum((rec[i] * W[i]).sum() for i in ATTN_LAYERS)
    if with_outputs:
        loss_r = loss_r + (seq_r * dseq).sum() + (pooled_r * dpool).sum() + sum((layers_r[k] * v).sum() for k, v in dh.items())
    loss_r.backward()
    gc = grid.to(cuda).requires_grad_(True)
    seq, pooled, hidden, attn = model(ids.to(cuda), gc, mask.to(cuda))
    assert all(a.requires_grad for a in attn)
    loss = sum((attn[i] * W[i].to(cuda)).sum() for i in ATTN_LAYERS)
    if with_outputs:
        loss = loss + (seq.float() * dseq.to(cuda)).sum() + (pooled.float() * dpool.to(cuda)).sum()
        loss = loss + sum((hidden[k].float() * v.to(cuda)).sum() for k, v in dh.items())
    loss.backward()
    checked = _compare_grads(model, sd, gc, gr)
    assert checked >= (12 * 15 + 2 if with_outputs else 12 * 4)


@pytest.mark.parametrize("with_outputs", [False, True])
@pytest.mark.parametrize("size", ["224px", "448px"])
def test_attention_loss_gradients_against_oracle(cuda, weights, size, with_outputs):
    run_attention_loss_gradients(cuda, weights, size, with_outputs)


def _grad_bits(model, gc):
    return [p.grad.detach().clone() for p in model.parameters()] + [gc.grad.detach().clone()]


def _rewind(eng, state):
    eng._call_count = state[0]
    eng._drop_counter.fill_(state[1])


def run_dropped_positions_do_not_matter(cuda, weights, size="448px"):
    """Train mode, attention dropout 0.1: a G that differs only where the returned attention is zero (the dropped elements)
    gives the same bits in every gradient (deterministic mode: a fixed accumulation order, same masks by rewinding the
    stream)."""
    model = _model(weights, cuda, attention_probs_dropout_prob=0.1, hidden_dropout_prob=0.1).train()
    eng = model._engine
    grid, ids, mask, L, W, g = _inputs(size, 93)
    ids, mask, gdev = ids.to(cuda), mask.to(cuda), grid.to(cuda)
    out = []
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        with torch.no_grad():
            model(ids, gdev, mask)                           # creates the dropout counter
        state = (eng._call_count, int(eng._drop_counter.reshape(-1)[0].item()))
        for variant in range(2):
            _rewind(eng, state)
            model.zero_grad(set_to_none=False)
            gc = gdev.clone().requires_grad_(True)
            seq, pooled, hidden, attn = model(ids, gc, mask)
            loss = (seq.float() * 0.01).sum()
            for i in ATTN_LAYERS:
                w = W[i].to(cuda)
                if variant:
                    dropped = attn[i].detach() == 0
                    assert bool(dropped.any())
                    w = torch.where(dropped, w + 5.0, w)
                loss = loss + (attn[i] * w).sum()
            loss.backward()
            out.append(_grad_bits(model, gc))
    finally:
        torch.use_deterministic_algorithms(prev)
    for a, b in zip(*out):
        assert torch.equal(a, b)


def test_gradient_at_dropped_positions_changes_nothing(cuda, weights):
    run_dropped_positions_do_not_matter(cuda, weights)


@contextlib.contextmanager
def _timing(cuda):
    from clipbert_b200 import ops
    ev = [] if cuda.type == "cuda" else None
    ops.set_op_timing(ev)
    try:
        yield ev
    finally:
        ops.set_op_timing(None)


def run_switch_semantics(cuda, weights, size="224px", launches=None):
    """Default: attentions do not require grad. Switch on, no loss on the attentions: the same launches (names, in order) and
    the same gradient bits as the switch off (deterministic mode). Under torch.no_grad the attentions are not differentiable.
    launches: the emulated-ops call counter on the CPU replay (the launch list there)."""
    grid, ids, mask, L, W, g = _inputs(size, 95)
    ids, mask = ids.to(cuda), mask.to(cuda)
    base = G._base(weights, cuda).train()
    assert base.differentiable_attentions is False
    assert not base(ids, grid.clone().to(cuda).requires_grad_(True), mask)[3][0].requires_grad
    res = []
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for on in (False, True):
            model = G._base(weights, cuda).train()
            model.differentiable_attentions = on
            gc = grid.clone().to(cuda).requires_grad_(True)
            before = dict(launches) if launches is not None else None
            with _timing(cuda) as ev:
                seq, pooled, hidden, attn = model(ids, gc, mask)
                assert attn[0].requires_grad == on
                (seq.float().sum() * 0.01 + pooled.float().sum()).backward()
                names = [e[0] for e in ev] if ev is not None else {k: v - before[k] for k, v in launches.items()}
            res.append((names, _grad_bits(model, gc)))
            with torch.no_grad():
                assert not any(a.requires_grad for a in model(ids, gc, mask)[3])
    finally:
        torch.use_deterministic_algorithms(prev)
    assert res[0][0] == res[1][0]
    for a, b in zip(res[0][1], res[1][1]):
        assert torch.equal(a, b)


def test_switch_off_and_unused_attentions_change_nothing(cuda, weights):
    run_switch_semantics(cuda, weights)


def run_head_bert_gradients_land_in_the_flat_buffer(cuda, weights, size="224px"):
    """model.transformer.bert inside a head: the switch on head.bert, and an attention loss writes its gradients into the
    head's flat gradient buffer (what the optimizer and the all-reduce read)."""
    import clipbert_b200 as cb
    from util import make_cfg
    cfg = make_cfg(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    cfg.output_attentions = True
    head = cb.ClipBertForVideoTextRetrieval(cfg)
    head.load_state_dict({k[len("transformer."):]: v for k, v in weights.items() if k.startswith("transformer.")})
    head = head.to(cuda).train()
    head.bert.differentiable_attentions = True
    grid, ids, mask, L, W, g = _inputs(size, 97)
    seq, pooled, attn = head.bert(ids.to(cuda), grid.to(cuda), mask.to(cuda))
    (attn[5] * W[5].to(cuda)).sum().backward()
    flat = head._flat
    lo, hi = flat.grad.data_ptr(), flat.grad.data_ptr() + 4 * flat.grad.numel()
    for p in head.bert.parameters():
        assert p.grad is None or lo <= p.grad.data_ptr() < hi
    q5, q6 = head.bert.encoder.layer[5].attention.self.query.weight, head.bert.encoder.layer[6].attention.self.query.weight
    assert float(q5.grad.abs().sum()) > 0 and float(q6.grad.abs().sum()) == 0
    assert float(head.bert.encoder.layer[5].attention.self.value.weight.grad.abs().sum()) == 0
    assert float(head.bert.encoder.layer[4].attention.self.value.weight.grad.abs().sum()) > 0


def test_head_bert_attention_gradients_land_in_the_flat_buffer(cuda, weights):
    run_head_bert_gradients_land_in_the_flat_buffer(cuda, weights)


def test_cuda_graph_replay_matches_eager(cuda, weights):
    """An attention loss with dropout, captured once: a replay rewound to an eager step's position gives that step's bits."""
    model = _model(weights, cuda, attention_probs_dropout_prob=0.1, hidden_dropout_prob=0.1).train()
    eng = model._engine
    grid, ids, mask, L, W, g = _inputs("224px", 99)
    ids, mask, gdev = ids.to(cuda), mask.to(cuda), grid.to(cuda).to(torch.bfloat16)
    Wd = {i: w.to(cuda) for i, w in W.items()}
    params = list(model.parameters())

    def step():
        model.zero_grad(set_to_none=False)
        seq, pooled, hidden, attn = model(ids, gdev, mask)
        loss = seq.float().sum() * 0.01 + sum((attn[i] * Wd[i]).sum() for i in ATTN_LAYERS)
        loss.backward()
        return loss

    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                step()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        calls0, w0 = eng._call_count, int(eng._drop_counter.item())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            step()
        eng._call_count = calls0
        eng._drop_counter.fill_(w0)
        step()
        torch.cuda.synchronize()
        eager = [p.grad.detach().clone() for p in params]
        eng._drop_counter.fill_(w0)
        graph.replay()
        torch.cuda.synchronize()
        replay = [p.grad.detach().clone() for p in params]
    finally:
        torch.use_deterministic_algorithms(prev)
    assert float(eager[0].abs().sum()) > 0
    for a, b in zip(eager, replay):
        assert torch.equal(a, b)


def test_deterministic_mode_three_runs_give_the_same_bits(cuda, weights):
    model = _model(weights, cuda, attention_probs_dropout_prob=0.1, hidden_dropout_prob=0.1).train()
    eng = model._engine
    grid, ids, mask, L, W, g = _inputs("448px", 101)
    ids, mask, gdev = ids.to(cuda), mask.to(cuda), grid.to(cuda)
    with torch.no_grad():
        model(ids, gdev, mask)
    state = (eng._call_count, int(eng._drop_counter.item()))
    runs = []
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(3):
            _rewind(eng, state)
            model.zero_grad(set_to_none=False)
            gc = gdev.clone().requires_grad_(True)
            seq, pooled, hidden, attn = model(ids, gc, mask)
            sum((attn[i] * W[i].to(cuda)).sum() for i in ATTN_LAYERS).backward()
            runs.append(_grad_bits(model, gc))
    finally:
        torch.use_deterministic_algorithms(prev)
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a, b)


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)
