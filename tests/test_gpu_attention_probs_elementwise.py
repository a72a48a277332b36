"""cb_attention_probs, the kernel behind every attention map ClipBertBaseModel hands out (output_attentions, the maps module
hooks see, A_k of layerwise_autograd's split at a differentiable map), element by element against float64.

Reference, from the same bf16 Q / K, the int64 text mask, the forward's OWN lse (fp32, as the kernel reads it) and the fp32
dropout multipliers r of tests/dropout_ref.py:

  S_ij = Q_i . K_j / 8 + madd_j  (madd_j = -10000 for a masked text key, else 0) ;  A = exp(S - lse) r

The kernel writes A in fp32 without a bf16 rounding (csrc/attention_tc.cu, attn_tc_probs_kernel).

Bound, per element (U = 2^-24; S, e_S and E as in test_gpu_attention_elementwise.py):
  |got - A| <= P (e_S + E(S - lse)) r + U |P r| + 2^-126 max(r, 1)
  e_S: the mma.sync dot product of 64 exact bf16 products and the roundings of s / 8 + madd; E: __expf, the subtraction of
  lse; U |P r|: the multiplication by r. The floor: --use_fast_math flushes a subnormal __expf result to zero, before the
  multiplication by r (<= 1 / (1 - p)).
Dropped elements (r = 0) must be +0 exactly, bit for bit; every element the mask keeps and whose reference is above the
floor must be non-zero, so the dropped set is exactly the one tests/dropout_ref.py restates.

Cases: L from 1 to 521, at each tile and staging regime (L mod 4 != 0 shifts the staged rows of tc_store_staged_rows);
heads 1, 3, 12, 16; lt = 0, L - 9, L; rows whose every text key is masked and sequences whose every key is masked; p = 0,
0.1, 1 and a bound dropout word; qkv with a row pitch, NaN in the pitch columns and in 64 rows either side, lse inside NaN;
the output inside guard bands (Guarded). Each case runs twice and must give the same bits; the rows with a live key sum to
one at p = 0, and the maps times V give the forward's ctx. Every case prints "RATIO probs <case> <max err / bound>". In the
peaked cases the largest ratio is close to 1 by construction: it is an element just below 2^-126 that the kernel flushes to
zero, whose error is the reference itself.

The maps a model returns: ClipBertBaseModel in train mode at 224 px (L = 41) and 448 px (L = 69), on the default path, on
the module path (an observe-only hook on every module) and with layerwise_autograd. Every layer's map is checked as above,
from the qkv and lse the engine's test capture (_capture["attn<i>"]) records where the maps are made, under the layer's
seed derived again from the engine's counters and the device word the call bound. Only the maps are checked here: the
backward arithmetic the module path and layerwise_autograd add of their own (the FFN and pooler splits, the residual
hand-over, the chain of the split at a map, the intakes of replaced tensors) is not.

The CPU half runs the unpitched cases and the three model paths (at CPU size) through the emulator's restatement
(tests/test_base_model_emulated.py, answering ops.attention_probs in the CPU replays). For the kernel cases that
restatement is the reference's own float64 formula, so those runs check the harness (shapes, masks, multipliers, the bound
word), not an independent computation; the model runs check that every path hands out the map of its own layer's qkv, lse,
seed and word. What shows that the bound rejects wrong results are the self-tests: three planted faults (an lse from the
neighbouring row, a key mask shifted by one key, a 1 % error confined to probabilities below 1e-4) must be rejected, and
the last one passes the normwise bound this kernel's earlier test used.
"""
import pytest
import torch

import dropout_ref as D
import ops_emulator as E
import test_base_model_emulated as BE
import test_gpu_attention_elementwise as A
import test_gpu_attention_probs_bwd as PB
from elementwise import BF16, F32, F64, U, Guarded, _INT, _record, check_bound
from util import TOL_BF16_OP, relerr

HD = 64
NSEQ = A.NSEQ
FLOOR = 2.0 ** -126                 # the smallest normal fp32: __expf flushes subnormal results to zero


# ------------------------------------------------------------------------------------------------ reference
def probs_ref(q, k, madd, lse, r):
    """(A, bound) [NSEQ, H, L, L] float64 from the bf16 Q / K [NSEQ, H, L, 64], the additive key mask, the kernel's lse and
    the multipliers r (see the module docstring)."""
    S, eS = A._scores(q, k, madd)
    lse = lse.detach().cpu().double()[..., None]
    P = torch.exp(S - lse)
    ref = P * r
    bound = P * (eS + A._E(S - lse)) * r + U * ref.abs() + FLOOR * r.clamp_min(1.0)
    return ref, bound


# ------------------------------------------------------------------------------------------------ cases
class Case:
    def __init__(self, L, lt_mode="pad", p=0.0, heads=3, pitched=False, word=False, text_masked=False, peaked=False):
        self.L, self.lt_mode, self.lt, self.p, self.heads = L, lt_mode, PB._lt(lt_mode, L), p, heads
        self.pitched, self.word, self.text_masked, self.peaked = pitched, word, text_masked, peaked
        assert not text_masked or 0 < self.lt < L, "every text key masked with visual keys live: 0 < lt < L"

    @property
    def id(self):
        s = "L%d-lt%d-p%g-H%d" % (self.L, self.lt, self.p, self.heads)
        for flag, name in ((self.peaked, "peaked"), (self.text_masked, "textmasked"), (self.pitched, "pitched"),
                           (self.word, "word")):
            if flag:
                s += "-" + name
        return s


LENGTHS = [1, 2, 3, 5, 9, 17, 41, 48, 63, 64, 65, 69, 127, 128, 129, 169, 521]
HEADS = (3, 12, 1, 16)


def _cases():
    out = []
    modes = ("pad", "lt0", "ltL")
    for n, L in enumerate(LENGTHS):
        out.append(Case(L, modes[n % 3], p=0.1 if n % 2 else 0.0, heads=3 if L > 512 else HEADS[n % 4], pitched=n % 4 == 1,
                        peaked=n % 3 == 2))
    out += [Case(L, "pad", p=1.0) for L in (5, 41, 65, 169)]
    out += [Case(L, "pad", p=0.1, word=True, heads=12) for L in (9, 48, 69, 129)]
    out += [Case(L, "pad", p=0.1 if n % 2 else 0.0, text_masked=True) for n, L in enumerate((17, 41, 64, 69, 128, 169))]
    out += [Case(L, "ltL", p=0.1, heads=h) for L in (41, 169) for h in (1, 16)]
    out += [Case(L, "pad", p=0.1, pitched=True, peaked=n % 2 == 1) for n, L in enumerate((3, 63, 127, 521))]
    out += [Case(L, "ltL", p=0.1, pitched=True, word=True) for L in (65, 128)]
    out += [Case(L, "lt0", p=0.1) for L in (65, 128)]
    return out


CASES = _cases()
EMU_CASES = [c for c in CASES if not c.pitched]           # the restatement reads an unpitched qkv


def _mask(case):
    """A._mask (masked tail keys, a masked first 64-key tile at long L, sequence 2 entirely masked when lt = L); with
    text_masked, sequence 2's every text key is masked while its visual keys stay live."""
    m = A._mask(case.L, case.lt)
    if case.text_masked:
        m[2] = 0
    return m


def _inputs(case):
    g = torch.Generator().manual_seed(7 * case.L + case.heads + int(10 * case.p) + 3 * case.text_masked)
    qkv = torch.randn(NSEQ * case.L, 3 * case.heads * HD, generator=g, dtype=F64)
    if case.peaked:                     # |S| up to ~100: probabilities over many decades, down to the flush floor
        qkv[:, :2 * case.heads * HD] *= 4
    return qkv.to(BF16), _mask(case)


def _bits(t):
    return t.detach().cpu().contiguous().view(_INT[t.dtype]).clone()


def _check_map(kind, tag, got, q, k, madd, lse, r):
    """got (fp32 [nseq, H, L, L]) against probs_ref: dropped elements +0 exactly, kept elements above the flush floor non-zero
    (the dropped set is the restated one), every element within its bound. Prints the RATIO line."""
    got = got.detach().cpu()
    ref, bound = probs_ref(q, k, madd, lse, r)
    dropped = r == 0
    assert bool((_bits(got)[dropped] == 0).all()), "%s: a dropped element is not +0" % tag
    assert bool((got[~dropped & (ref > 2.0 * FLOOR)] != 0).all()), "%s: a kept element is zero" % tag
    _record(kind, tag, check_bound(tag + " probs", got, ref, bound))


# ------------------------------------------------------------------------------------------------ running a case
def _run(be, case, qkv, mask, seed, word):
    """The forward (for ctx and lse), then cb_attention_probs into Guarded outputs: two runs on the device, one emulated."""
    n, L, H = NSEQ, case.L, case.heads
    hid = H * HD
    dev = be.dev
    with A._bound_word(be, word):
        if be.emulated:
            ctx = torch.empty(n * L, hid, dtype=BF16)
            lse = torch.empty(n, H, L, dtype=F32)
            E.attention_fwd(qkv, mask, ctx, lse, n, L, case.lt, H, case.p, seed)
            out = Guarded((n, H, L, L), F32, dev)
            BE.attention_probs(qkv, mask, lse, out.t, n, L, case.lt, H, case.p, seed)
            return ctx, lse, [out]
        from clipbert_b200 import ops
        ld = 3 * hid + 64 if case.pitched else 3 * hid
        xin = A._Window(qkv, ld, dev)
        mask_d = mask.to(dev)
        ctx = torch.empty(n * L, hid, dtype=BF16, device=dev)
        lse_t = torch.empty(n, H, L, dtype=F32, device=dev)
        ops._call("cb_attention_fwd", ops._p(xin.t), ld, ops._p(mask_d), ops._p(ctx), hid, ops._p(lse_t), n, L, case.lt, H, HD,
                  case.p, seed, ops._s())
        lse = PB._nan_window(lse_t, dev)
        outs = []
        for _ in range(2):
            out = Guarded((n, H, L, L), F32, dev)
            ops._call("cb_attention_probs", ops._p(xin.t), ld, ops._p(mask_d), ops._p(lse), ops._p(out.t), n, L, case.lt, H, HD,
                      case.p, seed, ops._s())
            outs.append(out)
        torch.cuda.synchronize()
        return ctx, lse_t, outs


def _probs_case(be, case):
    L, H = case.L, case.heads
    seed = 2024 + L
    word = 0x5A5A + L if case.word else None
    qkv, mask = _inputs(case)
    ctx, lse, outs = _run(be, case, qkv, mask, seed, word)
    for out in outs:
        out.check(case.id + " probs")
    if len(outs) == 2:
        assert torch.equal(_bits(outs[0].buf), _bits(outs[1].buf)), "%s: two identical runs differ" % case.id
    got = outs[0].t.cpu()
    r = A._mult(case, seed, word)
    q, k, v = A._split(qkv, H)
    madd = A._madd(mask, L, case.lt)
    _check_map("probs", case.id, got, q, k, madd, lse, r)
    if case.p >= 1:
        assert bool((r == 0).all())
    if case.p == 0:                                       # sequences with a live key: rows of a softmax
        live = (madd == 0).any(-1)
        assert float((got.double().sum(-1)[live] - 1).abs().max()) < 2e-5, case.id
    if case.p < 1:                                        # the maps times V give the forward's ctx
        pv = A._merge(got.double() @ v)
        assert relerr(pv, ctx.float()) < 2 * TOL_BF16_OP, (case.id, relerr(pv, ctx.float()))


@pytest.mark.parametrize("be_name,case", [pytest.param("device", c, marks=pytest.mark.gpu, id="device-" + c.id) for c in CASES]
                         + [pytest.param("emulator", c, id="emulator-" + c.id) for c in EMU_CASES])
def test_attention_probs_elementwise(be_name, case):
    if be_name == "device" and not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    _probs_case(A.Backend(be_name), case)


def test_case_matrix_covers_the_lengths_heads_masks_and_dropout():
    assert [c.L for c in CASES[:len(LENGTHS)]] == LENGTHS and {c.L % 4 for c in CASES} == {0, 1, 2, 3}
    assert {c.heads for c in CASES} == set(HEADS)
    assert {c.lt_mode for c in CASES} == {"pad", "lt0", "ltL"} and {c.p for c in CASES} == {0.0, 0.1, 1.0}
    assert any(c.word for c in CASES) and any(c.pitched for c in CASES) and any(c.text_masked for c in CASES)
    assert {c.peaked for c in CASES if c.L > 64} == {False, True}
    # every key of sequence 2 masked (lt = L), with and without dropout, on one tile and on several
    assert {(c.L > 64, c.p > 0) for c in CASES if c.lt == c.L and c.L > 1} == {(False, False), (False, True), (True, False),
                                                                              (True, True)}
    assert len({c.id for c in CASES}) == len(CASES)


# ------------------------------------------------------------------------------------------------ the maps a model returns
MAP_PATHS = ("default", "module", "layerwise")


def run_returned_maps(dev, weights, size, path):
    """Every layer's map that ClipBertBaseModel returns in train mode (attention and hidden dropout 0.1, differentiable maps),
    element by element against probs_ref from that layer's own qkv and lse, which the engine's test capture records where the
    maps are made (on every path). The seed, seed + 16 (i + 1) + 1, is derived again from the engine's counters, and the
    multipliers from it and the device word the call bound. default: no hook; module: an observe-only forward hook on every
    hookable module (the module path); layerwise: layerwise_autograd, no hook (the split at each map)."""
    import test_gpu_attention_retained_grads as RG
    import test_gpu_transformer_hooks as TH
    model = PB._model(weights, dev, attention_probs_dropout_prob=0.1, hidden_dropout_prob=0.1).train()
    model.layerwise_autograd = path == "layerwise"
    eng = model._engine
    grid, ids, mask, L, _ = RG._inputs(size, 141)
    nseq, lt = ids.shape
    handles = [m.register_forward_hook(lambda *a: None) for _, m in TH.site_modules(model)] if path == "module" else []
    eng._capture = {}
    try:
        seq, pooled, hidden, attn = model(ids.to(dev), grid.to(dev).requires_grad_(True), mask.to(dev))
    finally:
        cap, eng._capture = eng._capture, None
        for h in handles:
            h.remove()
    assert len(attn) == 12 and all(a.requires_grad for a in attn)
    seed = (eng._seed_base + eng._call_count * 1000003) & (2 ** 64 - 1)
    word = int(eng._drop_counter.reshape(-1)[0].item())
    madd = torch.cat([(mask == 0).double() * -10000.0, torch.zeros(nseq, L - lt, dtype=F64)], 1)
    idx = D.attention_index(nseq, 12, L)
    for i in range(12):
        c = cap["attn%d" % i]
        assert c["seed"] == seed + 16 * (i + 1) + 1 and int(c["word"].reshape(-1)[0].item()) == word, i
        q, k = (t.reshape(nseq, L, 12, HD).permute(0, 2, 1, 3) for t in c["qkv"].cpu().double().view(nseq, L, 3, 768).unbind(2)[:2])
        r = torch.from_numpy(D.multipliers(D.effective_seed(seed + 16 * (i + 1) + 1, word), idx, 0.1)).double()
        _check_map("maps-" + path, "%s-%s-layer%d" % (size, path, i), attn[i], q, k, madd, c["lse"], r)


@pytest.mark.gpu
@pytest.mark.parametrize("path", MAP_PATHS)
@pytest.mark.parametrize("size", ["224px", "448px"])
def test_returned_maps_elementwise(cuda, weights, size, path):
    run_returned_maps(cuda, weights, size, path)


@pytest.mark.parametrize("path", MAP_PATHS)
def test_returned_maps_elementwise_on_emulated_ops(weights, path):
    import test_transformer_hooks_emulated as THE
    with THE.emulated() as calls:                         # the emulated ops of every path, the module path's included
        run_returned_maps(torch.device("cpu"), weights, "cpu", path)
    assert calls["attention_probs"] == 12


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)


# ------------------------------------------------------------------------------------------------ CPU self-tests
def _fault_setup(L=65, heads=2, p=0.1, seed=99):
    case = Case(L, "pad", p=p, heads=heads, peaked=True)
    qkv, mask = _inputs(case)
    q, k, _ = A._split(qkv, heads)
    madd = A._madd(mask, L, case.lt)
    lse = torch.logsumexp(q @ k.transpose(-1, -2) / 8.0 + madd[:, None, None, :], -1).float()
    r = A._mult(case, seed, None)
    ref, bound = probs_ref(q, k, madd, lse, r)
    return dict(case=case, q=q, k=k, mask=mask, madd=madd, lse=lse, r=r, ref=ref, bound=bound)


def _ok(s, got64):
    check_bound("fault probs", got64.float(), s["ref"], s["bound"])


def _old_bound_passes(s, got64):
    """The normwise check this kernel's earlier test made: max |got - ref| < 2e-5 + 2e-4 max |ref|."""
    got = got64.float().double()
    return float((got - s["ref"]).abs().max()) < 2e-5 + 2e-4 * float(s["ref"].abs().max())


def test_reference_accepts_itself_in_fp32_and_is_the_softmax():
    """The reference rounded once to fp32 passes its own bound; from the exact log-sum-exp at p = 0 it is softmax(S)."""
    s = _fault_setup()
    _ok(s, s["ref"])
    s0 = _fault_setup(p=0.0)
    S = s0["q"] @ s0["k"].transpose(-1, -2) / 8.0 + s0["madd"][:, None, None, :]
    ref, _ = probs_ref(s0["q"], s0["k"], s0["madd"], torch.logsumexp(S, -1), s0["r"])
    assert torch.allclose(ref, torch.softmax(S, -1), rtol=1e-12, atol=0)


def test_fault_lse_of_the_neighbouring_row_is_rejected():
    s = _fault_setup()
    lse = torch.roll(s["lse"], 1, dims=-1)
    with pytest.raises(AssertionError, match="out of bound"):
        _ok(s, probs_ref(s["q"], s["k"], s["madd"], lse, s["r"])[0])


def test_fault_key_mask_shifted_by_one_key_is_rejected():
    s = _fault_setup()
    c = s["case"]
    mask = torch.roll(s["mask"], 1, dims=1)
    assert not torch.equal(mask, s["mask"])
    madd = A._madd(mask, c.L, c.lt)
    with pytest.raises(AssertionError, match="out of bound"):
        _ok(s, probs_ref(s["q"], s["k"], madd, s["lse"], s["r"])[0])


def test_fault_one_percent_on_probabilities_below_1e4_is_rejected_but_passes_the_old_normwise_bound():
    s = _fault_setup()
    small = (s["ref"] > 0) & (s["ref"] < 1e-4)
    assert bool(small.any())
    got = torch.where(small, s["ref"] * 1.01, s["ref"])
    with pytest.raises(AssertionError, match="out of bound"):
        _ok(s, got)
    assert _old_bound_passes(s, got)


def test_fault_dropped_element_kept_is_caught():
    """Elements the mask drops, written as their undropped probability, are out of bound."""
    s = _fault_setup()
    P = probs_ref(s["q"], s["k"], s["madd"], s["lse"], torch.ones_like(s["r"]))[0]
    with pytest.raises(AssertionError, match="out of bound"):
        _ok(s, torch.where(s["r"] == 0, P, s["ref"]))


def test_emulated_restatement_reads_the_given_lse_and_word():
    """BE.attention_probs, as the CPU replays answer ops.attention_probs: a perturbed lse and a bound word change its output."""
    case = Case(41, "pad", p=0.1, heads=2)
    qkv, mask = _inputs(case)
    n, L, H = NSEQ, case.L, case.heads
    ctx, lse = torch.empty(n * L, H * HD, dtype=BF16), torch.empty(n, H, L)
    E.attention_fwd(qkv, mask, ctx, lse, n, L, case.lt, H, 0.0, 0)
    outs = []
    for l_in, word in ((lse, None), (lse + 0.05, None), (lse, 7)):
        o = torch.empty(n, H, L, L)
        E.dropout_offset_bind(None if word is None else torch.tensor([word]))
        try:
            BE.attention_probs(qkv, mask, l_in, o, n, L, case.lt, H, case.p, 5)
        finally:
            E.dropout_offset_bind(None)
        outs.append(o)
    assert not torch.equal(outs[0], outs[1]) and not torch.equal(outs[0] == 0, outs[2] == 0)
