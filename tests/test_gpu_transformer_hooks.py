"""Module hooks on ClipBertBaseModel: with a hook on bert or a module below it, bert(...) and every head's forward run through the
modules (bert.embeddings, bert.visual_embeddings, bert.encoder, each BertLayer with its attention, attention.self,
attention.output, intermediate and output, bert.pooler), so torch's forward hooks, pre-hooks, replacements and tensor hooks on
their outputs apply, and the backward is a chain of nodes split at the hooked boundaries.

Against the oracle's fp32 autograd (oracle/clipbert_ref.py) with the run's own attention-dropout masks, through ref_bert below: a
restatement of clipbert_base_model with a tap at every site, pinned to the oracle on the CPU
(tests/test_transformer_hooks_emulated.py):
  - every site's forward-hook output and the gradient its tensor hook sees, on all 12 layers;
  - interventions run on both sides: token ablation, head ablation, layer patching, a gradient-rewriting tensor hook;
  - integrated gradients on bert.embeddings by forward-hook replacement and torch.autograd.grad.
The word-vector text-embedding kernels (cb_embed_text_fwd_vectors, cb_embed_text_bwd_vectors / _det, cb_embed_word_scatter)
against float64 and bit for bit against the id-based kernels on word[ids].
Bit for bit against the default path (deterministic mode): observe-only hooks on every site but intermediate, output and pooler
(those three move a fused derivative out of a GEMM epilogue: one bf16 rounding more), on bert(...), a head's forward with ragged
repeat counts, and ClipBert's forward / forward_clips; the launches after every hook is removed.
"""
import contextlib
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_gpu_attention_probs_bwd as PB
import test_gpu_attention_retained_grads as RG
import test_gpu_layerwise_autograd as LW
from util import TOL_GRAD, cosine, make_cfg, relerr

pytestmark = pytest.mark.gpu

PREFIX = "transformer.bert."


# ------------------------------------------------------------------------------------------------ oracle with taps
def ref_bert(ids, grid, mask, sd, mult=None, tap=None):
    """oracle.clipbert_ref.clipbert_base_model (eval, attention dropout by the multipliers mult[layer]) with tap(site, t) -> t at
    every module boundary the engine hands to hooks. Returns (sequence_output, pooled_output)."""
    from oracle import clipbert_ref as R
    cfg = R.BERT_CFG
    eps, nh = cfg["layer_norm_eps"], cfg["num_attention_heads"]
    tap = tap or (lambda site, t: t)
    e = PREFIX + "embeddings."
    wv = tap("word_embeddings", F.embedding(ids, sd[e + "word_embeddings.weight"]))
    te = tap("embeddings", R.layer_norm(wv + sd[e + "position_embeddings.weight"][:ids.shape[1]].unsqueeze(0)
                                        + sd[e + "token_type_embeddings.weight"][0].view(1, 1, -1), sd, e + "LayerNorm.", eps))
    ve = tap("visual_embeddings", R.visual_embeddings(grid, sd, PREFIX + "visual_embeddings.", eps))
    full = torch.cat([mask, mask.new_ones(ve.shape[:2])], dim=-1)
    h = torch.cat([te, ve], dim=1)
    ext = (1.0 - full[:, None, None, :].to(h.dtype)) * -10000.0
    for i in range(cfg["num_hidden_layers"]):
        p = "%sencoder.layer.%d." % (PREFIX, i)
        b, n, d = h.shape
        hd = d // nh

        def split(x):
            return x.view(b, n, nh, hd).permute(0, 2, 1, 3)
        q, k, v = (split(R.linear(h, sd, p + "attention.self.%s." % w)) for w in ("query", "key", "value"))
        pr = torch.softmax(torch.matmul(q, k.transpose(-1, -2)) / math.sqrt(hd) + ext, dim=-1)
        if mult is not None:
            pr = pr * mult[i]
        ctx = tap("layer.%d.attention.self" % i, torch.matmul(pr, v).permute(0, 2, 1, 3).reshape(b, n, d))
        a = tap("layer.%d.attention.output" % i,
                R.layer_norm(R.linear(ctx, sd, p + "attention.output.dense.") + h, sd, p + "attention.output.LayerNorm.", eps))
        gel = tap("layer.%d.intermediate" % i, F.gelu(R.linear(a, sd, p + "intermediate.dense.")))
        h = tap("layer.%d.output" % i, R.layer_norm(R.linear(gel, sd, p + "output.dense.") + a, sd, p + "output.LayerNorm.", eps))
    pooled = tap("pooler", torch.tanh(R.linear(h[:, 0], sd, PREFIX + "pooler.dense.")))
    return h, pooled


def site_modules(bert):
    """[(site, module)] for every hookable module of bert but bert itself; site names as ref_bert's taps."""
    out = [("embeddings", bert.embeddings), ("word_embeddings", bert.embeddings.word_embeddings),
           ("visual_embeddings", bert.visual_embeddings), ("encoder", bert.encoder),
           ("pooler", bert.pooler)]
    for i, ly in enumerate(bert.encoder.layer):
        out += [("layer.%d" % i, ly), ("layer.%d.attention" % i, ly.attention), ("layer.%d.attention.self" % i, ly.attention.self),
                ("layer.%d.attention.output" % i, ly.attention.output), ("layer.%d.intermediate" % i, ly.intermediate),
                ("layer.%d.output" % i, ly.output)]
    return out


def ref_site(site):
    """The ref_bert tap whose tensor a module hands to its hooks."""
    if site == "encoder":
        return "layer.11.output"
    parts = site.split(".")
    if len(parts) == 2:
        return site + ".output"
    if parts[-1] == "attention":
        return site + ".output"
    return site


def record_sites(sites):
    """Forward hooks recording each module's output (the first member of a tuple) and, through a tensor hook on it, the gradient
    it receives. Returns (outputs, grads, handles)."""
    outs, grads, handles = {}, {}, []
    for site, mod in sites:
        def hook(m, inp, out, site=site):
            t = out[0] if isinstance(out, tuple) else out
            outs[site] = t.detach().clone()
            if t.requires_grad:
                t.register_hook(lambda g, site=site: grads.__setitem__(site, g.detach().clone()))
        handles.append(mod.register_forward_hook(hook))
    return outs, grads, handles


def ref_recorder(interventions=None):
    rec = {}
    interventions = interventions or {}

    def tap(site, t):
        if t.requires_grad:
            t.retain_grad()
        rec[site] = t
        f = interventions.get(site)
        return t if f is None else f(t)
    return rec, tap


def close(what, got, ref):
    assert got is not None, what
    e, c = relerr(got, ref), cosine(got, ref)
    assert e < TOL_GRAD and c > 0.999, (what, e, c)


def compare_params(grads, sd, floor=None):
    """Every parameter gradient of bert ({name: .grad}) against the oracle's; returns the number compared. floor: {name: (relerr,
    cosine)} of the default path on the same pass - a gradient outside the tolerances passes when it is as close to the oracle
    as the default path's (up to a quarter more error)."""
    checked = 0
    for name, g in grads.items():
        ref = sd[PREFIX + name].grad
        if ref is None or float(ref.abs().sum()) == 0.0:
            assert g is None or float(g.abs().sum()) == 0.0, name
            continue
        if name.endswith("attention.self.key.bias"):       # mathematically zero: rounding noise on both sides
            continue
        e, c = relerr(g, ref), cosine(g, ref)
        if floor is not None and not (e < TOL_GRAD and c > 0.999):
            fe, fc = floor[name]
            assert e <= 1.25 * fe and 1 - c <= 1.25 * (1 - fc), (name, e, c, fe, fc)
        else:
            close(name, g, ref)
        checked += 1
    return checked


def _grads(model):
    return {n: (None if p.grad is None else p.grad.detach().clone()) for n, p in model.named_parameters()}


def _model(weights, dev, p=0.1, attn=False, **cfg):
    m = RG._model(weights, dev, attention_probs_dropout_prob=p, **cfg)
    m.differentiable_attentions = attn
    return m.train() if p > 0 else m.eval()


def _oracle_sd(weights):
    return {k: (v.clone().requires_grad_(True) if k.startswith(PREFIX) else v) for k, v in weights.items()}


def _weights_of(nseq, L, g, dev):
    ws = (torch.randn(nseq, L, 768, generator=g) * 0.1).to(torch.bfloat16).float()
    wp = torch.randn(nseq, 768, generator=g).to(torch.bfloat16).float()
    return (ws, wp), (ws.to(dev), wp.to(dev))


def _score(seq, pooled, ws, wp):
    return (seq.float() * ws).sum() + (pooled.float() * wp).sum()


@contextlib.contextmanager
def _deterministic():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


@contextlib.contextmanager
def hooks(handles):
    try:
        yield handles
    finally:
        for h in handles:
            h.remove()


# ------------------------------------------------------------------------------------------------ the word-vector kernels
def text_vectors_ref(vec, pos, typ, gamma, beta, nseq, lt, l, eps, p, seed):
    """float64 (out [nseq * lt, 768] before the bf16 rounding, mean, rstd, multipliers) of cb_embed_text_fwd_vectors (no bound word)."""
    import dropout_ref as D
    v = vec.double() + pos.double()[:lt].repeat(nseq, 1) + typ.double()[0]
    mean = v.mean(1, keepdim=True)
    var = ((v - mean) ** 2).mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    xhat = (v - mean) * rstd
    y = xhat * gamma.double() + beta.double()
    mult = torch.ones_like(y) if p == 0 else torch.from_numpy(
        D.multipliers(D.effective_seed(seed, None), D.embedding_index(nseq, l, range(lt)), p)).double().reshape(nseq * lt, -1)
    return y * mult, mean[:, 0], rstd[:, 0], mult, xhat


def run_vector_kernels(dev, lt, p, pitched):
    """cb_embed_text_fwd_vectors, cb_embed_text_bwd_vectors / _det and cb_embed_word_scatter: against float64 (output within one
    bf16 ulp plus the fp32 LayerNorm's rounding; d vec within fp32 rounding of the float64 LayerNorm backward), with NaN guard
    bands around every output, and bit for bit against cb_embed_text_fwd / cb_embed_text_bwd_det on vec = word[ids] (the table
    gradient through the scatter included); the default mode's d vec equals the deterministic one's (one writer per element)."""
    from clipbert_b200 import ops
    from elementwise import ulp_bf16
    g = torch.Generator().manual_seed(lt * 7 + int(p * 10))
    nseq, H, vocab, extra = 3 if lt < 512 else 1, 768, 97, 9
    L, R, eps, seed = lt + extra, (3 if lt < 512 else 1) * lt, 1e-12, 4242 + lt
    word = torch.randn(vocab, H, generator=g).to(dev)
    pos, typ = torch.randn(lt, H, generator=g).to(dev) * 0.1, torch.randn(1, H, generator=g).to(dev) * 0.1
    gamma, beta = (1 + 0.1 * torch.randn(H, generator=g)).to(dev), (0.1 * torch.randn(H, generator=g)).to(dev)
    ids = torch.randint(0, vocab, (nseq, lt), generator=g)
    ids[:, -1] = ids[:, 0]                                      # repeated tokens: the scatter sums rows in order
    ids = ids.to(dev)
    big = torch.full((R, H + (36 if pitched else 0)), float("nan"), device=dev)
    vec = big[:, :H]
    vec.copy_(word[ids.reshape(-1)])
    ops.dropout_offset_bind(None)

    def guarded(rows, cols, dtype):
        buf = torch.full((rows + 8, cols), float("nan"), dtype=dtype, device=dev)
        return buf, buf[4:4 + rows]
    obuf, out = guarded(nseq * L, H, torch.bfloat16)
    sbuf, stats = guarded(R, 2, torch.float32)
    ops.embed_text_fwd_vectors(vec, pos, typ, gamma, beta, out, stats, nseq, lt, L, eps, p, seed)
    torch.cuda.synchronize()
    ref, mean, rstd, mult, xhat = text_vectors_ref(vec.cpu(), pos.cpu(), typ.cpu(), gamma.cpu(), beta.cpu(), nseq, lt, L, eps, p, seed)
    got = out.view(nseq, L, H)[:, :lt].reshape(R, H).double().cpu()
    assert bool(torch.isnan(out.view(nseq, L, H)[:, lt:]).all()) and bool(torch.isnan(obuf[:4]).all() and torch.isnan(obuf[-4:]).all())
    assert bool(((got - ref).abs() <= ulp_bf16(ref) + 1e-5 * (1 + ref.abs())).all())
    assert torch.allclose(stats.double().cpu()[:, 0], mean, rtol=1e-5, atol=1e-6) and torch.allclose(stats.double().cpu()[:, 1], rstd, rtol=1e-5)
    assert bool(torch.isnan(sbuf[:4]).all() and torch.isnan(sbuf[-4:]).all())
    # the id kernel on word[ids]: the same bits
    out2, stats2 = torch.full_like(out, float("nan")), torch.empty_like(stats)
    ops.embed_text_fwd(ids, word, pos, typ, gamma, beta, out2, stats2, nseq, lt, L, eps, p, seed)
    assert torch.equal(out2.view(torch.int16), out.view(torch.int16)) and torch.equal(stats2, stats)
    # backward
    dh = torch.randn(nseq * L, H, generator=g).to(torch.bfloat16).to(dev)
    res = {}
    for det in (False, True):
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(det)
        try:
            dbuf, dvec = guarded(R, H, torch.float32)
            tabs = [torch.zeros_like(t) for t in (pos, typ, gamma, beta)]
            ops.embed_text_bwd_vectors(dh, vec, pos, typ, gamma, stats, dvec, *tabs, nseq, lt, L, p, seed)
            dword = torch.zeros_like(word)
            ops.embed_word_scatter(ids, dvec, dword)
            torch.cuda.synchronize()
            assert bool(torch.isnan(dbuf[:4]).all() and torch.isnan(dbuf[-4:]).all()) and not bool(torch.isnan(dvec).any())
            res[det] = [dvec.clone(), dword] + tabs
        finally:
            torch.use_deterministic_algorithms(prev)
    assert torch.equal(res[False][0], res[True][0])
    dy = dh.view(nseq, L, H)[:, :lt].reshape(R, H).double().cpu() * mult
    gx = dy * gamma.double().cpu()
    dref = rstd[:, None] * (gx - gx.mean(1, keepdim=True) - xhat * (gx * xhat).mean(1, keepdim=True))
    scale = dref.abs().amax(1, keepdim=True) + 1e-30
    assert bool(((res[True][0].double().cpu() - dref).abs() <= 1e-4 * scale).all())
    # deterministic: the id kernel's table and parameter gradients, bit for bit
    torch.use_deterministic_algorithms(True)
    try:
        tabs = [torch.zeros_like(t) for t in (word, pos, typ, gamma, beta)]
        ops.embed_text_bwd(dh, ids, word, pos, typ, gamma, stats, *tabs, nseq, lt, L, p, seed)
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(False)
    for a, b in zip(res[True][1:], tabs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("pitched", [False, True])
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("lt", [1, 20, 32, 512])
def test_word_vector_kernels(cuda, lt, p, pitched):
    run_vector_kernels(cuda, lt, p, pitched)


def test_word_vector_kernels_refuse_bad_arguments_and_launch_nothing(cuda):
    from clipbert_b200 import ops
    H, nseq, lt, L = 768, 2, 4, 6
    vec = torch.zeros(nseq * lt, H + 4, device=cuda)
    out = torch.full((nseq * L, H), 3.0, dtype=torch.bfloat16, device=cuda)
    stats, dvec = torch.zeros(nseq * lt, 2, device=cuda), torch.full((nseq * lt, H), 5.0, device=cuda)
    t = [torch.zeros(lt, H, device=cuda), torch.zeros(1, H, device=cuda), torch.ones(H, device=cuda), torch.zeros(H, device=cuda)]
    P, S = ops._p, ops._s

    def fwd(v=vec, ld=H + 4, hidden=H, lt_=lt, l=L):
        ops._call("cb_embed_text_fwd_vectors", P(v), ld, P(t[0]), P(t[1]), P(t[2]), P(t[3]), P(out), P(stats), nseq, lt_, l, hidden,
                  1e-12, 0.0, 1, S())

    def bwd(v=vec, ld=H + 4, dv=dvec, hidden=H, lt_=lt, l=L):
        ops._call("cb_embed_text_bwd_vectors", P(out), P(v), ld, P(t[0]), P(t[1]), P(t[2]), P(stats), P(dv), P(t[0]), P(t[1]),
                  P(t[2]), P(t[3]), nseq, lt_, l, hidden, 0.0, 1, S())
    for call in (fwd, bwd):
        for kw in (dict(ld=H - 4), dict(ld=H + 2), dict(v=vec.view(-1)[1:]), dict(v=None), dict(hidden=1024), dict(lt_=0), dict(l=lt - 1)):
            with pytest.raises(RuntimeError):
                call(**kw)
    with pytest.raises(RuntimeError):
        bwd(dv=None)
    with pytest.raises(RuntimeError):
        ops._call("cb_embed_word_scatter", P(stats), P(dvec), P(dvec), 0, 10, H, S())
    torch.cuda.synchronize()
    assert bool((out == 3.0).all()) and bool((dvec == 5.0).all()) and bool((stats == 0).all())


# ------------------------------------------------------------------------------------------------ every site against the oracle
def run_sites_against_oracle(dev, weights, size, diff_attn=False, subset=None):
    """Hooks on every site of every layer (or the sites in subset): each forward-hook output and the gradient its tensor hook
    sees, and every parameter and visual_inputs gradient, against the oracle's fp32 autograd with the run's attention masks."""
    model = _model(weights, dev, attn=diff_attn)
    eng = model._engine
    grid, ids, mask, L, g = RG._inputs(size, 151)
    nseq = ids.shape[0]
    (ws, wp), (wsd, wpd) = _weights_of(nseq, L, g, dev)
    sites = [s for s in site_modules(model) if subset is None or s[0] in subset]
    with torch.no_grad():
        model(ids.to(dev), grid.to(dev), mask.to(dev))
    state = (eng._call_count, int(eng._drop_counter.item()))
    gc = grid.clone().to(dev).requires_grad_(True)
    outs, grads, handles = record_sites(sites)
    with hooks(handles):
        seq, pooled = model(ids.to(dev), gc, mask.to(dev))[:2]
        _score(seq, pooled, wsd, wpd).backward()
    mult = LW._masks_of_last_call(eng, nseq, L, 0.1)
    hooked = _grads(model)
    PB._rewind(eng, state)                 # the default path on the same pass: the floor of the parameter comparison
    eng.zero_grad(set_to_none=False)
    seq0, pooled0 = model(ids.to(dev), grid.clone().to(dev).requires_grad_(True), mask.to(dev))[:2]
    _score(seq0, pooled0, wsd, wpd).backward()
    default = _grads(model)
    sd = _oracle_sd(weights)
    gr = grid.clone().requires_grad_(True)
    rec, tap = ref_recorder()
    seq_r, pooled_r = ref_bert(ids, gr, mask, sd, mult, tap)
    _score(seq_r, pooled_r, ws, wp).backward()
    assert sorted(outs) == sorted(s for s, _ in sites)
    for site, _ in sites:
        close(site, outs[site], rec[ref_site(site)])
        close(site + " grad", grads[site], rec[ref_site(site)].grad)
    close("visual_inputs grad", gc.grad, gr.grad)
    floor = {n: (relerr(g, sd[PREFIX + n].grad), cosine(g, sd[PREFIX + n].grad)) for n, g in default.items()
             if sd[PREFIX + n].grad is not None}
    assert compare_params(hooked, sd, floor) >= 12 * 14


@pytest.mark.parametrize("diff_attn", [False, True])
@pytest.mark.parametrize("size", ["224px", "448px", "512tok"])
def test_every_site_against_oracle(cuda, weights, size, diff_attn):
    run_sites_against_oracle(cuda, weights, size, diff_attn)


@pytest.mark.parametrize("subset", [("layer.3", "encoder"), ("layer.2.attention", "layer.9.attention.self"),
                                    ("layer.5.intermediate",), ("layer.7.attention.output", "layer.7.output", "pooler")])
def test_hooked_subsets_against_oracle(cuda, weights, subset):
    run_sites_against_oracle(cuda, weights, "224px", subset=set(subset))


# ------------------------------------------------------------------------------------------------ observe-only hooks keep the bits
def BIT_SITES(site):
    """The sites whose observe-only hooks keep every bit: all but intermediate, output (whose input is intermediate's output)
    and pooler."""
    ffn_out = site.endswith(".output") and not site.endswith("attention.output")
    return not (site.endswith("intermediate") or ffn_out or site == "pooler")


def _head(weights, dev, cls_name="ClipBertForVideoTextRetrieval", **cfg):
    import clipbert_b200 as cb
    c = make_cfg(**dict(dict(hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1), **cfg))
    h = getattr(cb, cls_name)(c)
    own = h.state_dict()
    h.load_state_dict({k[len("transformer."):]: v for k, v in weights.items()
                       if k.startswith("transformer.") and k[len("transformer."):] in own and own[k[len("transformer."):]].shape == v.shape},
                      strict=False)
    return h.to(dev).train()


def _flat_and_grid(eng, gc):
    return [eng._flat.grad.detach().clone(), None if gc.grad is None else gc.grad.detach().clone()]


def run_bits_observe_only(dev, weights, size, which, launches=None, sites=BIT_SITES):
    """Deterministic mode, dropout 0.1 (hidden and attention): observe-only forward hooks on every site selected by sites give
    the outputs, the flat gradient buffer and d visual_inputs of the no-hook pass, bit for bit. which: "bert" (bert(...)),
    "retrieval" (the head's forward) or "ragged" (the head with repeat counts [1, 3, 2], as forward_clips runs it)."""
    grid, ids, mask, L, g = RG._inputs(size, 153)
    counts = None
    if which == "bert":
        model = _model(weights, dev, hidden_dropout_prob=0.1)
        bert, eng = model, model._engine
    else:
        eng = _head(weights, dev)
        bert = eng.bert
        if which == "ragged":           # 3 videos with 1, 3 and 2 captions
            counts = [1, 3, 2]
            rows = torch.arange(6) % ids.shape[0]
            ids, mask, grid = ids[rows], mask[rows], grid[torch.arange(3) % grid.shape[0]]
    nseq = ids.shape[0]
    (_, _), (wsd, wpd) = _weights_of(nseq, L, g, dev)
    ids, mask = ids.to(dev), mask.to(dev)
    with torch.no_grad():
        if which == "bert":
            bert(ids, grid.to(dev), mask)
        else:
            eng(ids, grid.to(dev), mask, _repeat_counts=counts)
    state = (eng._call_count, int(eng._drop_counter.item()))
    res = []
    with _deterministic():
        for hooked in (False, True):
            PB._rewind(eng, state)
            eng.zero_grad(set_to_none=False)
            gc = grid.clone().to(dev).requires_grad_(True)
            chosen = [s for s in site_modules(bert) if sites(s[0])] if hooked else []
            outs, grads, handles = record_sites(chosen)
            with hooks(handles):
                if which == "bert":
                    seq, pooled = bert(ids, gc, mask)[:2]
                    out = [seq, pooled]
                    loss = _score(seq, pooled, wsd, wpd)
                else:
                    logits = eng(ids, gc, mask, _repeat_counts=counts)["logits"]
                    out = [logits]
                    loss = (logits.float() * torch.arange(1, logits.numel() + 1, device=dev).view(logits.shape).float()).sum()
                loss.backward()
            assert len(outs) == len(chosen) and (not hooked or len(grads) > 0)
            res.append([t.detach().clone() for t in out] + _flat_and_grid(eng, gc))
    for a, b in zip(res[0], res[1]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("which", ["bert", "retrieval", "ragged"])
@pytest.mark.parametrize("size", ["224px", "448px"])
def test_observe_only_hooks_keep_the_bits(cuda, weights, size, which):
    run_bits_observe_only(cuda, weights, size, which)


# ------------------------------------------------------------------------------------------------ interventions
def _head_scale():
    cols = torch.full((768,), 0.7)
    cols[4 * 64: 5 * 64] = 0                    # head 4 ablated, the other heads scaled
    return cols


def run_interventions(dev, weights, size, which):
    """One intervention on both sides, then the outputs, the parameter gradients and d visual_inputs against the oracle:
    "tokens": a forward hook zeroing visual tokens 0 and 2 of bert.visual_embeddings' output;
    "heads": a pre-hook on layer[5].attention.output scaling the context (head 4 zeroed, the others x 0.7);
    "patch": layer[6]'s output replaced by the same layer's output on a second input;
    "grad": a tensor hook on layer[7].intermediate's output zeroing the gradient of its first 1000 columns."""
    model = _model(weights, dev)
    eng = model._engine
    grid, ids, mask, L, g = RG._inputs(size, 155)
    nseq = ids.shape[0]
    (ws, wp), (wsd, wpd) = _weights_of(nseq, L, g, dev)
    lay = model.encoder.layer
    handles, interventions = [], {}
    if which == "tokens":
        keep = torch.ones(L - ids.shape[1], 1)
        keep[0] = keep[2] = 0
        handles.append(model.visual_embeddings.register_forward_hook(lambda m, i, o: o * keep.to(dev).to(o.dtype)))
        interventions["visual_embeddings"] = lambda t: t * keep
    elif which == "heads":
        cols = _head_scale()
        handles.append(lay[5].attention.output.register_forward_pre_hook(lambda m, a: (a[0] * cols.to(dev).to(a[0].dtype), a[1])))
        interventions["layer.5.attention.self"] = lambda t: t * cols
    elif which == "patch":
        grid2, ids2, mask2, _, _ = RG._inputs(size, 157)
        saved = {}
        h = lay[6].register_forward_hook(lambda m, i, o: saved.__setitem__("y", o[0].detach().clone()))
        with torch.no_grad():
            model.eval()
            model(ids2.to(dev), grid2.to(dev), mask2.to(dev))
            model.train()
        h.remove()
        handles.append(lay[6].register_forward_hook(lambda m, i, o: (saved["y"],) + tuple(o[1:])))
        with torch.no_grad():
            ref_bert(ids2, grid2, mask2, weights, None, _capture_at("layer.6.output", saved, "ref"))
        interventions["layer.6.output"] = lambda t: saved["ref"]
    elif which == "word":          # word vectors of tokens 1 and 3 replaced by token 5's (fp16, a strided view)
        def swap(t):
            t = t.clone()
            t[:, 1] = t[:, 5]
            t[:, 3] = t[:, 5]
            return t
        handles.append(model.embeddings.word_embeddings.register_forward_hook(
            lambda m, i, o: swap(o).to(torch.float16).transpose(0, 1).contiguous().transpose(0, 1)))
        interventions["word_embeddings"] = lambda t: swap(t.to(torch.float16).float())
    elif which == "grad":
        def rewrite(g):
            g = g.clone()
            g[..., :1000] = 0
            return g

        def fwd(m, i, o):
            o.register_hook(rewrite)
        handles.append(lay[7].intermediate.register_forward_hook(fwd))

        def ref_int(t):
            t.register_hook(rewrite)
            return t
        interventions["layer.7.intermediate"] = ref_int
    gc = grid.clone().to(dev).requires_grad_(True)
    with hooks(handles):
        seq, pooled = model(ids.to(dev), gc, mask.to(dev))[:2]
        _score(seq, pooled, wsd, wpd).backward()
    mult = LW._masks_of_last_call(eng, nseq, L, 0.1)
    sd = _oracle_sd(weights)
    gr = grid.clone().requires_grad_(True)
    rec, tap = ref_recorder(interventions)
    seq_r, pooled_r = ref_bert(ids, gr, mask, sd, mult, tap)
    _score(seq_r, pooled_r, ws, wp).backward()
    close("sequence_output", seq, seq_r)
    close("pooled_output", pooled, pooled_r)
    if which == "patch":
        assert gc.grad is None or float(gc.grad.abs().sum()) == 0
        assert float(lay[3].attention.self.query.weight.grad.abs().sum()) == 0
    else:
        close("visual_inputs grad", gc.grad, gr.grad)
    assert compare_params(_grads(model), sd) > 0


def _capture_at(site, saved, key):
    def tap(s, t):
        if s == site:
            saved[key] = t.detach().clone()
        return t
    return tap


@pytest.mark.parametrize("which", ["tokens", "heads", "patch", "word", "grad"])
def test_interventions_against_oracle(cuda, weights, which):
    run_interventions(cuda, weights, "224px", which)


# ------------------------------------------------------------------------------------------------ integrated gradients
def integrated_gradients(run, x, steps):
    """Integrated gradients of F (run(x') -> scalar, differentiable in x') from the zero baseline, right Riemann sum over steps.
    Returns (attributions, F(x) - F(0))."""
    total = torch.zeros_like(x, dtype=torch.float32)
    for k in range(1, steps + 1):
        xi = (x * (k / steps)).detach().requires_grad_(True)
        (gi,) = torch.autograd.grad(run(xi), xi)
        total += gi.float()
    with torch.no_grad():
        gap = float(run(x)) - float(run(torch.zeros_like(x)))
    return x.float() * total / steps, gap


def run_integrated_gradients(dev, weights, size, steps=20, site="embeddings"):
    """IG on bert.embeddings' output, F = <pooled_output, w>, written with a forward-hook replacement and autograd.grad: the
    attributions against the oracle's, and the completeness gap sum(attr) - (F(x) - F(0)) equal to the oracle's (the Riemann
    sum's own error, the same on both sides) within 2 % of F(x) - F(0)."""
    model = _model(weights, dev, p=0.0)
    mod = model.embeddings if site == "embeddings" else model.embeddings.word_embeddings
    grid, ids, mask, L, g = RG._inputs(size, 159)
    nseq = ids.shape[0]
    (_, wp), (_, wpd) = _weights_of(nseq, L, g, dev)
    ids_d, grid_d, mask_d = ids.to(dev), grid.to(dev), mask.to(dev)
    saved = {}
    with hooks([mod.register_forward_hook(lambda m, i, o: saved.__setitem__("x", o.detach().float().clone()))]):
        with torch.no_grad():
            model(ids_d, grid_d, mask_d)

    def run(xi):
        with hooks([mod.register_forward_hook(lambda m, i, o: xi)]):
            return (model(ids_d, grid_d, mask_d)[1].float() * wpd).sum()
    attr, gap = integrated_gradients(run, saved["x"], steps)
    sd = {k: v for k, v in weights.items()}
    with torch.no_grad():
        ref_bert(ids, grid, mask, sd, None, _capture_at(site, saved, "ref"))
    x_ref = saved["ref"]

    def run_ref(xi):
        return (ref_bert(ids, grid, mask, sd, None, lambda s, t: xi if s == site else t)[1] * wp).sum()
    attr_r, gap_r = integrated_gradients(run_ref, x_ref, steps)
    close("IG attributions", attr, attr_r)
    assert abs(gap - gap_r) <= 0.05 * abs(gap_r), (gap, gap_r)
    err, err_r = float(attr.sum()) - gap, float(attr_r.sum()) - gap_r
    assert abs(err - err_r) <= 0.02 * abs(gap_r), (err, err_r, gap_r)
    return attr, gap


@pytest.mark.parametrize("site", ["embeddings", "word_embeddings"])
def test_integrated_gradients(cuda, weights, site):
    run_integrated_gradients(cuda, weights, "224px", site=site)


# ------------------------------------------------------------------------------------------------ heads and ClipBert
HEADS = [("ClipBertForVideoTextRetrieval", {}), ("ClipBertForSequenceClassification", dict(num_labels=5, loss_type="ce")),
         ("ClipBertForMultipleChoice", dict(num_labels=1)), ("ClipBertForPreTraining", dict(pixel_random_sampling_size=3))]


def run_head_hooks(dev, weights, size, cls_name, cfg, sites=("layer.3", "layer.5.attention.self", "layer.5.attention.output")):
    """Observe-only hooks on head.bert's modules fire in the head's forward (train mode, dropout 0.1; pre-training with MLM + ITM
    and sampled visual tokens) and give the flat gradient buffer and d visual_inputs of the no-hook step, bit for bit."""
    head = _head(weights, dev, cls_name, **cfg)
    grid, ids, mask, L, g = RG._inputs(size, 161)
    ids, mask = ids.to(dev), mask.to(dev)
    with torch.no_grad():
        head(ids, grid.to(dev), mask)
    state = (head._call_count, int(head._drop_counter.item()))
    res = []
    with _deterministic():
        for hooked in (False, True):
            PB._rewind(head, state)
            np.random.seed(5)
            head.zero_grad(set_to_none=False)
            gc = grid.clone().to(dev).requires_grad_(True)
            chosen = [s for s in site_modules(head.bert) if hooked and s[0] in sites]
            outs, grads, handles = record_sites(chosen)
            with hooks(handles):
                out = head(ids, gc, mask)
                if cls_name == "ClipBertForPreTraining":
                    loss = (out["mlm_scores"].float() * 1e-3).sum() + (out["itm_scores"].float() * torch.tensor([1.0, -2.0], device=dev)).sum()
                else:
                    loss = (out["logits"].float() * torch.arange(1, out["logits"].numel() + 1, device=dev).view(out["logits"].shape)).sum()
                loss.backward()
            assert len(outs) == len(chosen) and len(grads) == len(chosen)
            res.append([head._flat.grad.detach().clone(), gc.grad.detach().clone()])
    for a, b in zip(res[0], res[1]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("cls_name,cfg", HEADS, ids=[h[0] for h in HEADS])
def test_hooks_on_head_bert_fire_and_keep_the_bits(cuda, weights, cls_name, cfg):
    run_head_hooks(cuda, weights, "224px", cls_name, cfg)


@pytest.mark.parametrize("path", ["forward", "forward_clips", "encode_clips"])
def test_clipbert_paths_fire_hooks_and_keep_the_bits(cuda, weights, path):
    """ClipBert.forward, forward_clips and forward_clips(grid=...): hooks on transformer.bert's modules fire, and the frame and
    parameter gradients are those of the no-hook pass (deterministic, eval)."""
    import test_gpu_input_grads as IG
    from oracle import synth
    model = IG.clipbert(cuda, weights, "none")
    clips = 1 if path == "forward" else 2
    batch = synth.synth_batch(2, 2 * clips, n_ex=2, size=160, seed=11)
    bert = model.transformer.bert
    res = []
    with _deterministic():
        for hooked in (False, True):
            model.zero_grad(set_to_none=False)
            xd = batch["visual_inputs"].to(cuda).requires_grad_(True)
            mb = {k: (v.to(cuda) if torch.is_tensor(v) else list(v)) for k, v in batch.items()}
            chosen = [s for s in site_modules(bert) if hooked and s[0] in ("layer.4", "layer.8.attention.self", "embeddings")]
            outs, grads, handles = record_sites(chosen)
            with hooks(handles):
                if path == "forward":
                    mb["visual_inputs"] = xd
                    logits = model(mb)["logits"]
                elif path == "forward_clips":
                    mb["visual_inputs"] = xd
                    logits = model.forward_clips(mb, clips)["logits"]
                else:
                    grid = model.encode_clips(xd, clips)
                    del mb["visual_inputs"]
                    logits = model.forward_clips(mb, clips, grid=grid)["logits"]
                (logits.float() * torch.linspace(-1, 1, logits.numel(), device=cuda).view(logits.shape)).sum().backward()
            assert len(outs) == len(chosen) and len(grads) == len(chosen)
            res.append([xd.grad.clone()] + [m._flat.grad.clone() for m in (model.transformer, model.cnn)])
    for a, b in zip(res[0], res[1]):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ semantics
def run_semantics(dev, weights, size, launches=None):
    """autograd.grad leaves the flat gradient buffer bit-identical; retain_graph allows a second backward (hooks see the same
    bits, parameter gradients double); no_grad fires forward hooks and builds no nodes; with every hook removed the pass issues
    the launches of a model that never had one."""
    model = _model(weights, dev, hidden_dropout_prob=0.1)
    eng = model._engine
    grid, ids, mask, L, g = RG._inputs(size, 163)
    nseq = ids.shape[0]
    (_, _), (wsd, wpd) = _weights_of(nseq, L, g, dev)
    ids, mask, gdev = ids.to(dev), mask.to(dev), grid.to(dev)
    sites = [s for s in site_modules(model) if s[0] in ("layer.5", "layer.7.attention.self", "layer.7.attention.output",
                                                          "layer.9.intermediate", "layer.9.output", "embeddings", "pooler")]
    with _deterministic():
        seq, pooled = model(ids, gdev.clone().requires_grad_(True), mask)[:2]
        _score(seq, pooled, wsd, wpd).backward()
        before = eng._flat.grad.clone()
        outs, grads, handles = record_sites(sites)
        with hooks(handles):
            got = {}
            ga = model.encoder.layer[5].register_forward_hook(lambda m, i, o: got.__setitem__("y5", o[0]))
            gc = gdev.clone().requires_grad_(True)
            seq, pooled = model(ids, gc, mask)[:2]
            ga.remove()
            score = _score(seq, pooled, wsd, wpd)
            (g5,) = torch.autograd.grad(score, [got["y5"]], retain_graph=True)
            assert torch.equal(eng._flat.grad, before) and gc.grad is None and float(g5.float().abs().sum()) > 0
            eng.zero_grad(set_to_none=False)
            score.backward(retain_graph=True)
            once = [grads[s].clone() for s, _ in sites] + [eng._flat.grad.clone(), gc.grad.clone()]
            score.backward()
            twice = [grads[s].clone() for s, _ in sites] + [eng._flat.grad.clone(), gc.grad.clone()]
            for a, b in zip(once[:-2], twice[:-2]):
                assert torch.equal(a, b)
            assert torch.equal(twice[-1].float(), 2 * once[-1].float())
            assert float((twice[-2] - 2 * once[-2]).abs().max()) <= 1e-6 * float(once[-2].abs().max())
            with pytest.raises(RuntimeError, match="second time"):
                score.backward()
            outs.clear()
            with torch.no_grad():
                seq, pooled = model(ids, gc, mask)[:2]
            assert len(outs) == len(sites) and seq.grad_fn is None and not pooled.requires_grad
    # every hook removed: the launches of the default path
    counts = []
    for fresh in (True, False):
        m = _model(weights, dev, hidden_dropout_prob=0.1) if fresh else model
        for _ in range(2):              # the second step of each: the same repack state
            before = dict(launches) if launches is not None else None
            with PB._timing(dev) as ev:
                seq, pooled = m(ids, gdev.clone().requires_grad_(True), mask)[:2]
                _score(seq, pooled, wsd, wpd).backward()
                names = [e[0] for e in ev] if ev is not None else \
                    {k: v - before[k] for k, v in launches.items() if k != "dropout_offset_bind"}
        counts.append(names)
    assert counts[0] == counts[1]


def test_semantics(cuda, weights):
    run_semantics(cuda, weights, "224px")


def test_memory_returns_to_its_baseline(cuda, weights):
    model = _model(weights, cuda)
    grid, ids, mask, L, g = RG._inputs("448px", 165)
    (_, _), (wsd, wpd) = _weights_of(ids.shape[0], L, g, cuda)
    ids, mask, gdev = ids.to(cuda), mask.to(cuda), grid.to(cuda)
    sites = [s for s in site_modules(model) if BIT_SITES(s[0]) or s[0].endswith("intermediate")]
    outs, grads, handles = record_sites(sites)

    def step(partial):
        gc = gdev.clone().requires_grad_(True)
        seq, pooled = model(ids, gc, mask)[:2]
        score = _score(seq, pooled, wsd, wpd)
        if partial:
            torch.autograd.grad(score, [seq])
        else:
            score.backward()
        outs.clear()
        grads.clear()
        return torch.cuda.memory_allocated()

    with hooks(handles):
        step(False)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        for partial in (False, True, False):
            step(partial)
            torch.cuda.synchronize()
            assert torch.cuda.memory_allocated() == base, partial


def run_refusals(dev, weights):
    """Every hook the module path cannot honour raises, naming the module."""
    model = _model(weights, dev, p=0.0)
    grid, ids, mask, L, g = RG._inputs("cpu" if dev.type == "cpu" else "224px", 167)
    ids, mask, grid = ids.to(dev), mask.to(dev), grid.to(dev)
    lay = model.encoder.layer[2]
    leaves = [(lay.attention.self.query, "attention.self.query", "layer.2.attention.self"),
              (lay.output.dense, "layer.2.output.dense", "layer.2.output"),
              (lay.attention.output.LayerNorm, "attention.output.LayerNorm", "attention.output"),
              (model.embeddings.position_embeddings, "embeddings.position_embeddings", "bert.embeddings"),
              (model.visual_embeddings.row_position_embeddings, "row_position_embeddings", "bert.visual_embeddings"),
              (model.pooler.dense, "pooler.dense", "bert.pooler"),
              (model.encoder.layer, "bert.encoder.layer", "bert.encoder")]
    for mod, name, parent in leaves:
        with hooks([mod.register_forward_hook(lambda m, i, o: None)]):
            with pytest.raises(RuntimeError, match=name) as e:
                model(ids, grid, mask)
            assert parent in str(e.value)
    with hooks([lay.register_forward_pre_hook(lambda m, a: (a[0], a[1] * 2.0, None))]):
        with pytest.raises(RuntimeError, match="BertLayer.*extended mask"):
            model(ids, grid, mask)
    with hooks([lay.attention.register_forward_pre_hook(lambda m, a: (a[0], a[1], torch.ones(12)))]):
        with pytest.raises(RuntimeError, match="BertAttention received a head_mask"):
            model(ids, grid, mask)
    assert model.output_hidden_states
    with hooks([model.encoder.register_forward_hook(lambda m, i, o: (o[0], tuple(t * 1 for t in o[1])) + tuple(o[2:]))]):
        with pytest.raises(RuntimeError, match="bert.encoder replaced a member"):
            model(ids, grid, mask)
    for mod in (model.encoder.layer[0], model.embeddings, model.pooler):
        with pytest.raises(RuntimeError, match="%s of ClipBertBaseModel runs only inside" % type(mod).__name__):
            mod(torch.zeros(1, 3, 768, device=dev))
    head = _head(weights, dev)
    with hooks([head.classifier.register_forward_hook(lambda m, i, o: None)]):
        with pytest.raises(RuntimeError, match="head's own module classifier"):
            head(ids, grid, mask)
    with hooks([head.bert.encoder.layer[0].register_forward_hook(lambda m, i, o: None)]):
        head._grad_ready_hook = lambda g: None
        try:
            with pytest.raises(RuntimeError, match="enable_overlapped_allreduce"):
                head(ids, grid, mask)
        finally:
            head._grad_ready_hook = None


def test_refusals(cuda, weights):
    run_refusals(cuda, weights)


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)
