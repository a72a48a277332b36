"""ClipBertBaseModel.forward (src/modeling/modeling.py:201-238) on the H100 path, and the argument checks of cb_attention_probs,
the kernel behind its output_attentions (its results are checked element by element in test_gpu_attention_probs_elementwise.py).

Module: outputs, hidden states and attentions against the reference-generated golden vectors and the oracle, gradients of
every transformer parameter and of visual_inputs against fp32 autograd, dropout pattern of train-mode attentions, CUDA-graph
replay, and the heads unchanged by the two flags. The test bodies take the device as an argument: tests/test_base_model_emulated.py replays them on CPU.
"""

import pytest
import torch

import dropout_ref as D
from util import TOL_FP32_E2E, TOL_GRAD, TOL_LOGITS, TOL_MATCHED, TOL_MATCHED_DEEP, cosine, make_cfg, relerr

pytestmark = pytest.mark.gpu

HEADS = 3


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)


def _qkv_case(L, padded, seed, nseq=2, dev="cpu"):
    g = torch.Generator().manual_seed(seed)
    lt = max(1, L - 9) if L > 9 else L
    qkv = torch.randn(nseq * L, 3 * HEADS * 64, generator=g).to(torch.bfloat16)
    mask = torch.ones(nseq, lt, dtype=torch.int64)
    if padded and lt > 2:
        mask[0, lt // 2:] = 0            # the [CLS] key stays live: a row never sees only masked keys
        mask[1, lt - 1] = 0
    return qkv.to(dev), mask.to(dev), lt


def test_attention_probs_rejects_bad_arguments(cuda):
    from clipbert_b200 import ops
    qkv, mask, lt = _qkv_case(41, False, 3, 2, cuda)
    lse = torch.zeros(2, HEADS, 41, device=cuda)
    buf = torch.empty(2 * HEADS * 41 * 41 + 1, device=cuda)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        ops.attention_probs(qkv, mask, lse, buf[1:].view(2, HEADS, 41, 41), 2, 41, lt, HEADS, 0.0, 1)
    with pytest.raises(RuntimeError, match="bad arguments"):
        ops._call("cb_attention_probs", ops._p(qkv), qkv.shape[1], ops._p(mask), ops._p(lse), ops._p(buf), 2, 41, 42, HEADS, 64, 0.0, 1, ops._s())


def test_attention_fwd_bwd_reject_bad_arguments(cuda):
    """cb_attention_fwd / _bwd check what cb_attention_probs checks, on the host, before any launch: 0 <= lt <= l, heads > 0,
    nseq and heads within the grid (65535), row pitches that hold Q | K | V and the merged heads, 16-byte aligned vectors."""
    from clipbert_b200 import ops
    n, L = 2, 41
    hid = HEADS * 64
    qkv, mask, lt = _qkv_case(L, False, 3, n, cuda)
    flat = torch.zeros(n * L * 3 * hid + 8, dtype=torch.bfloat16, device=cuda)
    ctx, dctx = (torch.zeros(n * L * hid + 8, dtype=torch.bfloat16, device=cuda) for _ in range(2))
    lse = torch.zeros(n, HEADS, L, device=cuda)
    P = ops._p

    def fwd(q=qkv, ld_q=3 * hid, c=ctx, ld_c=hid, nseq=n, lt_=lt, heads=HEADS):
        ops._call("cb_attention_fwd", P(q), ld_q, P(mask), P(c), ld_c, P(lse), nseq, L, lt_, heads, 64, 0.0, 1, ops._s())

    def bwd(q=qkv, ld_q=3 * hid, c=ctx, d=dctx, ld_c=hid, dq=flat, ld_dq=3 * hid, nseq=n, lt_=lt, heads=HEADS):
        ops._call("cb_attention_bwd", P(q), ld_q, P(mask), P(c), P(d), ld_c, P(lse), P(dq), ld_dq, nseq, L, lt_, heads, 64, 0.0, 1,
                  ops._s())

    for f in (fwd, bwd):
        for kw in (dict(lt_=L + 1), dict(lt_=-1), dict(heads=0), dict(nseq=65536), dict(heads=65536)):
            with pytest.raises(RuntimeError, match="bad arguments"):
                f(**kw)
        for kw in (dict(ld_q=3 * hid - 8), dict(ld_c=hid - 8)):
            with pytest.raises(RuntimeError, match="row pitches must hold"):
                f(**kw)
        for kw in (dict(q=flat[1:]), dict(c=ctx[1:])):
            with pytest.raises(RuntimeError, match="16-byte aligned"):
                f(**kw)
    with pytest.raises(RuntimeError, match="row pitches must hold"):
        bwd(ld_dq=3 * hid - 8)
    for kw in (dict(d=dctx[1:]), dict(dq=flat[1:])):
        with pytest.raises(RuntimeError, match="16-byte aligned"):
            bwd(**kw)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ module
def _base(sd, cuda, hidden=True, attn=True, **cfg_extra):
    import clipbert_b200 as cb
    cfg = make_cfg(**dict(dict(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0), **cfg_extra))
    cfg.output_hidden_states, cfg.output_attentions = hidden, attn
    model = cb.ClipBertBaseModel(cfg)
    res = model.load_state_dict({k[len("transformer.bert."):]: v for k, v in sd.items() if k.startswith("transformer.bert.")})
    assert not res.missing_keys and not res.unexpected_keys
    return model.to(cuda)


def _oracle_probs():
    """drop hook of oracle.clipbert_ref that records each layer's attention probabilities (and applies no dropout)."""
    rec = {}

    def drop(site, layer, x):
        if site == "attn_probs":
            rec[layer] = x
        return x
    return rec, drop


def test_base_model_against_reference_golden(cuda, weights):
    """tests/golden/transformer_base_outputs.pt: the reference's own ClipBertBaseModel with both flags on (fp32, eval)."""
    import os
    g = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "transformer_base_outputs.pt"),
                   map_location="cpu", weights_only=False)
    model = _base(weights, cuda).eval()
    for key in ("L41", "L69"):
        c = g[key]
        with torch.no_grad():
            seq, pooled, hidden, attn = model(c["ids"].to(cuda), c["grid"].to(cuda), c["mask"].to(cuda))
        L = c["L"]
        assert seq.shape == (2, L, 768) and pooled.shape == (2, 768) and len(hidden) == 13 and len(attn) == 12
        assert seq.dtype == pooled.dtype == hidden[0].dtype == torch.bfloat16 and attn[0].dtype == torch.float32
        assert attn[0].shape == (2, 12, L, L) and torch.equal(seq, hidden[-1])
        assert relerr(pooled, c["pooled"]) < TOL_FP32_E2E
        assert relerr(seq[:, :, :32], c["seq_slice"]) < TOL_FP32_E2E
        for k in range(13):
            assert relerr(hidden[k][:, :2, :32], c["hidden_slices"][k]) < TOL_FP32_E2E, (key, k)
            mean, std = c["hidden_stats"][k].tolist()
            got = hidden[k].float()
            assert abs(float(got.std()) / std - 1) < 1e-2 and abs(float(got.mean()) - mean) < 1e-2 * std, (key, k)
        for j, layer in enumerate(c["attn_layers"]):
            a = attn[layer][:1, :2]
            assert relerr(a, c["attentions"][j]) < TOL_FP32_E2E, (key, layer, relerr(a, c["attentions"][j]))


def _check_against_oracle(model, ids, grid, mask, weights, cuda):
    from oracle import clipbert_ref as R
    rec16, drop16 = _oracle_probs()
    rec32, drop32 = _oracle_probs()
    with torch.no_grad():
        seq16, pooled16, layers16 = R.clipbert_base_model(ids, grid, mask, weights, return_layers=True, rnd=R.Rounding.bf16(), drop=drop16)
        seq32, pooled32, layers32 = R.clipbert_base_model(ids, grid, mask, weights, return_layers=True, drop=drop32)
        seq, pooled, hidden, attn = model(ids.to(cuda), grid.to(cuda), mask.to(cuda))
    assert relerr(hidden[0], layers16[0]) < TOL_MATCHED
    for i in range(1, 13):
        e16, e32 = relerr(hidden[i], layers16[i]), relerr(hidden[i], layers32[i])
        assert e16 < TOL_MATCHED_DEEP * 1.5 and e32 < TOL_FP32_E2E, (i, e16, e32)
        a16, a32 = relerr(attn[i - 1], rec16[i - 1]), relerr(attn[i - 1], rec32[i - 1])
        assert a16 < TOL_MATCHED_DEEP * 1.5 and a32 < TOL_FP32_E2E, (i - 1, a16, a32)
    assert relerr(pooled, pooled16) < TOL_LOGITS and relerr(pooled, pooled32) < TOL_LOGITS
    assert torch.equal(seq, hidden[-1])


@pytest.mark.parametrize("size", ["224px", "448px", "512tok"])
def test_base_model_against_oracle(cuda, weights, size):
    from oracle import synth
    model = _base(weights, cuda).eval()
    g = torch.Generator().manual_seed(41)
    nseq, lt, gh = {"224px": (3, 32, 3), "448px": (2, 20, 7), "512tok": (1, 512, 3)}[size]
    grid = (torch.randn(nseq, 2, gh, gh, 768, generator=g).abs()).to(torch.bfloat16).float()
    ids, mask = synth.synth_text(nseq, lt, seed=43)
    _check_against_oracle(model, ids, grid, mask, weights, cuda)


def test_base_model_gradients(cuda, weights, nseq=3, lt=24, gh=3):
    """A mixed upstream gradient - d sequence_output, d pooled_output, d hidden_states[0 / 5 / 12] - into every transformer
    parameter and into visual_inputs, against fp32 autograd on the oracle."""
    from oracle import clipbert_ref as R, synth
    model = _base(weights, cuda).train()                  # dropout p = 0 (see _base)
    g = torch.Generator().manual_seed(51)
    grid = (torch.randn(nseq, 2, gh, gh, 768, generator=g).abs()).to(torch.bfloat16).float()
    ids, mask = synth.synth_text(nseq, lt, seed=52)
    L = lt + gh * gh
    dseq, dpool = torch.randn(nseq, L, 768, generator=g) * 0.1, torch.randn(nseq, 768, generator=g)
    dh = {0: torch.randn(nseq, L, 768, generator=g) * 0.1, 5: torch.randn(nseq, L, 768, generator=g) * 0.1,
          12: torch.randn(nseq, L, 768, generator=g) * 0.1}
    dseq, dpool = dseq.to(torch.bfloat16).float(), dpool.to(torch.bfloat16).float()
    dh = {k: v.to(torch.bfloat16).float() for k, v in dh.items()}
    sd = {k: (v.clone().requires_grad_(True) if k.startswith("transformer.bert.") else v) for k, v in weights.items()}
    gr = grid.clone().requires_grad_(True)
    seq_r, pooled_r, layers_r = R.clipbert_base_model(ids, gr, mask, sd, return_layers=True)
    (seq_r * dseq).sum().add_((pooled_r * dpool).sum()).add_(sum((layers_r[k] * v).sum() for k, v in dh.items())).backward()
    gc = grid.to(cuda).requires_grad_(True)               # fp32 visual_inputs: the cast to bf16 is part of the graph
    seq, pooled, hidden, attn = model(ids.to(cuda), gc, mask.to(cuda))
    assert seq.requires_grad and hidden[0].requires_grad and not attn[0].requires_grad
    loss = (seq.float() * dseq.to(cuda)).sum() + (pooled.float() * dpool.to(cuda)).sum()
    loss = loss + sum((hidden[k].float() * v.to(cuda)).sum() for k, v in dh.items())
    loss.backward()
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
    assert checked >= 12 * 15 + 2                        # every encoder parameter but key.bias, the pooler, the embeddings


def test_train_mode_attentions_carry_the_forward_dropout_mask(cuda, weights):
    """Train mode, attention dropout 0.1: each returned P is the post-dropout tensor of the reference (transformers.py:271,284),
    zero exactly where the fused forward dropped, at the step's seed and device word; the kept elements scaled by 1 / 0.9."""
    from oracle import synth
    p = 0.1
    model = _base(weights, cuda, attention_probs_dropout_prob=p, hidden_dropout_prob=0.1).train()
    eng = model._engine
    g = torch.Generator().manual_seed(61)
    nseq, lt = 2, 20
    grid = (torch.randn(nseq, 1, 7, 7, 768, generator=g).abs()).to(torch.bfloat16).float()
    ids, mask = synth.synth_text(nseq, lt, seed=62)
    with torch.no_grad():
        model(ids.to(cuda), grid.to(cuda), mask.to(cuda))        # advances the stream once: masks differ between calls
        seq, pooled, hidden, attn = model(ids.to(cuda), grid.to(cuda), mask.to(cuda))
    seed = (eng._seed_base + eng._call_count * 1000003) & (2 ** 64 - 1)
    word = int(eng._drop_counter.item())
    L = lt + 49
    idx = D.attention_index(nseq, 12, L)
    for i in (0, 7, 11):
        keep = torch.from_numpy(D.multipliers(D.effective_seed(seed + 16 * (i + 1) + 1, word), idx, p)) != 0
        a = attn[i].cpu()
        live = torch.cat([mask.bool(), torch.ones(nseq, L - lt, dtype=torch.bool)], 1)[:, None, None, :].expand_as(a)
        assert torch.equal(a[live] != 0, keep[live]), i
        assert float(a[live & ~keep].abs().max()) == 0.0
        # kept probabilities of a row sum to (1 / 0.9) x (1 - dropped mass): between 0 and 1 / 0.9
        assert float(a.sum(-1).max()) < 1 / (1 - p) + 1e-4


def test_cuda_graph_train_step_through_bert(cuda, weights):
    """A train-mode forward + backward through bert(...) captured once: replays draw fresh masks (the device word advances),
    and a replay rewound to an eager step's position reproduces that step's outputs and gradients."""
    from oracle import synth
    model = _base(weights, cuda, attn=False, attention_probs_dropout_prob=0.1, hidden_dropout_prob=0.1).train()
    eng = model._engine
    g = torch.Generator().manual_seed(71)
    grid = (torch.randn(2, 1, 3, 3, 768, generator=g).abs()).to(torch.bfloat16).to(cuda)
    ids, mask = synth.synth_text(2, 16, seed=72)
    ids, mask = ids.to(cuda), mask.to(cuda)
    w = torch.randn(2, 25, 768, generator=g).to(cuda)
    probe = model.encoder.layer[0].attention.self.query.weight

    def step():
        model.zero_grad(set_to_none=False)
        seq, pooled, hidden = model(ids, grid, mask)
        loss = (seq.float() * w).sum() + pooled.float().sum() + hidden[3].float().sum()
        loss.backward()
        return loss

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    calls0, w0 = eng._call_count, int(eng._drop_counter.item())
    g_ = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g_, stream=s):
        loss_dev = step().detach()                     # host seed of call calls0 + 1 baked in; the word advances on the device
    losses, words = [], []
    for _ in range(2):
        g_.replay()
        torch.cuda.synchronize()
        losses.append(float(loss_dev))
        words.append(int(eng._drop_counter.item()))
    assert words[1] == words[0] + 1 and losses[0] != losses[1]     # fresh masks at every replay
    # an eager step with the captured call's host seed at the first replay's position, then that replay again
    eng._call_count = calls0
    eng._drop_counter.fill_(w0)
    eager_loss = float(step().detach())
    eager_grad = probe.grad.detach().clone()
    eng._drop_counter.fill_(w0)
    g_.replay()
    torch.cuda.synchronize()
    assert abs(float(loss_dev) - eager_loss) <= 1e-5 * abs(eager_loss) and abs(losses[0] - eager_loss) <= 1e-5 * abs(eager_loss)
    assert relerr(probe.grad, eager_grad) < 1e-4


def test_heads_ignore_the_output_flags(cuda, weights):
    """output_hidden_states / output_attentions only shape bert(...): a head's forward, its launches and its logits are the same."""
    import clipbert_b200 as cb
    from clipbert_b200 import ops
    from oracle import synth
    g = torch.Generator().manual_seed(81)
    grid = (torch.randn(2, 1, 3, 3, 768, generator=g).abs()).to(torch.bfloat16).to(cuda)
    ids, mask = synth.synth_text(4, 16, seed=82)
    res = []
    for flags in (False, True):
        cfg = make_cfg(output_hidden_states=flags, output_attentions=flags)
        head = cb.ClipBertForVideoTextRetrieval(cfg)
        head.load_state_dict({k[len("transformer."):]: v for k, v in weights.items() if k.startswith("transformer.")})
        head = head.to(cuda).eval()
        with torch.no_grad():
            head(ids.to(cuda), grid, mask.to(cuda), _repeat_counts=[2, 2])     # warm-up
            n0 = ops.launch_count() if cuda.type == "cuda" else 0
            logits = head(ids.to(cuda), grid, mask.to(cuda), _repeat_counts=[2, 2])["logits"]
            n1 = ops.launch_count() if cuda.type == "cuda" else 0
        res.append((logits.clone(), n1 - n0))
    assert torch.equal(res[0][0], res[1][0]) and res[0][1] == res[1][1]
