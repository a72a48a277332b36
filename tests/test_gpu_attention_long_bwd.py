"""Tensor-core attention backward for sequences longer than 64 tokens (attn_tc_bwd_kv_kernel / attn_tc_bwd_q_kernel): against
fp32 torch autograd, against the CUDA-core backward (cb_debug_attention_general), with pitched buffers, run to run, under
dropout, and inside the full model at 768 px (L = 25 + 144 = 169)."""
import ctypes

import pytest
import torch

from util import TOL_BF16_OP, TOL_GRAD, TOL_LOGITS, cosine, make_cfg, relerr

pytestmark = pytest.mark.gpu

HEADS = 12


def _rnd(g, *shape, scale=1.0, dev="cuda"):
    return (torch.randn(*shape, generator=g) * scale).to(dev).to(torch.bfloat16)


def _mask(nseq, lt):
    """Text mask with some masked keys (as test_attention_fwd_bwd builds it); a [nseq, 1] dummy when there is no text."""
    mask = torch.ones(nseq, max(lt, 1), dtype=torch.int64)
    if lt > 4:
        mask[0, lt - 3:] = 0
        mask[-1, lt // 2:] = 0
    return mask if lt > 0 else torch.ones(nseq, 1, dtype=torch.int64)


def _general(on):
    from clipbert_b200 import _lib
    _lib.lib().cb_debug_attention_general(ctypes.c_int(on))


# (nseq, L, lt): one live row in the tail tile, the 448 px and 768 px shapes, exact tiles, 512-token text, no text
SHAPES = [(2, 65, 20), (2, 69, 20), (2, 128, 64), (2, 149, 100), (2, 169, 25), (1, 174, 30), (1, 521, 512), (2, 80, 0)]


@pytest.mark.parametrize("dims", SHAPES)
def test_long_attention_backward_matches_autograd(cuda, dims):
    from clipbert_b200 import ops
    nseq, L, lt = dims
    g = torch.Generator().manual_seed(31)
    qkv = _rnd(g, nseq * L, 3 * 768)
    dctx = _rnd(g, nseq * L, 768)
    mask = _mask(nseq, lt)
    mask_c = mask.to(cuda)
    ctx = torch.empty(nseq * L, 768, device=cuda, dtype=torch.bfloat16)
    lse = torch.empty(nseq, HEADS, L, device=cuda)
    ops.attention_fwd(qkv, mask_c, ctx, lse, nseq, L, lt, HEADS, 0.0, 0)
    dqkv = torch.empty_like(qkv)
    ops.attention_bwd(qkv, mask_c, ctx, dctx, lse, dqkv, nseq, L, lt, HEADS, 0.0, 0)

    x = qkv.float().view(nseq, L, 3, HEADS, 64).requires_grad_(True)
    q, k, v = (x[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    full = torch.cat([mask[:, :lt].to(cuda), torch.ones(nseq, L - lt, dtype=torch.int64, device=cuda)], 1)
    ext = (1.0 - full[:, None, None, :].float()) * -10000.0
    p = torch.softmax(q @ k.transpose(-1, -2) / 8.0 + ext, -1)
    ref = (p @ v).permute(0, 2, 1, 3).reshape(nseq * L, 768)
    ref.backward(dctx.float())
    e = relerr(dqkv, x.grad.reshape(nseq * L, 3 * 768))
    assert e < 2 * TOL_BF16_OP, e


@pytest.mark.parametrize("dims", [(2, 69, 20), (2, 149, 100), (1, 521, 512)])
def test_long_attention_backward_matches_cuda_core_backward(cuda, dims):
    """One forward, then the backward on the tensor-core kernels and on the CUDA-core kernels, with and without dropout (same
    seed: both regenerate the same dropout stream)."""
    from clipbert_b200 import ops
    nseq, L, lt = dims
    g = torch.Generator().manual_seed(32)
    qkv, dctx = _rnd(g, nseq * L, 3 * 768), _rnd(g, nseq * L, 768)
    mask = _mask(nseq, lt).to(cuda)
    for p, seed in ((0.0, 0), (0.1, 5)):
        ctx = torch.empty(nseq * L, 768, device=cuda, dtype=torch.bfloat16)
        lse = torch.empty(nseq, HEADS, L, device=cuda)
        ops.attention_fwd(qkv, mask, ctx, lse, nseq, L, lt, HEADS, p, seed)
        outs = []
        try:
            for general in (0, 1):
                _general(general)
                dqkv = torch.empty_like(qkv)
                ops.attention_bwd(qkv, mask, ctx, dctx, lse, dqkv, nseq, L, lt, HEADS, p, seed)
                outs.append(dqkv)
        finally:
            _general(0)
        e = relerr(outs[0], outs[1])
        assert e < 3 * TOL_BF16_OP, (p, e)


@pytest.mark.parametrize("dims", [(2, 69, 20), (2, 169, 25)])
def test_long_attention_backward_pitched_buffers(cuda, dims):
    """Row pitches wider than the packed width: the padding columns of dqkv are never written, every live row is, and the
    result equals the packed call's."""
    from clipbert_b200 import ops
    nseq, L, lt = dims
    g = torch.Generator().manual_seed(33)
    qkv, dctx = _rnd(g, nseq * L, 3 * 768), _rnd(g, nseq * L, 768)
    mask = _mask(nseq, lt).to(cuda)
    ctx = torch.empty(nseq * L, 768, device=cuda, dtype=torch.bfloat16)
    lse = torch.empty(nseq, HEADS, L, device=cuda)
    ops.attention_fwd(qkv, mask, ctx, lse, nseq, L, lt, HEADS, 0.1, 9)
    packed = torch.empty_like(qkv)
    ops.attention_bwd(qkv, mask, ctx, dctx, lse, packed, nseq, L, lt, HEADS, 0.1, 9)

    ld_qkv, ld_ctx, ld_dqkv = 3 * 768 + 64, 768 + 128, 3 * 768 + 192
    qkv_p = torch.zeros(nseq * L, ld_qkv, device=cuda, dtype=torch.bfloat16)
    qkv_p[:, :3 * 768] = qkv
    ctx_p = torch.zeros(nseq * L, ld_ctx, device=cuda, dtype=torch.bfloat16)
    ctx_p[:, :768] = ctx
    dctx_p = torch.zeros(nseq * L, ld_ctx, device=cuda, dtype=torch.bfloat16)
    dctx_p[:, :768] = dctx
    sentinel = 12345.0     # exact in bf16, never a gradient here
    dqkv_p = torch.full((nseq * L, ld_dqkv), sentinel, device=cuda, dtype=torch.bfloat16)
    ops._call("cb_attention_bwd", ops._p(qkv_p), ld_qkv, ops._p(mask), ops._p(ctx_p), ops._p(dctx_p), ld_ctx, ops._p(lse),
              ops._p(dqkv_p), ld_dqkv, nseq, L, lt, HEADS, 64, 0.1, 9, ops._s())
    torch.cuda.synchronize()
    assert bool((dqkv_p[:, 3 * 768:] == sentinel).all()), "padding columns written"
    assert not bool((dqkv_p[:, :3 * 768] == sentinel).any()), "a live element was not written"
    assert torch.equal(dqkv_p[:, :3 * 768], packed)


def test_long_attention_backward_is_repeatable(cuda):
    from clipbert_b200 import ops
    nseq, L, lt = 2, 149, 100
    g = torch.Generator().manual_seed(34)
    qkv, dctx = _rnd(g, nseq * L, 3 * 768), _rnd(g, nseq * L, 768)
    mask = _mask(nseq, lt).to(cuda)
    ctx = torch.empty(nseq * L, 768, device=cuda, dtype=torch.bfloat16)
    lse = torch.empty(nseq, HEADS, L, device=cuda)
    ops.attention_fwd(qkv, mask, ctx, lse, nseq, L, lt, HEADS, 0.1, 3)
    outs = []
    for _ in range(2):
        dqkv = torch.full_like(qkv, float("nan"))
        ops.attention_bwd(qkv, mask, ctx, dctx, lse, dqkv, nseq, L, lt, HEADS, 0.1, 3)
        outs.append(dqkv)
    assert torch.equal(outs[0], outs[1])


def test_long_attention_backward_dropout_is_linear_in_dout(cuda):
    """With p > 0 the backward regenerates the forward's dropout mask from the seed: for a fixed mask it is linear in dO."""
    from clipbert_b200 import ops
    nseq, L, lt = 2, 149, 100
    g = torch.Generator().manual_seed(35)
    qkv = _rnd(g, nseq * L, 3 * 768, scale=0.5)
    mask = _mask(nseq, lt).to(cuda)
    ctx = torch.empty(nseq * L, 768, device=cuda, dtype=torch.bfloat16)
    lse = torch.empty(nseq, HEADS, L, device=cuda)
    ops.attention_fwd(qkv, mask, ctx, lse, nseq, L, lt, HEADS, 0.1, 77)
    d1, d2 = _rnd(g, nseq * L, 768), _rnd(g, nseq * L, 768)
    outs = []
    for d in (d1, d2, (d1.float() + d2.float()).to(torch.bfloat16)):
        dq = torch.empty_like(qkv)
        ops.attention_bwd(qkv, mask, ctx, d, lse, dq, nseq, L, lt, HEADS, 0.1, 77)
        outs.append(dq.float())
    assert relerr(outs[2], outs[0] + outs[1]) < 3 * TOL_BF16_OP
    # and the dropout really changes the result
    dq0 = torch.empty_like(qkv)
    ops.attention_bwd(qkv, mask, ctx, d1, lse, dq0, nseq, L, lt, HEADS, 0.0, 77)
    assert relerr(outs[0], dq0.float()) > 1e-2


def test_model_768px_forward_backward(cuda):
    """1 video x 1 frame at 768 px (12 x 12 = 144 visual tokens) with 25-token captions: L = 169 through all 12 layers. Logits
    of the default path against the oracle; every transformer parameter gradient of the tensor-core attention backward against
    the CUDA-core one. For the gradients both runs use the same (CUDA-core) attention forward, so that they see the same
    activations: otherwise last-bit differences between the two forwards flip units of the classifier ReLU, and the gradients
    upstream of it then differ by far more than the backward kernels do."""
    import clipbert_b200 as cb
    from clipbert_b200 import ops
    from model_util import cnn_patterns
    from oracle import clipbert_ref as R, synth
    weights = synth.full_state_dict(42)
    model = cb.ClipBert(make_cfg(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0), detectron2_model_cfg="R-50-grid.yaml",
                        transformer_cls=cb.ClipBertForVideoTextRetrieval)
    assert not model.load_state_dict(weights).missing_keys
    model = model.to(cuda).train()
    batch = synth.synth_batch(1, 1, n_ex=2, size=768, max_len=25, seed=23)
    mb = {k: (v.to(cuda) if torch.is_tensor(v) else list(v)) for k, v in batch.items()}

    def run(general, capture=False):
        _general(general)
        model.zero_grad()
        if capture:
            model.cnn._capture, model.transformer._capture = {}, {}
        d = dict(mb)
        out = model(d)           # replaces d["visual_inputs"] by the grid features
        pat = None
        if capture:
            assert d["visual_inputs"].shape == (1, 1, 12, 12, 768)
            pat = cnn_patterns(model.cnn._capture["stash"], d["visual_inputs"])
            pat.relu_masks["transformer.classifier.relu"] = (model.transformer._capture["c1"] > 0).cpu()
            model.cnn._capture = model.transformer._capture = None
        out["loss"].mean().backward()
        torch.cuda.synchronize()
        grads = {n: p.grad.detach().clone() for n, p in model.named_parameters()
                 if n.startswith("transformer.") and p.grad is not None}
        return out, grads, pat

    try:
        out, _, pat = run(0, capture=True)       # the default path: tensor-core forward and backward
        ops.set_attention_flash(0)
        out_tc, g_tc, _ = run(0)                 # CUDA-core forward, tensor-core backward
        out_gen, g_gen, _ = run(1)               # CUDA-core forward and backward
    finally:
        ops.set_attention_flash(1)
        _general(0)
    assert torch.equal(out_tc["logits"], out_gen["logits"])
    with torch.no_grad():
        ref = R.clipbert_forward(dict(batch), weights, rnd=pat)
    assert relerr(out["logits"], ref["logits"]) < TOL_LOGITS, relerr(out["logits"], ref["logits"])

    assert set(g_tc) == set(g_gen) and any("encoder.layer.11.attention.self.query" in n for n in g_tc)
    bad = []
    for n, ref_g in g_gen.items():
        if float(ref_g.abs().sum()) == 0.0 or n.endswith("attention.self.key.bias"):
            continue       # the key bias gradient is zero in exact arithmetic (softmax is shift-invariant): only noise is left
        e, c = relerr(g_tc[n], ref_g), cosine(g_tc[n], ref_g)
        if not (e <= TOL_GRAD and c >= 0.999):
            bad.append((n, e, c))
    assert not bad, bad[:10]
