"""Model-level parity of the H100 path against the CPU oracle (same seeded weights and inputs).

Forward: per stage and end to end, against BOTH the plain fp32 oracle and the bf16-rounding-matched
oracle (oracle.clipbert_ref.Rounding.bf16). Backward: every trainable parameter gradient and the
gradient flowing into the CNN, against fp32 autograd on the oracle. Dropout is off (eval-mode
probabilities, p = 0); training with dropout on is compared with the oracle under the same masks in test_gpu_dropout.py.
"""
import pytest
import torch

from model_util import cnn_patterns
from util import TOL_FP32_E2E, TOL_GRAD, TOL_LOGITS, TOL_MATCHED, TOL_MATCHED_DEEP, cosine, make_cfg, relerr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)


def _build(cls_name, sd, cuda, **cfg_extra):
    import clipbert_b200 as cb
    cfg = make_cfg(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, **cfg_extra)
    model = cb.ClipBert(cfg, detectron2_model_cfg="R-50-grid.yaml", transformer_cls=getattr(cb, cls_name))
    missing = model.load_state_dict(sd)
    assert not missing.missing_keys, missing
    return model.to(cuda)


@pytest.mark.parametrize("size", [224, 96])
def test_cnn_forward_stages(cuda, weights, size):
    from oracle import clipbert_ref as R, synth
    model = _build("ClipBertForVideoTextRetrieval", weights, cuda).eval()
    x = synth.synth_images(2, 2, size=size, seed=5)
    with torch.no_grad():
        _, st32 = R.grid_feat_backbone(x, weights, return_stages=True)
        _, st16 = R.grid_feat_backbone(x, weights, return_stages=True, rnd=R.Rounding.bf16())
        model.cnn._capture = {}
        grid = model.cnn(x.to(cuda))
    cap = model.cnn._capture
    model.cnn._capture = None
    assert grid.shape == st32["grid"].shape
    for name in ("stem", "res2", "res3", "res4", "res5"):
        got = cap[name].float().permute(0, 3, 1, 2)
        assert relerr(got, st16[name]) < TOL_MATCHED_DEEP, (name, relerr(got, st16[name]))
        assert relerr(got, st32[name]) < TOL_FP32_E2E, (name, relerr(got, st32[name]))
    assert relerr(grid, st16["grid"]) < TOL_MATCHED_DEEP, relerr(grid, st16["grid"])
    assert relerr(grid, st32["grid"]) < TOL_FP32_E2E


def test_cnn_backward(cuda, weights):
    from oracle import clipbert_ref as R, synth
    model = _build("ClipBertForVideoTextRetrieval", weights, cuda).train()
    x = synth.synth_images(2, 2, size=224, seed=6)
    g = torch.Generator().manual_seed(1)
    sd = {k: (v.clone().requires_grad_(True) if (k.endswith(".weight") and "norm" not in k and k.startswith("cnn.")) else v)
          for k, v in weights.items()}
    model.cnn._capture = {}
    grid = model.cnn(x.to(cuda))
    # the oracle differentiates along the SAME ReLU / max-pool selection as the run (see Rounding.relu_masks)
    pat = cnn_patterns(model.cnn._capture["stash"], grid)
    model.cnn._capture = None
    grid_ref = R.grid_feat_backbone(x, sd, rnd=pat)
    assert relerr(grid, grid_ref) < TOL_FP32_E2E
    dgrid = torch.randn(grid_ref.shape, generator=g).to(torch.bfloat16).float()
    grid_ref.backward(dgrid)
    grid.backward(dgrid.to(cuda).to(grid.dtype))
    checked = 0
    for name, p in model.cnn.named_parameters():
        key = "cnn." + name
        ref = sd[key].grad
        if not p.requires_grad:
            assert ref is None or float(ref.abs().sum()) == 0.0 or "res2" in key or "stem" in key
            continue
        assert p.grad is not None, key
        assert cosine(p.grad, ref) > 0.999, (key, cosine(p.grad, ref))
        assert relerr(p.grad, ref) < TOL_GRAD, (key, relerr(p.grad, ref))
        checked += 1
    assert checked == 3 * 13 + 3 + 1        # res3-5 convs + 3 shortcuts + grid_encoder


@pytest.mark.parametrize("n_ex", [1, 2])
def test_transformer_forward_backward(cuda, weights, n_ex):
    from oracle import clipbert_ref as R, synth
    model = _build("ClipBertForVideoTextRetrieval", weights, cuda).train()
    tr = model.transformer
    nvid, T = 3, 2
    g = torch.Generator().manual_seed(2)
    grid = (torch.randn(nvid, T, 3, 3, 768, generator=g).abs() * 2).to(torch.bfloat16).float()
    ids, mask = synth.synth_text(nvid * n_ex, 32, seed=3)
    labels = torch.randint(0, 2, (nvid * n_ex,), generator=g)
    sd = {k: (v.clone().requires_grad_(True) if k.startswith("transformer.") else v) for k, v in weights.items()}
    gr = grid.clone().requires_grad_(True)
    rep = R.repeat_tensor_rows(gr, [n_ex] * nvid)
    seq, pooled, layers = R.clipbert_base_model(ids, rep, mask, sd, return_layers=True)
    logits_ref = R.mlp_head(pooled, sd)
    loss_ref = R.retrieval_loss(logits_ref, labels).mean()
    with torch.no_grad():
        _, _, layers16 = R.clipbert_base_model(ids, rep.detach(), mask, weights, return_layers=True, rnd=R.Rounding.bf16())
        out16 = R.video_text_retrieval(ids, rep.detach(), mask, weights, rnd=R.Rounding.bf16())

    gc = grid.to(cuda).to(torch.bfloat16).requires_grad_(True)
    tr._capture = {}
    out = tr(ids.to(cuda), gc, mask.to(cuda), labels=labels.to(cuda), sample_size=nvid, _repeat_counts=[n_ex] * nvid)
    cap, tr._capture = tr._capture, None
    assert relerr(cap["embeddings"], layers16[0]) < TOL_MATCHED
    assert relerr(cap["layer0"], layers16[1]) < 3 * TOL_MATCHED
    for i in range(12):
        e16, e32 = relerr(cap["layer%d" % i], layers16[i + 1]), relerr(cap["layer%d" % i], layers[i + 1])
        assert e16 < TOL_MATCHED_DEEP * 1.5 and e32 < TOL_FP32_E2E, (i, e16, e32)
    assert relerr(out["logits"], out16["logits"]) < TOL_LOGITS, relerr(out["logits"], out16["logits"])
    assert relerr(out["logits"], logits_ref) < TOL_LOGITS
    assert abs(float(out["loss"].mean()) - float(loss_ref)) < 2e-3
    # gradients: the oracle differentiates along the run's classifier ReLU pattern (see Rounding.relu_masks)
    hpat = R.Rounding(relu_masks={"transformer.classifier.relu": (cap["c1"] > 0).cpu()})
    R.retrieval_loss(R.mlp_head(pooled, sd, rnd=hpat), labels).mean().backward()
    out["loss"].mean().backward()
    assert relerr(gc.grad, gr.grad) < TOL_GRAD and cosine(gc.grad, gr.grad) > 0.999
    bad = []
    for name, p in tr.named_parameters():
        key = "transformer." + name
        ref = sd[key].grad
        if ref is None or float(ref.abs().sum()) == 0.0:
            assert p.grad is None or float(p.grad.abs().sum()) == 0.0, key
            continue
        if name.endswith("attention.self.key.bias"):
            # mathematically zero (softmax is invariant to a per-query constant): both sides are rounding noise
            qb = sd[key.replace("key.bias", "query.bias")].grad
            assert float(p.grad.norm()) < 0.05 * float(qb.norm()), key
            continue
        e, c = relerr(p.grad, ref), cosine(p.grad, ref)
        if not (e < TOL_GRAD and c > 0.999):
            bad.append((key, e, c))
    assert not bad, bad[:10]


def test_clipbert_end_to_end_two_clips_lse(cuda, weights):
    """ClipBert.forward per clip + the reference clip loop (run_video_retrieval.py:396-422), fwd+bwd."""
    from oracle import clipbert_ref as R, synth
    model = _build("ClipBertForVideoTextRetrieval", weights, cuda).train()
    n_clips, T, B, n_ex = 2, 2, 2, 2
    batch = synth.synth_batch(B, n_clips * T, n_ex=n_ex, size=224, seed=9)
    vis = batch["visual_inputs"].view(B, n_clips, T, 3, 224, 224)
    sd = {k: (v.clone().requires_grad_(True) if (k.endswith(("weight", "bias")) and "norm" not in k) else v) for k, v in weights.items()}
    logits, pats = [], []
    for c in range(n_clips):
        mb = {k: (v.to(cuda) if torch.is_tensor(v) else v) for k, v in batch.items()}
        mb["visual_inputs"] = vis[:, c].to(cuda)
        mb["n_examples_list"] = list(batch["n_examples_list"])
        model.cnn._capture, model.transformer._capture = {}, {}
        out = model(mb)
        assert "n_examples_list" not in mb and mb["sample_size"] == B      # reference dict mutations (e2e_model.py:31-37)
        logits.append(out["logits"])
        pat = cnn_patterns(model.cnn._capture["stash"], mb["visual_inputs"])
        pat.relu_masks["transformer.classifier.relu"] = (model.transformer._capture["c1"] > 0).cpu()
        pats.append(pat)
    model.cnn._capture = model.transformer._capture = None
    ref_logits = []
    for c in range(n_clips):
        mb = dict(batch, visual_inputs=vis[:, c])
        ref_logits.append(R.clipbert_forward(mb, sd, rnd=pats[c])["logits"])
    loss_ref = R.aggregate_clip_logits(ref_logits, batch["labels"], "lse")
    loss_ref.backward()
    lg = torch.stack(logits).permute(1, 0, 2).contiguous()
    o = torch.logsumexp(lg.view(lg.shape[0], -1), dim=-1, keepdim=True) - torch.logsumexp(lg, dim=1)
    loss = torch.gather(o, -1, batch["labels"].to(cuda).view(-1, 1)).mean()
    assert abs(float(loss) - float(loss_ref)) < 3e-3, (float(loss), float(loss_ref))
    for c in range(n_clips):
        assert relerr(logits[c], ref_logits[c]) < TOL_LOGITS
    loss.backward()
    bad = []
    for name, p in model.named_parameters():
        ref = sd[name].grad
        if not p.requires_grad or ref is None or float(ref.abs().sum()) == 0.0 or name.endswith("attention.self.key.bias"):
            continue
        e, c = relerr(p.grad, ref), cosine(p.grad, ref)
        if not (e < 2 * TOL_GRAD and c > 0.998):
            bad.append((name, e, c))
    assert not bad, bad[:10]
    # parameter-name contract used by setup_e2e_optimizer (src/optimization/utils.py:99-113)
    names = [n for n, _ in model.named_parameters()]
    assert any("grid_encoder" in n for n in names) and all(("cnn" in n) or ("transformer" in n) for n in names)


def test_multiple_choice_and_classification_heads(cuda, weights):
    from oracle import clipbert_ref as R, synth
    g = torch.Generator().manual_seed(4)
    grid = (torch.randn(2, 1, 3, 3, 768, generator=g).abs()).to(torch.bfloat16).float()
    # TGIF-QA style: 5 options per video, one score each, CE over options (modeling.py:430-451)
    sd = dict(weights)
    sd.update(synth.transformer_state_dict(50, num_labels=1))
    model = _build("ClipBertForMultipleChoice", sd, cuda, num_labels=5).eval()
    ids, mask = synth.synth_text(10, 25, seed=5)
    labels = torch.tensor([1, 4])
    with torch.no_grad():
        ref = R.multiple_choice(ids, R.repeat_tensor_rows(grid, [5, 5]), mask, sd, 5, labels, rnd=R.Rounding.bf16())
        out = model.transformer(ids.to(cuda), grid.to(cuda), mask.to(cuda), labels=labels.to(cuda), _repeat_counts=[5, 5])
    assert out["logits"].shape == (2, 5)
    assert relerr(out["logits"], ref["logits"]) < TOL_LOGITS and relerr(out["loss"], ref["loss"]) < 1e-2
    # VQA style: 3129-way BCE (num_labels not a multiple of 8 -> zero-padded head)
    sd.update(synth.transformer_state_dict(51, num_labels=3129))
    model = _build("ClipBertForSequenceClassification", sd, cuda, num_labels=3129, loss_type="bce").eval()
    ids, mask = synth.synth_text(2, 20, seed=6)
    tgt = (torch.rand(2, 3129, generator=g) > 0.99).float()
    with torch.no_grad():
        ref = R.sequence_classification(ids, grid, mask, sd, tgt, rnd=R.Rounding.bf16())
        out = model.transformer(ids.to(cuda), grid.to(cuda), mask.to(cuda), labels=tgt.to(cuda))
    assert out["logits"].shape == (2, 3129)
    assert relerr(out["logits"], ref["logits"]) < TOL_LOGITS and relerr(out["loss"], ref["loss"]) < 1e-2


def test_ragged_repeat_counts_and_eval_determinism(cuda, weights):
    from oracle import clipbert_ref as R, synth
    model = _build("ClipBertForVideoTextRetrieval", weights, cuda).eval()
    g = torch.Generator().manual_seed(7)
    grid = (torch.randn(3, 2, 3, 3, 768, generator=g).abs()).to(torch.bfloat16).float()
    counts = [1, 3, 2]
    ids, mask = synth.synth_text(6, 32, seed=8)
    with torch.no_grad():
        ref = R.video_text_retrieval(ids, R.repeat_tensor_rows(grid, counts), mask, weights, rnd=R.Rounding.bf16())
        a = model.transformer(ids.to(cuda), grid.to(cuda), mask.to(cuda), _repeat_counts=counts)["logits"]
        b = model.transformer(ids.to(cuda), grid.to(cuda), mask.to(cuda), _repeat_counts=counts)["logits"]
        # pre-repeated rows through the public signature give the same bits as the fused gather
        c = model.transformer(ids.to(cuda), R.repeat_tensor_rows(grid, counts).to(cuda), mask.to(cuda))["logits"]
    assert torch.equal(a, b) and torch.equal(a, c)
    assert relerr(a, ref["logits"]) < TOL_LOGITS


def _golden(name):
    import os
    return torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name), map_location="cpu", weights_only=False)


def test_against_reference_generated_golden_vectors(cuda, weights):
    """tests/golden/*.pt were produced by the reference's own classes (tools/make_golden.py)."""
    g = _golden("transformer_retrieval.pt")
    model = _build("ClipBertForVideoTextRetrieval", weights, cuda).train()
    tr = model.transformer
    grid = g["grid"].clone().to(cuda).requires_grad_(True)
    tr._capture = {}
    out = tr(g["ids"].to(cuda), grid, g["mask"].to(cuda), labels=g["labels"].to(cuda), sample_size=2, _repeat_counts=[g["n_ex"]] * 2)
    cap, tr._capture = tr._capture, None
    assert relerr(out["logits"], g["logits"]) < TOL_LOGITS and relerr(out["loss"], g["loss"]) < 5e-3
    assert relerr(cap["pooled"], g["pooled"]) < TOL_FP32_E2E
    assert relerr(cap["layer11"][:, :2, :32], g["seq_first_rows"]) < TOL_FP32_E2E
    out["loss"].mean().backward()
    # the classifier ReLU pattern of a bf16 run differs from the fp32 reference's on a few units (see Rounding.relu_masks),
    # so gradients upstream of it are compared loosely here and tightly in test_transformer_forward_backward
    assert cosine(grid.grad, g["dgrid"]) > 0.98
    named = dict(tr.named_parameters())
    for k, n in g["grad_norms"].items():
        assert abs(float(named[k].grad.norm()) / n - 1) < 0.2, k
    g = _golden("transformer_multiple_choice.pt")
    from oracle import synth
    sd = dict(weights)
    sd.update(synth.transformer_state_dict(50, num_labels=1))
    model = _build("ClipBertForMultipleChoice", sd, cuda, num_labels=5).eval()
    with torch.no_grad():
        o = model.transformer(g["ids"].to(cuda), g["grid"].to(cuda), g["mask"].to(cuda), labels=g["labels"].to(cuda), _repeat_counts=[5, 5])
    assert relerr(o["logits"], g["logits"]) < TOL_LOGITS and relerr(o["loss"], g["loss"]) < 1e-2
    g = _golden("cnn_grid.pt")
    model = _build("ClipBertForVideoTextRetrieval", weights, cuda).eval()
    with torch.no_grad():
        g96 = model.cnn(synth.synth_images(1, 2, size=96, seed=21).to(cuda))
        g224 = model.cnn(synth.synth_images(1, 1, size=224, seed=22).to(cuda))
    assert g96.shape == (1, 2, 1, 1, 768) and g224.shape == (1, 1, 3, 3, 768)
    assert relerr(g96, g["grid96"]) < TOL_FP32_E2E and relerr(g224, g["grid224"]) < TOL_FP32_E2E


def test_pretraining_heads_mlm_itm(cuda, weights):
    import clipbert_b200 as cb
    from oracle import clipbert_ref as R, synth
    g = _golden("transformer_pretraining.pt")
    sd = {k: v for k, v in weights.items() if not k.startswith("transformer.classifier.")}
    sd.update({k: v for k, v in synth.transformer_state_dict(60, head="pretraining").items() if k.startswith("transformer.cls.")})
    cfg = make_cfg(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    model = cb.ClipBertForPreTraining(cfg)
    res = model.load_state_dict({k[len("transformer."):]: v for k, v in sd.items() if k.startswith("transformer.")}, strict=False)
    assert set(res.missing_keys) <= {"cls.predictions.decoder.weight", "cls.predictions.decoder.bias"} and not res.unexpected_keys
    model = model.to(cuda).train()
    grid = g["grid"].clone().to(cuda).requires_grad_(True)
    out = model(g["ids"].to(cuda), grid, g["mask"].to(cuda), mlm_labels=g["mlm_labels"].to(cuda), itm_labels=g["itm_labels"].to(cuda),
                _repeat_counts=[g["n_ex"]] * 2)
    assert out["mlm_scores"].shape == (4, 32, 30522) and out["itm_scores"].shape == (4, 2)
    # forward against the reference-generated golden
    assert relerr(out["itm_scores"], g["itm_scores"]) < TOL_LOGITS
    assert relerr(out["mlm_scores"][:, :4, :64], g["mlm_scores_slice"]) < TOL_LOGITS
    assert relerr(out["mlm_loss"][g["mlm_labels"].view(-1) != -100], g["mlm_loss"][g["mlm_labels"].view(-1) != -100]) < 1e-2
    assert float((out["mlm_scores"].argmax(-1).cpu() == g["mlm_argmax"]).float().mean()) > 0.97
    # backward against fp32 autograd on the oracle (no ReLU on this head: smooth, no pattern matching needed)
    sdr = {k: (v.clone().requires_grad_(True) if k.startswith("transformer.") else v) for k, v in sd.items()}
    gr = g["grid"].float().requires_grad_(True)
    o = R.pretraining(g["ids"], R.repeat_tensor_rows(gr, [g["n_ex"]] * 2), g["mask"], sdr, g["mlm_labels"], g["itm_labels"])
    n_mlm = int((g["mlm_labels"] != -100).sum())
    (o["mlm_loss"].sum() / n_mlm + o["itm_loss"].mean()).backward()
    (out["mlm_loss"].sum() / n_mlm + out["itm_loss"].mean()).backward()
    assert cosine(grid.grad, gr.grad) > 0.999 and relerr(grid.grad, gr.grad) < TOL_GRAD
    bad = []
    for name, p in model.named_parameters():
        ref = sdr["transformer." + name].grad
        if ref is None or float(ref.abs().sum()) == 0.0 or name.endswith("attention.self.key.bias"):
            continue
        e, c = relerr(p.grad, ref), cosine(p.grad, ref)
        if not (e < TOL_GRAD and c > 0.999):
            bad.append((name, e, c))
    assert not bad, bad[:10]


def test_native_resolution_448_and_long_text(cuda, weights):
    """The reference's native MSRVTT setting is 448 px (7x7 = 49 visual tokens, the paper's grid; SURVEY §0.3) and its
    paragraph-retrieval inference uses long captions: L = 20 + 49 = 69 and L = 512 + 9 = 521 both take the general
    (multi-tile) attention kernels."""
    from oracle import clipbert_ref as R, synth
    model = _build("ClipBertForVideoTextRetrieval", weights, cuda).train()
    # ---- 448 px, 1 video x 2 frames, 2 captions of 20 tokens: forward + backward ----
    batch = synth.synth_batch(1, 2, n_ex=2, size=448, max_len=20, seed=13)
    mb = {k: (v.to(cuda) if torch.is_tensor(v) else list(v)) for k, v in batch.items()}
    model.cnn._capture, model.transformer._capture = {}, {}
    out = model(mb)
    assert mb["visual_inputs"].shape == (1, 2, 7, 7, 768)
    pat = cnn_patterns(model.cnn._capture["stash"], mb["visual_inputs"])
    pat.relu_masks["transformer.classifier.relu"] = (model.transformer._capture["c1"] > 0).cpu()
    model.cnn._capture = model.transformer._capture = None
    sd = {k: (v.clone().requires_grad_(True) if k in ("cnn.grid_encoder.0.weight", "transformer.bert.encoder.layer.0.attention.self.query.weight",
                                                       "cnn.feature.backbone.res4.0.conv2.weight") else v) for k, v in weights.items()}
    ref = R.clipbert_forward(dict(batch), sd, rnd=pat)
    assert relerr(out["logits"], ref["logits"]) < TOL_LOGITS
    out["loss"].mean().backward()
    ref["loss"].mean().backward()
    named = dict(model.named_parameters())
    for k in ("cnn.grid_encoder.0.weight", "transformer.bert.encoder.layer.0.attention.self.query.weight", "cnn.feature.backbone.res4.0.conv2.weight"):
        assert cosine(named[k].grad, sd[k].grad) > 0.995, (k, cosine(named[k].grad, sd[k].grad))
    # ---- 512-token captions at 224 px (C5-style inference, L = 521) ----
    model.eval()
    g = torch.Generator().manual_seed(17)
    grid = (torch.randn(1, 1, 3, 3, 768, generator=g).abs()).to(torch.bfloat16).float()
    ids, mask = synth.synth_text(2, 512, seed=19)
    with torch.no_grad():
        ref = R.video_text_retrieval(ids, R.repeat_tensor_rows(grid, [2]), mask, weights, rnd=R.Rounding.bf16())
        got = model.transformer(ids.to(cuda), grid.to(cuda), mask.to(cuda), _repeat_counts=[2])
    assert relerr(got["logits"], ref["logits"]) < TOL_LOGITS


def test_forward_clips_equals_the_reference_clip_loop(cuda, weights):
    """SURVEY §8 f1: ClipBert.forward_clips (all clips in one pass) against the per-clip loop of
    run_video_retrieval.py:396-404 on the same model - logits and every parameter gradient - with ragged
    n_examples_list, and with programmatic dependent launch off vs on (must be bit-identical: every kernel
    waits for its producers before its first global access)."""
    from clipbert_b200 import ops
    from oracle import synth
    model = _build("ClipBertForVideoTextRetrieval", weights, cuda).train()      # dropout p = 0 (see _build)
    n_clips, T, B = 2, 2, 3
    counts = [2, 1, 3]
    batch = synth.synth_batch(B, n_clips * T, n_ex=1, size=96, seed=11)
    ids, mask = synth.synth_text(sum(counts), 24, seed=12)
    labels = torch.tensor([1, 0, 1, 0, 0, 1])
    dev_batch = dict(visual_inputs=batch["visual_inputs"].to(cuda), text_input_ids=ids.to(cuda), text_input_mask=mask.to(cuda))

    def lse(lg):
        lg = lg.permute(1, 0, 2).contiguous()
        o = torch.logsumexp(lg.view(lg.shape[0], -1), dim=-1, keepdim=True) - torch.logsumexp(lg, dim=1)
        return torch.gather(o, -1, labels.to(cuda).view(-1, 1)).mean()

    def grads():
        return {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.requires_grad and p.grad is not None}

    # reference loop
    model.zero_grad()
    vis = dev_batch["visual_inputs"].view(B, n_clips, T, 3, 96, 96)
    per_clip = []
    for c in range(n_clips):
        mb = dict(dev_batch, visual_inputs=vis[:, c], n_examples_list=list(counts))
        per_clip.append(model(mb)["logits"])
    loop_logits = torch.stack(per_clip)
    lse(loop_logits).backward()
    g_loop = grads()
    # one batched pass, PDL on and off
    res = {}
    for pdl in (1, 0):
        prev = ops.set_pdl(pdl)
        model.zero_grad()
        out = model.forward_clips(dict(dev_batch, n_examples_list=list(counts)), n_clips)["logits"]
        lse(out).backward()
        if cuda.type == "cuda":
            torch.cuda.synchronize()
        res[pdl] = (out.detach().clone(), grads())
        ops.set_pdl(prev)
    out, g_b = res[1]
    assert out.shape == loop_logits.shape == (n_clips, sum(counts), 2)
    assert relerr(out, loop_logits) < 1e-3, relerr(out, loop_logits)
    assert set(g_b) == set(g_loop)
    bad = [(n, relerr(g_b[n], g_loop[n])) for n in g_loop if float(g_loop[n].abs().sum()) > 0 and
           not (relerr(g_b[n], g_loop[n]) < 2e-2 and cosine(g_b[n], g_loop[n]) > 0.999)]
    assert not bad, bad[:8]
    assert torch.equal(res[0][0], res[1][0]), "PDL changed the forward result"
    # wgrad accumulates with fp32 red.add (order is not deterministic), so gradients are compared to a tight tolerance
    assert all(relerr(res[0][1][n], res[1][1][n]) < 1e-4 for n in g_loop if float(g_loop[n].abs().sum()) > 0)
