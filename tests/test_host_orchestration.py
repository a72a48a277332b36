"""Host-side orchestration of clipbert_b200/modeling.py on CPU: the real Python engine (flat parameter buffers, stash, call
order, epilogue flags, index bookkeeping) driven through tests/ops_emulator.py - torch restatements of what include/
clipbert_b200.h says each entry point computes - and compared with the oracle's autograd. This checks the host logic
without a GPU; the kernels behind the same calls are checked on an H100 by tests/test_gpu_*.py.
"""
import numpy as np
import pytest
import torch

from ops_emulator import emulated_transformer_ops
from util import TOL_GRAD, TOL_LOGITS, cosine, make_cfg, relerr


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)


def _transformer(cls_name, sd, **cfg_extra):
    import clipbert_b200 as cb
    cfg = make_cfg(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, **cfg_extra)
    model = getattr(cb, cls_name)(cfg)
    res = model.load_state_dict({k[len("transformer."):]: v for k, v in sd.items() if k.startswith("transformer.")}, strict=False)
    assert set(res.missing_keys) <= {"cls.predictions.decoder.weight", "cls.predictions.decoder.bias"} and not res.unexpected_keys
    return model.train()


def _check_grads(model, sdr, skip=()):
    bad = []
    for name, p in model.named_parameters():
        ref = sdr["transformer." + name].grad
        if ref is None or float(ref.abs().sum()) == 0.0 or name.endswith("attention.self.key.bias") or name in skip:
            continue
        e, c = relerr(p.grad, ref), cosine(p.grad, ref)
        if not (e < TOL_GRAD and c > 0.999):
            bad.append((name, e, c))
    assert not bad, bad[:10]


@pytest.mark.parametrize("counts", [[2, 2, 2], [1, 3, 2]])
def test_retrieval_engine_forward_backward_on_emulated_ops(weights, counts):
    from oracle import clipbert_ref as R, synth
    nvid, nseq = len(counts), sum(counts)
    g = torch.Generator().manual_seed(2)
    grid = (torch.randn(nvid, 2, 3, 3, 768, generator=g).abs() * 2).to(torch.bfloat16)
    ids, mask = synth.synth_text(nseq, 14, seed=3)
    labels = torch.randint(0, 2, (nseq,), generator=g)
    model = _transformer("ClipBertForVideoTextRetrieval", weights)
    gc = grid.clone().requires_grad_(True)
    with emulated_transformer_ops() as calls:
        model._capture = {}
        out = model(ids, gc, mask, labels=labels, sample_size=nvid, _repeat_counts=list(counts))
        cap, model._capture = model._capture, None
        out["loss"].mean().backward()
    assert calls["gemm"] == 12 * 4 + 3 + (12 * 8 + 2 + 2 + 2) and calls["attention_fwd"] == 12 and calls["attention_bwd"] == 12
    sdr = {k: (v.clone().requires_grad_(True) if k.startswith("transformer.") else v) for k, v in weights.items()}
    gr = grid.float().requires_grad_(True)
    rep = R.repeat_tensor_rows(gr, counts)
    _, pooled = R.clipbert_base_model(ids, rep, mask, sdr)
    hpat = R.Rounding(relu_masks={"transformer.classifier.relu": cap["c1"] > 0})
    logits_ref = R.mlp_head(pooled, sdr, rnd=hpat)
    R.retrieval_loss(logits_ref, labels).mean().backward()
    assert relerr(out["logits"], logits_ref) < TOL_LOGITS
    assert relerr(gc.grad, gr.grad) < TOL_GRAD and cosine(gc.grad, gr.grad) > 0.999
    _check_grads(model, sdr)


def test_pretraining_engine_with_visual_token_sampling_on_emulated_ops(weights):
    """MLM + ITM heads and pre-training's train-mode random sampling of visual tokens (modeling.py:15-34,80-88): same numpy
    seed -> same kept tokens as the oracle; dropped tokens get no gradient; row / column tables receive the scattered sums."""
    from oracle import clipbert_ref as R, synth
    sd = {k: v for k, v in weights.items() if not k.startswith("transformer.classifier.")}
    sd.update({k: v for k, v in synth.transformer_state_dict(60, head="pretraining").items() if k.startswith("transformer.cls.")})
    model = _transformer("ClipBertForPreTraining", sd, pixel_random_sampling_size=7)
    g = torch.Generator().manual_seed(5)
    grid0 = torch.randn(2, 2, 4, 5, 768, generator=g).abs().bfloat16()
    ids, mask = synth.synth_text(4, 12, seed=9)
    mlm = torch.full((4, 12), -100, dtype=torch.long)
    mlm[:, 3], mlm[:, 7] = ids[:, 3], ids[:, 7]
    itm = torch.tensor([1, 1, 1, 0])      # mostly one sign: alternating signs make dW_itm a difference of near-equal pooled rows (ill-conditioned under bf16)
    grid = grid0.clone().requires_grad_(True)
    with emulated_transformer_ops():
        np.random.seed(77)
        out = model(ids, grid, mask, mlm_labels=mlm, itm_labels=itm, _repeat_counts=[2, 2])
        (out["mlm_loss"].sum() / 8 + out["itm_loss"].mean()).backward()
    assert out["mlm_scores"].shape == (4, 12, 30522)
    sdr = {k: (v.clone().requires_grad_(True) if k.startswith("transformer.") else v) for k, v in sd.items()}
    gr = grid0.float().requires_grad_(True)
    np.random.seed(77)
    ref = R.pretraining(ids, R.repeat_tensor_rows(gr, [2, 2]), mask, sdr, mlm, itm, pixel_random_sampling_size=7)
    (ref["mlm_loss"].sum() / 8 + ref["itm_loss"].mean()).backward()
    assert relerr(out["itm_scores"], ref["itm_scores"]) < TOL_LOGITS
    assert relerr(out["mlm_scores"], ref["mlm_scores"]) < TOL_LOGITS
    np.random.seed(77)
    kept = set(R.random_sample_indices(20, 7).tolist())
    dropped = torch.tensor([j for j in range(20) if j not in kept])
    assert float(grid.grad.float().view(2, 2, 20, 768)[:, :, dropped].abs().max()) == 0.0
    assert cosine(grid.grad, gr.grad) > 0.999 and relerr(grid.grad, gr.grad) < TOL_GRAD
    _check_grads(model, sdr)
    # eval mode: the whole grid (no sampling), L = 12 + 20
    model.eval()
    with emulated_transformer_ops(), torch.no_grad():
        ev = model(ids, grid0, mask, _repeat_counts=[2, 2])
        ref_ev = R.pretraining(ids, R.repeat_tensor_rows(grid0.float(), [2, 2]), mask, sd)
    assert relerr(ev["itm_scores"], ref_ev["itm_scores"]) < TOL_LOGITS


def test_multiple_choice_engine_on_emulated_ops(weights):
    from oracle import clipbert_ref as R, synth
    sd = dict(weights)
    sd.update(synth.transformer_state_dict(50, num_labels=1))
    model = _transformer("ClipBertForMultipleChoice", sd, num_labels=5).eval()
    g = torch.Generator().manual_seed(4)
    grid = torch.randn(2, 1, 3, 3, 768, generator=g).abs().to(torch.bfloat16)
    ids, mask = synth.synth_text(10, 16, seed=5)
    labels = torch.tensor([1, 4])
    with emulated_transformer_ops(), torch.no_grad():
        out = model(ids, grid, mask, labels=labels, _repeat_counts=[5, 5])
        ref = R.multiple_choice(ids, R.repeat_tensor_rows(grid.float(), [5, 5]), mask, sd, 5, labels, rnd=R.Rounding.bf16())
    assert out["logits"].shape == (2, 5)
    assert relerr(out["logits"], ref["logits"]) < TOL_LOGITS and relerr(out["loss"], ref["loss"]) < 1e-2


# ---------------------------------------------------------------------------------------------------
# CNN engine (clipbert_b200/grid_feat.py) and the full ClipBert module on the emulated ABI
# ---------------------------------------------------------------------------------------------------
def _clipbert(sd, cls_name="ClipBertForVideoTextRetrieval", **cfg_extra):
    import clipbert_b200 as cb
    cfg = make_cfg(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, **cfg_extra)
    model = cb.ClipBert(cfg, detectron2_model_cfg="R-50-grid.yaml", transformer_cls=getattr(cb, cls_name))
    assert not model.load_state_dict(sd).missing_keys
    return model


@pytest.mark.parametrize("stem", ["s2d", "im2col"])
def test_cnn_engine_forward_backward_on_emulated_ops(weights, stem):
    """GridFeatBackbone's host logic: zero-bordered buffers and their recycling, row maps, stride-2 subsampling, the
    space-to-depth / patch-matrix stem, the backward walk with FREEZE_AT = 2, the mid-backward bucket hook."""
    from model_util import cnn_patterns
    from oracle import clipbert_ref as R, synth
    from util import TOL_FP32_E2E, TOL_MATCHED_DEEP
    model = _clipbert(weights).train()
    cnn = model.cnn
    cnn.stem_mode = stem
    x = synth.synth_images(1, 2, size=64, seed=6)
    sd = {k: (v.clone().requires_grad_(True) if (k.endswith(".weight") and "norm" not in k and k.startswith("cnn.")) else v)
          for k, v in weights.items()}
    hook_calls = []
    cnn._bucket_hook = lambda flat_grad, lo, side: hook_calls.append((lo, side, float(flat_grad[lo:].abs().sum()) > 0))
    with emulated_transformer_ops() as calls:
        cnn._capture = {}
        grid = cnn(x)
        cap, cnn._capture = cnn._capture, None
        with torch.no_grad():
            _, st16 = R.grid_feat_backbone(x, weights, return_stages=True, rnd=R.Rounding.bf16())
        for name in ("stem", "res2", "res3", "res4", "res5"):
            got = cap[name].float().permute(0, 3, 1, 2)
            assert relerr(got, st16[name]) < TOL_MATCHED_DEEP, (name, relerr(got, st16[name]))
        assert relerr(grid, st16["grid"]) < TOL_MATCHED_DEEP
        pat = cnn_patterns(cap["stash"], grid)
        grid_ref = R.grid_feat_backbone(x, sd, rnd=pat)
        assert relerr(grid, grid_ref) < TOL_FP32_E2E
        dgrid = torch.randn(grid_ref.shape, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16).float()
        grid_ref.backward(dgrid)
        grid.backward(dgrid.to(grid.dtype))
    assert calls["stem_s2d" if stem == "s2d" else "stem_im2col"] == 1 and calls["stem_im2col" if stem == "s2d" else "stem_s2d"] == 0
    # the bucket hook fired once, after res5.0, with the tail of the flat buffer = res5 + grid_encoder already holding gradients
    res5_0 = cnn.feature.backbone.res5[0]
    assert hook_calls == [(res5_0.shortcut._e["offset"], None, True)]
    assert cnn._pending_backward == 0
    checked = 0
    for name, p in cnn.named_parameters():
        ref = sd["cnn." + name].grad
        if not p.requires_grad:
            continue
        assert cosine(p.grad, ref) > 0.999 and relerr(p.grad, ref) < TOL_GRAD, (name, cosine(p.grad, ref), relerr(p.grad, ref))
        checked += 1
    assert checked == 3 * 13 + 3 + 1


def test_clipbert_forward_clips_and_clip_loop_on_emulated_ops(weights):
    """ClipBert.forward_clips against the reference-order clip loop and the oracle, ragged n_examples_list, end to end
    (CNN + transformer + LSE aggregation), including the dict mutations of ClipBert.forward (e2e_model.py:29-39)."""
    from oracle import clipbert_ref as R, synth
    model = _clipbert(weights).eval()
    n_clips, T, B, size = 2, 1, 2, 64
    counts = [2, 1]
    batch = synth.synth_batch(B, n_clips * T, n_ex=1, size=size, seed=11)
    ids, mask = synth.synth_text(sum(counts), 10, seed=12)
    vis = batch["visual_inputs"].view(B, n_clips, T, 3, size, size)
    with emulated_transformer_ops(), torch.no_grad():
        out = model.forward_clips(dict(visual_inputs=batch["visual_inputs"], text_input_ids=ids, text_input_mask=mask,
                                       n_examples_list=list(counts)), n_clips)["logits"]
        loop = []
        for c in range(n_clips):
            mb = dict(visual_inputs=vis[:, c], text_input_ids=ids, text_input_mask=mask, labels=None, n_examples_list=list(counts))
            loop.append(model(mb)["logits"])
            assert "n_examples_list" not in mb and mb["sample_size"] == B and mb["visual_inputs"].shape == (B, T, 1, 1, 768)
        ref = [R.clipbert_forward(dict(visual_inputs=vis[:, c], text_input_ids=ids, text_input_mask=mask, n_examples_list=list(counts)),
                                  weights, rnd=R.Rounding.bf16())["logits"] for c in range(n_clips)]
    assert out.shape == (n_clips, sum(counts), 2)
    assert torch.equal(out, torch.stack(loop))          # float64 accumulation in the emulator: batching must not change a bit
    assert relerr(out, torch.stack(ref)) < TOL_LOGITS


def test_fused_clip_lse_loss_function_on_emulated_ops():
    """clipbert_b200.clip_lse_loss (autograd wrapper of cb_clip_lse_loss) against the oracle's clip aggregation
    (run_video_retrieval.py:404-422) - value, gradient, upstream scaling, list input."""
    import clipbert_b200 as cb
    from oracle import clipbert_ref as R
    g = torch.Generator().manual_seed(3)
    for n_clips, nseq, ncls in ((2, 5, 2), (4, 7, 5), (1, 3, 2)):
        z = torch.randn(n_clips, nseq, ncls, generator=g)
        y = torch.randint(0, ncls, (nseq,), generator=g)
        zr = z.clone().requires_grad_(True)
        ref = R.aggregate_clip_logits(list(zr.unbind(0)), y, "lse")
        (3.0 * ref).backward()
        zt = z.clone().requires_grad_(True)
        with emulated_transformer_ops() as calls:
            loss = cb.clip_lse_loss(zt, y)
            (3.0 * loss).backward()
            loss_list = cb.clip_lse_loss(list(z.unbind(0)), y)
        assert calls["clip_lse_loss"] == 2
        assert loss.shape == () and torch.allclose(loss, ref.detach(), atol=1e-6) and torch.allclose(loss_list, ref.detach(), atol=1e-6)
        assert torch.allclose(zt.grad, zr.grad, atol=1e-6)


def test_training_step_clip_loop_vs_batched_pass_on_emulated_ops(weights):
    """One training step both ways - the reference's per-clip loop (n_clips forward calls, one backward through all of them)
    and ONE batched pass (forward_clips) - must give the same gradients in both halves; the data-parallel hooks fire once per
    step, after the LAST outstanding backward of each half (gradients of all clips accumulated)."""
    import clipbert_b200 as cb
    from oracle import synth
    model = _clipbert(weights).train()
    n_clips, T, B, size = 2, 1, 2, 64
    batch = synth.synth_batch(B, n_clips * T, n_ex=1, size=size, seed=21)
    vis = batch["visual_inputs"].view(B, n_clips, T, 3, size, size)
    fired = []
    model.transformer._grad_ready_hook = lambda g: fired.append(("transformer", float(g.abs().sum())))
    model.cnn._bucket_hook = lambda g, lo, side: fired.append(("cnn", lo, model.transformer._pending_backward, model.cnn._pending_backward))

    def grads():
        return {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.requires_grad and p.grad is not None}

    with emulated_transformer_ops():
        model.zero_grad()
        logits = [model(dict(visual_inputs=vis[:, c], text_input_ids=batch["text_input_ids"], text_input_mask=batch["text_input_mask"],
                             labels=batch["labels"], n_examples_list=[1] * B))["logits"] for c in range(n_clips)]
        cb.clip_lse_loss(logits, batch["labels"]).backward()
        g_loop, fired_loop = grads(), list(fired)
        fired.clear()
        model.zero_grad()
        out = model.forward_clips(dict(visual_inputs=batch["visual_inputs"], text_input_ids=batch["text_input_ids"],
                                       text_input_mask=batch["text_input_mask"], n_examples_list=[1] * B), n_clips)["logits"]
        cb.clip_lse_loss(out, batch["labels"]).backward()
        g_batched = grads()
    # hooks: once per half per step, when nothing else of that half is pending
    for events in (fired_loop, fired):
        assert [e[0] for e in events] == ["transformer", "cnn"], events
        assert events[0][1] > 0 and events[1][2] == 0 and events[1][3] == 0
    assert set(g_loop) == set(g_batched) and len(g_loop) > 200
    bad = [(n, relerr(g_batched[n], g_loop[n])) for n in g_loop
           if float(g_loop[n].abs().sum()) > 0 and not (relerr(g_batched[n], g_loop[n]) < 2e-2 and cosine(g_batched[n], g_loop[n]) > 0.999)]
    assert not bad, bad[:8]


def test_zero_grad_in_forward_replaces_the_serial_zero_grad_on_emulated_ops(weights):
    """ClipBert.zero_grad_in_forward: the step clears the flat gradient buffers itself (on the GPU: on a side stream beside the
    transformer forward). Two steps on the same batch without any model.zero_grad() must leave the gradient of ONE step, in eval
    / no_grad passes nothing is cleared, and with the switch off the second step accumulates."""
    import clipbert_b200 as cb
    from oracle import synth
    model = _clipbert(weights).train()
    for m in model.modules():
        if hasattr(m, "p") and isinstance(getattr(m, "p"), float):
            m.p = 0.0
    model.transformer.config.hidden_dropout_prob = 0.0
    model.transformer.config.attention_probs_dropout_prob = 0.0
    n_clips, B, size = 2, 2, 64
    batch = synth.synth_batch(B, n_clips, n_ex=1, size=size, seed=23)

    def step():
        out = model.forward_clips(dict(visual_inputs=batch["visual_inputs"], text_input_ids=batch["text_input_ids"],
                                       text_input_mask=batch["text_input_mask"], n_examples_list=[1] * B), n_clips)["logits"]
        cb.clip_lse_loss(out, batch["labels"]).backward()
        return [g.detach().clone() for g in model.flat_grads()]

    with emulated_transformer_ops():
        model.zero_grad()
        g1 = step()
        assert len(g1) == 2 and all(float(g.abs().sum()) > 0 for g in g1)
        model.zero_grad_in_forward = True
        g2 = step()                                # no zero_grad() in between
        for a, b in zip(g1, g2):
            assert relerr(b, a) < 1e-6
        with torch.no_grad():                      # an evaluation pass between two steps clears nothing
            model.eval()
            model.forward_clips(dict(visual_inputs=batch["visual_inputs"], text_input_ids=batch["text_input_ids"],
                                     text_input_mask=batch["text_input_mask"], n_examples_list=[1] * B), n_clips)
            model.train()
        for a, b in zip(g2, model.flat_grads()):
            assert torch.equal(a, b)
        model.zero_grad_in_forward = False
        g3 = step()                                # accumulates on top of g2
        for a, b in zip(g1, g3):
            assert relerr(b, 2 * a) < 1e-6


def test_bf16_operand_refresh_contract_on_emulated_ops(weights):
    """When the bf16 operand copy is refreshed (INTEGRATION.md, "Weight updates"): after a backward (reference AdamW edits
    p.data in place), on version-counted writes, on mark_weights_updated(); an unannounced p.data edit between two
    forward-only passes is the documented exception."""
    from oracle import synth
    model = _clipbert(weights).eval()
    batch = synth.synth_batch(1, 1, n_ex=1, size=64, seed=5)

    def fwd():
        with torch.no_grad():
            return model({k: (v.clone() if torch.is_tensor(v) else list(v)) for k, v in batch.items()})["logits"]

    w_cls = model.transformer.classifier[2].weight
    w_ge = model.cnn.grid_encoder[0].weight
    with emulated_transformer_ops():
        base = fwd()
        with torch.no_grad():
            w_cls.mul_(1.5)                      # version-counted write: picked up
            w_ge.mul_(1.5)
        a = fwd()
        assert not torch.equal(a, base)
        w_cls.data.mul_(2.0)                     # p.data edit, no backward in between: NOT seen ...
        w_ge.data.mul_(2.0)
        assert torch.equal(fwd(), a)
        model.cnn.mark_weights_updated()         # ... until announced
        model.transformer.mark_weights_updated()
        b = fwd()
        assert not torch.equal(b, a)
        model.train()                            # reference training order: forward, backward, p.data update, forward
        out = model({k: (v.clone() if torch.is_tensor(v) else list(v)) for k, v in batch.items()})
        out["loss"].mean().backward()
        w_cls.data.mul_(0.5)
        w_ge.data.mul_(0.5)
        model.eval()
        assert torch.allclose(fwd(), a, atol=1e-6)


@pytest.mark.parametrize("freeze_at", [1, 3])
def test_cnn_engine_other_freeze_points_on_emulated_ops(weights, freeze_at):
    """detectron2's BACKBONE.FREEZE_AT other than the shipped 2: res2 trainable (1) / res3 frozen too (3). FREEZE_AT = 0 (a
    trainable stem) has no backward on this path and must be refused rather than return a silent zero gradient."""
    import clipbert_b200 as cb
    from model_util import cnn_patterns
    from oracle import clipbert_ref as R, synth
    cfg = make_cfg(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    with pytest.raises(NotImplementedError):
        cb.GridFeatBackbone(detectron2_model_cfg="R-50-grid.yaml", config=cfg, freeze_at=0)
    model = cb.ClipBert(cfg, detectron2_model_cfg="R-50-grid.yaml", freeze_at=freeze_at)
    model.load_state_dict(weights)
    model.train()
    x = synth.synth_images(1, 2, size=64, seed=6)
    sd = {k: (v.clone().requires_grad_(True) if (k.endswith(".weight") and "norm" not in k and k.startswith("cnn.")) else v)
          for k, v in weights.items()}
    with emulated_transformer_ops():
        model.cnn._capture = {}
        grid = model.cnn(x)
        cap, model.cnn._capture = model.cnn._capture, None
        ref = R.grid_feat_backbone(x, sd, rnd=cnn_patterns(cap["stash"], grid), freeze_at=freeze_at)
        dg = torch.randn(ref.shape, generator=torch.Generator().manual_seed(1)).bfloat16().float()
        ref.backward(dg)
        grid.backward(dg.to(grid.dtype))
    checked = 0
    for name, p in model.cnn.named_parameters():
        r = sd["cnn." + name].grad
        if not p.requires_grad:
            assert p.grad is None or float(p.grad.abs().sum()) == 0.0
            continue
        assert cosine(p.grad, r) > 0.999 and relerr(p.grad, r) < TOL_GRAD, name
        checked += 1
    assert checked == {1: 53, 3: 30}[freeze_at]


def test_inference_retrieval_grid_reuse_on_emulated_ops(weights):
    """inference_retrieval (src/tasks/run_video_retrieval.py:628-666): one video, its captions in mini-batches, every clip
    scored per mini-batch. encode_clips once + forward_clips(grid=...) per mini-batch must equal the reference-order loop
    (which re-runs the CNN for every mini-batch and clip) bit for bit, and the oracle within bf16 tolerance."""
    from oracle import clipbert_ref as R, synth
    model = _clipbert(weights).eval()
    n_clips, T, size, n_caps, eval_bsz = 3, 1, 64, 5, 2
    vis = synth.synth_images(1, n_clips * T, size=size, seed=31)
    ids, mask = synth.synth_text(n_caps, 10, seed=32)
    clips = vis.view(1, n_clips, T, 3, size, size)
    with emulated_transformer_ops() as calls, torch.no_grad():
        loop = []
        for i in range(0, n_caps, eval_bsz):
            per_clip = [model(dict(visual_inputs=clips[:, c], text_input_ids=ids[i:i + eval_bsz], text_input_mask=mask[i:i + eval_bsz],
                                   labels=None, n_examples_list=[len(ids[i:i + eval_bsz])]))["logits"] for c in range(n_clips)]
            loop.append(torch.stack(per_clip))
        stems_loop = calls["stem_s2d"]
        grid = model.encode_clips(vis, n_clips)
        fast = [model.forward_clips(dict(text_input_ids=ids[i:i + eval_bsz], text_input_mask=mask[i:i + eval_bsz],
                                         n_examples_list=[len(ids[i:i + eval_bsz])]), n_clips, grid=grid)["logits"]
                for i in range(0, n_caps, eval_bsz)]
        assert stems_loop == 9 and calls["stem_s2d"] == 10          # 3 mini-batches x 3 clips vs one CNN pass
        ref = torch.stack([R.clipbert_forward(dict(visual_inputs=clips[:, c], text_input_ids=ids, text_input_mask=mask, n_examples_list=[n_caps]),
                                              weights, rnd=R.Rounding.bf16())["logits"] for c in range(n_clips)])
    assert grid.shape == (n_clips, T, 1, 1, 768)
    for a, b in zip(fast, loop):
        assert a.shape == b.shape and torch.equal(a, b)
    assert relerr(torch.cat(fast, dim=1), ref) < TOL_LOGITS


def test_dropout_stream_word_is_bound_only_for_the_duration_of_a_pass(weights):
    """The dropout stream position (cb_dropout_offset_bind) is process-wide library state: a training forward advances the model's
    device counter into a fresh per-call word and binds it, the backward re-binds THAT word (it must regenerate the forward's
    masks even if another forward ran in between - the reference's per-clip loop), and both unbind on the way out, so no later
    launch can read a word whose tensor has been freed."""
    import ops_emulator as E
    from oracle import synth
    g = torch.Generator().manual_seed(4)
    grid = (torch.randn(2, 2, 3, 3, 768, generator=g).abs()).to(torch.bfloat16)
    ids, mask = synth.synth_text(2, 10, seed=5)
    labels = torch.tensor([1, 0])
    model = _transformer("ClipBertForVideoTextRetrieval", weights)
    model.config.hidden_dropout_prob = 0.1                       # (the helper builds p = 0 models; the emulator ignores the masks)
    seen = []
    with emulated_transformer_ops(ignore_dropout=True):
        from clipbert_b200 import ops
        real_bind = ops.dropout_offset_bind

        def spy(word):
            seen.append(None if word is None else int(word.item()))
            real_bind(word)
        ops.dropout_offset_bind = spy
        try:
            out1 = model(ids, grid.clone().requires_grad_(True), mask, labels=labels, sample_size=2)
            assert E.BOUND_DROPOUT_WORD is None and seen == [1, None]
            out2 = model(ids, grid.clone().requires_grad_(True), mask, labels=labels, sample_size=2)     # a second forward before any backward
            assert seen == [1, None, 2, None]
            out1["loss"].mean().backward()                       # ... and the FIRST pass' backward re-binds the first pass' word
            assert seen[-2:] == [1, None] and E.BOUND_DROPOUT_WORD is None
            out2["loss"].mean().backward()
            assert seen[-2:] == [2, None]
        finally:
            ops.dropout_offset_bind = real_bind
    assert int(model._drop_counter.item()) == 2
    model.eval()
    with emulated_transformer_ops(), torch.no_grad():
        model(ids, grid, mask)                                   # eval: no stream position is consumed
    assert int(model._drop_counter.item()) == 2


def test_input_stage_on_emulated_ops(weights):
    """clipbert_b200.input_stage: resize_pad (ImageResize + ImagePad) through the emulated cb_resize_pad, and ImageNorm's mean /
    std fused into the stem (mean in the gather, 1 / std folded into the stem weights at pack time) against the oracle fed with
    the explicitly normalised frames."""
    import torch.nn.functional as F
    from clipbert_b200 import input_stage as IS
    from oracle import clipbert_ref as R
    g = torch.Generator().manual_seed(9)
    mean, std = (123.675, 116.28, 103.53), (58.395, 57.12, 57.375)
    raw = torch.randint(0, 256, (1, 2, 3, 40, 72), generator=g, dtype=torch.uint8)
    model = _clipbert(weights).eval()
    IS.set_image_norm(model, mean, std)
    with emulated_transformer_ops():
        frames = torch.empty(1, 2, 3, 64, 64)          # (input_stage.resize_pad itself asserts CUDA tensors: call the op it wraps)
        from clipbert_b200 import ops
        nh, nw = IS.get_resize_size(40, 72, 64)
        ops.resize_pad(raw, frames, nh, nw)
        ref = F.pad(F.interpolate(raw.view(-1, 3, 40, 72).float(), size=(nh, nw), mode="bilinear", align_corners=False), (0, 64 - nw, 0, 64 - nh))
        assert torch.equal(frames.view(-1, 3, 64, 64), ref) and (nh, nw) == (35, 64)
        model.cnn._capture = {}
        with torch.no_grad():
            model.cnn(frames)
        cap, model.cnn._capture = model.cnn._capture, None
    xn = (frames - torch.tensor(mean).view(1, 1, 3, 1, 1)) / torch.tensor(std).view(1, 1, 3, 1, 1)
    with torch.no_grad():
        _, st = R.grid_feat_backbone(xn, weights, return_stages=True, rnd=R.Rounding.bf16())
    assert relerr(cap["stem"].float().permute(0, 3, 1, 2), st["stem"]) < 1e-2
