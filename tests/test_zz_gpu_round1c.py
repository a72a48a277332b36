"""GPU parity tests of the clip-batched, long-sequence and loss-kernel paths (written against the CPU oracle). They sort last so
that a surprise here cannot hide the result of the established suites.
Every kernel they launch is one the earlier suites already cover; what is new is the host-side index bookkeeping.
"""
import os

import numpy as np
import pytest
import torch

from util import TOL_GRAD, TOL_LOGITS, cosine, make_cfg, relerr

pytestmark = pytest.mark.gpu

# Everything else in this file exercises the default kernels through host logic that was validated on CPU.


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)


def _pretraining_model(weights, cuda, **cfg_extra):
    import clipbert_b200 as cb
    from oracle import synth
    sd = {k: v for k, v in weights.items() if not k.startswith("transformer.classifier.")}
    sd.update({k: v for k, v in synth.transformer_state_dict(60, head="pretraining").items() if k.startswith("transformer.cls.")})
    cfg = make_cfg(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, **cfg_extra)
    model = cb.ClipBertForPreTraining(cfg)
    res = model.load_state_dict({k[len("transformer."):]: v for k, v in sd.items() if k.startswith("transformer.")}, strict=False)
    assert set(res.missing_keys) <= {"cls.predictions.decoder.weight", "cls.predictions.decoder.bias"} and not res.unexpected_keys
    return model.to(cuda), sd


def test_pretraining_random_visual_token_sampling(cuda, weights):
    """VisualInputEmbedding's train-mode sampling (src/modeling/modeling.py:15-34,80-88): with numpy seeded like the oracle's
    draw the H100 path keeps the same sorted subset; forward, the scattered grid gradient and the row / column position
    table gradients (index_add of the virtual-grid gradient) against fp32 autograd on the oracle."""
    from oracle import clipbert_ref as R, synth
    model, sd = _pretraining_model(weights, cuda, pixel_random_sampling_size=7)
    model.train()
    g = torch.Generator().manual_seed(5)
    grid0 = torch.randn(2, 2, 4, 5, 768, generator=g).abs().bfloat16()          # 20 visual tokens, keep 7
    ids, mask = synth.synth_text(4, 12, seed=9)                                 # 2 captions per video
    mlm = torch.full((4, 12), -100, dtype=torch.long)
    mlm[:, 3] = ids[:, 3]
    mlm[:, 7] = ids[:, 7]
    itm = torch.tensor([1, 1, 1, 0])      # mostly one sign: alternating signs make dW_itm a difference of near-equal pooled rows (ill-conditioned under bf16)
    grid = grid0.clone().to(cuda).requires_grad_(True)
    np.random.seed(77)
    out = model(ids.to(cuda), grid, mask.to(cuda), mlm_labels=mlm.to(cuda), itm_labels=itm.to(cuda), _repeat_counts=[2, 2])
    assert out["mlm_scores"].shape == (4, 12, 30522)
    sdr = {k: (v.clone().requires_grad_(True) if k.startswith("transformer.") else v) for k, v in sd.items()}
    gr = grid0.float().requires_grad_(True)
    np.random.seed(77)
    ref = R.pretraining(ids, R.repeat_tensor_rows(gr, [2, 2]), mask, sdr, mlm, itm, pixel_random_sampling_size=7)
    # 19-token sequences of a 4-sequence batch: fewer, smaller logits than the 41-token cases TOL_LOGITS was set on (the CPU
    # replay of this test through the ABI emulator sits at 1.5e-2 / 1.2e-2)
    assert relerr(out["itm_scores"], ref["itm_scores"]) < 1.6 * TOL_LOGITS
    assert relerr(out["mlm_scores"][:, :, :256], ref["mlm_scores"][:, :, :256]) < 1.6 * TOL_LOGITS
    (out["mlm_loss"].sum() / 8 + out["itm_loss"].mean()).backward()
    (ref["mlm_loss"].sum() / 8 + ref["itm_loss"].mean()).backward()
    np.random.seed(77)
    kept = R.random_sample_indices(20, 7)
    dropped = torch.tensor([j for j in range(20) if j not in set(kept.tolist())])
    gg = grid.grad.float().cpu().view(2, 2, 20, 768)
    assert float(gg[:, :, dropped].abs().max()) == 0.0, "dropped visual tokens must receive no gradient"
    assert cosine(grid.grad, gr.grad) > 0.999 and relerr(grid.grad, gr.grad) < TOL_GRAD
    named = dict(model.named_parameters())
    for name in ("bert.visual_embeddings.row_position_embeddings.weight", "bert.visual_embeddings.col_position_embeddings.weight",
                 "bert.visual_embeddings.LayerNorm.weight", "bert.visual_embeddings.token_type_embeddings.weight",
                 "bert.encoder.layer.0.attention.self.query.weight", "bert.encoder.layer.11.output.dense.weight"):
        r = sdr["transformer." + name].grad
        assert relerr(named[name].grad, r) < TOL_GRAD and cosine(named[name].grad, r) > 0.999, name
    # eval mode and sample sizes >= the token count leave the sequence whole (reference: self.training / num_samples >= seq_len)
    model.eval()
    with torch.no_grad():
        e1 = model(ids.to(cuda), grid0.to(cuda), mask.to(cuda), _repeat_counts=[2, 2])
    model.config.pixel_random_sampling_size = 0
    with torch.no_grad():
        e0 = model(ids.to(cuda), grid0.to(cuda), mask.to(cuda), _repeat_counts=[2, 2])
    assert torch.equal(e1["itm_scores"], e0["itm_scores"])


def _clipbert(cls_name, sd, cuda, **cfg_extra):
    import clipbert_b200 as cb
    cfg = make_cfg(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, **cfg_extra)
    model = cb.ClipBert(cfg, detectron2_model_cfg="R-50-grid.yaml", transformer_cls=getattr(cb, cls_name))
    assert not model.load_state_dict(sd).missing_keys
    return model.to(cuda)


def test_config4_tgif_qa_multiple_choice_clip_batched(cuda, weights):
    """BASELINE config 4 in miniature (TGIF-QA action: 2 clips x 1 frame, 5 options per video, ClipBertForMultipleChoice):
    forward_clips folds the (video, clip) units into one pass and returns the (n_clips, B, 5) tensor the reference stacks
    (run_video_qa.py:470-486); checked against the oracle's per-clip loop and against this path's own loop."""
    from oracle import clipbert_ref as R, synth
    sd = dict(weights)
    sd.update(synth.transformer_state_dict(50, num_labels=1))
    model = _clipbert("ClipBertForMultipleChoice", sd, cuda, num_labels=5).eval()
    B, n_clips, T, n_ex, size = 3, 2, 1, 5, 128
    batch = synth.synth_batch(B, n_clips * T, n_ex=n_ex, size=size, max_len=16, seed=21)
    labels = torch.tensor([0, 3, 4])
    vis = batch["visual_inputs"].view(B, n_clips, T, 3, size, size)
    dev = {k: v.to(cuda) for k, v in batch.items() if torch.is_tensor(v)}
    with torch.no_grad():
        out = model.forward_clips(dict(visual_inputs=dev["visual_inputs"], text_input_ids=dev["text_input_ids"],
                                       text_input_mask=dev["text_input_mask"], n_examples_list=[n_ex] * B), n_clips)["logits"]
        loop = torch.stack([model(dict(visual_inputs=dev["visual_inputs"].view(B, n_clips, T, 3, size, size)[:, c],
                                       text_input_ids=dev["text_input_ids"], text_input_mask=dev["text_input_mask"], labels=None,
                                       n_examples_list=[n_ex] * B))["logits"] for c in range(n_clips)])
        ref = torch.stack([R.clipbert_forward(dict(batch, visual_inputs=vis[:, c], labels=labels), sd, head="multiple_choice", num_labels=5,
                                              rnd=R.Rounding.bf16())["logits"] for c in range(n_clips)])
    assert out.shape == loop.shape == ref.shape == (n_clips, B, 5)
    assert relerr(out, loop) < 1e-3, relerr(out, loop)
    assert relerr(out, ref) < TOL_LOGITS, relerr(out, ref)
    # clip aggregation + CE over the options as the task script does it (mean pooling of the clip scores, run_video_qa.py:488-501)
    loss = torch.nn.functional.cross_entropy(out.mean(0), labels.to(cuda))
    loss_ref = torch.nn.functional.cross_entropy(ref.mean(0), labels)
    assert abs(float(loss) - float(loss_ref)) < 5e-3


def test_config3_four_clips_two_frames_clip_batched(cuda, weights):
    """BASELINE config 3's per-GPU shape in miniature (4 clips x 2 frames, one caption per video): one batched pass of the 8
    (video, clip) units against the oracle's clip loop, logits and the LSE-aggregated loss (run_video_retrieval.py:404-422)."""
    from oracle import clipbert_ref as R, synth
    model = _clipbert("ClipBertForVideoTextRetrieval", weights, cuda).eval()
    B, n_clips, T, size = 2, 4, 2, 96
    batch = synth.synth_batch(B, n_clips * T, n_ex=1, size=size, seed=31)
    vis = batch["visual_inputs"].view(B, n_clips, T, 3, size, size)
    with torch.no_grad():
        out = model.forward_clips(dict(visual_inputs=batch["visual_inputs"].to(cuda), text_input_ids=batch["text_input_ids"].to(cuda),
                                       text_input_mask=batch["text_input_mask"].to(cuda), n_examples_list=[1] * B), n_clips)["logits"]
        ref = [R.clipbert_forward(dict(batch, visual_inputs=vis[:, c]), weights, rnd=R.Rounding.bf16())["logits"] for c in range(n_clips)]
    assert out.shape == (n_clips, B, 2)
    assert relerr(out, torch.stack(ref)) < TOL_LOGITS
    loss_ref = R.aggregate_clip_logits(ref, batch["labels"], "lse")
    lg = out.permute(1, 0, 2).contiguous()
    o = torch.logsumexp(lg.view(B, -1), dim=-1, keepdim=True) - torch.logsumexp(lg, dim=1)
    loss = torch.gather(o, -1, batch["labels"].to(cuda).view(-1, 1)).mean()
    assert abs(float(loss) - float(loss_ref)) < 3e-3


def test_fused_clip_lse_loss_kernel(cuda):
    """cb_clip_lse_loss (forward + backward of the "lse" clip aggregation, run_video_retrieval.py:404-422) against the oracle:
    fp32 in / fp32 out, so the tolerance is accumulation-order noise (fast-math exp / log: 1e-5 relative)."""
    import clipbert_b200 as cb
    from oracle import clipbert_ref as R
    g = torch.Generator().manual_seed(3)
    for n_clips, nseq, ncls, scale in ((2, 32, 2, 1.0), (4, 320, 5, 3.0), (16, 8, 2, 0.2), (1, 1, 2, 1.0), (2, 700, 3, 10.0)):
        z = torch.randn(n_clips, nseq, ncls, generator=g) * scale
        y = torch.randint(0, ncls, (nseq,), generator=g)
        zr = z.clone().requires_grad_(True)
        ref = R.aggregate_clip_logits(list(zr.unbind(0)), y, "lse")
        (2.0 * ref).backward()
        zt = z.to(cuda).requires_grad_(True)
        loss = cb.clip_lse_loss(zt, y.to(cuda))
        (2.0 * loss).backward()
        assert abs(float(loss) - float(ref)) < 2e-5 * max(1.0, abs(float(ref))), (n_clips, nseq, ncls, float(loss), float(ref))
        assert relerr(zt.grad, zr.grad) < 2e-5, (n_clips, nseq, ncls, relerr(zt.grad, zr.grad))
        with torch.no_grad():                      # forward only (no gradient buffer)
            assert abs(float(cb.clip_lse_loss(z.to(cuda), y.to(cuda))) - float(ref)) < 2e-5 * max(1.0, abs(float(ref)))


@pytest.mark.parametrize("variant", [1, 0])     # 1: cp.async double-buffered key tiles (default), 0: synchronous loads
@pytest.mark.parametrize("dims", [(2, 69, 20), (2, 150, 100), (1, 521, 512), (3, 128, 64), (1, 65, 0)])
def test_attention_tensor_core_forward_for_long_sequences(cuda, dims, variant):
    """The mma.sync online-softmax forward for L > 64 (attn_tc_fwd_flash_kernel; 448 px frames L = 69, paragraph retrieval
    L = 521) against fp32 torch attention and against the CUDA-core kernel it replaces: context, saved log-sum-exp (the general
    backward consumes it), and the same dropout stream. Default for L > 64."""
    from clipbert_b200 import ops
    from util import TOL_BF16_OP
    nseq, L, lt = dims
    heads = 12
    g = torch.Generator().manual_seed(31)
    qkv = (torch.randn(nseq * L, 3 * 768, generator=g)).to(cuda).to(torch.bfloat16)
    mask = torch.ones(nseq, max(lt, 1), dtype=torch.int64, device=cuda)
    if lt > 4:
        mask[0, lt - 3:] = 0
        mask[-1, lt // 2:] = 0
    ref_mask = mask[:, :lt]
    outs = {}
    try:
        ops.set_attention_flash_pipe(variant)
        for flash in (0, 1):
            ops.set_attention_flash(flash)
            for p, seed in ((0.0, 0), (0.1, 5)):
                ctx = torch.zeros(nseq * L, 768, device=cuda, dtype=torch.bfloat16)
                lse = torch.zeros(nseq, heads, L, device=cuda)
                ops.attention_fwd(qkv, mask, ctx, lse, nseq, L, lt, heads, p, seed)
                outs[(flash, p)] = (ctx, lse)
    finally:
        ops.set_attention_flash(1)
        ops.set_attention_flash_pipe(1)
    x = qkv.float().view(nseq, L, 3, heads, 64)
    q, k, v = (x[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    full = torch.cat([ref_mask, torch.ones(nseq, L - lt, dtype=torch.int64, device=cuda)], 1)
    s = q @ k.transpose(-1, -2) / 8.0 + (1.0 - full[:, None, None, :].float()) * -10000.0
    ref = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(nseq * L, 768)
    ref_lse = torch.logsumexp(s, -1)
    ctx, lse = outs[(1, 0.0)]
    assert relerr(ctx, ref) < TOL_BF16_OP, relerr(ctx, ref)
    assert float((lse - ref_lse).abs().max()) < 2e-2 and relerr(lse, outs[(0, 0.0)][1]) < 1e-3
    assert relerr(ctx, outs[(0, 0.0)][0]) < 2 * TOL_BF16_OP
    # same (seed, element) dropout stream as the general kernel: P is rounded to bf16 here and kept fp32 there
    assert relerr(outs[(1, 0.1)][0], outs[(0, 0.1)][0]) < 3 * TOL_BF16_OP
    assert relerr(outs[(1, 0.1)][1], outs[(0, 0.1)][1]) < 1e-3


def test_forward_error_sits_at_the_bf16_noise_floor_of_the_reference_ops(cuda, weights):
    """How far may a correct bf16 implementation be from the fp32 reference? Run the ORACLE's own ops (plain torch: cuDNN /
    cuBLAS bf16 under autocast, fp32 LayerNorm / softmax - the mixed precision the reference trains in) on the same GPU and
    measure its distance from the fp32 oracle; this path must not be further away than a small multiple of that floor."""
    from oracle import clipbert_ref as R, synth
    model = _clipbert("ClipBertForVideoTextRetrieval", weights, cuda).eval()
    batch = synth.synth_batch(2, 2, n_ex=2, size=224, seed=41)
    with torch.no_grad():
        ref32 = R.clipbert_forward(dict(batch), weights)["logits"]
        sd_gpu = {k: v.to(cuda) for k, v in weights.items()}
        gb = {k: (v.to(cuda) if torch.is_tensor(v) else list(v)) for k, v in batch.items()}
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ref16 = R.clipbert_forward(gb, sd_gpu)["logits"].float().cpu()
        mb = {k: (v.to(cuda) if torch.is_tensor(v) else list(v)) for k, v in batch.items()}
        out = model(mb)["logits"]
    e_floor, e_ours = relerr(ref16, ref32), relerr(out, ref32)
    print("bf16 noise floor of the reference ops %.3e | this path %.3e" % (e_floor, e_ours))
    assert e_ours < TOL_LOGITS
    assert e_ours < 3.0 * e_floor + 5e-3, (e_ours, e_floor)


# Last on purpose: if the driver accepts the 3-D tensor map but the hardware disagrees with the layout, a TMA fault would poison
# the CUDA context for every test after it.
def test_gemm_mn_major_operands_through_3d_tma_boxes(cuda):
    """ops.set_mn3d(1): the MN-major operands of the dgrad (NN) and wgrad GEMMs arrive as one 3-D TMA box per k-chunk instead of
    BN/64 2-D boxes. Same bytes in the same shared-memory layout, so NN results must be bit-identical to the 2-D path and the
    wgrad (fp32 red.add, order not deterministic) equal to accumulation noise; also against fp32 torch. Shapes whose column
    count is not a multiple of 64 keep the 2-D boxes automatically."""
    import torch.nn.functional as F
    from clipbert_b200 import ops
    from util import TOL_BF16_OP, TOL_FP32_OP
    g = torch.Generator().manual_seed(2)

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g) * scale).to(cuda).to(torch.bfloat16)

    def both(fn):
        outs = []
        try:
            for on in (0, 1):
                ops.set_mn3d(on)
                outs.append(fn())
        finally:
            ops.set_mn3d(1)
        return outs

    # ---- NN (dgrad of Linear / 1x1 conv): out [M, N] = A [M, K] @ B [K, N] ----
    for M, N, K, bn in ((500, 384, 256, 0), (1312, 2304, 768, 256), (2624, 768, 3072, 128), (64, 768, 3072, 64), (700, 264, 512, 0)):
        A, B = rnd(M, K), rnd(K, N, scale=0.1)

        def run():
            C = torch.zeros(M, N, device=cuda)
            ops.gemm(mode=ops.CB_GEMM_NN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=K, b_ld=N, out=C, out_ld=N, out_fp32=1, block_n=bn)
            return C
        c2d, c3d = both(run)
        assert relerr(c3d, A.float() @ B.float()) < TOL_FP32_OP, (M, N, K)
        assert torch.equal(c2d, c3d), (M, N, K)
    # ---- NN with 9 taps: dgrad of a 3x3 conv over the zero-bordered layout, bf16 output through the UNPAD row map ----
    for NB, H, W, Cin, Cout in ((2, 7, 7, 64, 128), (3, 14, 14, 256, 256), (1, 3, 5, 512, 64)):
        x = rnd(NB, H, W, Cin)
        wf = rnd(Cin, Cout, 3, 3, scale=0.05)
        xp = torch.zeros(NB, H + 2, W + 2, Cin, device=cuda, dtype=torch.bfloat16)
        xp[:, 1:-1, 1:-1] = x
        P = NB * (H + 2) * (W + 2)
        wfk = wf.permute(0, 2, 3, 1).contiguous().view(Cin, 9 * Cout)

        def run():
            y = torch.zeros(NB * H * W, Cout, device=cuda, dtype=torch.bfloat16)
            ops.gemm(mode=ops.CB_GEMM_NN, m=P, n=Cout, k=Cin, a=xp, a_rows=P, a_ld=Cin, b=wfk, b_rows=Cin, b_ld=9 * Cout, ntaps=9,
                     tap_w=W + 2, tap_sign=-1, out=y, out_ld=Cout, rowmap=ops.ROWMAP_UNPAD, map_h=H, map_w=W)
            return y
        y2d, y3d = both(run)
        ref = F.conv_transpose2d(x.float().permute(0, 3, 1, 2), wf.float(), padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
        assert relerr(y3d, ref) < TOL_BF16_OP and torch.equal(y2d, y3d), (NB, H, W, Cin, Cout)
    # ---- WGRAD: dW [Mo, No] += dY^T X (both operands MN-major), plain and 9-tap ----
    for P, Mo, No, bn, sk in ((1312, 768, 768, 128, 1), (2624, 3072, 768, 0, 0), (5000, 256, 256, 128, 7), (50176, 512, 128, 0, 0), (333, 136, 72, 64, 1)):
        dY, X = rnd(P, Mo), rnd(P, No)

        def run():
            dW = torch.zeros(Mo, No, device=cuda)
            ops.gemm(mode=ops.CB_GEMM_WGRAD, m=Mo, n=No, k=P, a=dY, a_rows=P, a_ld=Mo, b=X, b_rows=P, b_ld=No, split_k=sk, out=dW, out_ld=No,
                     out_fp32=1, block_n=bn)
            return dW
        w2d, w3d = both(run)
        assert relerr(w3d, dY.float().t() @ X.float()) < TOL_FP32_OP and relerr(w3d, w2d) < TOL_FP32_OP, (P, Mo, No)
    for NB, H, W, Cin, Cout, sk in ((2, 7, 7, 64, 128, 1), (4, 14, 14, 128, 128, 3)):
        x, dy = rnd(NB, H, W, Cin), rnd(NB, H, W, Cout)
        xp = torch.zeros(NB, H + 2, W + 2, Cin, device=cuda, dtype=torch.bfloat16)
        dyp = torch.zeros(NB, H + 2, W + 2, Cout, device=cuda, dtype=torch.bfloat16)
        xp[:, 1:-1, 1:-1], dyp[:, 1:-1, 1:-1] = x, dy
        P = NB * (H + 2) * (W + 2)

        def run():
            dW = torch.zeros(Cout, 9 * Cin, device=cuda)
            ops.gemm(mode=ops.CB_GEMM_WGRAD, m=Cout, n=Cin, k=P, a=dyp, a_rows=P, a_ld=Cout, b=xp, b_rows=P, b_ld=Cin, ntaps=9, tap_w=W + 2,
                     tap_sign=1, split_k=sk, out=dW, out_ld=9 * Cin, out_fp32=1)
            return dW
        w2d, w3d = both(run)
        wz = torch.zeros(Cout, Cin, 3, 3, device=cuda, requires_grad=True)
        F.conv2d(x.float().permute(0, 3, 1, 2), wz, padding=1).backward(dy.float().permute(0, 3, 1, 2))
        assert relerr(w3d, wz.grad.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin)) < TOL_FP32_OP and relerr(w3d, w2d) < TOL_FP32_OP
