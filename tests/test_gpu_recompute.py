"""Activation recomputation: GridFeatBackbone.recompute_activations (each ResNet stage re-run from its kept input before its
backward) and ClipBertBaseModel.recompute_activations (each encoder layer re-run from its kept input hidden state).

The recomputed tensors come from the forward's own launches with the forward's seeds and dropout word, so in deterministic mode
(torch.use_deterministic_algorithms(True)) the switch on gives the switch off's bits: logits, loss, every parameter gradient and
the frame / grid gradient, on both stem modes, FREEZE_AT 1 - 3, frames requiring grad or not, every head's default path, ragged
n_examples_list, two FusedAdamW steps and a CUDA-graph replay. In default mode the two agree within the fp32-atomic noise of the
weight gradients. Peak memory drops by at least the stash the switch removes, computed from shapes; the three combinations the
switch refuses raise. tests/test_recompute_emulated.py replays the runners below on a CPU and checks launch order and buffer
lifetimes.
"""
import contextlib

import numpy as np
import pytest
import torch

from util import make_cfg, relerr

BF16 = torch.bfloat16
TOL_DEFAULT = 1e-4      # default mode: fp32 atomic accumulation order in the weight gradients, LN / bias sums
STAGES = (("res2", 3, 64, 256, 1), ("res3", 4, 128, 512, 2), ("res4", 6, 256, 1024, 2), ("res5", 3, 512, 2048, 2))


@contextlib.contextmanager
def deterministic(on=True):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(bool(on))
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


@contextlib.contextmanager
def recompute(cnn=False, bert=False):
    """Both switches as class defaults, so that models built inside a runner pick them up."""
    import clipbert_b200 as cb
    prev = cb.GridFeatBackbone.recompute_activations, cb.ClipBertBaseModel.recompute_activations
    cb.GridFeatBackbone.recompute_activations, cb.ClipBertBaseModel.recompute_activations = bool(cnn), bool(bert)
    try:
        yield
    finally:
        cb.GridFeatBackbone.recompute_activations, cb.ClipBertBaseModel.recompute_activations = prev


def compare(off, on, det, what=""):
    assert len(off) == len(on)
    for i, (a, b) in enumerate(zip(off, on)):
        if a is None:
            assert b is None, (what, i)
            continue
        assert a.shape == b.shape and a.dtype == b.dtype, (what, i)
        if det:
            assert torch.equal(a, b), "%s: output %d differs with the switch on" % (what, i)
        else:
            assert relerr(b, a) < TOL_DEFAULT, (what, i, relerr(b, a))
        assert bool(torch.isfinite(a.float()).all()), (what, i)


def off_and_on(run, det=True, cnn=True, bert=True):
    with deterministic(det):
        with recompute():
            off = run()
        with recompute(cnn, bert):
            on = run()
    return off, on


# ------------------------------------------------------------------------------------------------ CNN
def cnn_step(dev, sd, size, stem_mode, freeze_at, frames_grad, n_frms=2):
    """Two backward passes of one GridFeatBackbone: [grid, every parameter gradient (accumulated twice), frame gradient]."""
    import test_gpu_cnn_hooks as H
    m = H.backbone(dev, sd, freeze_at)
    m.stem_mode = stem_mode
    x = H.frames(dev, size, n_frms=n_frms)
    out = []
    for step in range(2):
        xg = x.clone().requires_grad_(frames_grad)
        grid = m(xg)
        dgrid = torch.randn(grid.shape, generator=torch.Generator().manual_seed(step)).to(BF16).to(dev)
        grid.backward(dgrid)
        out += [grid.detach().clone(), xg.grad.clone() if frames_grad else None]
    return out + [p.grad.clone() for p in m.parameters() if p.grad is not None]


def run_cnn(dev, sd, size, stem_mode, freeze_at, frames_grad, det=True):
    off, on = off_and_on(lambda: cnn_step(dev, sd, size, stem_mode, freeze_at, frames_grad), det, bert=False)
    compare(off, on, det, "cnn %d %s FREEZE_AT %d frames_grad %s" % (size, stem_mode, freeze_at, frames_grad))


@pytest.fixture(scope="module")
def cnn_sd():
    from oracle import synth
    return synth.cnn_state_dict(42)


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)


CNN_CASES = [(size, mode, fa, fg) for size in (224, 448) for mode in ("s2d", "im2col") for fa in (1, 2, 3) for fg in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("size,stem_mode,freeze_at,frames_grad", CNN_CASES,
                         ids=["%d-%s-fa%d-%s" % (s, m, f, "frames" if g else "noframes") for s, m, f, g in CNN_CASES])
def test_cnn_bits_switch_on_equal_off(cuda, cnn_sd, size, stem_mode, freeze_at, frames_grad):
    run_cnn(cuda, cnn_sd, size, stem_mode, freeze_at, frames_grad)


@pytest.mark.gpu
@pytest.mark.parametrize("freeze_at,frames_grad", [(2, False), (1, True)])
def test_cnn_default_mode_within_atomic_noise(cuda, cnn_sd, freeze_at, frames_grad):
    run_cnn(cuda, cnn_sd, 224, "s2d", freeze_at, frames_grad, det=False)


# ------------------------------------------------------------------------------------------------ transformer heads
def _zero(engine):
    f = getattr(engine, "_flat", None)
    if f is not None:
        f.attach_grads()
        f.grad.zero_()


def head_step(dev, weights, kind, gh=3, lt=20, counts=(1, 3, 2), p=0.1, steps=2):
    """Two training steps of a transformer head at dropout p on a fixed grid (visual tokens gh x gh, L = lt + gh * gh), with ragged
    repeat counts: [loss, flat gradient, grid gradient] per step."""
    import clipbert_b200 as cb
    from oracle import synth
    torch.manual_seed(0)
    nvid = len(counts)
    nseq = sum(counts)
    g = torch.Generator().manual_seed(3)
    grid0 = torch.randn(nvid, 2, gh, gh, 768, generator=g).abs().to(BF16).float()
    extra = {}
    if kind == "mc":
        extra = dict(num_labels=3)
    if kind == "pretrain":
        extra = dict(pixel_random_sampling_size=gh * gh - 2)
    cfg = make_cfg(hidden_dropout_prob=p, attention_probs_dropout_prob=p, **extra)
    cls = {"retrieval": cb.ClipBertForVideoTextRetrieval, "qa": cb.ClipBertForSequenceClassification,
           "mc": cb.ClipBertForMultipleChoice, "pretrain": cb.ClipBertForPreTraining}[kind]
    model = cls(cfg)
    sd = {k[len("transformer."):]: v for k, v in weights.items() if k.startswith("transformer.")}
    if kind != "retrieval":
        sd = {k: v for k, v in sd.items() if not k.startswith("classifier.")}
    model.load_state_dict(sd, strict=False)
    model.to(dev).train()
    if kind == "mc":
        counts = [3] * nvid
        nseq = 3 * nvid
    ids, mask = synth.synth_text(nseq, lt, seed=5)
    ids, mask = ids.to(dev), mask.to(dev)
    out = []
    for step in range(steps):
        _zero(model)
        grid = grid0.clone().to(dev).requires_grad_(True)
        if kind == "pretrain":
            np.random.seed(77 + step)
            mlm = torch.full((nseq, lt), -100, dtype=torch.long)
            mlm[:, 3], mlm[:, 7] = ids[:, 3].cpu(), ids[:, 7].cpu()
            itm = torch.tensor([1, 0] * nseq)[:nseq]
            o = model(ids, grid, mask, mlm_labels=mlm.to(dev), itm_labels=itm.to(dev), _repeat_counts=list(counts))
            loss = o["mlm_loss"].sum() / 8 + o["itm_loss"].mean()
        else:
            labels = torch.arange(nvid if kind == "mc" else nseq) % (3 if kind == "mc" else 2)
            o = model(ids, grid, mask, labels=labels.to(dev), _repeat_counts=list(counts))
            loss = o["loss"].mean()
        loss.backward()
        out += [loss.detach().clone(), model._flat.grad.clone(), grid.grad.clone()]
    return out


def base_step(dev, weights, gh=3, lt=20, p=0.1):
    """ClipBertBaseModel(...) with hidden states: a loss on sequence_output, pooled_output and a hidden state."""
    import clipbert_b200 as cb
    from oracle import synth
    torch.manual_seed(0)
    cfg = make_cfg(hidden_dropout_prob=p, attention_probs_dropout_prob=p, output_hidden_states=True)
    bert = cb.ClipBertBaseModel(cfg)
    bert.load_state_dict({k[len("transformer.bert."):]: v for k, v in weights.items() if k.startswith("transformer.bert.")})
    bert.to(dev).train()
    g = torch.Generator().manual_seed(8)
    grid0 = torch.randn(4, 1, gh, gh, 768, generator=g).abs().to(BF16).float()
    ids, mask = synth.synth_text(4, lt, seed=3)
    out = []
    for _ in range(2):
        bert.zero_grad()
        grid = grid0.clone().to(dev).requires_grad_(True)
        seq, pooled, hidden = bert(ids.to(dev), grid, mask.to(dev))
        loss = seq.float().square().mean() + pooled.float().sum() + hidden[5].float().mean()
        loss.backward()
        out += [seq.detach().clone(), loss.detach().clone(), grid.grad.clone()]
        out += [p.grad.clone() for p in bert.parameters() if p.grad is not None]
    return out


HEADS = ["retrieval", "qa", "mc", "pretrain"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", HEADS)
@pytest.mark.parametrize("gh", [3, 7], ids=["L29", "L69"])
def test_heads_bits_switch_on_equal_off(cuda, weights, kind, gh):
    off, on = off_and_on(lambda: head_step(cuda, weights, kind, gh=gh), cnn=False)
    compare(off, on, True, kind)


@pytest.mark.gpu
@pytest.mark.parametrize("L", [41, 69])
def test_lengths_41_and_69(cuda, weights, L):
    """L = 41 (one-tile attention) and 69 (the long-sequence kernels): lt + gh * gh."""
    gh = 3 if L == 41 else 7
    off, on = off_and_on(lambda: head_step(cuda, weights, "retrieval", gh=gh, lt=L - gh * gh), cnn=False)
    compare(off, on, True, "L%d" % L)


@pytest.mark.gpu
def test_base_model_with_hidden_states_bits(cuda, weights):
    off, on = off_and_on(lambda: base_step(cuda, weights), cnn=False)
    compare(off, on, True, "base")


@pytest.mark.gpu
def test_heads_default_mode_within_atomic_noise(cuda, weights):
    off, on = off_and_on(lambda: head_step(cuda, weights, "retrieval", gh=7), det=False, cnn=False)
    compare(off, on, False, "retrieval default mode")


# ------------------------------------------------------------------------------------------------ end to end
def e2e_steps(dev, weights, kind="ClipBertForSequenceClassification", size=224, counts=(2, 1), n_clips=2, frames=2):
    """ClipBert with both halves, dropout 0.1, forward_clips over ragged n_examples_list, clip-mean cross entropy, FusedAdamW
    (clip + step), two steps: [logits, loss, flat gradients] per step, then the optimizer's masters and moments."""
    import clipbert_b200 as cb
    from clipbert_b200.optim import FusedAdamW
    from oracle import synth
    from test_gpu_optim import e2e_param_groups
    from test_zz2_gpu_round2 import _clipbert
    torch.manual_seed(0)
    model = _clipbert(kind, weights, dev, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1).train()
    opt = FusedAdamW([g for g in e2e_param_groups(model) if g["params"]], lr=5e-5, betas=(0.9, 0.98), model=model)
    batch = synth.synth_batch(len(counts), n_clips * frames, n_ex=1, size=size, seed=9)
    ids, mask = synth.synth_text(sum(counts), 20, seed=4)
    res = []
    for _ in range(2):
        model.zero_grad()
        mb = dict(visual_inputs=batch["visual_inputs"].to(dev), text_input_ids=ids.to(dev), text_input_mask=mask.to(dev),
                  n_examples_list=list(counts))
        logits = model.forward_clips(mb, n_clips)["logits"]
        loss = torch.nn.functional.cross_entropy(logits.float().mean(0), (torch.arange(sum(counts)) % 2).to(dev))
        loss.backward()
        opt.clip_grad_norm(1.0)
        res += [logits.detach().clone(), loss.detach().clone()]
        res += [m._flat.grad.clone() for m in (model.transformer, model.cnn) if getattr(m, "_flat", None) is not None]
        opt.step()
    for h in opt._plan:
        res += [h["flat"].master.clone(), h["exp_avg"].clone(), h["exp_avg_sq"].clone()]
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ClipBertForSequenceClassification", "ClipBertForVideoTextRetrieval"], ids=["qa", "retrieval"])
def test_e2e_two_fused_adamw_steps_bits(cuda, weights, kind):
    off, on = off_and_on(lambda: e2e_steps(cuda, weights, kind))
    compare(off, on, True, kind)


def graph_step_runs(dev, weights, replays=3):
    """A retrieval training step captured in a CUDA graph and replayed: [loss, a weight gradient] of each replay, then of a
    replay rewound to the first replay's dropout position."""
    from oracle import synth
    from test_zz2_gpu_round2 import _clipbert, _to
    torch.manual_seed(0)
    model = _clipbert("ClipBertForVideoTextRetrieval", weights, dev, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1).train()
    batch = _to(synth.synth_batch(2, 2, n_ex=1, size=96, seed=61), dev)
    tr = model.transformer

    def step():
        model.zero_grad()
        loss = model(dict(batch))["loss"].mean()
        loss.backward()
        return loss
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        loss_dev = step().detach()
    w0 = int(tr._drop_counter.item())
    out = []
    for _ in range(replays):
        g.replay()
        torch.cuda.synchronize()
        out += [loss_dev.clone(), tr.bert.encoder.layer[0].output.dense.weight.grad.detach().clone(),
                model.cnn.feature.backbone.res5[0].conv1.weight.grad.detach().clone()]
    tr._drop_counter.fill_(w0)
    g.replay()
    torch.cuda.synchronize()
    out += [loss_dev.clone(), tr.bert.encoder.layer[0].output.dense.weight.grad.detach().clone()]
    del g
    return out


@pytest.mark.gpu
def test_cuda_graph_replay_fresh_masks_and_equal_to_switch_off(cuda, weights):
    off, on = off_and_on(lambda: graph_step_runs(cuda, weights))
    compare(off, on, True, "graph")
    losses = [float(on[3 * k]) for k in range(3)]
    assert len(set(losses)) == 3, losses                           # fresh masks on every replay
    assert torch.equal(on[-2], on[0]) and torch.equal(on[-1], on[1])   # rewound: replay 0's masks again


# ------------------------------------------------------------------------------------------------ memory
def cnn_stash_removed(n, size, freeze_at, frames_grad):
    """Bytes of the CNN stash the switch removes, from shapes: for every stage that runs a backward, its blocks' subsampled
    inputs (stride 2), 3x3-conv outputs and block outputs except the stage's last (the next stage's kept input); the recompute
    then holds one such stage at a time, so the largest comes back."""
    h = ((size - 1) // 2 + 1 - 1) // 2 + 1
    per_stage = []
    for si, (name, nb, mid, cout, stride) in enumerate(STAGES):
        cin = 64 if si == 0 else STAGES[si - 1][3]
        if stride == 2:
            h = (h - 1) // 2 + 1
        if not (frames_grad or freeze_at <= si + 1):
            continue
        px = n * h * h
        b = px * cin if stride == 2 else 0            # xs of block 0
        b += nb * px * mid                            # b
        b += (nb - 1) * px * cout                     # y of all but the last
        per_stage.append(2 * b)
    return sum(per_stage) - max(per_stage)


def cnn_peak(dev, sd, size, n_frms, freeze_at, frames_grad, on):
    import test_gpu_cnn_hooks as H
    m = H.backbone(dev, sd, freeze_at)
    m.recompute_activations = on
    x = H.frames(dev, size, n_frms=n_frms)
    for step in range(2):          # the second step runs with the pool of zero-bordered buffers already filled
        xg = x.clone().requires_grad_(frames_grad)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        grid = m(xg)
        grid.backward(torch.ones_like(grid))
        del grid, xg
        torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


@pytest.mark.gpu
@pytest.mark.parametrize("freeze_at,frames_grad", [(2, False), (1, True)])
def test_cnn_peak_memory_drops_by_the_removed_stash(cuda, cnn_sd, freeze_at, frames_grad):
    size, n_frms = 448, 8
    off = cnn_peak(cuda, cnn_sd, size, n_frms, freeze_at, frames_grad, False)
    on = cnn_peak(cuda, cnn_sd, size, n_frms, freeze_at, frames_grad, True)
    removed = cnn_stash_removed(n_frms, size, freeze_at, frames_grad)
    assert off - on >= removed, (off, on, removed)


def bert_peak(dev, weights, on, nseq=32, gh=7, lt=40):
    import clipbert_b200 as cb
    from oracle import synth
    cfg = make_cfg(hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
    bert = cb.ClipBertBaseModel(cfg).to(dev).train()
    bert.recompute_activations = on
    grid = torch.randn(nseq, 1, gh, gh, 768, device=dev).abs().to(BF16)
    ids, mask = synth.synth_text(nseq, lt, seed=3)
    for _ in range(2):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        seq, pooled = bert(ids.to(dev), grid, mask.to(dev))
        (seq.float().mean() + pooled.float().mean()).backward()
        del seq, pooled
        torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


@pytest.mark.gpu
def test_bert_peak_memory_drops_by_the_removed_stash(cuda, weights):
    """The layers' stash but the input (qkv 3H, ctx, s1, a, s2 H each, gel and u 4H each as bf16; lse and two LN stats fp32), less
    the two layers the backward holds at once (the one it runs and the one above, whose weight gradients are still in flight)."""
    nseq, gh, lt = 32, 7, 40
    L, H, heads = lt + gh * gh, 768, 12
    M = nseq * L
    per_layer = 2 * M * (3 * H + 4 * H + 8 * H) + 4 * (nseq * heads * L + 4 * M)
    removed = (12 - 2) * per_layer
    off, on = bert_peak(cuda, weights, False), bert_peak(cuda, weights, True)
    assert off - on >= removed, (off, on, removed)


# ------------------------------------------------------------------------------------------------ refusals
def run_refusals(dev, weights, cnn_sd):
    import clipbert_b200 as cb
    import test_gpu_cnn_hooks as H
    from oracle import synth
    cfg = make_cfg(output_attentions=True)
    bert = cb.ClipBertBaseModel(cfg).to(dev)
    bert.recompute_activations = True
    grid = torch.randn(2, 1, 3, 3, 768).abs().to(BF16).to(dev)
    ids, mask = synth.synth_text(2, 12, seed=3)
    ids, mask = ids.to(dev), mask.to(dev)
    for attr in ("differentiable_attentions", "layerwise_autograd"):
        setattr(bert, attr, True)
        with pytest.raises(RuntimeError, match="recompute_activations cannot be combined with %s" % attr):
            bert(ids, grid, mask)
        with torch.no_grad():
            bert(ids, grid, mask)                       # a pass that records no autograd recomputes nothing
        setattr(bert, attr, False)
    h = bert.encoder.layer[3].register_forward_hook(lambda *a: None)
    with pytest.raises(RuntimeError, match="recompute_activations cannot be combined with hooks"):
        bert(ids, grid, mask)
    h.remove()
    bert(ids, grid, mask)                               # the switch alone runs
    m = H.backbone(dev, cnn_sd)
    m.recompute_activations = True
    h = m.feature.backbone.res3[1].register_forward_hook(lambda *a: None)
    with pytest.raises(RuntimeError, match="recompute_activations cannot be combined with hooks"):
        m(H.frames(dev, 64, n_frms=1))
    h.remove()


@pytest.mark.gpu
def test_refusals(cuda, weights, cnn_sd):
    run_refusals(cuda, weights, cnn_sd)


def test_switches_default_off():
    import clipbert_b200 as cb
    assert cb.GridFeatBackbone.recompute_activations is False and cb.ClipBertBaseModel.recompute_activations is False
