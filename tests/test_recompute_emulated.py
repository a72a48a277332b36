"""Activation recomputation on CPU: the runners of tests/test_gpu_recompute.py replayed with the C-ABI calls answered by
tests/ops_emulator.py (and the frame-gradient restatements of tests/test_input_grads_emulated.py), plus what only a recording of
the calls shows: the order in which the engines issue the recompute launches, that every zero-bordered buffer goes back to the
pool only after the weight gradient that reads it, and that the overlapped exchange's CNN bucket still fires once, after res5.
Planted faults (a recompute that draws the next step's dropout masks, a stage buffer recycled before its weight gradient) must
make the checks fail."""
import contextlib

import pytest
import torch

import test_gpu_recompute as R
import test_input_grads_emulated as IGE

CPU = torch.device("cpu")
SIZE = 64


@pytest.fixture(scope="module")
def cnn_sd():
    from oracle import synth
    return synth.cnn_state_dict(42)


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)


# ------------------------------------------------------------------------------------------------ bits, switch on against off
@pytest.mark.parametrize("stem_mode,freeze_at,frames_grad", [("s2d", 1, True), ("im2col", 2, False), ("s2d", 3, False),
                                                             ("im2col", 3, True)])
def test_cnn_bits_on_emulated_ops(cnn_sd, stem_mode, freeze_at, frames_grad):
    with IGE.emulated_ops():
        R.run_cnn(CPU, cnn_sd, SIZE, stem_mode, freeze_at, frames_grad)


@pytest.mark.parametrize("kind", R.HEADS)
def test_heads_bits_on_emulated_ops(weights, kind):
    with IGE.emulated_ops():
        off, on = R.off_and_on(lambda: R.head_step(CPU, weights, kind, gh=3, lt=8, counts=(1, 2)), cnn=False)
    R.compare(off, on, True, kind)


def test_base_model_bits_on_emulated_ops(weights):
    with IGE.emulated_ops():
        off, on = R.off_and_on(lambda: R.base_step(CPU, weights, gh=2, lt=8), cnn=False)
    R.compare(off, on, True, "base")


def test_refusals_on_emulated_ops(weights, cnn_sd):
    import test_layerwise_autograd_emulated as LWE
    with LWE.emulated_ops():
        R.run_refusals(CPU, weights, cnn_sd)


# ------------------------------------------------------------------------------------------------ launch order and lifetimes
@contextlib.contextmanager
def recorded():
    """The emulated ops, with every GEMM launch, side-queue launch, join and pool return logged in issue order."""
    from clipbert_b200 import grid_feat, ops
    log = []
    with IGE.emulated_ops():
        gemm, run, join, put = ops.gemm, ops.SideQueue.run, ops.SideQueue.join, grid_feat.GridFeatBackbone._pad_put

        def gemm_(**kw):
            log.append(("gemm", kw["mode"], kw["m"], kw["n"], kw["k"], kw.get("ntaps", 1)))
            return gemm(**kw)

        def run_(self, fn, *keep):
            log.append(("side", {id(t) for t in keep}))
            return run(self, fn, *keep)

        def join_(self):
            log.append(("join",))
            return join(self)

        def put_(self, t, *a):
            log.append(("put", id(t)))
            return put(self, t, *a)
        ops.gemm, ops.SideQueue.run, ops.SideQueue.join, grid_feat.GridFeatBackbone._pad_put = gemm_, run_, join_, put_
        try:
            yield log
        finally:
            ops.gemm, ops.SideQueue.run, ops.SideQueue.join, grid_feat.GridFeatBackbone._pad_put = gemm, run, join, put


def _cnn_train(cnn_sd, freeze_at=2, bucket=None):
    import test_gpu_cnn_hooks as H
    m = H.backbone(CPU, cnn_sd, freeze_at)
    m.recompute_activations = True
    m._bucket_hook = bucket
    x = H.frames(CPU, SIZE, n_frms=1)
    grid = m(x)
    return m, grid


def check_recycled_after_reader(log):
    """Every buffer returned to the pool is read by no side-queue launch issued before it unless a join lies between them."""
    pending = set()
    for e in log:
        if e[0] == "side":
            pending |= e[1]
        elif e[0] == "join":
            pending.clear()
        elif e[0] == "put":
            assert e[1] not in pending, "a buffer went back to the pool before the weight gradient that reads it ran"


def test_cnn_recompute_launch_order(cnn_sd):
    """The backward re-issues, stage by stage from res5 down to res3 (FREEZE_AT 2), exactly the forward's convolution launches
    of that stage, each stage's recompute before its first dgrad launch and after the previous stage's join."""
    from clipbert_b200 import ops
    with recorded() as log:
        m, grid = _cnn_train(cnn_sd)
        n_fwd = len(log)
        grid.backward(torch.ones_like(grid))
    fwd = [e for e in log[:n_fwd] if e[0] == "gemm"]
    bwd = log[n_fwd:]
    # the forward's TN launches per stage: res2's blocks start after the stem GEMM; every block is 3 or 4 convolutions
    conv = [e for e in fwd if e[1] == ops.CB_GEMM_TN][1:-1]          # less the stem and the grid_encoder conv
    per_stage, i = {}, 0
    for name, nb, *_ in R.STAGES:
        k = nb * 3 + 1
        per_stage[name], i = conv[i:i + k], i + k
    assert i == len(conv)
    runs, cur = [], None
    for e in bwd:
        if e[0] == "gemm" and e[1] == ops.CB_GEMM_TN:
            if cur is None:
                cur = []
                runs.append(cur)
            cur.append(e)
        elif e[0] == "gemm" or e[0] == "join":
            cur = None
    # all but the stage's last conv3, whose output is the next stage's kept input (or res5_pad)
    assert runs == [per_stage["res5"][:-1], per_stage["res4"][:-1], per_stage["res3"][:-1]]
    joins = [k for k, e in enumerate(bwd) if e[0] == "join"]
    assert len(joins) >= 3
    check_recycled_after_reader(bwd)


def test_transformer_recompute_launch_order(weights):
    """Before each layer's backward, top-down, the backward re-issues that layer's four forward GEMMs (QKV, attention output,
    intermediate, output) with the forward's shapes, and joins the side queue before the layer's first dgrad."""
    from clipbert_b200 import ops
    with recorded() as log, R.recompute(bert=True):
        R.head_step(CPU, weights, "retrieval", gh=2, lt=8, counts=(1, 2), steps=1)
    tn = [k for k, e in enumerate(log) if e[0] == "gemm" and e[1] == ops.CB_GEMM_TN]
    start = next(k for k, e in enumerate(log) if e[0] == "gemm" and e[1] == ops.CB_GEMM_WGRAD)
    fwd_layers = [log[k][2:] for k in tn if k < start][:48]
    bwd_tn = [log[k][2:] for k in tn if k > start]
    assert len(bwd_tn) == 48
    for j in range(12):
        assert bwd_tn[4 * j: 4 * j + 4] == fwd_layers[4 * (11 - j): 4 * (11 - j) + 4], j
    # each group of four is followed by a join before the next NN (dgrad) launch
    last = max(k for k in tn if k > start)
    after = [e for e in log[last + 1:] if e[0] in ("join", "gemm")]
    assert after[0] == ("join",)


def test_recycled_buffers_check_rejects_a_premature_recycle(cnn_sd):
    """Planted fault: the stage's join left out, so its zero-bordered buffers go back to the pool while its weight gradients may
    still read them."""
    from clipbert_b200 import ops
    with recorded() as log:
        logged_join = ops.SideQueue.join          # recorded()'s logging join, restored before recorded() restores the real one
        try:
            m, grid = _cnn_train(cnn_sd)
            n_fwd = len(log)
            real = m._blocks_backward

            def no_join(*a, **k):
                g = real(*a, **k)
                ops.SideQueue.join = lambda self: None
                return g
            m._blocks_backward = no_join
            grid.backward(torch.ones_like(grid))
        finally:
            ops.SideQueue.join = logged_join
    with pytest.raises(AssertionError, match="before the weight gradient"):
        check_recycled_after_reader(log[n_fwd:])


def test_bucket_hook_fires_once_after_res5(cnn_sd):
    """The overlapped exchange's CNN bucket: one call, after res5.0's weight gradients are enqueued and before res4 recomputes,
    with the offset of res5's first parameter."""
    from clipbert_b200 import ops
    calls = []
    with recorded() as log:
        m, grid = _cnn_train(cnn_sd, bucket=lambda g, off, side: (calls.append(off), log.append(("bucket",))))
        n_fwd = len(log)
        grid.backward(torch.ones_like(grid))
    bb = m.feature.backbone
    assert calls == [bb.res5[0].shortcut._e["offset"]]
    bwd = log[n_fwd:]
    k = bwd.index(("bucket",))
    res4_conv1 = (ops.CB_GEMM_TN, None)
    before = [e for e in bwd[:k] if e[0] == "side"]
    assert len(before) == 4                     # grid_encoder + res5.2, res5.1, res5.0
    joins_before = [e for e in bwd[:k] if e[0] == "join"]
    assert not joins_before                     # res5's weight gradients may still run under the exchange's start
    assert any(e[0] == "gemm" and e[1] == res4_conv1[0] for e in bwd[k:])


# ------------------------------------------------------------------------------------------------ planted fault: dropout word
def test_recompute_with_the_next_steps_dropout_word_fails(weights, monkeypatch):
    """Planted fault: the recompute binds a different dropout word (the one the next step would draw) - its masks are not the
    forward's, and the comparison with the switch off must fail."""
    from clipbert_b200 import modeling, ops
    real = modeling._ClipBertHeadModel._recompute_layer

    def next_word(self, st, i, ly):
        word = st["drop_word"] + 1
        ops.dropout_offset_bind(word)
        try:
            return real(self, st, i, ly)
        finally:
            ops.dropout_offset_bind(st["drop_word"])
    with IGE.emulated_ops():
        monkeypatch.setattr(modeling._ClipBertHeadModel, "_recompute_layer", next_word)
        off, on = R.off_and_on(lambda: R.head_step(CPU, weights, "retrieval", gh=2, lt=8, counts=(1, 2), steps=1), cnn=False)
    with pytest.raises(AssertionError, match="differs with the switch on"):
        R.compare(off, on, True, "planted")


# ------------------------------------------------------------------------------------------------ data parallel, gloo
def _accumulated_step(weights, rank):
    """ClipBert retrieval (dropout 0.1) with the overlapped exchange and the mid-backward CNN bucket: two micro-steps under
    no_sync(), then one that exchanges; both flat gradient buffers after each micro-step."""
    from oracle import synth
    from test_zz2_gpu_round2 import _clipbert
    torch.manual_seed(0)
    model = _clipbert("ClipBertForVideoTextRetrieval", weights, CPU, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1).train()
    model.enable_overlapped_allreduce(cnn_buckets=True)
    out = []
    model.zero_grad()
    for micro in range(3):
        batch = synth.synth_batch(1, 2, n_ex=2, size=SIZE, seed=10 * rank + micro)
        with model.no_sync() if micro < 2 else contextlib.nullcontext():
            model(dict(batch))["loss"].mean().backward()
            model.allreduce_grads()
        out += [model.transformer._flat.grad.clone(), model.cnn._flat.grad.clone()]
    return out


def _no_sync_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from oracle import synth
        weights = synth.full_state_dict(42)
        runs = {}
        for on in (False, True):
            with IGE.emulated_ops(), R.recompute(on, on):
                runs[on] = _accumulated_step(weights, rank)
        same = [torch.equal(a, b) for a, b in zip(runs[False], runs[True])]
        q.put((rank, same, [float(t.double().abs().sum()) for t in runs[True]]))
    finally:
        dist.destroy_process_group()


def test_gloo_two_ranks_no_sync_accumulation_equals_switch_off():
    """Two ranks over gloo, each accumulating two micro-steps under no_sync() and exchanging on the third (overlapped exchange,
    CNN bucket after res5): with both switches on, every micro-step's accumulated buffers are the switch off's, bit for bit, and
    after the exchange both ranks hold the same buffers."""
    import os

    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() + 421) % 1000
    procs = [ctx.Process(target=_no_sync_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=1500) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, same, sums in res:
        assert all(same), (rank, same)
    (_, _, s0), (_, _, s1) = res
    assert s0[:4] != s1[:4]                  # the micro-steps under no_sync() accumulate each rank's own gradients
    assert s0[4:] == s1[4:]                  # the third exchanges: both ranks hold the mean
