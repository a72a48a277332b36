"""Deterministic mode (torch.use_deterministic_algorithms(True)): every accumulation of the library runs in a fixed order, so a
training step gives the same bits on every run.

Per kernel, with inputs for which the atomic order matters (K-splits, many blocks per column, repeated token ids, ragged repeat
counts) and outputs pre-filled with non-zero values: three runs are bit-identical, agree with a float64 restatement within the
op tolerance, and with the default (atomic) mode. Then invariance of the bits under the grid cap, the side queue, PDL and CUDA
graph replay, and two training steps of each head run twice from the same state."""
import contextlib
import os
import sys

import numpy as np
import pytest
import torch

from util import TOL_FP32_OP, make_cfg, relerr

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu
BF16, F32 = torch.bfloat16, torch.float32
# accumulation-order noise of one fp32 reduction over a few thousand bf16 terms, and of the LN / embedding backwards (their
# per-row arithmetic is fp32 with approximate rsqrt), relative to a float64 restatement
TOL_REDUCE = 1e-4


@contextlib.contextmanager
def deterministic(on=True):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _three_runs(fn):
    """fn() -> list of output tensors; run three times in deterministic mode, assert bit equality, return the first run."""
    runs = []
    for _ in range(3):
        with deterministic():
            runs.append([t.clone() for t in fn()])
    torch.cuda.synchronize()
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a, b), "deterministic mode gave different bits on a re-run"
    return runs[0]


# ---------------------------------------------------------------------------------------------------------------------------------
# weight-gradient GEMM
# ---------------------------------------------------------------------------------------------------------------------------------
def _wgrad_problem(cuda, m, n, p, ntaps=1, tap_w=0, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(p, m, generator=g).to(BF16).to(cuda)
    b = torch.randn(p, n, generator=g).to(BF16).to(cuda)
    out0 = torch.randn(m, ntaps * n, generator=g).to(cuda)          # accumulate semantics: out += dW
    ref = out0.double().cpu().clone()
    A, B = a.double().cpu(), b.double().cpu()
    for t in range(ntaps):
        shift = ((t // 3 - 1) * tap_w + (t % 3 - 1)) if ntaps == 9 else 0
        idx = torch.arange(p) + shift
        ok = (idx >= 0) & (idx < p)
        Bs = torch.zeros(p, n, dtype=torch.float64)
        Bs[ok] = B[idx[ok]]
        ref[:, t * n:(t + 1) * n] += A.t() @ Bs
    kw = dict(mode=1, m=m, n=n, k=p, a=a, a_rows=p, a_ld=m, b=b, b_rows=p, b_ld=n, ntaps=ntaps, tap_w=tap_w, tap_sign=1, out_ld=ntaps * n,
              out_fp32=1)
    return kw, out0, ref


@pytest.mark.parametrize("split_k", [1, 2, 3, 7, 0])
@pytest.mark.parametrize("block_n", [64, 128, 256])
def test_wgrad_gemm_bits(cuda, split_k, block_n):
    from clipbert_b200 import ops
    kw, out0, ref = _wgrad_problem(cuda, 200, 256, 2600, seed=split_k * 7 + block_n)      # m = 200: a ragged row tile

    def run():
        out = out0.clone()
        ops.gemm(**dict(kw, out=out, split_k=split_k, block_n=block_n))
        return [out]
    det = _three_runs(run)[0]
    with deterministic(False):
        dflt = run()[0]
    assert relerr(det, ref) < TOL_FP32_OP and relerr(det, dflt) < TOL_FP32_OP
    if split_k > 1:
        kw2 = dict(kw, out=out0.clone(), split_k=split_k, block_n=block_n)
        assert ops.gemm_workspace_bytes(kw2) == split_k * 200 * 256 * 4


@pytest.mark.parametrize("ntaps", [1, 9])
def test_wgrad_gemm_taps_bits(cuda, ntaps):
    """1-tap and 9-tap (3x3 conv / grid encoder) weight gradients over zero-bordered 14 x 14 images."""
    from clipbert_b200 import ops
    p = 4 * 16 * 16
    kw, out0, ref = _wgrad_problem(cuda, 128, 192, p, ntaps=ntaps, tap_w=16, seed=ntaps)

    def run():
        out = out0.clone()
        ops.gemm(**dict(kw, out=out, split_k=3))
        auto = out0.clone()
        ops.gemm(**dict(kw, out=auto))
        return [out, auto]
    det, auto = _three_runs(run)
    assert relerr(det, ref) < TOL_FP32_OP and relerr(auto, ref) < TOL_FP32_OP


@pytest.mark.parametrize("split_k", [0, 3])
def test_wgrad_group_bits(cuda, split_k):
    """The grouped launch (the four Linear layers of a BertLayer) with one and with three K-splits."""
    from clipbert_b200 import ops
    probs = [_wgrad_problem(cuda, m, n, 2624, seed=i) for i, (m, n) in enumerate([(768, 3072), (3072, 768), (768, 768), (2304, 768)])]

    def run():
        outs = [o.clone() for _, o, _ in probs]
        kws = [dict(kw, out=o) for (kw, _, _), o in zip(probs, outs)]
        kws[0]["split_k"] = split_k
        ops.gemm_wgrad_group(kws)
        return outs
    det = _three_runs(run)
    with deterministic(False):
        dflt = run()
    for d, f, (_, _, ref) in zip(det, dflt, probs):
        assert relerr(d, ref) < TOL_FP32_OP and relerr(d, f) < TOL_FP32_OP


def test_wgrad_without_workspace_is_an_error(cuda):
    from clipbert_b200 import _lib as L, ops
    kw, out0, _ = _wgrad_problem(cuda, 128, 128, 2048)
    d = ops._gemm_descs([dict(kw, out=out0, split_k=4)])
    prev = ops.set_deterministic(True)
    try:
        assert L.lib().cb_gemm(d, ops._s()) == -1
        assert b"workspace" in L.lib().cb_last_error()
        cs = torch.zeros(256, device=cuda)
        assert ops._fn("cb_colsum")(out0.data_ptr(), 256, cs.data_ptr(), 64, 256, ops._s()) == -1     # the atomic entry point refuses
    finally:
        ops.set_deterministic(prev)
        ops._lib_deterministic = prev


# ---------------------------------------------------------------------------------------------------------------------------------
# bias column sums, LayerNorm / embedding parameter gradients, word-table scatter, sumsq, loss scalars
# ---------------------------------------------------------------------------------------------------------------------------------
def test_colsum_bits(cuda):
    from clipbert_b200 import ops
    g = torch.Generator().manual_seed(1)
    x = torch.randn(5000, 2304, generator=g).to(BF16).to(cuda)        # 40 slabs per column
    out0 = torch.randn(2304, generator=g).to(cuda)
    ref = out0.double().cpu() + x.double().cpu().sum(0)

    def run():
        out = out0.clone()
        ops.colsum(x, out, 5000, 2304)
        return [out]
    det = _three_runs(run)[0]
    assert relerr(det, ref) < TOL_FP32_OP


def _cpu(*ts):
    return [None if t is None else t.detach().cpu().clone() for t in ts]


def test_layernorm_bwd_bits(cuda):
    import ops_emulator as E
    from clipbert_b200 import ops
    g = torch.Generator().manual_seed(2)
    m = 3000                                    # 264 blocks, several rows per warp
    x = torch.randn(m, 768, generator=g).to(BF16).to(cuda)
    gamma = (1 + 0.1 * torch.randn(768, generator=g)).to(cuda)
    beta = (0.1 * torch.randn(768, generator=g)).to(cuda)
    y = torch.empty_like(x)
    stats = torch.empty(m, 2, device=cuda)
    ops.layernorm_fwd(x, gamma, beta, y, stats, 1e-12)
    dy = torch.randn(m, 768, generator=g).to(BF16).to(cuda)
    pre = [torch.randn(768, generator=g).to(cuda) for _ in range(3)]

    def run(fn=ops.layernorm_bwd, tensors=(dy, x, stats, gamma)):
        dx, dxd = torch.empty(m, 768, dtype=BF16, device=tensors[0].device), torch.empty(m, 768, dtype=BF16, device=tensors[0].device)
        acc = [t.clone().to(tensors[0].device) for t in pre]
        fn(*tensors, dx, dxd, acc[0], acc[1], acc[2], 0.1, 77)
        return [dx, dxd] + acc
    det = _three_runs(run)
    ref = run(E.layernorm_bwd, _cpu(dy, x, stats, gamma))
    for d, r in zip(det[2:], ref[2:]):
        assert relerr(d, r) < TOL_REDUCE
    assert relerr(det[0], ref[0]) < 4e-3


def _embed_text_case(cuda, same_ids):
    from clipbert_b200 import ops
    g = torch.Generator().manual_seed(3)
    nseq, lt, L, V = 64, 20, 29, 1000
    ids = torch.randint(0, V, (nseq, lt), generator=g)
    if same_ids:
        ids[:] = ids[0]                          # the same ids in every sequence: every table row has 64 writers
    ids[:, 0], ids[:, -1] = 101, 102             # [CLS] / [SEP]
    ids = ids.to(cuda)
    word, pos, typ = (0.02 * torch.randn(V, 768, generator=g)).to(cuda), (0.02 * torch.randn(64, 768, generator=g)).to(cuda), \
        (0.02 * torch.randn(2, 768, generator=g)).to(cuda)
    gamma, beta = (1 + 0.1 * torch.randn(768, generator=g)).to(cuda), (0.1 * torch.randn(768, generator=g)).to(cuda)
    out = torch.zeros(nseq * L, 768, dtype=BF16, device=cuda)
    stats = torch.empty(nseq * lt, 2, device=cuda)
    ops.embed_text_fwd(ids, word, pos, typ, gamma, beta, out, stats, nseq, lt, L, 1e-12, 0.1, 5)
    dh = torch.randn(nseq * L, 768, generator=g).to(BF16).to(cuda)
    pre = [torch.randn(*s, generator=g).to(cuda) for s in ((V, 768), (64, 768), (2, 768), (768,), (768,))]
    return dict(args=(dh, ids, word, pos, typ, gamma, stats), pre=pre, dims=(nseq, lt, L))


@pytest.mark.parametrize("same_ids", [False, True])
def test_embed_text_bwd_bits(cuda, same_ids):
    import ops_emulator as E
    from clipbert_b200 import ops
    c = _embed_text_case(cuda, same_ids)

    def run(fn=ops.embed_text_bwd, args=c["args"]):
        acc = [t.clone().to(args[0].device) for t in c["pre"]]
        fn(*args, *acc, *c["dims"], 0.1, 5)
        return acc
    det = _three_runs(run)
    ref = run(E.embed_text_bwd, _cpu(*c["args"]))
    with deterministic(False):
        dflt = run()
    for d, r, f in zip(det, ref, dflt):
        assert relerr(d, r) < TOL_REDUCE and relerr(d, f) < TOL_REDUCE


@pytest.mark.parametrize("counts,gh", [([4] * 16, 3), ([1, 3, 2, 7, 1, 5, 2, 3], 7)])
def test_embed_visual_bwd_bits(cuda, counts, gh):
    """Uniform and ragged repeat counts (seq2vid / vid_start), 3 x 3 and 7 x 7 grids, many blocks per cell."""
    import ops_emulator as E
    from clipbert_b200 import ops
    g = torch.Generator().manual_seed(4)
    nvid, T, lt = len(counts), 2, 12
    nseq, L = sum(counts), lt + gh * gh
    uniform = len(set(counts)) == 1
    s2v = None if uniform else torch.tensor(np.repeat(np.arange(nvid), counts), dtype=torch.int32).to(cuda)
    starts = None if uniform else torch.tensor(np.concatenate([[0], np.cumsum(counts)]), dtype=torch.int32).to(cuda)
    n_ex = counts[0] if uniform else 0
    grid = torch.randn(nvid, T, gh, gh, 768, generator=g).abs().to(BF16).to(cuda)
    row, col, typ = ((0.02 * torch.randn(r, 768, generator=g)).to(cuda) for r in (gh, gh, 2))
    gamma, beta = (1 + 0.1 * torch.randn(768, generator=g)).to(cuda), (0.1 * torch.randn(768, generator=g)).to(cuda)
    out = torch.zeros(nseq * L, 768, dtype=BF16, device=cuda)
    stats = torch.empty(nseq * gh * gh, 2, device=cuda)
    ops.embed_visual_fwd(grid, s2v, n_ex, row, col, typ, gamma, beta, out, stats, nseq, T, gh, gh, lt, L, 1e-12, 0.1, 9)
    dh = torch.randn(nseq * L, 768, generator=g).to(BF16).to(cuda)
    pre = [torch.randn(*s, generator=g).to(cuda) for s in ((gh, 768), (gh, 768), (2, 768), (768,), (768,))]
    tensors = (dh, grid, s2v, starts, n_ex, row, col, typ, gamma, stats)

    def run(fn=ops.embed_visual_bwd, ts=tensors):
        dev = ts[0].device
        dv_tmp = torch.empty(nseq * gh * gh, 768, device=dev)
        dgrid = torch.empty(nvid, T, gh, gh, 768, dtype=BF16, device=dev)
        acc = [t.clone().to(dev) for t in pre]
        fn(*ts, dv_tmp, dgrid, *acc, nseq, nvid, T, gh, gh, lt, L, 0.1, 9)
        return [dgrid] + acc
    det = _three_runs(run)
    ref = run(E.embed_visual_bwd, tuple(t if not torch.is_tensor(t) else t.cpu() for t in tensors))
    for d, r in zip(det[1:], ref[1:]):
        assert relerr(d, r) < TOL_REDUCE
    assert relerr(det[0], ref[0]) < 4e-3


def test_sumsq_and_clip_loss_bits(cuda):
    from clipbert_b200 import ops, optim
    g = torch.Generator().manual_seed(6)
    x = torch.randn(3_000_000, generator=g).to(cuda)
    rows = [[o, min(65536, 3_000_000 - o), 0, 0, -1, 0, 0, 0] for o in range(0, 3_000_000, 65536)]
    chunks = torch.tensor(rows, dtype=torch.int64, device=cuda)
    z = torch.randn(2, 600, 5, generator=g).to(cuda)           # 600 examples: three loss blocks
    y = torch.randint(0, 5, (600,), generator=g).to(cuda)

    def run():
        o1 = torch.full((1,), 3.0, device=cuda)
        optim.sumsq(x, chunks, len(rows), o1)
        o2 = torch.full((1,), 3.0, device=cuda)
        ops.sumsq_det(x, x.numel(), None, 0, o2, ops._scratch(ops.sumsq_scratch_bytes(x.numel(), None, 0), x))
        outs = [o1, o2]
        for pool in (0, 1, 2):
            loss, dz = torch.empty(1, device=cuda), torch.empty_like(z)
            if pool == 0:
                ops.clip_lse_loss(z, y, loss, dz, 2, 600, 5)
            else:
                ops.clip_pool_ce_loss(z, y, loss, dz, 2, 600, 5, pool)
            outs += [loss, dz]
        return outs
    det = _three_runs(run)
    ss = float((x.double() ** 2).sum()) + 3.0
    assert abs(float(det[0]) / ss - 1) < TOL_FP32_OP and abs(float(det[1]) / ss - 1) < TOL_FP32_OP
    zl = z.double().cpu().permute(1, 0, 2)
    lse = torch.logsumexp(zl.reshape(600, -1), -1) - torch.logsumexp(zl[torch.arange(600), :, y.cpu()], -1)
    assert abs(float(det[2]) / float(lse.mean()) - 1) < TOL_FP32_OP


# ---------------------------------------------------------------------------------------------------------------------------------
# invariance: grid cap, side queue, PDL, CUDA-graph replay
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)


def _retrieval_transformer(weights, cuda, p=0.1):
    from test_gpu_model import _build
    model = _build("ClipBertForVideoTextRetrieval", weights, cuda).train()
    tr = model.transformer
    tr.config.hidden_dropout_prob = tr.config.attention_probs_dropout_prob = p
    return model


def _zero_flat_grad(engine):
    """zero an engine's flat gradient buffer (it exists once the engine has run a forward)"""
    f = getattr(engine, "_flat", None)
    if f is not None:
        f.attach_grads()
        f.grad.zero_()


def _transformer_step(model, cuda, gh=3, lt=20, seed=1):
    """forward + backward of the retrieval head on a fixed synthetic grid -> [loss, flat transformer gradient, d grid]"""
    from oracle import synth
    g = torch.Generator().manual_seed(seed)
    grid = torch.randn(4, 1, gh, gh, 768, generator=g).abs().to(BF16).float().to(cuda).requires_grad_(True)
    ids, mask = synth.synth_text(8, lt, seed=seed)
    labels = torch.tensor([1, 0] * 4)
    _zero_flat_grad(model.transformer)
    out = model.transformer(ids.to(cuda), grid, mask.to(cuda), labels=labels.to(cuda), _repeat_counts=[2] * 4)
    out["loss"].mean().backward()
    return [out["loss"].detach(), model.transformer._flat.grad, grid.grad]


def test_bits_do_not_depend_on_grid_cap_side_queue_or_pdl(cuda, weights):
    from clipbert_b200 import ops
    runs = {}
    settings = [("base", {}), ("sm_limit_66", dict(sm=66)), ("no_overlap", dict(overlap=False)), ("pdl1", dict(pdl=1)),
                ("pdl2", dict(pdl=2))]
    for name, s in settings:
        torch.manual_seed(0)
        model = _retrieval_transformer(weights, cuda)
        ops.set_sm_limit(s.get("sm", 0))
        prev_overlap, ops.overlap_wgrad = ops.overlap_wgrad, s.get("overlap", True)
        prev_pdl = ops.set_pdl(s.get("pdl", 0))
        try:
            with deterministic():
                runs[name] = [t.clone() for t in _transformer_step(model, cuda)]
            torch.cuda.synchronize()
        finally:
            ops.set_sm_limit(0)
            ops.overlap_wgrad = prev_overlap
            ops.set_pdl(prev_pdl)
    for name, r in runs.items():
        for a, b in zip(runs["base"], r):
            assert torch.equal(a, b), name


def test_graph_replay_gives_the_eager_bits(cuda):
    """A captured sequence of deterministic accumulations (split weight gradient, group, column sums, LayerNorm backward)
    replays to the bits of the eager run."""
    from clipbert_b200 import ops
    kw, out0, _ = _wgrad_problem(cuda, 768, 768, 2600, seed=11)
    g = torch.Generator().manual_seed(12)
    x = torch.randn(3000, 768, generator=g).to(BF16).to(cuda)
    stats = torch.empty(3000, 2, device=cuda)
    gamma = torch.ones(768, device=cuda)
    y = torch.empty_like(x)
    ops.layernorm_fwd(x, gamma, gamma * 0, y, stats, 1e-12)
    outs = [out0.clone(), torch.zeros(768, device=cuda), torch.zeros(768, device=cuda), torch.zeros(768, device=cuda)]
    dx = torch.empty_like(x)

    def body():
        ops.gemm(**dict(kw, out=outs[0], split_k=5))
        ops.colsum(x, outs[1], 3000, 768)
        ops.layernorm_bwd(x, y, stats, gamma, dx, None, outs[2], outs[3], None, 0.0, 0)

    def reset():
        outs[0].copy_(out0)
        for t in outs[1:]:
            t.zero_()
    with deterministic():
        reset()
        body()
        eager = [t.clone() for t in outs]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):          # warm-up on a side stream, as torch.cuda.graphs asks
            reset()
            body()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            body()
        for _ in range(2):
            reset()
            graph.replay()
            torch.cuda.synchronize()
            for a, b in zip(eager, outs):
                assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------------------
# model level: two training steps from the same state, twice
# ---------------------------------------------------------------------------------------------------------------------------------
def _assert_same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), "output %d differs between two deterministic runs" % i
        assert bool(torch.isfinite(x.float()).all()), "output %d is not finite" % i


def _clipbert_retrieval_run(weights, cuda, toggle=False):
    """ClipBert retrieval, dropout 0.1, forward_clips + clip_lse_loss + FusedAdamW (clip + step), two steps."""
    import clipbert_b200 as cb
    from clipbert_b200 import ops
    from clipbert_b200.optim import FusedAdamW
    from oracle import synth
    from test_gpu_optim import e2e_param_groups
    torch.manual_seed(0)
    model = _retrieval_transformer(weights, cuda)
    opt = FusedAdamW([g for g in e2e_param_groups(model) if g["params"]], lr=5e-5, betas=(0.9, 0.98), model=model)
    batch = synth.synth_batch(2, 4, n_ex=2, size=224, seed=9)
    res, modes = [], []
    for step in range(2):
        on = not (toggle and step == 1)
        with deterministic(on):
            model.zero_grad()
            mb = {k: (v.to(cuda) if torch.is_tensor(v) else list(v)) for k, v in batch.items()}
            logits = model.forward_clips(mb, 2)["logits"]
            loss = cb.clip_lse_loss(logits, batch["labels"].to(cuda))
            loss.backward()
            gn = opt.clip_grad_norm(1.0)
            grads = [m._flat.grad.clone() for m in (model.transformer, model.cnn) if getattr(m, "_flat", None) is not None and m._flat.grad is not None]
            opt.step()
            modes.append(ops._lib_deterministic)
        res += [loss.detach().clone(), gn.clone()] + grads
    for h in opt._plan:
        res += [h["flat"].master.clone(), h["exp_avg"].clone(), h["exp_avg_sq"].clone()]
    torch.cuda.synchronize()
    return res, modes


def test_clipbert_retrieval_training_steps_repeat_bit_for_bit(cuda, weights):
    a, modes = _clipbert_retrieval_run(weights, cuda)
    b, _ = _clipbert_retrieval_run(weights, cuda)
    assert modes == [True, True]
    _assert_same(a, b)


def test_toggling_the_flag_between_steps_switches_the_mode(cuda, weights):
    a, modes = _clipbert_retrieval_run(weights, cuda, toggle=True)
    assert modes == [True, False]
    b, _ = _clipbert_retrieval_run(weights, cuda)
    _assert_same(a[:4], b[:4])           # the first (deterministic) step is the same; the second used the atomics


def test_pretraining_with_sampled_visual_tokens_repeats_bit_for_bit(cuda, weights):
    """ClipBertForPreTraining with pixel_random_sampling_size and MLM labels: the tied word table gets two writers (decoder
    weight gradient and the embedding scatter) and the sampled tokens go through index_add_."""
    from oracle import synth
    from test_zz_gpu_round1c import _pretraining_model
    g = torch.Generator().manual_seed(5)
    grid0 = torch.randn(2, 2, 4, 5, 768, generator=g).abs().bfloat16()
    ids, mask = synth.synth_text(4, 12, seed=9)
    mlm = torch.full((4, 12), -100, dtype=torch.long)
    mlm[:, 3], mlm[:, 7] = ids[:, 3], ids[:, 7]
    itm = torch.tensor([1, 1, 1, 0])

    def run():
        torch.manual_seed(0)
        model, _ = _pretraining_model(weights, cuda, pixel_random_sampling_size=7)
        model.config.hidden_dropout_prob = model.config.attention_probs_dropout_prob = 0.1
        model.train()
        res = []
        with deterministic():
            for step in range(2):
                _zero_flat_grad(model)
                grid = grid0.clone().to(cuda).requires_grad_(True)
                np.random.seed(77 + step)
                out = model(ids.to(cuda), grid, mask.to(cuda), mlm_labels=mlm.to(cuda), itm_labels=itm.to(cuda), _repeat_counts=[2, 2])
                loss = out["mlm_loss"].sum() / 8 + out["itm_loss"].mean()
                loss.backward()
                res += [loss.detach().clone(), model._flat.grad.clone(), grid.grad.clone()]
        torch.cuda.synchronize()
        return res
    _assert_same(run(), run())


def test_multiple_choice_repeats_bit_for_bit(cuda, weights):
    from oracle import synth
    from test_gpu_model import _build
    sd = dict(weights)
    sd.update(synth.transformer_state_dict(50, num_labels=1))
    g = torch.Generator().manual_seed(4)
    grid0 = torch.randn(2, 1, 3, 3, 768, generator=g).abs().to(BF16).float()
    ids, mask = synth.synth_text(10, 25, seed=5)
    labels = torch.tensor([1, 4])

    def run():
        torch.manual_seed(0)
        model = _build("ClipBertForMultipleChoice", sd, cuda, num_labels=5).train()
        model.transformer.config.hidden_dropout_prob = 0.1
        res = []
        with deterministic():
            for _ in range(2):
                tr = model.transformer
                _zero_flat_grad(tr)
                grid = grid0.clone().to(cuda).requires_grad_(True)
                out = tr(ids.to(cuda), grid, mask.to(cuda), labels=labels.to(cuda), _repeat_counts=[5, 5])
                out["loss"].mean().backward()
                res += [out["loss"].detach().clone(), tr._flat.grad.clone(), grid.grad.clone()]
        torch.cuda.synchronize()
        return res
    _assert_same(run(), run())


def test_base_model_with_hidden_states_repeats_bit_for_bit(cuda, weights):
    import clipbert_b200 as cb
    from oracle import synth
    g = torch.Generator().manual_seed(8)
    grid0 = torch.randn(4, 1, 3, 3, 768, generator=g).abs().to(BF16).float()
    ids, mask = synth.synth_text(4, 16, seed=3)

    def run():
        torch.manual_seed(0)
        cfg = make_cfg(hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1, output_hidden_states=True)
        bert = cb.ClipBertBaseModel(cfg).to(cuda).train()
        res = []
        with deterministic():
            for _ in range(2):
                bert.zero_grad()
                grid = grid0.clone().to(cuda).requires_grad_(True)
                out = bert(ids.to(cuda), grid, mask.to(cuda))
                seq, pooled, hidden = out[0], out[1], out[2]
                loss = seq.float().square().mean() + pooled.float().sum() + hidden[5].float().mean()
                loss.backward()
                res += [loss.detach().clone(), grid.grad.clone()] + [p.grad.clone() for p in bert.parameters() if p.grad is not None]
        torch.cuda.synchronize()
        return res
    _assert_same(run(), run())


def test_long_sequence_step_repeats_bit_for_bit(cuda, weights):
    """L = 20 + 49 = 69 > 64: the long-sequence attention kernels in the step."""
    def run():
        torch.manual_seed(0)
        model = _retrieval_transformer(weights, cuda)
        with deterministic():
            r = [t.clone() for t in _transformer_step(model, cuda, gh=7)]
        torch.cuda.synchronize()
        return r
    _assert_same(run(), run())
