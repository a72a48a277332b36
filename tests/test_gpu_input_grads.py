"""Gradients with respect to the input frames: d score / d frames through the grid encoder, every ResNet block (frozen ones
too), the stem max pool + ReLU and the stem convolution, as the reference gets them from autograd (d2's FREEZE_AT and
freeze_cnn_backbone set requires_grad = False on parameters and detach no activation, src/modeling/grid_feat.py:89-105).

Kernels, element by element against float64 from the launch's own bf16 inputs (the error model of
tests/test_gpu_cnn_elementwise.py, U = 2^-24), each output between NaN guard bands that must stay untouched:
  cb_maxpool3x3s2_bwd[_strided]  F.max_pool2d's arg-max (first maximum, last NaN) of the pool input, the window gradients that
                                  pick an element summed, ReLU' = (x > 0): bit-exact where at most one window picks the element,
                                  else 3 U sum|dy| (three fp32 adds) + 1 ulp_bf16 of the result;
  cb_stem_dgrad                   torch.nn.grad.conv2d_input in float64 on the stem operand _stem_w reshaped to [64, 3, 7, 7]
                                  (BGR input channels), flipped back to RGB: 3 n U conv(|dc1|, |w|) with n = 16 taps x 64
                                  channels, + U |v| for the fp32 result.
Module: GridFeatBackbone's frame gradient against the oracle's fp32 autograd called with freeze_at = 0 and weights that do not
require grad, so it detaches nothing, differentiating along the run's ReLU patterns and max-pool selections (the stem's too:
the ReLU net's gradient is discontinuous in its activation pattern, see oracle Rounding.relu_masks). End to end: the same
through ClipBert.forward, forward_clips and encode_clips + forward_clips(grid=...) on the retrieval head.

Every element-wise check prints "RATIO <kernel> <case> <max err / bound>". tests/test_input_grads_emulated.py replays the module
and end-to-end cases that fit a CPU on the emulated ops and shows the kernel checks reject planted faults.
"""
import contextlib

import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input

from elementwise import BF16, F32, F64, U, Guarded, _record, check_bound, ulp_bf16
from model_util import cnn_patterns
from util import TOL_GRAD, cosine, make_cfg, relerr

FTZ = 2.0 ** -126
PIXEL_STD = (58.395, 57.12, 57.375)
STEM_TERMS = 16 * 64          # taps x channels of one stem input gradient element


@contextlib.contextmanager
def _deterministic(on=True):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(bool(on))
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.int16 if t.dtype in (BF16, torch.float16) else torch.int32)


# ------------------------------------------------------------------------------------------------ kernel references
def pool_bwd_ref(dy, x):
    """dy: [n, ho, wo, c], x: the pool input [n, h, w, c] (bf16). float64 NHWC value and bound of the bf16 result: the sum of the
    window gradients whose F.max_pool2d(3, 2, 1) arg-max is the element, kept where x > 0; bound 0 (bit-exact) where at most one
    window picks it."""
    x64 = x.detach().cpu().double().permute(0, 3, 1, 2)
    n, c, h, w = x64.shape
    _, idx = F.max_pool2d(x64, 3, 2, 1, return_indices=True)
    idx = idx.flatten(2)
    d = dy.detach().cpu().double().permute(0, 3, 1, 2).flatten(2)

    def scatter(v):
        return torch.zeros(n, c, h * w, dtype=F64).scatter_add_(2, idx, v).view(n, c, h, w)
    v, T, cnt = scatter(d), scatter(d.abs()), scatter(torch.ones_like(d))
    keep = x64 > 0
    v = torch.where(keep, v, torch.zeros_like(v))
    bound = torch.where(keep & (cnt > 1), 3 * U * T + ulp_bf16(v) + FTZ, torch.zeros_like(v))
    return v.permute(0, 2, 3, 1), bound.permute(0, 2, 3, 1)


def stem_weight64(w):
    """The stem operand [64, >= 147] (columns (r, s, c), c in BGR order) as a float64 [64, 3, 7, 7] convolution weight."""
    return w[:, :147].detach().cpu().double().reshape(64, 7, 7, 3).permute(0, 3, 1, 2)


def stem_dgrad_ref(dc1, w, n, h, wimg):
    """float64 RGB NCHW value and bound of cb_stem_dgrad: the 7x7/s2/p3 input gradient of the BGR frames, flipped back."""
    ho, wo = (h - 1) // 2 + 1, (wimg - 1) // 2 + 1
    wk = stem_weight64(w)
    d = dc1.detach().cpu().double().reshape(n, ho, wo, 64).permute(0, 3, 1, 2)
    v = conv2d_input((n, 3, h, wimg), wk, d, stride=2, padding=3)
    T = conv2d_input((n, 3, h, wimg), wk.abs(), d.abs(), stride=2, padding=3)
    return v[:, [2, 1, 0]], (3 * STEM_TERMS * U * T + U * v.abs() + FTZ)[:, [2, 1, 0]]


# ------------------------------------------------------------------------------------------------ kernel inputs
def pool_inputs(n, h, w, seed, c=64):
    """A post-ReLU-like pool input with many equal bf16 maxima (a few levels), all-zero windows, -0 and one NaN, and its dy."""
    g = torch.Generator().manual_seed(seed)
    x = (torch.randint(-3, 5, (n, h, w, c), generator=g).double() * 0.5).clamp_min(0.0)
    x[:, : min(h, 5), : min(w, 5)] = 0.0                              # all-zero windows
    neg0 = torch.rand(n, h, w, c, generator=g) < 0.05
    x = torch.where(neg0 & (x == 0), torch.full_like(x, -0.0), x)
    x[0, h // 2, w // 2, 3] = float("nan")
    dy = torch.randn(n, (h - 1) // 2 + 1, (w - 1) // 2 + 1, c, generator=g).to(BF16)
    return dy, x.to(BF16)


def stem_operand(dev, pixel_std=None):
    """A real stem operand (_stem_w: FrozenBN scale folded in, and 1 / std with pixel_std)."""
    import clipbert_b200 as cb
    from oracle import synth
    m = cb.GridFeatBackbone()
    m.load_state_dict(synth.cnn_state_dict(42))
    m = m.to(dev)
    if pixel_std is not None:
        from clipbert_b200 import input_stage
        from clipbert_b200.workload import IMAGE_MEAN
        input_stage.set_image_norm(m, IMAGE_MEAN, pixel_std)
    m._ensure_ready(torch.device(dev))
    return m._stem_w


def dc1_input(n, ho, wo, seed):
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(n * ho * wo, 64, generator=g)
    return torch.where(torch.rand(n * ho * wo, 64, generator=g) < 0.4, torch.zeros_like(d), d).to(BF16)


POOL_CASES = [(2, 224, False), (2, 200, False), (2, 160, False), (1, 97, False), (3, 33, False), (2, 224, True), (1, 97, True),
              (2, 33, True)]
STEM_CASES = [(2, 224, False), (2, 224, True), (2, 200, False), (2, 160, True), (1, 448, False), (1, 224, False), (1, 97, True)]


def _conv_out(size):
    return (size - 1) // 2 + 1


def run_pool_bwd(dev, n, size, strided, seed):
    """One launch (the strided form reads x on the s2d stem's (h+3) x (w+3) grid, NaN outside the image). Returns (dx, ref, bound)."""
    from clipbert_b200 import ops
    h = w = _conv_out(size)
    dy, x = pool_inputs(n, h, w, seed)
    out = Guarded((n * h * w, 64), BF16, dev)
    if strided:
        grid = torch.full((n, h + 3, w + 3, 64), float("nan"), dtype=BF16)
        grid[:, :h, :w] = x
        ops.maxpool3x3s2_bwd(dy.to(dev), grid.to(dev), out.t, n, h, w, 64, row_pitch=w + 3, img_pitch=(h + 3) * (w + 3))
    else:
        ops.maxpool3x3s2_bwd(dy.to(dev), x.to(dev), out.t, n, h, w, 64)
    ref, bound = pool_bwd_ref(dy, x)
    return out, ref, bound


def run_stem_dgrad(dev, n, size, std, seed):
    from clipbert_b200 import ops
    w = stem_operand(dev, PIXEL_STD if std else None)
    ho = _conv_out(size)
    dc1 = dc1_input(n, ho, ho, seed).to(dev)
    out = Guarded((n, 3, size, size), F32, dev)
    ops.stem_dgrad(dc1, w, out.t, n, size, size)
    ref, bound = stem_dgrad_ref(dc1, w, n, size, size)
    return out, ref, bound, (dc1, w)


def _pool_id(c):
    return "%dx%d%s" % (c[0], c[1], "-strided" if c[2] else "")


def _stem_id(c):
    return "%dx%d%s" % (c[0], c[1], "-std" if c[2] else "")


@pytest.mark.gpu
@pytest.mark.parametrize("case", POOL_CASES, ids=[_pool_id(c) for c in POOL_CASES])
def test_maxpool3x3s2_bwd_elementwise(cuda, case):
    n, size, strided = case
    out, ref, bound = run_pool_bwd(cuda, n, size, strided, seed=size + n)
    torch.cuda.synchronize()
    out.check("cb_maxpool3x3s2_bwd " + _pool_id(case))
    h = _conv_out(size)
    r = check_bound("cb_maxpool3x3s2_bwd " + _pool_id(case), out.t.view(n, h, h, 64), ref, bound)
    _record("cb_maxpool3x3s2_bwd", _pool_id(case), r)
    # the case has both kinds of element: picked by one window (bit-exact) and by several (sum)
    assert bool((bound == 0).any()) and bool((bound > 0).any())


@pytest.mark.gpu
@pytest.mark.parametrize("case", STEM_CASES, ids=[_stem_id(c) for c in STEM_CASES])
def test_stem_dgrad_elementwise(cuda, case):
    n, size, std = case
    out, ref, bound, _ = run_stem_dgrad(cuda, n, size, std, seed=7 * size + n)
    torch.cuda.synchronize()
    out.check("cb_stem_dgrad " + _stem_id(case))
    r = check_bound("cb_stem_dgrad " + _stem_id(case), out.t, ref, bound)
    _record("cb_stem_dgrad", _stem_id(case), r)


@pytest.mark.gpu
def test_input_grad_kernels_are_reproducible(cuda):
    """The same inputs give the same bits on every run, with torch's deterministic flag and without."""
    from clipbert_b200 import ops
    runs = []
    for det in (False, True, False):
        with _deterministic(det):
            out, _, _ = run_pool_bwd(cuda, 2, 200, True, seed=5)
            s_out, _, _, (dc1, w) = run_stem_dgrad(cuda, 2, 200, True, seed=6)
            again = torch.empty_like(s_out.t)
            ops.stem_dgrad(dc1, w, again, 2, 200, 200)
            torch.cuda.synchronize()
            runs.append((_bits(out.t), _bits(s_out.t), _bits(again)))
    for a in runs[1:]:
        for x, y in zip(runs[0], a):
            assert torch.equal(x, y)
    assert torch.equal(runs[0][1], runs[0][2])


# ------------------------------------------------------------------------------------------------ module against the oracle
class ModuleCase:
    def __init__(self, videos, frames, size, stem="s2d16", freeze_at=2, inputs="float"):
        self.videos, self.frames, self.size, self.stem, self.freeze_at, self.inputs = videos, frames, size, stem, freeze_at, inputs
        self.id = "%dx%dx%d-%s-fa%d-%s" % (videos, frames, size, stem, freeze_at, inputs)

    @property
    def pixels(self):
        return self.videos * self.frames * self.size * self.size


MODULE_CASES = [ModuleCase(2, 2, 224), ModuleCase(2, 2, 224, stem="s2d64"), ModuleCase(2, 2, 224, stem="im2col"),
                ModuleCase(1, 1, 448), ModuleCase(1, 2, 200, freeze_at=1, inputs="raw"), ModuleCase(1, 2, 200, "im2col", 3, "bf16"),
                ModuleCase(2, 1, 224, freeze_at=3, inputs="raw"), ModuleCase(1, 2, 224, "im2col", 1, "bf16"),
                ModuleCase(1, 2, 200, "s2d64", 2, "raw")]


def stem_patterns(stash):
    """The run's stem ReLU pattern and max-pool selection (NCHW, CPU) from the stash of a forward whose frames required grad."""
    fr = stash["frames"]
    n, ho, wo = stash["n"], fr["ho"], fr["wo"]
    c1 = fr["c1"].view(n, -1, fr["pitch"][0] or wo, 64)[:, :ho, :wo] if fr["pitch"][0] else fr["c1"].view(n, ho, wo, 64)
    c1 = c1.float().permute(0, 3, 1, 2).cpu()
    return c1 > 0, F.max_pool2d(c1, 3, 2, 1, return_indices=True)[1]


@contextlib.contextmanager
def oracle_stem(mask, idx):
    """The oracle's BasicStem differentiated along the run's ReLU pattern and max-pool selection (oracle/ is not edited: its
    resnet50_res5 looks basic_stem up at call time)."""
    from oracle import clipbert_ref as R
    orig = R.basic_stem

    def basic_stem(x, sd, prefix, rnd=R.EXACT):
        z = R.conv_bn(rnd.act(x), sd, prefix + "conv1.", stride=2, padding=3, rnd=rnd)
        z = rnd.act(z * mask.to(z.dtype))
        n, c = z.shape[:2]
        return z.flatten(2).gather(2, idx.flatten(2)).view(n, c, idx.shape[2], idx.shape[3])
    R.basic_stem = basic_stem
    try:
        yield
    finally:
        R.basic_stem = orig


def _frames(case, seed):
    """(frames handed to the module, the oracle's normalised fp32 input as a function of the same CPU leaf, the leaf)."""
    from oracle import synth
    from clipbert_b200.workload import IMAGE_MEAN
    if case.inputs == "raw":
        raw = synth.synth_images(case.videos, case.frames, size=case.size, seed=seed, as_uint8=True).float()
        leaf = raw.clone().requires_grad_(True)
        mean = torch.tensor(IMAGE_MEAN).view(1, 1, 3, 1, 1)
        std = torch.tensor(PIXEL_STD).view(1, 1, 3, 1, 1)
        return raw, leaf, lambda: (leaf - mean) / std
    x = synth.synth_images(case.videos, case.frames, size=case.size, seed=seed)
    if case.inputs == "bf16":
        x = x.to(BF16)
    leaf = x.clone().requires_grad_(True)
    return x, leaf, lambda: leaf.float()


def backbone(dev, case, sd):
    import clipbert_b200 as cb
    m = cb.GridFeatBackbone(freeze_at=case.freeze_at)
    assert not m.load_state_dict(sd).missing_keys
    m = m.to(dev)
    m.stem_mode = "im2col" if case.stem == "im2col" else "s2d"
    m._s2d_ld = 64 if case.stem == "s2d64" else 16
    if case.inputs == "raw":
        from clipbert_b200 import input_stage
        from clipbert_b200.workload import IMAGE_MEAN
        input_stage.set_image_norm(m, IMAGE_MEAN, PIXEL_STD)
    return m


def run_module_against_oracle(dev, case, sd):
    """d <grid, dgrid> / d frames of GridFeatBackbone against the oracle's fp32 autograd. Returns (relerr, cosine)."""
    from oracle import clipbert_ref as R
    m = backbone(dev, case, sd)
    x, leaf, oracle_in = _frames(case, seed=case.size + case.frames)
    xd = x.to(dev).requires_grad_(True)
    m._capture = {}
    grid = m(xd)
    stash = m._capture["stash"]
    m._capture = None
    dgrid = torch.randn(grid.shape, generator=torch.Generator().manual_seed(3)).to(BF16)
    (dx,) = torch.autograd.grad(grid, xd, dgrid.to(dev))
    assert dx.dtype == xd.dtype and dx.shape == xd.shape
    pat = cnn_patterns(stash, grid)
    with oracle_stem(*stem_patterns(stash)), torch.enable_grad():
        ref = R.grid_feat_backbone(oracle_in(), sd, freeze_at=0, rnd=pat)
        ref.backward(dgrid.float())
    e, c = relerr(dx, leaf.grad), cosine(dx, leaf.grad)
    print("RELERR module %s relerr %.3g cosine %.6f" % (case.id, e, c))
    assert e < TOL_GRAD and c > 0.999, (case.id, e, c)
    assert all(p.grad is None for p in m.parameters() if not p.requires_grad)
    return e, c


@pytest.fixture(scope="module")
def cnn_sd():
    from oracle import synth
    return synth.cnn_state_dict(42)


@pytest.mark.gpu
@pytest.mark.parametrize("case", MODULE_CASES, ids=[c.id for c in MODULE_CASES])
def test_backbone_frame_gradient_matches_oracle(cuda, cnn_sd, case):
    run_module_against_oracle(cuda, case, cnn_sd)


# ------------------------------------------------------------------------------------------------ end to end
E2E_PATHS = ("forward", "forward_clips", "encode_clips")


def clipbert(dev, sd, frozen):
    import clipbert_b200 as cb
    model = cb.ClipBert(make_cfg(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0), detectron2_model_cfg="R-50-grid.yaml")
    assert not model.load_state_dict(sd).missing_keys
    model = model.to(dev).eval()
    if frozen == "all":
        for p in model.parameters():
            p.requires_grad_(False)
    elif frozen == "cnn":
        model.freeze_cnn_backbone()
    return model


def run_e2e_against_oracle(dev, sd, path, frozen, size=224, frames=2, videos=2, tol=TOL_GRAD):
    """d score / d frames, score = <logits, fixed weights>, through ClipBert on the retrieval head, by torch.autograd.grad,
    against the oracle's clipbert_forward on the same units. Returns (relerr, cosine)."""
    from oracle import clipbert_ref as R, synth
    model = clipbert(dev, sd, frozen)
    clips = 1 if path == "forward" else 2
    batch = synth.synth_batch(videos, frames * clips, n_ex=2, size=size, seed=11)
    leaf = batch["visual_inputs"].clone().requires_grad_(True)
    xd = batch["visual_inputs"].to(dev).requires_grad_(True)
    mb = {k: (v.to(dev) if torch.is_tensor(v) else list(v)) for k, v in batch.items()}
    model.cnn._capture, model.transformer._capture = {}, {}
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
    stash, c1 = model.cnn._capture["stash"], model.transformer._capture["c1"]
    model.cnn._capture = model.transformer._capture = None
    wl = torch.randn(logits.shape, generator=torch.Generator().manual_seed(4))
    score = (logits * wl.to(dev)).sum()
    (dx,) = torch.autograd.grad(score, xd)
    # the oracle on the units the engine ran (one clip, or the B * clips units of forward_clips in pass order)
    if path == "forward":
        units, ids, mask, counts = leaf, batch["text_input_ids"], batch["text_input_mask"], list(batch["n_examples_list"])
    else:
        _, gather, scatter, counts = model._clip_plan
        gather, scatter = gather.cpu(), scatter.cpu()
        units = leaf.reshape((videos * clips, frames) + tuple(leaf.shape[2:]))
        ids, mask = batch["text_input_ids"].index_select(0, gather), batch["text_input_mask"].index_select(0, gather)
    pat = cnn_patterns(stash, _grid_of(stash))
    pat.relu_masks["transformer.classifier.relu"] = (c1 > 0).cpu()
    with oracle_stem(*stem_patterns(stash)), torch.enable_grad():
        ref = R.clipbert_forward(dict(visual_inputs=units, text_input_ids=ids, text_input_mask=mask, n_examples_list=counts), sd,
                                 freeze_at=0, rnd=pat)["logits"]
        if path != "forward":
            ref = ref.index_select(0, scatter).view(clips, -1, ref.shape[-1])
        (ref * wl).sum().backward()
    e, c = relerr(dx, leaf.grad), cosine(dx, leaf.grad)
    print("RELERR e2e %s-%s relerr %.3g cosine %.6f" % (path, frozen, e, c))
    assert e < tol and c > 0.999, (path, frozen, e, c)
    return dx


def _grid_of(stash):
    """The grid of the pass (forward_clips does not return it), from the stash's grid encoder conv: relu(max_pool2d(2, 2))."""
    n, h, w = stash["n"], stash["h"], stash["w"]
    g = stash["gconv"].float().view(n, h, w, -1).permute(0, 3, 1, 2)
    return torch.relu(F.max_pool2d(g, 2, 2)).permute(0, 2, 3, 1).reshape(n, 1, h // 2, w // 2, -1)


@pytest.fixture(scope="module")
def full_sd():
    from oracle import synth
    return synth.full_state_dict(42)


@pytest.mark.gpu
@pytest.mark.parametrize("path", E2E_PATHS)
@pytest.mark.parametrize("frozen", ["all", "cnn"])
def test_clipbert_frame_gradient_matches_oracle(cuda, full_sd, path, frozen):
    run_e2e_against_oracle(cuda, full_sd, path, frozen)


# ------------------------------------------------------------------------------------------------ nothing else changes
def run_parameter_gradients_unchanged(dev, sd, size=160, frames=2):
    """Under deterministic mode a training backward with frames that require grad leaves every parameter gradient bit-identical
    to the same step without, frozen parameters keep .grad None and their slice of the flat gradient buffer is never written."""
    from oracle import synth
    case = ModuleCase(1, frames, size)
    m = backbone(dev, case, sd)
    x = synth.synth_images(1, frames, size=size, seed=21).to(dev)
    with _deterministic():
        grid = m(x)
        dgrid = torch.randn(grid.shape, generator=torch.Generator().manual_seed(8)).to(BF16).to(dev)
        grid.backward(dgrid)
        want = {n: p.grad.clone() for n, p in m.named_parameters() if p.requires_grad}
        frozen = [mod for _, mod in m._convs() if not mod.weight.requires_grad]
        for mod in frozen:
            e = mod._e
            m._flat.grad[e["offset"]: e["offset"] + e["numel"]].fill_(float("nan"))
        for p in m.parameters():
            if p.grad is not None:
                p.grad.zero_()
        xg = x.clone().requires_grad_(True)
        grid = m(xg)
        grid.backward(dgrid)
    assert xg.grad is not None and float(xg.grad.abs().sum()) > 0
    for n, p in m.named_parameters():
        if p.requires_grad:
            assert torch.equal(_bits(p.grad), _bits(want[n])), n
        else:
            assert p.grad is None, n
    for mod in frozen:
        e = mod._e
        assert bool(torch.isnan(m._flat.grad[e["offset"]: e["offset"] + e["numel"]]).all())
    assert len(frozen) == 1 + 3 * 3 + 1          # stem + res2 (FREEZE_AT 2)


@pytest.mark.gpu
def test_parameter_gradients_unchanged_by_frame_gradients(cuda, cnn_sd):
    run_parameter_gradients_unchanged(cuda, cnn_sd)


@pytest.mark.gpu
def test_no_frame_gradient_no_extra_launches(cuda, cnn_sd):
    """Frames that do not require grad: no stem backward launch; with them, exactly the two stem kernels plus the frozen
    blocks' dgrad chain are added, and every pooled zero-bordered buffer comes back."""
    from clipbert_b200 import ops
    from oracle import synth
    m = backbone(cuda, ModuleCase(1, 2, 96), cnn_sd)
    x = synth.synth_images(1, 2, size=96, seed=2).to(cuda)
    counts = []
    for req in (False, True, False):
        xi = x.clone().requires_grad_(req)
        n0 = ops.launch_count()
        grid = m(xi)
        grid.backward(torch.ones_like(grid))
        torch.cuda.synchronize()
        counts.append(ops.launch_count() - n0)
    assert counts[0] == counts[2] and counts[1] > counts[0]


# ------------------------------------------------------------------------------------------------ reproducible and capturable
@pytest.mark.gpu
def test_end_to_end_frame_gradient_is_bit_reproducible(cuda, full_sd):
    with _deterministic():
        a = run_e2e_against_oracle(cuda, full_sd, "forward", "all", size=160)
        b = run_e2e_against_oracle(cuda, full_sd, "forward", "all", size=160)
    assert torch.equal(_bits(a), _bits(b))


@pytest.mark.gpu
def test_cuda_graph_capture_replays_eager_bits(cuda, cnn_sd):
    """An eval forward + backward to the frames of a frozen backbone, captured once, replays to the eager step's bits."""
    from oracle import synth
    m = backbone(cuda, ModuleCase(1, 2, 160), cnn_sd)
    for p in m.parameters():
        p.requires_grad_(False)
    m.eval()
    x = synth.synth_images(1, 2, size=160, seed=31).to(cuda).requires_grad_(True)
    dgrid = None

    def step():
        grid = m(x)
        return torch.autograd.grad(grid, x, dgrid)[0]
    with _deterministic():
        dgrid = torch.randn(m(x.detach()).shape, generator=torch.Generator().manual_seed(9)).to(BF16).to(cuda)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step()
        torch.cuda.current_stream().wait_stream(s)
        eager = step().clone()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            captured = step()
        graph.replay()
        torch.cuda.synchronize()
    assert float(eager.abs().sum()) > 0
    assert torch.equal(_bits(eager), _bits(captured))
