"""Gradients through the input stage: cb_resize_pad_bwd, the adjoint of cb_resize_pad (ImageResize = F.interpolate(bilinear,
align_corners=False) + ImagePad = zeros at the bottom / right, src/datasets/data_utils.py:136-160,202-234), and
input_stage.resize_pad as an autograd op, so that d score / d frames reaches the decoded frames as in the reference.

Kernel, element by element, with NaN guard bands around dx that must stay untouched (overwrite mode starts from NaN, so an
element never written fails):
  - against float64 R^T dy, R built per axis from the fp32 taps the forward kernel computes (f = fma(o + 0.5, s, -0.5) rounded
    once, clamped at 0; s = fl32(in / out); i0 = min(int f, n - 1); i1 = min(i0 + 1, n - 1); weights fl32(1 - l) and l). The
    kernel sums at most kx products per row of taps and ky rows: |err| <= (kx + ky + 2) U (|R|^T |dy|), U = 2^-24;
  - against torch.autograd.grad through float64 F.interpolate + F.pad on the CPU, with the fp32 rounding of the taps added: a
    source coordinate off by eps moves each weight by at most eps, eps = 4 (n + 2) U per axis, over every output whose
    coordinate lies within two pixels;
  - the adjoint identity <R x, y> = <x, R^T y> between the forward and backward kernels, in float64.
End to end, decoded fp32 frames go through resize_pad, a set_image_norm model and ClipBert, against the oracle's fp32 autograd
through F.interpolate + F.pad + (x - mean) / std + clipbert_forward (as tests/test_gpu_input_grads.py). Every element-wise check
prints "RATIO cb_resize_pad_bwd <case> <max err / bound>". tests/test_resize_pad_bwd_emulated.py runs the references, the
autograd op on the emulated entry points and planted faults on the CPU.
"""
import contextlib
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_gpu_input_grads as IG
from elementwise import F32, F64, U, Guarded, _record, check_bound
from model_util import cnn_patterns
from util import TOL_GRAD, cosine, relerr

FTZ = 2.0 ** -126


# ------------------------------------------------------------------------------------------------ references
def taps64(n_out, n_in, scale=None, clamp=True, merge=True, half_pixel=True):
    """float64 [n_out, n_in] matrix of one axis of cb_resize_pad from the kernel's fp32 taps. The keywords plant the faults of
    tests/test_resize_pad_bwd_emulated.py: no clamp at the top / left edge, no merge of the two taps at the bottom / right (the
    second is lost), the source coordinate without the half-pixel offset, and another axis' scale."""
    s = np.float32(n_in) / np.float32(n_out) if scale is None else np.float32(scale)
    o = np.arange(n_out, dtype=np.float64)
    # (o + 0.5) * s is exact in float64, and so is the - 0.5 wherever the result is >= 0: one rounding, as the kernel's FFMA
    f = (((o + 0.5) * np.float64(s) - 0.5) if half_pixel else o * np.float64(s)).astype(np.float32)
    if clamp:
        f = np.maximum(f, np.float32(0))
    i0 = np.minimum(f.astype(np.int64), n_in - 1)          # truncation, as the kernel's static_cast<int>
    i1 = i0 + 1
    l = (f - i0.astype(np.float32)).astype(np.float32)
    w0 = (np.float32(1) - l).astype(np.float32)
    m = np.zeros((n_out, n_in + 1))
    rows = np.arange(n_out)
    np.add.at(m, (rows, i0), w0.astype(np.float64))
    if merge:
        i1 = np.minimum(i1, n_in - 1)
    np.add.at(m, (rows, i1), l.astype(np.float64))
    return torch.from_numpy(m[:, :n_in].copy())


def neighbours(n_out, n_in):
    """[n_out, n_in] 0 / 1: the input pixels within two of each output's float64 source coordinate (where either weight set
    can be non-zero)."""
    f = np.maximum((np.arange(n_out) + 0.5) * n_in / n_out - 0.5, 0.0)
    base = np.floor(f).astype(np.int64)
    m = np.zeros((n_out, n_in))
    for d in (-1, 0, 1, 2):
        idx = np.clip(base + d, 0, n_in - 1)
        m[np.arange(n_out), idx] = 1.0
    return torch.from_numpy(m)


def sum_depth(my, mx):
    """kx + ky + 2: at most kx fp32 products added per row of taps (two per output column that taps the pixel), ky per pixel."""
    return 2 * int((mx != 0).sum(0).max()) + 2 * int((my != 0).sum(0).max()) + 2


def adjoint_ref(dy, h, w, nh, nw, my=None, mx=None):
    """float64 R^T dy for dy [planes, S, S] (its pad region ignored) and the bound of the kernel's fp32 sums."""
    my = taps64(nh, h) if my is None else my
    mx = taps64(nw, w) if mx is None else mx
    d = dy.detach().cpu().double()[:, :nh, :nw]
    ref = my.t() @ d @ mx
    terms = my.abs().t() @ d.abs() @ mx.abs()
    return ref, sum_depth(my, mx) * U * terms + FTZ


def interp_ref(dy, h, w, nh, nw):
    """torch.autograd.grad of <F.pad(F.interpolate(x, (nh, nw), bilinear, align_corners=False)), dy> in float64, and the bound
    of the kernel's fp32 taps and sums against it."""
    planes, s = dy.shape[0], dy.shape[-1]
    d = dy.detach().cpu().double()
    x = torch.zeros(planes, 1, h, w, dtype=F64, requires_grad=True)
    with torch.enable_grad():
        y = F.pad(F.interpolate(x, size=(nh, nw), mode="bilinear", align_corners=False), (0, s - nw, 0, s - nh))
        (g,) = torch.autograd.grad(y, x, d[:, None])
    _, bound = adjoint_ref(dy, h, w, nh, nw)
    ey, ex = 4 * (h + 2) * U, 4 * (w + 2) * U
    reach = neighbours(nh, h).t() @ d[:, :nh, :nw].abs() @ neighbours(nw, w)
    return g[:, 0], bound + (ey + ex + ey * ex) * reach


# ------------------------------------------------------------------------------------------------ kernel cases
class Case:
    def __init__(self, planes, h, w, nh, nw, s, what):
        self.planes, self.h, self.w, self.nh, self.nw, self.s = planes, h, w, nh, nw, s
        self.id = "%dx%dx%d-to-%dx%d-S%d-%s" % (planes, h, w, nh, nw, s, what)


def _fit(planes, h, w, s, what):
    from clipbert_b200.input_stage import get_resize_size
    return Case(planes, h, w, *get_resize_size(h, w, s), s, what)


KERNEL_CASES = [
    _fit(2, 240, 320, 448, "up1.4"), _fit(2, 720, 1280, 448, "down2.9"), _fit(1, 1080, 1920, 768, "down2.5"),
    _fit(1, 2160, 3840, 448, "down8.6"), _fit(2, 50, 40, 448, "up9"), _fit(2, 1344, 1000, 448, "down3"),
    Case(3, 100, 300, 30, 90, 96, "down3.3"), Case(2, 13, 17, 117, 40, 128, "up9-x2.4"),
    Case(3, 1, 600, 1, 32, 32, "1x600"), Case(3, 600, 1, 32, 1, 32, "600x1"), Case(2, 3, 5, 19, 32, 32, "3x5-up"),
    Case(3, 360, 640, 252, 448, 448, "360p"), Case(2, 64, 100, 64, 77, 128, "identity-rows"),
    Case(2, 90, 48, 60, 48, 64, "identity-cols"), Case(2, 1, 1, 7, 7, 9, "1x1"), Case(2, 1, 17, 5, 40, 41, "1xN"),
    Case(2, 37, 53, 31, 45, 47, "odd-S"),
]


def _dy(case, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(case.planes, case.s, case.s, generator=g)      # the pad region too: it must not leak


def run_kernel(dev, case, seed, accumulate=False):
    """One launch into a guarded dx (NaN in overwrite mode, random values to add onto). Returns (out, dy, dx0)."""
    from clipbert_b200 import ops
    dy = _dy(case, seed)
    dx0 = torch.randn(case.planes, case.h, case.w, generator=torch.Generator().manual_seed(seed + 1)) * 3 if accumulate else None
    out = Guarded((case.planes, case.h, case.w), F32, dev, init=dx0)
    ops.resize_pad_bwd(dy.to(dev), out.t, case.nh, case.nw, accumulate=accumulate)
    return out, dy, dx0


@pytest.mark.gpu
@pytest.mark.parametrize("case", KERNEL_CASES, ids=[c.id for c in KERNEL_CASES])
@pytest.mark.parametrize("accumulate", [False, True], ids=["overwrite", "accumulate"])
def test_resize_pad_bwd_elementwise(cuda, case, accumulate):
    out, dy, dx0 = run_kernel(cuda, case, seed=case.h + 7 * case.w, accumulate=accumulate)
    torch.cuda.synchronize()
    out.check("cb_resize_pad_bwd " + case.id)
    ref, bound = adjoint_ref(dy, case.h, case.w, case.nh, case.nw)
    if accumulate:
        ref = ref + dx0.double()
        bound = bound + U * (ref.abs() + bound)
    r = check_bound("cb_resize_pad_bwd " + case.id, out.t, ref, bound)
    _record("cb_resize_pad_bwd", case.id + ("-acc" if accumulate else ""), r)
    if not accumulate:
        g, gb = interp_ref(dy, case.h, case.w, case.nh, case.nw)
        check_bound("cb_resize_pad_bwd vs F.interpolate " + case.id, out.t, g, gb)


def _adjoint_gap(dev, case, seed):
    """(|<R x, y> - <x, R^T y>|, its bound) with R x from cb_resize_pad and R^T y from cb_resize_pad_bwd."""
    from clipbert_b200 import ops
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(case.planes, case.h, case.w, generator=g) * 50
    y = torch.randn(case.planes, case.s, case.s, generator=g)
    rx = torch.empty(case.planes, case.s, case.s, device=dev)
    rty = torch.empty(case.planes, case.h, case.w, device=dev)
    ops.resize_pad(x.to(dev), rx, case.nh, case.nw)
    ops.resize_pad_bwd(y.to(dev), rty, case.nh, case.nw)
    lhs = float((rx.cpu().double() * y.double()).sum())
    rhs = float((x.double() * rty.cpu().double()).sum())
    my, mx = taps64(case.nh, case.h), taps64(case.nw, case.w)
    mag = float((my.abs() @ x.double().abs() @ mx.abs().t() * y.double()[:, :case.nh, :case.nw].abs()).sum())
    _, b = adjoint_ref(y, case.h, case.w, case.nh, case.nw)
    # the backward's bound, and the forward's (at most 8 fp32 operations per output), on every product
    tol = float((b * x.double().abs()).sum()) + 10 * U * mag + 1e-9
    return abs(lhs - rhs), tol


@pytest.mark.gpu
@pytest.mark.parametrize("case", KERNEL_CASES, ids=[c.id for c in KERNEL_CASES])
def test_adjoint_identity(cuda, case):
    gap, tol = _adjoint_gap(cuda, case, seed=case.w)
    print("ADJOINT %s gap %.3g bound %.3g" % (case.id, gap, tol))
    assert gap <= tol, (case.id, gap, tol)


@pytest.mark.gpu
def test_index_arithmetic_past_2_31_elements(cuda):
    """dx with more than 2^31 elements (2^31 + 4096 here; just below 2^31 when the card lacks the memory), checked element by
    element on the device against float64 R^T dy (per chunk of planes), with guard bands on both ends."""
    from clipbert_b200 import ops
    h = w = 64
    nh = nw = s = 8
    free = torch.cuda.mem_get_info()[0]
    planes = (2 ** 31) // (h * w) + 1 if free > 24e9 else (2 ** 31) // (h * w) - 1
    n = planes * h * w
    print("LARGE planes %d elements %d (2^31 = %d)" % (planes, n, 2 ** 31))
    buf = torch.full((n + 2 * 64,), float("nan"), device=cuda)
    dx = buf[64:64 + n].view(planes, h, w)
    dy = torch.randn(planes, s, s, device=cuda, generator=torch.Generator(device=cuda).manual_seed(5))
    ops.resize_pad_bwd(dy, dx, nh, nw)
    torch.cuda.synchronize()
    assert bool(torch.isnan(buf[:64]).all()) and bool(torch.isnan(buf[-64:]).all())
    my, mx = taps64(nh, h), taps64(nw, w)
    c = sum_depth(my, mx) * U
    my, mx = my.to(cuda), mx.to(cuda)
    worst = 0.0
    for p0 in range(0, planes, 1 << 16):
        d = dy[p0:p0 + (1 << 16)].double()
        ref = my.t() @ d @ mx
        bound = c * (my.abs().t() @ d.abs() @ mx.abs()) + FTZ
        got = dx[p0:p0 + (1 << 16)].double()
        err = (got - ref).abs()
        assert bool((err <= bound).all()), p0          # NaN (never written) fails too
        worst = max(worst, float((err / bound).max()))
    _record("cb_resize_pad_bwd", "large-%d-planes" % planes, worst)


def _status(name, *args):
    from clipbert_b200 import _lib as L, ops
    n0 = ops.launch_count()
    rc = ops._fn(name)(*args)
    assert rc != 0 and name in L.lib().cb_last_error().decode()
    assert ops.launch_count() == n0


def test_resize_pad_bwd_rejects_bad_arguments():
    """Checked before any launch, so this runs without a GPU."""
    p = ctypes.c_void_p(16)
    _status("cb_resize_pad_bwd", None, p, 1, 8, 8, 4, 4, 4, 0, None)           # null dy
    _status("cb_resize_pad_bwd", p, None, 1, 8, 8, 4, 4, 4, 0, None)           # null dx
    _status("cb_resize_pad_bwd", p, p, 0, 8, 8, 4, 4, 4, 0, None)              # no planes
    _status("cb_resize_pad_bwd", p, p, 1, 0, 8, 4, 4, 4, 0, None)              # empty source
    _status("cb_resize_pad_bwd", p, p, 1, 8, 8, 5, 4, 4, 0, None)              # resized frame taller than max_size
    _status("cb_resize_pad_bwd", p, p, 1, 8, 8, 4, 0, 4, 0, None)              # zero width
    _status("cb_resize_pad_bwd", p, p, 1, 8, 8, 4, 4, 4, 2, None)              # accumulate not 0 / 1


# ------------------------------------------------------------------------------------------------ reproducible and capturable
@contextlib.contextmanager
def _deterministic(on=True):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(bool(on))
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


@pytest.mark.gpu
def test_bits_reproducible_and_graph_replay_matches_eager(cuda):
    from clipbert_b200 import ops
    case = KERNEL_CASES[0]
    dy = _dy(case, 3).to(cuda)
    runs = []
    for det in (False, True, False):
        with _deterministic(det):
            dx = torch.empty(case.planes, case.h, case.w, device=cuda)
            ops.resize_pad_bwd(dy, dx, case.nh, case.nw)
            torch.cuda.synchronize()
            runs.append(dx.cpu())
    for r in runs[1:]:
        assert torch.equal(r.view(torch.int32), runs[0].view(torch.int32))
    dx = torch.full((case.planes, case.h, case.w), 5.0, device=cuda)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        ops.resize_pad_bwd(dy, dx, case.nh, case.nw, accumulate=True)
    dx.fill_(5.0)
    graph.replay()
    torch.cuda.synchronize()
    want = torch.full_like(dx, 5.0)
    ops.resize_pad_bwd(dy, want, case.nh, case.nw, accumulate=True)
    torch.cuda.synchronize()
    assert torch.equal(dx.cpu().view(torch.int32), want.cpu().view(torch.int32))


# ------------------------------------------------------------------------------------------------ end to end
IMAGE_STD = (1.0, 1.0, 1.0)          # the config's img_pixel_std (src/configs/msrvtt_ret_base_resnet50.json)


def decoded_frames(videos, frames, h, w, seed):
    """fp32 0..255 frames at their decoded resolution."""
    return torch.randint(0, 256, (videos, frames, 3, h, w), generator=torch.Generator().manual_seed(seed)).float()


def oracle_frames(raw, size):
    """The reference's tensor path: ImageResize (F.interpolate) + ImagePad (F.pad) + ImageNorm, differentiable."""
    from clipbert_b200.input_stage import get_resize_size
    from clipbert_b200.workload import IMAGE_MEAN
    h, w = raw.shape[-2:]
    nh, nw = get_resize_size(h, w, size)
    x = F.interpolate(raw.reshape(-1, 3, h, w), size=(nh, nw), mode="bilinear", align_corners=False)
    x = F.pad(x, (0, size - nw, 0, size - nh))
    x = (x - torch.tensor(IMAGE_MEAN).view(1, 3, 1, 1)) / torch.tensor(IMAGE_STD).view(1, 3, 1, 1)
    return x.view(tuple(raw.shape[:-2]) + (size, size))


def model_for(dev, sd, frozen, train):
    from clipbert_b200 import input_stage
    from clipbert_b200.workload import IMAGE_MEAN
    model = IG.clipbert(dev, sd, frozen)
    input_stage.set_image_norm(model, IMAGE_MEAN, IMAGE_STD)
    return model.train(train)


def run_e2e(dev, sd, path, frozen, train=False, h=150, w=200, size=224, frames=2, videos=2):
    """d score / d decoded frames through resize_pad and ClipBert (score = <logits, fixed weights>) against the oracle. Returns
    (frame gradient, model, the source tensor)."""
    from clipbert_b200 import input_stage
    from oracle import clipbert_ref as R, synth
    model = model_for(dev, sd, frozen, train)
    clips = 1 if path == "forward" else 2
    batch = synth.synth_batch(videos, frames * clips, n_ex=2, size=size, seed=11)
    raw = decoded_frames(videos, frames * clips, h, w, seed=h + w)
    leaf = raw.clone().requires_grad_(True)
    xd = raw.to(dev).requires_grad_(True)
    mb = {k: (v.to(dev) if torch.is_tensor(v) else list(v)) for k, v in batch.items() if k != "visual_inputs"}
    model.cnn._capture, model.transformer._capture = {}, {}
    frames_dev = input_stage.resize_pad(xd, size)
    if path == "forward":
        logits = model(dict(mb, visual_inputs=frames_dev))["logits"]
    elif path == "forward_clips":
        logits = model.forward_clips(dict(mb, visual_inputs=frames_dev), clips)["logits"]
    else:
        logits = model.forward_clips(mb, clips, grid=model.encode_clips(frames_dev, clips))["logits"]
    stash, c1 = model.cnn._capture["stash"], model.transformer._capture["c1"]
    model.cnn._capture = model.transformer._capture = None
    wl = torch.randn(logits.shape, generator=torch.Generator().manual_seed(4))
    score = (logits * wl.to(dev)).sum()
    if train:
        score.backward()
        dx = xd.grad
    else:
        (dx,) = torch.autograd.grad(score, xd)
    assert dx.shape == raw.shape and dx.dtype == torch.float32
    if path == "forward":
        units, ids, mask, counts = leaf, batch["text_input_ids"], batch["text_input_mask"], list(batch["n_examples_list"])
    else:
        _, gather, scatter, counts = model._clip_plan
        gather, scatter = gather.cpu(), scatter.cpu()
        units = leaf.reshape((videos * clips, frames) + tuple(leaf.shape[2:]))
        ids, mask = batch["text_input_ids"].index_select(0, gather), batch["text_input_mask"].index_select(0, gather)
    pat = cnn_patterns(stash, IG._grid_of(stash))
    pat.relu_masks["transformer.classifier.relu"] = (c1 > 0).cpu()
    with IG.oracle_stem(*IG.stem_patterns(stash)), torch.enable_grad():
        ref = R.clipbert_forward(dict(visual_inputs=oracle_frames(units, size), text_input_ids=ids, text_input_mask=mask,
                                      n_examples_list=counts), sd, freeze_at=0, rnd=pat)["logits"]
        if path != "forward":
            ref = ref.index_select(0, scatter).view(clips, -1, ref.shape[-1])
        (ref * wl).sum().backward()
    e, c = relerr(dx, leaf.grad), cosine(dx, leaf.grad)
    print("RELERR e2e %s-%s%s relerr %.3g cosine %.6f" % (path, frozen, "-train" if train else "", e, c))
    assert e < TOL_GRAD and c > 0.999, (path, frozen, e, c)
    return dx, model, xd


@pytest.fixture(scope="module")
def full_sd():
    from oracle import synth
    return synth.full_state_dict(42)


@pytest.mark.gpu
@pytest.mark.parametrize("path", IG.E2E_PATHS)
def test_decoded_frame_gradient_matches_oracle_frozen(cuda, full_sd, path):
    run_e2e(cuda, full_sd, path, "all")


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["forward", "forward_clips"])
def test_decoded_frame_gradient_matches_oracle_training(cuda, full_sd, path):
    """A training-mode model with trainable parameters (the transformer; the CNN frozen): the frame gradient matches the oracle,
    and every parameter gradient is bit-identical to the same step with source frames that do not require grad."""
    from clipbert_b200 import input_stage
    from oracle import synth
    with IG._deterministic():
        _, model, xd = run_e2e(cuda, full_sd, path, "cnn", train=True)
    want = {n: p.grad.clone() for n, p in model.named_parameters() if p.requires_grad}
    assert want and all(g is not None for g in want.values())
    for p in model.parameters():
        if p.grad is not None:
            p.grad.zero_()
    # the same step on the same model, with source frames that do not require grad
    clips = 1 if path == "forward" else 2
    batch = synth.synth_batch(2, 2 * clips, n_ex=2, size=224, seed=11)
    mb = {k: (v.to(cuda) if torch.is_tensor(v) else list(v)) for k, v in batch.items() if k != "visual_inputs"}
    with IG._deterministic():
        frames = input_stage.resize_pad(xd.detach(), 224)
        assert not frames.requires_grad
        mb["visual_inputs"] = frames
        logits = (model(mb) if path == "forward" else model.forward_clips(mb, clips))["logits"]
        wl = torch.randn(logits.shape, generator=torch.Generator().manual_seed(4))
        (logits * wl.to(cuda)).sum().backward()
    for n, p in model.named_parameters():
        if p.requires_grad:
            assert torch.equal(IG._bits(p.grad), IG._bits(want[n])), n
        else:
            assert p.grad is None, n


@pytest.mark.gpu
def test_end_to_end_is_bit_reproducible(cuda, full_sd):
    with IG._deterministic():
        a, _, _ = run_e2e(cuda, full_sd, "forward", "all", h=120, w=90, size=160)
        b, _, _ = run_e2e(cuda, full_sd, "forward", "all", h=120, w=90, size=160)
    assert torch.equal(IG._bits(a), IG._bits(b))


# ------------------------------------------------------------------------------------------------ launch semantics
def _launches(fn):
    from clipbert_b200 import ops
    events = []
    ops.set_op_timing(events)
    try:
        out = fn()
        torch.cuda.synchronize()
    finally:
        ops.set_op_timing(None)
    return [e[0] for e in events], out


@pytest.mark.gpu
def test_launches_without_and_with_frame_gradients(cuda, full_sd):
    """uint8 frames, fp32 frames without grad and frames that require grad under no_grad: exactly the one cb_resize_pad
    launch and the bits of the entry point itself. Frames that require grad: a model step issues what the same step with the
    padded frames as the leaf issues, plus exactly one cb_resize_pad_bwd; a non-contiguous source gets its gradient back in its
    own shape."""
    from clipbert_b200 import input_stage, ops
    raw = decoded_frames(1, 2, 150, 200, seed=1)
    for x in (raw.to(torch.uint8).to(cuda), raw.to(cuda), raw.to(cuda).requires_grad_(True)):
        want = torch.empty(1, 2, 3, 224, 224, device=cuda)
        ops.resize_pad(x.detach().contiguous(), want, 168, 224)
        if x.requires_grad:
            with torch.no_grad():
                names, out = _launches(lambda: input_stage.resize_pad(x, 224))
        else:
            names, out = _launches(lambda: input_stage.resize_pad(x, 224))
        assert names == ["cb_resize_pad"] and not out.requires_grad
        assert out.shape == (1, 2, 3, 224, 224) and out.dtype == torch.float32
        assert torch.equal(out.view(torch.int32), want.view(torch.int32))

    model = model_for(cuda, full_sd, "all", False)
    from oracle import synth
    batch = synth.synth_batch(1, 2, n_ex=2, size=224, seed=11)
    mb = {k: (v.to(cuda) if torch.is_tensor(v) else list(v)) for k, v in batch.items() if k != "visual_inputs"}
    src = raw.to(cuda)

    def step(source_grad):
        def run():
            if source_grad:
                x = src.clone().requires_grad_(True)
                frames = input_stage.resize_pad(x, 224)
            else:
                x = frames = input_stage.resize_pad(src, 224).requires_grad_(True)
            score = model(dict(mb, visual_inputs=frames))["logits"].sum()
            return torch.autograd.grad(score, x)[0]
        return _launches(run)
    with IG._deterministic():
        step(False)                                   # the first call prepares the weights (one-off launches)
        plain, g_pad = step(False)
        names, g_src = step(True)
    assert names == plain + ["cb_resize_pad_bwd"]
    assert g_pad.shape == (1, 2, 3, 224, 224) and g_src.shape == raw.shape
    want = torch.empty_like(g_src)
    ops.resize_pad_bwd(g_pad.contiguous(), want, 168, 224)
    assert torch.equal(g_src.view(torch.int32), want.view(torch.int32))

    nc = src.permute(0, 1, 2, 4, 3).contiguous().permute(0, 1, 2, 4, 3).requires_grad_(True)   # (..., H, W), W-major storage
    assert not nc.is_contiguous()
    out = input_stage.resize_pad(nc, 224)
    (g,) = torch.autograd.grad(out, nc, g_pad)
    assert g.shape == nc.shape and torch.equal(g.contiguous().view(torch.int32), want.view(torch.int32))
