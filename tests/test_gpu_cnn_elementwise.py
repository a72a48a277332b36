"""GridFeatBackbone (clipbert_b200/grid_feat.py): every convolution of a forward and a training backward, element by element,
against float64 computed from what the module means, not from the launch descriptors it builds.

Reference. Each convolution is restated with float64 F.conv2d and its gradients (torch.nn.grad.conv2d_input / conv2d_weight),
with the module's stride and padding, where padding means real zeros and not the run's buffer border. It is fed the run's
own bf16 input of that convolution (the module's _capture hooks), the packed bf16 operand m._w reshaped to [cout, cin, kh, kw],
and the fp32 m._scale / m._shift. So every convolution is checked on its own (no drift accumulates through 50 layers), while a
wrong tap, row map, border, mask source, residual or stale buffer still shows. The packed operands themselves are checked
against the fp32 masters and float64 FrozenBN.

Bounds, per element (U = 2^-24), the error model of tests/test_gpu_gemm_elementwise.py:
  accumulation  3 n U T, T = conv(|x|, |w|), n = the launch's K times its taps (cin kh kw; 256 for the space-to-depth stem,
                152 for the patch-matrix stem, cout kh kw for a dgrad);
  each fp32 add (BN shift, residual)  + U |v|;  ReLU and the ReLU-mask select add nothing (0 where the select gives 0);
  the stored bf16 result  + 1 ulp_bf16(ref) + 2^-126;
  weight gradients  |s| T U (3 P + 1) + (S + 1) U |s| T + 2^-126, P the launch's reduction length (pixels, padded pixels for
                3x3), S <= ceil(P / 64) the K-split (the gradient starts from zero).
Pure selections are bit-exact: subsample2, both pools (F.max_pool2d semantics; the 2x2 forward writes +0 for a -0 maximum),
the pool backward scatter, unsubsample2_mask / relu_mask, and the zero border of every padded buffer (+0 bits).

Workloads: 2 frames at 224 px (the reference size: res5 7x7, grid 3x3), 2 frames at 200 px and 1 at 160 px (odd maps into
every stride-2 subsample; a 2x2 pool that drops a row and a column), 1 frame at 448 px (native resolution), 3 frames at 96 px
(small M, GEMM tile tails), and 2 frames at 224 px under torch.use_deterministic_algorithms(True) (split-plane weight
gradients). The stem runs separately in each of its modes (space-to-depth with 16- and 64-element rows, patch matrix) on float
and uint8 frames with a fused ImageNorm. The geometry-reuse cases run one module at two geometries with the same padded row
count: the second call must pass every check and equal a fresh module's run bit for bit.

Backends: "h100" (marked gpu) and "emulator", tests/ops_emulator.py replaying the same module on the CPU (the cases that fit
its budget). Every checked tensor prints "RATIO <fwd|dgrad|wgrad|stem> <case>-<tensor> <max err / bound>". The CPU fault
self-tests plant faults in real activations and gradients and show that the checks reject them: a stale border row (which
stays under the norm-wise tolerance of the stage-by-stage model tests), a 3x3 tap row pitch off by one, a weight gradient
missing the last frame, and one missing its FrozenBN scale.
"""
import contextlib

import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

import ops_emulator as E
from elementwise import BF16, F64, U, _record, check_bitexact, check_bound, rne_bf16, ulp_bf16
from util import TOL_MATCHED_DEEP, relerr

FTZ = 2.0 ** -126
BK = 64                      # weight-gradient K-split granularity (pixels)
STAGES = (("res2", 3, 1), ("res3", 4, 2), ("res4", 6, 2), ("res5", 3, 2))
PIXEL_STD = (58.395, 57.12, 57.375)


# ------------------------------------------------------------------------------------------------ backends and runs
class Backend:
    def __init__(self, name):
        if name == "h100" and not torch.cuda.is_available():
            pytest.skip("no CUDA device")
        self.emulated = name == "emulator"
        self.dev = torch.device("cpu") if self.emulated else torch.device("cuda:0")

    @contextlib.contextmanager
    def ops(self):
        if self.emulated:
            with E.emulated_ops():
                yield
        else:
            yield
            torch.cuda.synchronize()


_SD = {}


def _module(be, train):
    import clipbert_b200 as cb
    from oracle import synth
    if "sd" not in _SD:
        _SD["sd"] = synth.cnn_state_dict(42)
    m = cb.GridFeatBackbone()
    assert not m.load_state_dict(_SD["sd"]).missing_keys
    return m.to(be.dev).train(train)


def _images(frames, size, seed, uint8=False):
    from oracle import synth
    return synth.synth_images(1, frames, size=size, seed=seed, as_uint8=uint8)


def _dgrid(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).to(BF16)


@contextlib.contextmanager
def _deterministic(on):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(bool(on) or prev)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _run(be, m, x, train, det=False, seed=1):
    """One forward (and, in training, a backward of a random bf16 dgrid from zeroed gradients) with every capture."""
    x = x.to(be.dev)
    dgrid = None
    with be.ops(), _deterministic(det):
        m._capture = {}
        try:
            if train:
                m.zero_grad(set_to_none=True)
                grid = m(x)
                dgrid = _dgrid(grid.shape, seed).to(be.dev)
                grid.backward(dgrid)
            else:
                with torch.no_grad():
                    grid = m(x)
            cap = m._capture
        finally:
            m._capture = None
    return grid.detach(), cap, dgrid


# ------------------------------------------------------------------------------------------------ layouts
def _nchw(t, n, h, w, padded=False):
    """bf16 NHWC rows (compact, or zero-bordered with padded=True: the interior) -> bf16 NCHW, contiguous."""
    if padded:
        t = t.reshape(n, h + 2, w + 2, -1)[:, 1:-1, 1:-1]
    return t.reshape(n, h, w, -1).permute(0, 3, 1, 2).contiguous()


def _weight(conv):
    """The packed bf16 operand [cout, (r, s, c)] as a float64 [cout, cin, kh, kw] convolution weight."""
    return conv._w.reshape(conv.cout, conv.k, conv.k, conv.cin).permute(0, 3, 1, 2).double()


def _relu_pos(x):
    """CB_AUX_RELU_MASK's (aux > 0): a positive normal bf16 or +inf."""
    b = x.view(torch.int16).to(torch.int64) & 0xFFFF
    return (b >= 0x0080) & (b <= 0x7F80)


def check_border(what, t, n, h, w):
    """Every border row of the zero-bordered [n, h + 2, w + 2, c] buffer t holds +0 bits."""
    bits = t.detach().reshape(n, h + 2, w + 2, -1).cpu().view(torch.int16)
    border = torch.ones(h + 2, w + 2, dtype=torch.bool)
    border[1:-1, 1:-1] = False
    bad = bits[:, border] != 0
    if bad.any():
        img, pix, ch = (int(v) for v in bad.nonzero()[0])
        y, x = (int(v) for v in border.nonzero()[pix])
        raise AssertionError("%s: %d border elements of the zero-bordered buffer are not +0; first at image %d, padded pixel "
                             "(%d, %d), channel %d: 0x%04x" % (what, int(bad.sum()), img, y, x, ch, int(bits[:, border][img, pix, ch]) & 0xFFFF))


# ------------------------------------------------------------------------------------------------ references and bounds
def fwd_ref(x, w, shift=None, stride=1, pad=0, residual=None, relu=True, n_acc=None):
    """Forward conv + FrozenBN shift (+ residual) (+ ReLU): float64 value and per-element bound of the bf16 result."""
    v = F.conv2d(x, w, stride=stride, padding=pad)
    e = 3.0 * (n_acc or w[0].numel()) * U * F.conv2d(x.abs(), w.abs(), stride=stride, padding=pad)
    if shift is not None:
        v = v + shift.double().view(1, -1, 1, 1)
        e = e + U * v.abs()
    if residual is not None:
        v = v + residual
        e = e + U * v.abs()
    if relu:
        v = torch.where(v <= 0, torch.zeros_like(v), v)
    return v, e + ulp_bf16(v) + FTZ


def dgrad_ref(dy, w, x_shape, stride=1, pad=0, residual=None, mask=None):
    """Input gradient of a conv (+ residual) (* ReLU-mask select): float64 value and bound of the bf16 result."""
    v = conv2d_input(x_shape, w, dy, stride=stride, padding=pad)
    e = 3.0 * w.shape[0] * w.shape[2] * w.shape[3] * U * conv2d_input(x_shape, w.abs(), dy.abs(), stride=stride, padding=pad)
    if residual is not None:
        v = v + residual
        e = e + U * v.abs()
    if mask is not None:
        v, e = torch.where(mask, v, torch.zeros_like(v)), torch.where(mask, e, torch.zeros_like(e))
    return v, e + ulp_bf16(v) + FTZ


def wgrad_ref(x, dy, w_shape, scale, P, stride=1, pad=0):
    """scale[cout] * dL/dW from zero: float64 value and bound of the fp32 result of a P-long reduction."""
    v = conv2d_weight(x, w_shape, dy, stride=stride, padding=pad)
    T = conv2d_weight(x.abs(), w_shape, dy.abs(), stride=stride, padding=pad)
    if scale is not None:
        s = scale.double().view(-1, 1, 1, 1)
        v, T = v * s, T * s.abs()
    S = -(-P // BK)
    return v, T * U * (3.0 * P + 1.0) + (S + 1.0) * U * T + FTZ


class Checker:
    """Runs the checks of one case and prints a RATIO line per checked tensor."""

    def __init__(self, case):
        self.case = case
        self.worst = {}

    def bound(self, kind, what, got, ref_bound):
        r = check_bound("%s %s" % (self.case, what), got, *ref_bound)
        _record(kind, "%s-%s" % (self.case, what), r)
        self.worst[kind] = max(self.worst.get(kind, 0.0), r)

    def exact(self, what, got, ref):
        check_bitexact("%s %s" % (self.case, what), got, ref)


# ------------------------------------------------------------------------------------------------ the checks
def check_packing(m):
    """m._w = RNE_bf16(w * scale) in [cout, (r, s, c)]; m._scale / m._shift within a few fp32 ulp of float64 FrozenBN; the stem
    operands: 1 / pixel_std folded in (BGR input channels), 152-pitch copy with zero columns, and the space-to-depth operand,
    the kernel zero-extended to 8 x 8 x 4 and permuted to [64, (r', x', dy, dx, c4)] with r = 2 r' + dy, s = 2 x' + dx."""
    for name, conv in m._convs():
        wk = conv.weight.detach().permute(0, 2, 3, 1).reshape(conv.cout, -1)
        if hasattr(conv, "norm"):
            nb = conv.norm
            s64 = nb.weight.double() / torch.sqrt(nb.running_var.double() + 1e-5)
            sh64 = nb.bias.double() - nb.running_mean.double() * s64
            check_bound(name + " scale", conv._scale, s64, 8 * U * s64.abs())
            check_bound(name + " shift", conv._shift, sh64, 10 * U * (nb.running_mean.double() * s64).abs() + 2 * U * sh64.abs())
            want = wk * conv._scale[:, None]
        else:
            assert conv._scale is None and conv._shift is None
            want = wk
        if name == "stem.conv1":
            if m.pixel_std is not None:
                r, g, b = (float(v) for v in m.pixel_std)
                inv = torch.tensor([1.0 / b, 1.0 / g, 1.0 / r], dtype=torch.float32, device=want.device)
                want = (want.view(64, 49, 3) * inv).reshape(64, 147)
            got = m._stem_w
            assert torch.equal(got[:, 147:].cpu().view(torch.int16), torch.zeros(64, 5, dtype=torch.int16)), "stem operand pitch columns"
            got = got[:, :147]
        else:
            got = conv._w
        assert torch.equal(got.cpu().view(torch.int16), want.to(BF16).cpu().view(torch.int16)), "%s: packed operand" % name
    j = torch.arange(256)
    rp, xp, dy, dx, c = j // 64, (j // 16) % 4, (j // 8) % 2, (j // 4) % 2, j % 4
    w8 = torch.zeros(64, 8, 8, 4, dtype=BF16)
    w8[:, :7, :7, :3] = m._stem_w[:, :147].cpu().view(64, 7, 7, 3)
    want = w8[:, 2 * rp + dy, 2 * xp + dx, c]
    assert torch.equal(m._stem_w_s2d.cpu().view(torch.int16), want.view(torch.int16)), "space-to-depth stem operand"


def check_stem(ck, m, images, cap):
    """c1 = relu(conv7x7/s2/p3(bf16(x - mean) in BGR, w') + shift); the pooled stem bit-exact from c1."""
    n = images.shape[0] * images.shape[1]
    x = images.reshape(n, 3, images.shape[-2], images.shape[-1])
    raw = x.dtype == torch.uint8 or m.raw_float_inputs
    mean = torch.tensor(m.pixel_mean if raw else (0.0, 0.0, 0.0), dtype=torch.float32, device=x.device).view(1, 3, 1, 1)
    xb = (x.float() - mean).to(BF16)[:, [2, 1, 0]].double()
    w = m._stem_w[:, :147].reshape(64, 7, 7, 3).permute(0, 3, 1, 2).double()
    c1 = cap["c1"].permute(0, 3, 1, 2).contiguous()
    stem = m.feature.backbone.stem.conv1
    ck.bound("stem", "c1", c1, fwd_ref(xb, w, stem._shift, stride=2, pad=3, n_acc=256 if m.stem_mode == "s2d" else 152))
    ck.exact("stem pool", cap["stem"].permute(0, 3, 1, 2).contiguous(), F.max_pool2d(c1.double(), 3, 2, 1))


def check_forward(ck, m, cap, n):
    """Every block (xs, sc, a_pad, b, y), the grid encoder conv and the grid. Returns the float64 / bf16 activations the
    backward checks need."""
    bb = m.feature.backbone
    stem = cap["stem"]
    h, w = stem.shape[1], stem.shape[2]
    x_in = stem.permute(0, 3, 1, 2).contiguous()
    acts = {}
    for name, nblocks, stride in STAGES:
        for bi, blk in enumerate(getattr(bb, name)):
            key = "%s.%d" % (name, bi)
            c = cap[key]
            s = blk.stride
            h_in, w_in = h, w
            h, w = (h - 1) // s + 1, (w - 1) // s + 1
            x64 = x_in.double()
            xs = _nchw(c["xs"], n, h, w)
            ck.exact(key + " xs", xs, x64[:, :, ::s, ::s])
            sc = _nchw(c["sc"], n, h, w)
            if blk.has_shortcut:
                ck.bound("fwd", key + ".shortcut", sc, fwd_ref(x64, _weight(blk.shortcut), blk.shortcut._shift, stride=s, relu=False))
            else:
                ck.exact(key + " sc", sc, x64)
            check_border(ck.case + " " + key + " a_pad", c["a_pad"], n, h, w)
            a = _nchw(c["a_pad"], n, h, w, padded=True)
            ck.bound("fwd", key + ".conv1", a, fwd_ref(x64, _weight(blk.conv1), blk.conv1._shift, stride=s))
            b = _nchw(c["b"], n, h, w)
            ck.bound("fwd", key + ".conv2", b, fwd_ref(a.double(), _weight(blk.conv2), blk.conv2._shift, pad=1))
            last = key == "res5.2"
            if last:
                check_border(ck.case + " " + key + " y", c["y"], n, h, w)
            y = _nchw(c["y"], n, h, w, padded=last)
            ck.bound("fwd", key + ".conv3", y, fwd_ref(b.double(), _weight(blk.conv3), blk.conv3._shift, residual=sc.double()))
            acts[key] = dict(x_in=x_in, h_in=h_in, w_in=w_in, h=h, w=w, xs=xs, a=a, b=b, y=y)
            x_in = y
    ge = m.grid_encoder[0]
    gconv = _nchw(cap["gconv"], n, h, w)
    ck.bound("fwd", "grid_encoder", gconv, fwd_ref(x_in.double(), _weight(ge), pad=1, relu=False))
    acts["gconv"] = gconv
    return acts


def check_grid(ck, grid, gconv):
    n, c = gconv.shape[0], gconv.shape[1]
    ref = torch.relu(F.max_pool2d(gconv.double(), 2, 2)) + 0.0          # + 0.0: a -0 maximum gives +0
    ck.exact("grid", grid.reshape(n, grid.shape[-3], grid.shape[-2], c).permute(0, 3, 1, 2).contiguous(), ref)


def check_backward(ck, m, cap, acts, dgrid, n):
    """dg_pad, the grid encoder's dgrad and weight gradient, and for every trainable block g, db_pad, da, dxs, its input
    gradient and its weight gradients (through p.grad, as PyTorch sees them)."""
    bw = cap["bwd"]
    bb = m.feature.backbone
    ge = m.grid_encoder[0]
    y5 = acts["res5.2"]
    h, w = y5["h"], y5["w"]
    gconv = acts["gconv"].double().requires_grad_(True)
    with torch.enable_grad():
        pooled = F.max_pool2d(gconv, 2, 2)
        up = dgrid.reshape(n, h // 2, w // 2, -1).permute(0, 3, 1, 2).double()
        pooled.backward(torch.where(pooled.detach() > 0, up, torch.zeros_like(up)))
    ref = torch.zeros(n, h + 2, w + 2, ge.cout, dtype=F64, device=gconv.device)
    ref[:, 1:-1, 1:-1] = gconv.grad.permute(0, 2, 3, 1)
    ck.exact("grid_encoder dg_pad", bw["grid_encoder"]["dg_pad"].reshape(n, h + 2, w + 2, -1), ref)
    dg = ref[:, 1:-1, 1:-1].permute(0, 3, 1, 2)
    y5d = y5["y"].double()
    ck.bound("dgrad", "grid_encoder", _nchw(bw["res5.2"]["g"], n, h, w),
             dgrad_ref(dg, _weight(ge), y5d.shape, pad=1, mask=_relu_pos(y5["y"])))
    ck.bound("wgrad", "grid_encoder", ge.weight.grad, wgrad_ref(y5d, dg, ge.weight.shape, None, n * (h + 2) * (w + 2), pad=1))
    checked = [ge.weight]
    names = [("%s.%d" % (name, bi), blk) for name, nb, _ in STAGES for bi, blk in enumerate(getattr(bb, name))]
    trainable = [(k, blk) for k, blk in names if blk.conv1.weight.requires_grad]
    assert set(bw) == {"grid_encoder"} | {k for k, _ in trainable}
    for i, (key, blk) in reversed(list(enumerate(trainable))):
        a, c = acts[key], bw[key]
        h, w, s = a["h"], a["w"], blk.stride
        rows, P3 = n * h * w, n * (h + 2) * (w + 2)
        g = _nchw(c["g"], n, h, w)
        if i + 1 < len(trainable):
            assert c["g"] is bw[trainable[i + 1][0]]["gin"], key + ": g is not the input gradient of the block above"
        g64, x64 = g.double(), a["x_in"].double()
        check_border(ck.case + " " + key + " db_pad", c["db_pad"], n, h, w)
        db = _nchw(c["db_pad"], n, h, w, padded=True)
        ck.bound("dgrad", key + ".conv3", db, dgrad_ref(g64, _weight(blk.conv3), a["b"].shape, mask=_relu_pos(a["b"])))
        da = _nchw(c["da"], n, h, w)
        ck.bound("dgrad", key + ".conv2", da, dgrad_ref(db.double(), _weight(blk.conv2), a["a"].shape, pad=1, mask=_relu_pos(a["a"])))
        wg = [(blk.conv3, a["b"].double(), g64, 1, 0, rows), (blk.conv2, a["a"].double(), db.double(), 1, 1, P3),
              (blk.conv1, x64, da.double(), s, 0, rows)]
        if blk.has_shortcut:
            wg.append((blk.shortcut, x64, g64, s, 0, rows))
        for conv, x, dy, st, pad, P in wg:
            part = [k for k, v in blk.named_children() if v is conv][0]
            ck.bound("wgrad", "%s.%s" % (key, part), conv.weight.grad, wgrad_ref(x, dy, conv.weight.shape, conv._scale, P, stride=st, pad=pad))
            checked.append(conv.weight)
        if i == 0:
            assert "gin" not in c, key + ": a gradient was computed below the first trainable block"
            continue
        xs_shape = a["xs"].shape
        if blk.has_shortcut:
            dxs_sc = _nchw(c["dxs_sc"], n, h, w)
            ck.bound("dgrad", key + ".shortcut", dxs_sc, dgrad_ref(g64, _weight(blk.shortcut), xs_shape))
            dxs = _nchw(c["dxs"], n, h, w)
            ck.bound("dgrad", key + ".conv1", dxs, dgrad_ref(da.double(), _weight(blk.conv1), xs_shape, residual=dxs_sc.double()))
            full = torch.zeros_like(x64)
            full[:, :, ::s, ::s] = dxs.double()
            ck.exact(key + " gin", _nchw(c["gin"], n, a["h_in"], a["w_in"]), torch.where(x64 > 0, full, torch.zeros_like(full)))
        else:
            ck.bound("dgrad", key + ".conv1", _nchw(c["gin"], n, h, w),
                     dgrad_ref(da.double(), _weight(blk.conv1), xs_shape, residual=g64, mask=_relu_pos(a["x_in"])))
    params = [p for p in m.parameters() if p.requires_grad]
    assert len(checked) == len(params) == 3 * 13 + 3 + 1 and {id(p) for p in checked} == {id(p) for p in params}
    assert all(p.grad is None for p in m.parameters() if not p.requires_grad)


def check_pool(m):
    """Every buffer the zero-bordered pool holds still has a +0 border for the geometry it is filed under."""
    for (n, h, w, c), lst in m._pad_pool.items():
        for t in lst:
            check_border("pooled buffer %dx%dx%dx%d" % (n, h, w, c), t, n, h, w)


def check_run(be, m, case, images, grid, cap, dgrid, train):
    ck = Checker(case)
    n = images.shape[0] * images.shape[1]
    check_packing(m)
    check_stem(ck, m, images.to(be.dev), cap)
    acts = check_forward(ck, m, cap, n)
    check_grid(ck, grid, acts["gconv"])
    if train:
        check_backward(ck, m, cap, acts, dgrid, n)
    check_pool(m)
    return ck


# ------------------------------------------------------------------------------------------------ workloads
class Case:
    def __init__(self, frames, size, det=False):
        self.frames, self.size, self.det = frames, size, det
        self.id = "%dx%d%s" % (frames, size, "-det" if det else "")

    @property
    def pixels(self):
        return self.frames * self.size * self.size


CASES = [Case(2, 224), Case(2, 200), Case(1, 160), Case(1, 448), Case(3, 96), Case(2, 224, det=True)]
_EMU_MAX = 2 * 224 * 224            # frame pixels of the emulated cases (CPU float64 run and reference)
EMU_CASES = [c for c in CASES if c.pixels <= _EMU_MAX]


def _params(cases, ids):
    return ([pytest.param("h100", c, marks=pytest.mark.gpu, id="h100-" + i) for c, i in zip(cases, ids)]
            + [pytest.param("emulator", c, id="emulator-" + i) for c, i in zip(cases, ids) if c in EMU_CASES])


@pytest.mark.parametrize("be_name,case", _params(CASES, [c.id for c in CASES]))
def test_cnn_training_step_elementwise(be_name, case):
    be = Backend(be_name)
    m = _module(be, train=True)
    images = _images(case.frames, case.size, seed=case.size + case.frames)
    grid, cap, dgrid = _run(be, m, images, train=True, det=case.det)
    check_run(be, m, case.id, images, grid, cap, dgrid, train=True)


STEMS = [("s2d16", "float"), ("s2d16", "uint8"), ("s2d64", "float"), ("s2d64", "uint8"), ("im2col", "float"), ("im2col", "uint8")]


@pytest.mark.parametrize("be_name,stem,frames", [pytest.param("h100", s, f, marks=pytest.mark.gpu, id="h100-%s-%s" % (s, f)) for s, f in STEMS]
                         + [pytest.param("emulator", s, f, id="emulator-%s-%s" % (s, f)) for s, f in STEMS if s != "s2d64"])
def test_cnn_stem_modes_elementwise(be_name, stem, frames):
    """Each stem mode on float frames (already normalised) and on uint8 frames with ImageNorm fused (mean in the gather,
    1 / std in the weights), 2 frames at 118 px (odd conv output, 59 x 59)."""
    from clipbert_b200 import input_stage
    from clipbert_b200.workload import IMAGE_MEAN
    be = Backend(be_name)
    m = _module(be, train=False)
    m.stem_mode = "im2col" if stem == "im2col" else "s2d"
    m._s2d_ld = 64 if stem == "s2d64" else 16
    uint8 = frames == "uint8"
    if uint8:
        input_stage.set_image_norm(m, IMAGE_MEAN, PIXEL_STD, raw_float_inputs=False)
    images = _images(2, 118, seed=11, uint8=uint8)
    grid, cap, _ = _run(be, m, images, train=False)
    assert m._s2d_ld == (64 if stem == "s2d64" else 16)
    ck = Checker("%s-%s" % (stem, frames))
    check_packing(m)
    check_stem(ck, m, images.to(be.dev), cap)


# ------------------------------------------------------------------------------------------------ geometry reuse
class Reuse:
    """A module runs geometry `first` and then `second`, whose zero-bordered buffers have the same row counts."""

    def __init__(self, first, second, train, emu):
        self.first, self.second, self.train, self.emu = first, second, train, emu
        self.id = "%dx%d-then-%dx%d-%s" % (first + second + ("train" if train else "eval",))


def _padded_rows(frames, size):
    ho = (size - 1) // 2 + 1
    h = (ho - 1) // 2 + 1
    for s in (2, 2, 2):
        h = (h - 1) // s + 1
    return frames * (h + 2) ** 2


REUSE = [Reuse((1, 192), (4, 64), t, True) for t in (False, True)] + [Reuse((2, 448), (8, 192), t, False) for t in (False, True)]


@pytest.mark.parametrize("be_name,r", [pytest.param("h100", r, marks=pytest.mark.gpu, id="h100-" + r.id) for r in REUSE]
                         + [pytest.param("emulator", r, id="emulator-" + r.id) for r in REUSE if r.emu])
def test_cnn_geometry_reuse(be_name, r):
    """The second geometry's res5 / grid-encoder buffers have the first's row count but other border rows: the second call
    must pass every check, keep every pooled border at +0, and give a fresh module's forward bit for bit (one writer per
    element) and, under deterministic mode, its weight gradients bit for bit."""
    assert _padded_rows(*r.first) == _padded_rows(*r.second)
    be = Backend(be_name)
    m = _module(be, r.train)
    _run(be, m, _images(*r.first, seed=3), r.train, det=True)
    images = _images(*r.second, seed=4)
    grid, cap, dgrid = _run(be, m, images, r.train, det=True, seed=5)
    check_run(be, m, r.id, images, grid, cap, dgrid, r.train)
    fresh = _module(be, r.train)
    grid0, cap0, _ = _run(be, fresh, images, r.train, det=True, seed=5)

    def same(a, b, what):
        assert torch.equal(a.detach().cpu().view(torch.int16), b.detach().cpu().view(torch.int16)), "%s: %s differs from a fresh module's" % (r.id, what)

    same(grid, grid0, "the grid")
    same(cap["gconv"], cap0["gconv"], "the grid encoder conv")
    for key in (k for k in cap if k[:3] == "res" and "." in k):
        for t in ("a_pad", "b", "y"):
            same(cap[key][t], cap0[key][t], "%s %s" % (key, t))
    if r.train:
        for (name, p), p0 in zip(m.named_parameters(), fresh.parameters()):
            if p.requires_grad:
                assert torch.equal(p.grad.cpu().view(torch.int32), p0.grad.cpu().view(torch.int32)), \
                    "%s: the weight gradient of %s differs from a fresh module's" % (r.id, name)


# ------------------------------------------------------------------------------------------------ CPU fault self-tests
@pytest.fixture(scope="module")
def emu_run():
    """An emulated training step of 8 frames at 64 px: real activations and gradients to plant faults in."""
    be = Backend("emulator")
    m = _module(be, train=True)
    _, cap, _ = _run(be, m, _images(8, 64, seed=7), train=True)
    return m, cap, 8


def _conv2_case(emu_run):
    m, cap, n = emu_run
    blk = m.feature.backbone.res2[1]
    a_pad = cap["res2.1"]["a_pad"]
    return m, blk, a_pad, n, 16, 16, fwd_ref(_nchw(a_pad, n, 16, 16, padded=True).double(), _weight(blk.conv2), blk.conv2._shift, pad=1)


def test_fault_stale_border_row_is_rejected_but_passes_the_normwise_check(emu_run):
    """One border row of res2.1's zero-bordered conv2 input holds an interior row (what a buffer recycled from another
    geometry holds): the border check and the conv check reject it; the output's norm-wise error stays under
    TOL_MATCHED_DEEP, the tolerance of the stage-by-stage model tests."""
    m, blk, a_pad, n, h, w, (ref, bound) = _conv2_case(emu_run)
    bad = a_pad.clone().view(n, h + 2, w + 2, -1)
    bad[-1, 0, 0] = bad[-1, 5, 5]
    with pytest.raises(AssertionError, match=r"border .* not \+0; first at image 7, padded pixel \(0, 0\)"):
        check_border("fault", bad, n, h, w)
    got = rne_bf16(fwd_ref(bad.permute(0, 3, 1, 2).double(), _weight(blk.conv2), blk.conv2._shift)[0])   # the buffer's border as padding
    with pytest.raises(AssertionError, match="out of bound"):
        check_bound("fault", got, ref, bound)
    assert relerr(got, ref) < TOL_MATCHED_DEEP


def test_fault_tap_row_pitch_off_by_one_is_rejected(emu_run):
    """res2.1's 3x3 conv run with tap_w = w + 1 (the taps of the rows above and below one pixel off) is rejected; the same
    launch with tap_w = w + 2 passes."""
    m, blk, a_pad, n, h, w, (ref, bound) = _conv2_case(emu_run)
    p = n * (h + 2) * (w + 2)
    for tap_w, ok in ((w + 2, True), (w + 1, False)):
        out = torch.empty(n * h * w, blk.mid, dtype=BF16)
        E.gemm(mode=0, m=p, n=blk.mid, k=blk.mid, a=a_pad, a_rows=p, a_ld=blk.mid, b=blk.conv2._w, b_rows=blk.mid, b_ld=9 * blk.mid,
               ntaps=9, tap_w=tap_w, tap_sign=1, shift=blk.conv2._shift, act=1, out=out, out_ld=blk.mid, rowmap=2, map_h=h, map_w=w)
        if ok:
            check_bound("tap_w %d" % tap_w, _nchw(out, n, h, w), ref, bound)
        else:
            with pytest.raises(AssertionError, match="out of bound"):
                check_bound("tap_w %d" % tap_w, _nchw(out, n, h, w), ref, bound)


def _res52_conv3_wgrad(emu_run, g_last_zero=False, scale=True):
    m, cap, n = emu_run
    blk = m.feature.backbone.res5[2]
    g = _nchw(cap["bwd"]["res5.2"]["g"], n, 2, 2).double()
    if g_last_zero:
        g[-1] = 0
    b = _nchw(cap["res5.2"]["b"], n, 2, 2).double()
    return wgrad_ref(b, g, blk.conv3.weight.shape, blk.conv3._scale if scale else None, n * 4)


def test_fault_last_frame_gradient_left_at_zero_is_rejected(emu_run):
    """res5.2 conv3's weight gradient without the last of 8 frames (its dY rows never reached the reduction) is rejected,
    the correct one rounded to fp32 passes."""
    ref, bound = _res52_conv3_wgrad(emu_run)
    check_bound("wgrad", ref.float(), ref, bound)
    got, _ = _res52_conv3_wgrad(emu_run, g_last_zero=True)
    with pytest.raises(AssertionError, match="out of bound"):
        check_bound("fault", got.float(), ref, bound)


def test_fault_weight_gradient_missing_its_bn_scale_is_rejected(emu_run):
    """res5.2 conv3's weight gradient without the FrozenBN scale folded into its operand (dL/dW' instead of s dL/dW') is
    rejected."""
    ref, bound = _res52_conv3_wgrad(emu_run)
    got, _ = _res52_conv3_wgrad(emu_run, scale=False)
    with pytest.raises(AssertionError, match="out of bound"):
        check_bound("fault", got.float(), ref, bound)
