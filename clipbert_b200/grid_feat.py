"""GridFeatBackbone on H100: detectron2 MSRA ResNet-50 (res5) + grid_encoder, forward and backward,
as wgmma implicit-GEMM convolutions over NHWC bf16 activations.

Mirrors the reference module ``src/modeling/grid_feat.py:GridFeatBackbone`` (same constructor
arguments, ``forward(x: (B,T,3,H,W)) -> (B,T,h,w,768)``, ``.feature``, ``.grid_encoder``,
``.config_file``) and its state_dict keys (SURVEY.md App. B), but none of its code: the d2 model is
not built; only the parameters of ``feature.backbone`` and ``grid_encoder`` exist.

Data layout in HBM
  * activations: NHWC bf16, "compact" rows = pixels (img, y, x); the input of every 3x3 conv (and the
    dY of its backward) is kept "padded": [img, H+2, W+2, C] with a zero border, so that the 3x3
    conv is 9 row-shifted K-slabs of ONE 2D TMA-loaded matrix (no im2col, no halo logic);
  * weights: KRSC bf16 with the FrozenBN scale folded in (w' = w * gamma * rsqrt(var + 1e-5)); the
    BN shift is a per-channel fp32 vector applied in the GEMM epilogue; fp32 masters stay KRSC too;
  * backward: ReLU masks are re-derived from the stored forward activations inside the dgrad
    epilogues; wgrad accumulates fp32 directly into the flat gradient buffer.
"""
import contextlib
import math

import torch
from torch import nn

from . import ops
from .modeling import _engine_runs
from .params import FlatGroup

RESNET50_STAGES = (("res2", 3, 64, 256, 1), ("res3", 4, 128, 512, 2), ("res4", 6, 256, 1024, 2), ("res5", 3, 512, 2048, 2))
RESNET50_LAST_BLOCK = "res5.2"     # its output is kept zero-bordered: the grid_encoder conv reads it
FROZEN_BN_EPS = 1e-5
STEM_KP = 152  # 7*7*3 = 147 zero-padded to a multiple of 8 (16-byte TMA row pitch)

_D2_CONFIG_TEXT = """MODEL:
  META_ARCHITECTURE: GeneralizedRCNN
  BACKBONE: {NAME: build_resnet_backbone, FREEZE_AT: %d}
  RESNETS: {DEPTH: 50, OUT_FEATURES: [res5], RES5_DILATION: 1, STRIDE_IN_1X1: true, NORM: FrozenBN}
  WEIGHTS: detectron2://ImageNetPretrained/MSRA/R-50.pkl
"""


def _require_cuda(t):
    assert t.is_cuda, "GridFeatBackbone runs on CUDA only (no CPU fallback)"


def _unmasked(kw):
    """A dgrad launch without its ReLU' mask, on the tile the masked launch runs on: the same fp32 sums rounded once to the same
    bf16 (the mask only selects +0), so cb_nhwc_intake can apply the mask later and give the default path's bits."""
    width = ops.gemm_tile_width(kw)
    kw = {k: v for k, v in kw.items() if k not in ("aux", "aux_ld", "aux_mode")}
    return dict(kw, block_n=0, reserved=ops.GEMM_FORCE_WIDE) if width == 256 else dict(kw, block_n=width)


def _nchw(buf, n, h, w, bordered=False):
    """The (n, c, h, w) view of an NHWC buffer, compact [n*h*w, c] or zero-bordered [n*(h+2)*(w+2), c] (its interior)."""
    if bordered:
        return buf.view(n, h + 2, w + 2, -1)[:, 1:-1, 1:-1].permute(0, 3, 1, 2)
    return buf.view(n, h, w, -1).permute(0, 3, 1, 2)


def _same_view(t, v):
    return t.dtype == v.dtype and t.device == v.device and t.data_ptr() == v.data_ptr() and t.shape == v.shape and t.stride() == v.stride()


def _check_shape(t, shape, what):
    if not torch.is_tensor(t) or tuple(t.shape) != tuple(shape):
        raise ValueError("GridFeatBackbone: %s must be a tensor of shape %s, got %s" % (what, tuple(shape),
                                                                                      tuple(t.shape) if torch.is_tensor(t) else type(t).__name__))


def _compact(t, c, h, w, act=None, what="input"):
    """t (n, c, h, w), any strides and float dtype, as the engine's compact NHWC bf16 [n*h*w, c]: t's own memory when it is already
    that layout and no mask is asked for, else one cb_nhwc_intake (act: masked by act > 0)."""
    n = t.shape[0]
    _check_shape(t, (n, c, h, w), what)
    t = t.detach()
    if act is None and t.dtype == torch.bfloat16 and t.permute(0, 2, 3, 1).is_contiguous() and t.data_ptr() % 16 == 0:
        return t.permute(0, 2, 3, 1).reshape(n * h * w, c)
    out = torch.empty(n * h * w, c, dtype=torch.bfloat16, device=t.device)
    ops.nhwc_intake(t, out, act=act, act_bordered=act is not None and act.shape[0] != n * h * w)
    return out


def _bordered(t, c, h, w, known=None, what="input"):
    """t (n, c, h, w) as a zero-bordered NHWC bf16 [n*(h+2)*(w+2), c]: ``known`` (such a buffer) when t is its interior view, else
    one cb_nhwc_intake into a fresh zeroed buffer."""
    n = t.shape[0]
    _check_shape(t, (n, c, h, w), what)
    if known is not None and _same_view(t, _nchw(known, n, h, w, bordered=True)):
        return known
    out = torch.zeros(n * (h + 2) * (w + 2), c, dtype=torch.bfloat16, device=t.device)
    ops.nhwc_intake(t.detach(), out, out_bordered=True)
    return out


def _anchor(mod):
    return next((p for p in mod.parameters() if p.requires_grad), None)


class _CnnPass:
    """One GridFeatBackbone.forward on the module path: each module the forward calls runs its part of the engine here, from the
    tensor it was handed (the previous module's output, or what a hook replaced it with) to an (N, C, h, w) view of the NHWC bf16
    buffer it writes. A pass that records autograd runs each part as a node (_StemNode, _BlockNode, _GridConvNode, _GridPoolNode)
    whose activations are its saved tensors."""

    def __init__(self, m, n):
        self.m, self.n = m, n
        self.h = self.w = None     # spatial size of the last output
        self.res5 = None           # the last block's zero-bordered output
        self.dg_pad = None         # the pool node's zero-bordered gradient at the grid_encoder conv output

    @staticmethod
    def records(x, anchor):
        return torch.is_grad_enabled() and (x.requires_grad or anchor is not None)

    def stem(self, x):
        if self.records(x, None):
            return _StemNode.apply(self, x)
        cur, _, self.h, self.w = self.m._stem_forward(x.detach(), False)
        return _nchw(cur, self.n, self.h, self.w)

    def run_block(self, blk, x):
        m, n = self.m, self.n
        x_in = _compact(x, blk.cin, self.h, self.w, what="the input of %s" % blk.block_name)
        last = blk.block_name == RESNET50_LAST_BLOCK
        st = m._block_forward(blk, x_in, n, self.h, self.w, last)
        self.h, self.w = st["h"], st["w"]
        if last:
            self.res5 = st["y"]
        return st, _nchw(st["y"], n, self.h, self.w, bordered=last)

    def block(self, blk, x):
        anchor = _anchor(blk)
        if self.records(x, anchor):
            return _BlockNode.apply(self, blk, x, anchor)
        st, y = self.run_block(blk, x)
        self.m._pad_put(st["a_pad"], self.n, self.h, self.w)     # consumed by conv2; the block output is handed out, never recycled
        return y

    def run_grid_conv(self, x):
        ge = self.m.grid_encoder[0]
        res5 = _bordered(x, ge.cin, self.h, self.w, known=self.res5, what="the input of grid_encoder")
        return res5, self.m._conv3x3(ge, res5, self.n, self.h, self.w, ops.ACT_NONE)

    def grid_conv(self, x):
        anchor = _anchor(self.m.grid_encoder[0])
        if self.records(x, anchor):
            return _GridConvNode.apply(self, x, anchor)
        return _nchw(self.run_grid_conv(x)[1], self.n, self.h, self.w)

    def run_grid_pool(self, x):
        c = self.m.grid_encoder[0].cout
        gconv = _compact(x, c, self.h, self.w, what="the input of grid_encoder's pool")
        grid = torch.empty(self.n * (self.h // 2) * (self.w // 2), c, dtype=torch.bfloat16, device=gconv.device)
        ops.maxpool2x2_relu_fwd(gconv, grid, self.n, self.h, self.w, c)
        return gconv, _nchw(grid, self.n, self.h // 2, self.w // 2)

    def grid_pool(self, x):
        if self.records(x, None):
            return _GridPoolNode.apply(self, x)
        return self.run_grid_pool(x)[1]


class _StemNode(torch.autograd.Function):
    """frames (N, 3, H, W) -> the pooled stem output; its backward is the frame gradient."""

    @staticmethod
    def forward(ctx, ps, x):
        cur, frames, ps.h, ps.w = ps.m._stem_forward(x.detach(), True)
        ctx.ps, ctx.hw, ctx.x = ps, (ps.h, ps.w), (x.shape, x.dtype)
        ctx.frames = {k: v for k, v in frames.items() if k != "c1"}
        ctx.save_for_backward(frames["c1"])
        return _nchw(cur, ps.n, ps.h, ps.w)

    @staticmethod
    def backward(ctx, dy):
        ps, (h, w) = ctx.ps, ctx.hw
        c1, = ctx.saved_tensors
        with ps.m._node_backward(False):
            g = _compact(dy, 64, h, w, what="the gradient of stem")
            dx = ps.m._stem_backward(g, dict(ctx.frames, c1=c1), ps.n)
        shape, dtype = ctx.x
        return None, dx.view(shape).to(dtype)


class _BlockNode(torch.autograd.Function):
    """Bottleneck block: its input -> its output. The backward takes the gradient at the output, applies the block's ReLU' on
    entry (cb_nhwc_intake), and returns the unmasked gradient at the input: the block below applies its own ReLU'."""

    @staticmethod
    def forward(ctx, ps, blk, x, anchor):
        st, y = ps.run_block(blk, x)
        ctx.ps, ctx.blk, ctx.has_anchor = ps, blk, anchor is not None
        ctx.geom = (st["h"], st["w"], st["h_in"], st["w_in"])
        ctx.save_for_backward(st["xs"], st["a_pad"], st["b"], st["y"])
        return y

    @staticmethod
    def backward(ctx, dy):
        ps, blk = ctx.ps, ctx.blk
        need_dx = _engine_runs(ctx.next_functions[0][0], False)
        grads = ctx.has_anchor and _engine_runs(ctx.next_functions[1][0], False)
        if not (need_dx or grads):
            return None, None, None, None
        xs, a_pad, b, y = ctx.saved_tensors
        h, w, h_in, w_in = ctx.geom
        st = dict(name=blk.block_name, blk=blk, x_in=xs if blk.stride == 1 else None, xs=xs, a_pad=a_pad, b=b, y=y, h=h, w=w,
                  h_in=h_in, w_in=w_in, trainable=blk.conv1.weight.requires_grad)
        with ps.m._node_backward(grads) as (sq, recycle):
            g = _compact(dy, blk.cout, h, w, act=y, what="the gradient of %s" % blk.block_name)
            gin = ps.m._block_backward(st, g, ps.n, sq, recycle, wgrad=grads, need_dx=need_dx, mask=False)
        return None, None, (None if gin is None else _nchw(gin, ps.n, h_in, w_in)), None


class _GridConvNode(torch.autograd.Function):
    """grid_encoder[0]: res5 output -> the conv output before pool and ReLU."""

    @staticmethod
    def forward(ctx, ps, x, anchor):
        res5, gconv = ps.run_grid_conv(x)
        ctx.ps, ctx.hw, ctx.has_anchor = ps, (ps.h, ps.w), anchor is not None
        ctx.save_for_backward(res5)
        return _nchw(gconv, ps.n, ps.h, ps.w)

    @staticmethod
    def backward(ctx, dg):
        ps, (h, w) = ctx.ps, ctx.hw
        need_dx = _engine_runs(ctx.next_functions[0][0], False)
        grads = ctx.has_anchor and _engine_runs(ctx.next_functions[1][0], False)
        if not (need_dx or grads):
            return None, None, None
        res5, = ctx.saved_tensors
        ge = ps.m.grid_encoder[0]
        with ps.m._node_backward(grads) as (sq, recycle):
            dg_pad = _bordered(dg, ge.cout, h, w, known=ps.dg_pad, what="the gradient of grid_encoder.0")
            g = ps.m._grid_conv_backward(dg_pad, res5, ps.n, h, w, sq, grads, need_dx, mask=False)
        return None, (None if g is None else _nchw(g, ps.n, h, w)), None


class _GridPoolNode(torch.autograd.Function):
    """grid_encoder's MaxPool2d(2, 2) + ReLU: the conv output -> the grid."""

    @staticmethod
    def forward(ctx, ps, x):
        gconv, grid = ps.run_grid_pool(x)
        ctx.ps, ctx.hw = ps, (ps.h, ps.w)
        ctx.save_for_backward(gconv)
        return grid

    @staticmethod
    def backward(ctx, dgrid):
        ps, (h, w) = ctx.ps, ctx.hw
        gconv, = ctx.saved_tensors
        c = gconv.shape[1]
        dgc = _compact(dgrid, c, h // 2, w // 2, what="the gradient of grid_encoder")
        ps.dg_pad = torch.empty(ps.n * (h + 2) * (w + 2), c, dtype=torch.bfloat16, device=gconv.device)
        ops.maxpool2x2_relu_bwd(dgc, gconv, ps.dg_pad, ps.n, h, w, c)
        return None, _nchw(ps.dg_pad, ps.n, h, w, bordered=True)


_PASSES = []     # the module-path passes running (GridFeatBackbone._module_forward), innermost last


def _active(module):
    """The module-path pass that is calling ``module``: the backbone's modules run only inside GridFeatBackbone.forward."""
    if not _PASSES:
        raise RuntimeError("%s of GridFeatBackbone runs only inside GridFeatBackbone.forward (call the GridFeatBackbone on (B, T, 3, H, W) "
                           "frames; calling feature.backbone, its stem, stages or blocks directly is not supported)" % type(module).__name__)
    return _PASSES[-1]


class FrozenBatchNorm2d(nn.Module):
    """Parameter container with detectron2's buffer names; applied as scale/shift in GEMM epilogues."""

    def __init__(self, c):
        super().__init__()
        self.register_buffer("weight", torch.ones(c))
        self.register_buffer("bias", torch.zeros(c))
        self.register_buffer("running_mean", torch.zeros(c))
        self.register_buffer("running_var", torch.ones(c))


class ConvBN(nn.Module):
    """d2 ``Conv2d(..., bias=False, norm=FrozenBN)`` parameter container (weight is KCRS like torch)."""

    def __init__(self, cin, cout, k, norm=True):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin, k, k))
        nn.init.kaiming_normal_(self.weight, mode="fan_out", nonlinearity="relu")   # d2 c2_msra_fill
        if norm:
            self.norm = FrozenBatchNorm2d(cout)
        self.cin, self.cout, self.k = cin, cout, k


class BottleneckBlock(nn.Module):
    def __init__(self, cin, mid, cout, stride, has_shortcut):
        super().__init__()
        if has_shortcut:
            self.shortcut = ConvBN(cin, cout, 1)
        self.conv1 = ConvBN(cin, mid, 1)
        self.conv2 = ConvBN(mid, mid, 3)
        self.conv3 = ConvBN(mid, cout, 1)
        self.stride, self.has_shortcut = stride, has_shortcut
        self.cin, self.mid, self.cout = cin, mid, cout
        self.block_name = None    # "res3.1": set by _Backbone

    def forward(self, x):
        """The block output, post-ReLU, (N, cout, h, w): runs when a hook on the CNN selects the module path."""
        return _active(self).block(self, x)


class _Stem(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = ConvBN(3, 64, 7)

    def forward(self, x):
        """The pooled stem output (N, 64, H/4, W/4) of (N, 3, H, W) frames (RGB, as GridFeatBackbone.forward was given them)."""
        return _active(self).stem(x)


class _Backbone(nn.Module):
    def __init__(self):
        super().__init__()
        self.stem = _Stem()
        cin = 64
        for name, nblocks, mid, cout, stride in RESNET50_STAGES:
            blocks = []
            for b in range(nblocks):
                blocks.append(BottleneckBlock(cin, mid, cout, stride if b == 0 else 1, b == 0))
                blocks[-1].block_name = "%s.%d" % (name, b)
                cin = cout
            setattr(self, name, nn.Sequential(*blocks))

    def forward(self, x):
        """d2's backbone with OUT_FEATURES [res5]: {"res5": (N, 2048, H/32, W/32)}."""
        _active(self)
        x = self.stem(x)
        for name, *_r in RESNET50_STAGES:
            x = getattr(self, name)(x)
        return {"res5": x}


class _Feature(nn.Module):
    """Stands in for the d2 GeneralizedRCNN: only ``backbone`` exists (RPN / ROI heads are dead
    parameters on this path, SURVEY.md §0.10, and are neither allocated nor all-reduced)."""

    def __init__(self):
        super().__init__()
        self.backbone = _Backbone()


class _GridEncoderConv(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin, 3, 3))
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))      # nn.Conv2d default (grid_feat.py:19-21)
        self.cin, self.cout, self.k = cin, cout, 3

    def forward(self, x):
        """The 3x3 conv output (N, cout, h, w), before the pool and the ReLU."""
        return _active(self).grid_conv(x)


class _GridEncoder(nn.Sequential):
    """grid_encoder: its conv is child 0 (key grid_encoder.0.weight); MaxPool2d(2, 2) and ReLU, which hold no parameters, run fused
    after it. Returns the grid (N, cout, h/2, w/2)."""

    def forward(self, x):
        return _active(self).grid_pool(self[0](x))


class _CnnFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, images, anchor):
        grid, stash = module._forward_impl(images, need_backward=True, frames_grad=ctx.needs_input_grad[1])
        module._pending_backward += 1
        ctx.module = module
        ctx.stash = stash
        ctx.frames = (images.shape, images.dtype)
        return grid

    @staticmethod
    def backward(ctx, dgrid):
        stash, ctx.stash = ctx.stash, None
        m = ctx.module
        m._pending_backward = max(0, m._pending_backward - 1)
        dx = None
        if stash is not None:
            dx = m._backward_impl(stash, dgrid, last=m._pending_backward == 0)
        if dx is not None:
            shape, dtype = ctx.frames
            dx = dx.view(shape).to(dtype)
        return None, dx, None


class GridFeatBackbone(nn.Module):
    """``model.recompute_activations = True`` (default False) trades compute for activation memory, as wrapping each ResNet stage
    in ``torch.utils.checkpoint`` does on the reference: a pass that records autograd keeps only each stage's input (the pooled
    stem output for res2, the previous stage's output for the others) instead of every block's activations, and the backward
    re-runs the stage's blocks from it, with the forward's launches, just before that stage's backward. One stage's activations
    are alive at a time; the gradients are bit-identical to the switch off in deterministic mode. Refused together with hooks on
    the CNN's modules (the module path keeps every block's activations as its nodes' saved tensors)."""

    recompute_activations = False

    def __init__(self, detectron2_model_cfg=None, config=None, input_format="BGR", freeze_at=2):
        super().__init__()
        assert input_format == "BGR", "detectron 2 image input format should be BGR"
        hidden = getattr(config, "hidden_size", 768) if config is not None else 768
        cin = getattr(config, "backbone_channel_in_size", 2048) if config is not None else 2048
        self.feature = _Feature()
        self.grid_encoder = _GridEncoder(_GridEncoderConv(cin, hidden))   # key: grid_encoder.0.weight
        self.input_format = input_format
        self.config = config
        self.freeze_at = freeze_at
        self.detectron2_model_cfg = detectron2_model_cfg
        self._flat = None
        self._bn = None
        self._dirty = True
        self._capture = None     # tests set this to a dict to receive per-stage / per-block activations (and, in backward, gradients)
        self._inject = None      # tests: {"res5.2": NHWC activation} makes that block start from the given tensor
        self._pending_backward = 0
        self._bucket_hook = None   # data-parallel: called as hook(flat_grad, first_finished_element, side_stream) mid-backward
        self._segments = None
        self._pad_pool = {}
        self._sites = None       # (name, module) of every module of feature.backbone and grid_encoder: where hooks are looked for
        self.pixel_mean = None   # set to (r,g,b) to take uint8 frames and fuse ImageNorm into the stem gather
        self.raw_float_inputs = False   # True: fp32 frames are RAW (0..255) and get the fused ImageNorm too (input_stage.set_image_norm)
        self.pixel_std = None    # (r,g,b) of ImageNorm's div_(std) (data_utils.py:276): folded into the stem conv weights at pack time
        self.stem_mode = "s2d"   # "s2d": space-to-depth implicit GEMM (no patch matrix); "im2col": patch gather + GEMM
        self._s2d_ld = 16        # 16: overlapping tensor-map rows; 64: explicit windows (set automatically if the driver refuses)
        self._optimizer_emits_packed = False   # FusedAdamW writes the bf16 operands itself (clipbert_b200/optim.py)
        # d2 FREEZE_AT: stem (1) and res2 (2) get no gradient
        if freeze_at < 1:
            # the reference ships FREEZE_AT: 2 (Base-RCNN-grid.yaml) and only ever freezes more (freeze_cnn_backbone); the
            # stem's weight gradient (7x7 wgrad over the patch matrix) is not built, and silently returning no gradient is worse
            raise NotImplementedError("GridFeatBackbone: FREEZE_AT = 0 (trainable stem) is not supported on the H100 path")
        bb = self.feature.backbone
        if freeze_at >= 1:
            for p in bb.stem.parameters():
                p.requires_grad = False
        for si, (name, *_r) in enumerate(RESNET50_STAGES):
            if freeze_at >= si + 2:
                for p in getattr(bb, name).parameters():
                    p.requires_grad = False

    # ---- reference API surface ------------------------------------------------------------------
    @property
    def config_file(self):
        return _D2_CONFIG_TEXT % self.freeze_at

    def load_state_dict(self, state_dict, strict=False, **kw):
        """``GridFeatBackbone.load_state_dict(path)`` in the reference (src/modeling/grid_feat.py:72-80) hands a checkpoint PATH to
        d2's DetectionCheckpointer: ``.pth`` or the MSRA ``R-50.pkl`` pickles, d2 key names relative to ``feature``. A dict is
        taken as a state dict (module keys, bare d2 keys, or ``cnn.``-prefixed). Shapes must match; keys of the dead d2 heads are
        ignored and returned in ``.ignored``. A missing path is an error that names it."""
        import os

        from . import load_save
        if isinstance(state_dict, (str, bytes, os.PathLike)):
            if not os.path.exists(state_dict):
                raise FileNotFoundError("GridFeatBackbone.load_state_dict: checkpoint %r does not exist (the reference falls back to the d2 "
                                        "config's MODEL.WEIGHTS URL, which this offline path cannot download)" % (state_dict,))
        loaded, ignored = load_save.load_detectron2_checkpoint(self, state_dict)
        self._dirty = True
        missing = sorted(k for k in self.state_dict() if k not in loaded)
        if strict and missing:
            raise RuntimeError("GridFeatBackbone.load_state_dict: missing keys %s" % missing[:8])
        return torch.nn.modules.module._IncompatibleKeys(missing, ignored)

    def mark_weights_updated(self):
        self._dirty = True

    # ---- internals --------------------------------------------------------------------------------
    def _convs(self):
        """Ordered (name, module, has_norm)."""
        bb = self.feature.backbone
        out = [("stem.conv1", bb.stem.conv1)]
        for name, *_r in RESNET50_STAGES:
            for bi, blk in enumerate(getattr(bb, name)):
                if blk.has_shortcut:
                    out.append(("%s.%d.shortcut" % (name, bi), blk.shortcut))
                out.append(("%s.%d.conv1" % (name, bi), blk.conv1))
                out.append(("%s.%d.conv2" % (name, bi), blk.conv2))
                out.append(("%s.%d.conv3" % (name, bi), blk.conv3))
        out.append(("grid_encoder.0", self.grid_encoder[0]))
        return out

    def _any_trainable(self):
        return any(m.weight.requires_grad for _, m in self._convs())

    def _ensure_ready(self, device):
        if self._flat is None or not self._flat.is_current() or self._flat.device != device:
            flat = FlatGroup(device)
            for name, m in self._convs():
                m._e = flat.add(name, m.weight, kind="conv")
            flat.materialize()
            self._flat = flat
            # FrozenBN buffers in four flat vectors so that scale/shift are 4 elementwise ops in total
            convs = [m for _, m in self._convs() if hasattr(m, "norm")]
            ctot = sum(m.cout for m in convs)
            bufs = {k: torch.empty(ctot, dtype=torch.float32, device=device) for k in ("weight", "bias", "running_mean", "running_var")}
            off = 0
            for m in convs:
                for k in bufs:
                    v = bufs[k][off: off + m.cout]
                    v.copy_(getattr(m.norm, k).to(device))
                    setattr(m.norm, k, v)          # buffers become views (state_dict keys unchanged)
                m._bn_off = off
                off += m.cout
            self._bn = bufs
            self._bn_scale = torch.empty(ctot, dtype=torch.float32, device=device)
            self._bn_shift = torch.empty(ctot, dtype=torch.float32, device=device)
            self._stem_w = torch.zeros(64, STEM_KP, dtype=torch.bfloat16, device=device)
            self._stem_w_s2d = torch.zeros(64, 256, dtype=torch.bfloat16, device=device)
            self._segments = None
            self._pad_pool = {}
            self._dirty = True
        if self._dirty or self._flat.needs_repack():
            self._repack()
            self._dirty = False
            self._flat.needs_repack()

    @torch.no_grad()
    def _repack(self):
        """fp32 masters -> bf16 KRSC operands with the FrozenBN scale folded in (runs when weights change)."""
        b = self._bn
        torch.rsqrt(b["running_var"] + FROZEN_BN_EPS, out=self._bn_scale)
        self._bn_scale.mul_(b["weight"])
        torch.addcmul(b["bias"], b["running_mean"], self._bn_scale, value=-1.0, out=self._bn_shift)
        flat = self._flat
        if self._segments is None:
            rows = []
            for name, m in self._convs():
                e = m._e
                rows.append([e["offset"], e["numel"], m.k * m.k * m.cin, m._bn_off if hasattr(m, "norm") else -1])
            self._segments = torch.tensor(rows, dtype=torch.int64, device=flat.master.device)
        ops.cast_scale_segments(flat.master, flat.packed, self._segments, self._bn_scale)     # all 54 convs, one launch
        for name, m in self._convs():
            e = m._e
            n = e["numel"]
            row_len = m.k * m.k * m.cin
            if hasattr(m, "norm"):
                m._scale, m._shift = self._bn_scale[m._bn_off: m._bn_off + m.cout], self._bn_shift[m._bn_off: m._bn_off + m.cout]
            else:
                m._scale = m._shift = None
            m._w = flat.packed[e["offset"]: e["offset"] + n].view(m.cout, row_len)
            m._gw = flat.grad[e["offset"]: e["offset"] + n].view(m.cout, row_len)
        stem = self.feature.backbone.stem.conv1
        if self.pixel_std is not None and any(float(v) != 1.0 for v in self.pixel_std):
            # conv(w, (x - mean) / std) == conv(w / std[c], x - mean): ImageNorm's division lives in the (frozen) stem weights, so the
            # gather kernel only subtracts the mean. Input channels of the stem are in BGR order (grid_feat.py:92-94).
            e = stem._e
            w32 = flat.master[e["offset"]: e["offset"] + e["numel"]].view(64, 49, 3) * self._bn_scale[stem._bn_off: stem._bn_off + 64].view(64, 1, 1)
            r, g, b_ = (float(v) for v in self.pixel_std)
            inv = torch.tensor([1.0 / b_, 1.0 / g, 1.0 / r], dtype=torch.float32, device=w32.device)
            stem._w.copy_((w32 * inv).reshape(64, 147))
        self._stem_w[:, :147] = stem._w      # [64, (r,s,c)] -> row pitch 152
        self._pack_stem_s2d(stem._w)
        stem._w = self._stem_w

    # ---- FusedAdamW hooks (clipbert_b200/optim.py) -------------------------------------------------
    def optimizer_segments(self):
        """Per conv weight: where its bf16 operand lives and which FrozenBN scale row-block folds into it."""
        return [dict(param=m.weight, row_len=m.k * m.k * m.cin, scale_off=m._bn_off if hasattr(m, "norm") else -1, emit=True)
                for _, m in self._convs()]

    def optimizer_scales(self):
        return self._bn_scale

    def packed_written_by_optimizer(self):
        """The optimizer kernel refreshed ``_flat.packed`` for every trainable conv: no re-cast on the next forward."""
        stem = self.feature.backbone.stem.conv1
        if stem.weight.requires_grad:       # FREEZE_AT = 0 only: the stem GEMM reads a 152-pitch copy
            e = stem._e
            self._stem_w[:, :147] = self._flat.packed[e["offset"]: e["offset"] + e["numel"]].view(64, 147)
            self._pack_stem_s2d(self._stem_w[:, :147])
        self._dirty = False
        self._flat.needs_repack()

    def _pack_stem_s2d(self, w147):
        """[64, (r, s, c)] 7x7x3 (BN scale folded) -> [64, (r', x', dy, dx, c4)] = [64, 256] for the space-to-depth stem:
        kernel zero-extended to 8x8x4, row r = 2r' + dy, column s = 2x' + dx (see cb_stem_s2d in the C header)."""
        w = torch.zeros(64, 8, 8, 4, dtype=w147.dtype, device=w147.device)
        w[:, :7, :7, :3] = w147.reshape(64, 7, 7, 3)
        self._stem_w_s2d.copy_(w.view(64, 4, 2, 4, 2, 4).permute(0, 1, 3, 2, 4, 5).reshape(64, 256))

    # ---- zero-bordered buffers --------------------------------------------------------------------
    # Only interior rows of a padded activation are ever written (CB_ROWMAP_PAD epilogues), so a buffer that was
    # zeroed once keeps a valid zero border for its whole life: recycle instead of re-zeroing every step. Which rows
    # are border depends on (n, h, w), not on the row count alone (1 x 6 x 6 and 4 x 2 x 2 both pad to 64 rows), so
    # the pool is keyed by the full geometry.
    def _pad_get(self, n, h, w, ch, device):
        lst = self._pad_pool.setdefault((n, h, w, ch), [])
        return lst.pop() if lst else torch.zeros(n * (h + 2) * (w + 2), ch, dtype=torch.bfloat16, device=device)

    def _pad_put(self, t, n, h, w):
        assert t.shape[0] == n * (h + 2) * (w + 2)
        self._pad_pool.setdefault((n, h, w, t.shape[1]), []).append(t)

    # ---- forward ----------------------------------------------------------------------------------
    def forward(self, x):
        """x: (B, T, 3, H, W) RGB, float (mean-subtracted) or uint8 if ``pixel_mean`` is set."""
        _require_cuda(x)
        self._ensure_ready(x.device)
        if self._hooked():
            if self.recompute_activations and torch.is_grad_enabled():
                raise RuntimeError("GridFeatBackbone: recompute_activations cannot be combined with hooks on the CNN's modules: the "
                                   "module path keeps every block's activations for its nodes' backward; remove the hooks or turn "
                                   "the switch off")
            return self._module_forward(x)
        if not (torch.is_grad_enabled() and (x.requires_grad or self._any_trainable())):
            return self._forward_impl(x, need_backward=False)[0]
        # a trainable parameter is passed only as an autograd anchor so that backward is scheduled; frames that require grad
        # (pixel attribution, attacks on the input) anchor the node themselves and receive d grid / d frames
        anchor = next((m.weight for _, m in self._convs() if m.weight.requires_grad), None)
        return _CnnFn.apply(self, x, anchor)

    # ---- module path: hooks on the backbone's modules ------------------------------------------------
    def _hook_sites(self):
        if self._sites is None:
            self._sites = ([("feature.backbone." + k if k else "feature.backbone", v) for k, v in self.feature.backbone.named_modules()]
                           + [("grid_encoder." + k if k else "grid_encoder", v) for k, v in self.grid_encoder.named_modules()])
        return self._sites

    def _hooked(self):
        """Whether a hook is registered on a module of the CNN (or a global module hook): the forward then runs the modules. Raises
        for hooks that cannot be honoured."""
        g = torch.nn.modules.module
        found = any(getattr(g, k, None) for k in ("_global_forward_hooks", "_global_forward_pre_hooks", "_global_backward_hooks",
                                                  "_global_backward_pre_hooks"))
        bb = self.feature.backbone
        for name, mod in self._hook_sites():
            if not (mod._forward_hooks or mod._forward_pre_hooks or mod._backward_hooks or mod._backward_pre_hooks):
                continue
            if isinstance(mod, (ConvBN, FrozenBatchNorm2d)):
                raise RuntimeError("GridFeatBackbone: hooks on %s are not supported: a convolution's output before the block's ReLU "
                                   "is fused into its GEMM epilogue and never exists in memory; hook the block instead" % name)
            if mod._forward_pre_hooks and (mod is bb or mod is bb.stem):
                raise RuntimeError("GridFeatBackbone: forward pre-hooks on %s are not supported: the frames it receives are the "
                                   "(N, 3, H, W) RGB frames, not the reference's BGR tensor" % name)
            found = True
        if found and self._bucket_hook is not None:
            raise RuntimeError("GridFeatBackbone: hooks on the CNN's modules are for analysis, not data-parallel training: they cannot "
                               "run while the overlapped gradient exchange (enable_overlapped_allreduce) is enabled")
        return found

    def _module_forward(self, x):
        """forward() through the modules, so that torch's hooks on them fire: feature.backbone -> stem -> res2..res5 -> blocks,
        then grid_encoder -> grid_encoder[0]. The same launches as the default path, plus one cb_nhwc_intake wherever a hook
        hands over a tensor that is not already in the engine's layout."""
        bsz, n_frms, c, h, w = x.shape
        ps = _CnnPass(self, bsz * n_frms)
        _PASSES.append(ps)
        try:
            feats = self.feature.backbone(x.reshape(bsz * n_frms, c, h, w))
            grid = self.grid_encoder(feats["res5"])
        finally:
            _PASSES.pop()
        return grid.reshape(bsz, n_frms, *grid.shape[1:]).permute(0, 1, 3, 4, 2)

    @contextlib.contextmanager
    def _node_backward(self, grads):
        """Around the backward of one module-path node: the flat gradient buffer attached and the bf16 operands due a repack when
        it writes parameter gradients, its side-queue weight gradients joined before it returns (a partial backward may run no
        later node), its scratch buffers back to the pool after the join."""
        sq = ops.SideQueue()
        recycle = []
        try:
            if grads:
                self._flat.attach_grads()
            yield sq, recycle
            if grads and not self._optimizer_emits_packed:
                self._dirty = True
        finally:
            sq.join()
            for t, tn, th, tw in recycle:
                self._pad_put(t, tn, th, tw)

    def _conv1x1(self, m, x, rows, act, residual=None, rowmap=ops.ROWMAP_NONE, hw=None, out=None):
        if out is None:
            out = torch.empty(rows, m.cout, dtype=torch.bfloat16, device=x.device)
        kw = dict(mode=ops.CB_GEMM_TN, m=rows, n=m.cout, k=m.cin, a=x, a_rows=rows, a_ld=m.cin, b=m._w, b_rows=m.cout,
                  b_ld=m.cin, shift=m._shift, act=act, out=out, out_ld=m.cout, rowmap=rowmap)
        if residual is not None:
            kw.update(residual=residual, res_ld=m.cout)
        if hw is not None:
            kw.update(map_h=hw[0], map_w=hw[1])
        ops.gemm(**kw)
        return out

    def _conv3x3(self, m, x_pad, n, h, w, act):
        """x_pad: [n, h+2, w+2, cin] zero-bordered; returns compact [n*h*w, cout]."""
        p = n * (h + 2) * (w + 2)
        out = torch.empty(n * h * w, m.cout, dtype=torch.bfloat16, device=x_pad.device)
        ops.gemm(mode=ops.CB_GEMM_TN, m=p, n=m.cout, k=m.cin, a=x_pad, a_rows=p, a_ld=m.cin, b=m._w, b_rows=m.cout,
                 b_ld=9 * m.cin, ntaps=9, tap_w=w + 2, tap_sign=1, shift=m._shift, act=act, out=out, out_ld=m.cout,
                 rowmap=ops.ROWMAP_UNPAD, map_h=h, map_w=w)
        return out

    def _forward_impl(self, images, need_backward, frames_grad=False):
        """``frames_grad``: the backward also computes the gradient with respect to the frames, so the stem output and every
        block's activations (frozen blocks too) are kept. With ``recompute_activations`` the stash keeps each such stage's input
        instead of its blocks' activations (``stages``); _backward_impl re-runs the blocks."""
        bsz, n_frms, c, h, w = images.shape
        assert c == 3
        n = bsz * n_frms
        cur, frames, hh, ww = self._stem_forward(images.reshape(n, c, h, w), need_backward and frames_grad)
        recompute = need_backward and self.recompute_activations
        # ---- res2..res5 ----
        blocks, stages = [], []
        bb = self.feature.backbone
        stage_names = [s[0] for s in RESNET50_STAGES]
        for si, name in enumerate(stage_names):
            stage = getattr(bb, name)
            for bi, blk in enumerate(stage):
                last = (si == len(stage_names) - 1) and (bi == len(stage) - 1)
                cur = self._injected(name, bi, cur, n, hh, ww)
                if bi == 0:
                    stage_in = dict(name=name, x=cur, h=hh, w=ww)
                st = self._block_forward(blk, cur, n, hh, ww, last)
                hh, ww = st["h"], st["w"]
                keep = need_backward and (st["trainable"] or frames is not None)     # a frozen block's dgrad chain leads to the frames
                if not keep or recompute:
                    self._pad_put(st["a_pad"], n, hh, ww)     # consumed by conv2 above; stream order makes the reuse safe
                else:
                    blocks.append(st)
                if keep and recompute and bi == 0:
                    stages.append(stage_in)
                cur = st["y"]
            if self._capture is not None:
                self._capture[name] = (cur.view(n, hh + 2, ww + 2, -1)[:, 1:-1, 1:-1] if name == "res5" else cur.view(n, hh, ww, -1))
        # ---- grid_encoder: conv3x3 (no norm) -> maxpool 2x2 -> ReLU ----
        ge = self.grid_encoder[0]
        gconv = self._conv3x3(ge, cur, n, hh, ww, ops.ACT_NONE)
        gh, gw = hh // 2, ww // 2
        grid = torch.empty(bsz, n_frms, gh, gw, ge.cout, dtype=torch.bfloat16, device=cur.device)
        ops.maxpool2x2_relu_fwd(gconv, grid, n, hh, ww, ge.cout)
        if self._capture is not None:
            self._capture["gconv"] = gconv
        stash = None
        if not need_backward:
            self._pad_put(cur, n, hh, ww)           # res5 output (padded), consumed by the grid_encoder conv
        if need_backward:
            stash = dict(n=n, h=hh, w=ww, res5_pad=cur, gconv=gconv, blocks=blocks, stages=stages, frames=frames)
            if self._capture is not None:
                self._capture["stash"] = stash
        return grid, stash

    def _injected(self, name, bi, cur, n, h, w):
        """The input of block name.bi: cur, or the NHWC activation a test injected there (layer-local parity: both implementations
        see the same input)."""
        key = "%s.%d" % (name, bi)
        if self._inject is None or key not in self._inject:
            return cur
        return self._inject[key].to(device=cur.device, dtype=torch.bfloat16).reshape(n * h * w, -1).contiguous()

    def _recompute_stage(self, sg, n):
        """The activations of one stage's blocks as _block_forward returned them in the forward, re-run from the stage's kept
        input with the same launches (recompute_activations). The last block's conv3 is not re-run: its output is the next stage's
        kept input, or res5_pad, and no block backward reads a block's own output."""
        blocks = []
        cur, hh, ww = sg["x"], sg["h"], sg["w"]
        stage = getattr(self.feature.backbone, sg["name"])
        for bi, blk in enumerate(stage):
            cur = self._injected(sg["name"], bi, cur, n, hh, ww)
            st = self._block_forward(blk, cur, n, hh, ww, blk.block_name == RESNET50_LAST_BLOCK, need_y=bi < len(stage) - 1)
            hh, ww, cur = st["h"], st["w"], st["y"]
            blocks.append(st)
        return blocks

    def _stem_forward(self, x, keep_frames):
        """x: (n, 3, h, w) frames. Returns (pooled stem output, compact [n*hh*ww, 64]; what the frame gradient needs when
        keep_frames, else None; hh; ww)."""
        dev = x.device
        n, c, h, w = x.shape
        if x.dtype == torch.uint8 or self.raw_float_inputs:
            # raw frames (uint8, or the fp32 output of input_stage.resize_pad): ImageNorm is fused - mean in the stem gather, 1 / std in
            # the stem weights. Float frames are otherwise taken as already normalised (what the reference's PrefetchLoader hands over).
            assert self.pixel_mean is not None, "raw frames need pixel_mean (fused ImageNorm)"
            mean = tuple(float(v) for v in self.pixel_mean)
            x = x if x.dtype in (torch.uint8, torch.float32) else x.float()
        else:
            x = x.float() if x.dtype != torch.float32 else x
            mean = (0.0, 0.0, 0.0)
        x = x.contiguous()
        bb = self.feature.backbone
        bf16 = torch.bfloat16
        # ---- stem: 7x7/s2 conv (+BN shift, ReLU) -> maxpool 3x3/s2 ----
        ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        hh, ww = (ho - 1) // 2 + 1, (wo - 1) // 2 + 1
        stem = bb.stem.conv1
        cur = torch.empty(n * hh * ww, 64, dtype=bf16, device=dev)
        mode = self.stem_mode
        if mode == "s2d":
            # space-to-depth frame (no patch matrix) -> 4-row-tap wgmma GEMM over its overlapping 64-element rows; the
            # output keeps the (ho+3) x (wo+3) grid of the s2d frame, the pool reads it with those pitches
            hs, ws = ho + 3, wo + 3
            rows = n * hs * ws
            ld = self._s2d_ld
            s2d = torch.empty((rows + 4) * ld, dtype=bf16, device=dev)        # + slack: the last rows' windows run past the frame
            ops.stem_s2d(x, s2d, n, h, w, ld, mean)
            c1 = torch.empty(rows, 64, dtype=bf16, device=dev)
            kw = dict(mode=ops.CB_GEMM_TN, m=rows, n=64, k=64, a=s2d, a_rows=rows, a_ld=ld, b=self._stem_w_s2d, b_rows=64, b_ld=256,
                      ntaps=4, tap_w=ws, tap_sign=1, shift=stem._shift, act=ops.ACT_RELU, out=c1, out_ld=64)
            try:
                ops.gemm(**kw)
            except RuntimeError as e:      # a driver that rejects overlapping tensor-map rows: store the windows explicitly
                if ld == 64 or "cuTensorMapEncodeTiled" not in str(e):
                    raise
                self._s2d_ld = ld = 64
                s2d = torch.empty((rows + 4) * ld, dtype=bf16, device=dev)
                ops.stem_s2d(x, s2d, n, h, w, ld, mean)
                ops.gemm(**dict(kw, a=s2d, a_ld=ld))
            del s2d
            pitch = (ws, hs * ws)
            ops.maxpool3x3s2(c1, cur, n, ho, wo, 64, row_pitch=ws, img_pitch=hs * ws)
            if self._capture is not None:
                self._capture["c1"] = c1.view(n, hs, ws, 64)[:, :ho, :wo]     # the pool's view of the s2d output grid
        else:
            # im2col gather (BGR flip + cast fused) -> GEMM over the [pixels, 152] patch matrix
            col = torch.empty(n * ho * wo, STEM_KP, dtype=bf16, device=dev)
            ops.stem_im2col(x, col, n, h, w, STEM_KP, mean)
            c1 = torch.empty(n * ho * wo, 64, dtype=bf16, device=dev)
            ops.gemm(mode=ops.CB_GEMM_TN, m=n * ho * wo, n=64, k=STEM_KP, a=col, a_rows=n * ho * wo, a_ld=STEM_KP, b=stem._w,
                     b_rows=64, b_ld=STEM_KP, shift=stem._shift, act=ops.ACT_RELU, out=c1, out_ld=64)
            del col
            pitch = (None, None)
            ops.maxpool3x3s2(c1, cur, n, ho, wo, 64)
            if self._capture is not None:
                self._capture["c1"] = c1.view(n, ho, wo, 64)
        frames = dict(c1=c1, pitch=pitch, ho=ho, wo=wo, h=h, w=w) if keep_frames else None
        del c1
        if self._capture is not None:
            self._capture["stem"] = cur.view(n, hh, ww, 64)
        return cur, frames, hh, ww

    def _block_forward(self, blk, x_in, n, h_in, w_in, last, need_y=True):
        """One bottleneck block from x_in (compact [n*h_in*w_in, cin]). Its output y is compact, or zero-bordered for the last
        block (the grid_encoder conv reads it); need_y = False (a recompute whose output is kept elsewhere): no shortcut and
        conv3 launches, y None. Returns the block's activations as its backward reads them."""
        dev, bf16 = x_in.device, torch.bfloat16
        hh, ww = h_in, w_in
        if blk.stride == 2:
            hh, ww = (hh - 1) // 2 + 1, (ww - 1) // 2 + 1
            xs = torch.empty(n * hh * ww, blk.cin, dtype=bf16, device=dev)
            ops.subsample2(x_in, xs, n, h_in, w_in, blk.cin)
        else:
            xs = x_in
        rows = n * hh * ww
        sc = self._conv1x1(blk.shortcut, xs, rows, ops.ACT_NONE) if blk.has_shortcut and need_y else xs
        a_pad = self._pad_get(n, hh, ww, blk.mid, dev)
        self._conv1x1(blk.conv1, xs, rows, ops.ACT_RELU, rowmap=ops.ROWMAP_PAD, hw=(hh, ww), out=a_pad)
        b = self._conv3x3(blk.conv2, a_pad, n, hh, ww, ops.ACT_RELU)
        if not need_y:
            return dict(name=blk.block_name, blk=blk, x_in=x_in, xs=xs, a_pad=a_pad, b=b, y=None, h=hh, w=ww, h_in=h_in, w_in=w_in,
                        trainable=blk.conv1.weight.requires_grad)
        if last:
            y = self._pad_get(n, hh, ww, blk.cout, dev)
            self._conv1x1(blk.conv3, b, rows, ops.ACT_RELU, residual=sc, rowmap=ops.ROWMAP_PAD, hw=(hh, ww), out=y)
        else:
            y = self._conv1x1(blk.conv3, b, rows, ops.ACT_RELU, residual=sc)
        if self._capture is not None:
            # clones of the pooled buffers: the pool hands them to a later call
            self._capture[blk.block_name] = dict(xs=xs, sc=sc, a_pad=a_pad.clone(), b=b, y=y.clone() if last else y)
        return dict(name=blk.block_name, blk=blk, x_in=x_in, xs=xs, a_pad=a_pad, b=b, y=y, h=hh, w=ww, h_in=h_in, w_in=w_in,
                    trainable=blk.conv1.weight.requires_grad)

    # ---- backward ---------------------------------------------------------------------------------
    def _wgrad_kw(self, m, dy, x, p, ntaps=1, tap_w=0):
        """dW[cout, t*cin + c] += scale[cout] * sum_p dy[p, cout] * x[p + shift_t, c]."""
        return dict(mode=ops.CB_GEMM_WGRAD, m=m.cout, n=m.cin, k=p, a=dy, a_rows=p, a_ld=m.cout, b=x, b_rows=p, b_ld=m.cin,
                    ntaps=ntaps, tap_w=tap_w, tap_sign=1, scale=m._scale, out=m._gw, out_ld=ntaps * m.cin, out_fp32=1)

    def _wgrad(self, m, dy, x, p, ntaps=1, tap_w=0):
        ops.gemm(**self._wgrad_kw(m, dy, x, p, ntaps, tap_w))

    def _dgrad1x1(self, m, dy, rows, residual=None, aux=None, rowmap=ops.ROWMAP_NONE, hw=None, out=None, mask=True):
        """dx[rows, cin] = dy[rows, cout] @ w'[cout, cin]  (+residual) (* relu mask of aux; not applied when mask is False)."""
        if out is None:
            out = torch.empty(rows, m.cin, dtype=torch.bfloat16, device=dy.device)
        kw = dict(mode=ops.CB_GEMM_NN, m=rows, n=m.cin, k=m.cout, a=dy, a_rows=rows, a_ld=m.cout, b=m._w, b_rows=m.cout,
                  b_ld=m.cin, out=out, out_ld=m.cin, rowmap=rowmap)
        if residual is not None:
            kw.update(residual=residual, res_ld=m.cin)
        if aux is not None:
            kw.update(aux=aux, aux_ld=m.cin, aux_mode=ops.AUX_RELU_MASK)
        if hw is not None:
            kw.update(map_h=hw[0], map_w=hw[1])
        ops.gemm(**(kw if mask else _unmasked(kw)))
        return out

    def _dgrad3x3(self, m, dy_pad, n, h, w, aux_pad, mask=True):
        p = n * (h + 2) * (w + 2)
        out = torch.empty(n * h * w, m.cin, dtype=torch.bfloat16, device=dy_pad.device)
        kw = dict(mode=ops.CB_GEMM_NN, m=p, n=m.cin, k=m.cout, a=dy_pad, a_rows=p, a_ld=m.cout, b=m._w, b_rows=m.cout,
                  b_ld=9 * m.cin, ntaps=9, tap_w=w + 2, tap_sign=-1, aux=aux_pad, aux_ld=m.cin, aux_mode=ops.AUX_RELU_MASK,
                  out=out, out_ld=m.cin, rowmap=ops.ROWMAP_UNPAD, map_h=h, map_w=w)
        ops.gemm(**(kw if mask else _unmasked(kw)))
        return out

    def _backward_impl(self, stash, dgrid, last=True):
        """``last``: no other backward of this step is outstanding (the reference's per-clip loop runs one per clip and the
        gradients accumulate), so a finished slice of the gradient buffer may be handed to ``_bucket_hook`` early."""
        self._flat.attach_grads()
        dev = dgrid.device
        bf16 = torch.bfloat16
        n, h, w = stash["n"], stash["h"], stash["w"]
        ge = self.grid_encoder[0]
        dgrid = dgrid.to(bf16).contiguous()
        p = n * (h + 2) * (w + 2)
        # wgrad GEMMs run on the side queue beside the dgrad chain; zero-bordered buffers they read go back to the pool
        # only after the join at the end (a recycled buffer would be overwritten by a later main-stream launch)
        sq = ops.SideQueue()
        recycle = []          # (zero-bordered buffer, n, h, w)
        cap = None if self._capture is None else self._capture.setdefault("bwd", {})
        dg_pad = torch.empty(p, ge.cout, dtype=bf16, device=dev)
        ops.maxpool2x2_relu_bwd(dgrid, stash["gconv"], dg_pad, n, h, w, ge.cout)
        res5_pad = stash["res5_pad"]
        recycle.append((res5_pad, n, h, w))
        if cap is not None:
            cap["grid_encoder"] = dict(dg_pad=dg_pad)
        blocks = stash["blocks"]
        stages = stash["stages"]
        frames = stash["frames"]
        g = self._grid_conv_backward(dg_pad, res5_pad, n, h, w, sq, ge.weight.requires_grad, bool(blocks or stages))
        del dg_pad
        if stages:
            # recompute_activations: top-down, each stage's blocks re-run from its kept input, then its backward. The join makes
            # the main stream wait for the stage's weight gradients, the last readers of its activations, before those are
            # released; the next stage then recomputes into that memory. Of the stage's zero-bordered buffers (a_pad, db_pad of
            # each block) the pool keeps one, the buffer the next forward reuses block by block; the others go back to the
            # allocator, since no other stage has their geometry, and the next backward allocates them zeroed again
            for sg in reversed(stages):
                blocks = self._recompute_stage(sg, n)
                stage_recycle = []
                g = self._blocks_backward(blocks, g, n, sq, stage_recycle, cap, frames, last, lowest=sg is stages[0])
                sq.join()
                for t, tn, th, tw in stage_recycle:
                    if not self._pad_pool.get((tn, th, tw, t.shape[1])):
                        self._pad_put(t, tn, th, tw)
                del blocks, stage_recycle
        else:
            g = self._blocks_backward(blocks, g, n, sq, recycle, cap, frames, last, lowest=True)
        dx = None
        if frames is not None:
            dx = self._stem_backward(g, frames, n, cap)
        sq.join()
        for t, tn, th, tw in recycle:
            self._pad_put(t, tn, th, tw)
        if not self._optimizer_emits_packed and self._any_trainable():
            self._dirty = True   # an optimizer step normally follows: repack bf16 operands on the next forward
        return dx

    def _blocks_backward(self, blocks, g, n, sq, recycle, cap, frames, last, lowest):
        """The backward of consecutive blocks, top-down from g; returns the gradient below the first of them, or None when none
        is needed. ``lowest``: blocks[0] is the lowest block that runs a backward."""
        for st in reversed(blocks):
            bucket = None
            if st["trainable"] and last and self._bucket_hook is not None and st["name"] == "res5.0":
                # every weight gradient of res5 + grid_encoder (78 % of the CNN's trainable parameters, the tail of the
                # flat buffer) has been enqueued: its exchange can overlap the res4 / res3 backward
                bucket = lambda blk=st["blk"]: self._bucket_hook(self._flat.grad, blk.shortcut._e["offset"], sq.side if sq.forked else None)  # noqa: E731
            # d2 FREEZE_AT: no gradient below the lowest block, unless it leads to the frames
            need_dx = not (lowest and st is blocks[0]) or (st["blk"].has_shortcut and frames is not None)
            gin = self._block_backward(st, g, n, sq, recycle, cap=cap, need_dx=need_dx, bucket=bucket)
            recycle.append((st["a_pad"], n, st["h"], st["w"]))
            if gin is None:
                return None
            g = gin
        return g

    def _grid_conv_backward(self, dg_pad, res5_pad, n, h, w, sq, wgrad, need_dx, mask=True):
        """grid_encoder conv from dg_pad (zero-bordered gradient at its output): its weight gradient on the side queue (wgrad) and
        the gradient at the res5 output, compact (need_dx), masked by res5's ReLU' unless mask is False."""
        ge = self.grid_encoder[0]
        if wgrad:
            sq.run(lambda: self._wgrad(ge, dg_pad, res5_pad, n * (h + 2) * (w + 2), ntaps=9, tap_w=w + 2), dg_pad, res5_pad)
        return self._dgrad3x3(ge, dg_pad, n, h, w, res5_pad, mask=mask) if need_dx else None

    def _block_backward(self, st, g, n, sq, recycle, cap=None, wgrad=True, need_dx=True, mask=True, bucket=None):
        """One bottleneck block's backward from g, the gradient at its pre-ReLU output (compact). Enqueues its weight gradients
        on the side queue (wgrad, trainable blocks) and returns the gradient at its input: for res2.0 the gradient at the stem's
        pooled output (the pool's backward applies the stem's ReLU'), otherwise the gradient at the previous block's pre-ReLU
        output, masked by that block's ReLU' (mask) or not (the module path: the previous block's node applies it). None
        unless need_dx. ``bucket`` is called once the weight gradients of a block with a shortcut are enqueued."""
        blk, hh, ww = st["blk"], st["h"], st["w"]
        dev, bf16 = g.device, torch.bfloat16
        rows = n * hh * ww
        pp = n * (hh + 2) * (ww + 2)
        db_pad = self._pad_get(n, hh, ww, blk.mid, dev)
        recycle.append((db_pad, n, hh, ww))
        self._dgrad1x1(blk.conv3, g, rows, aux=st["b"], rowmap=ops.ROWMAP_PAD, hw=(hh, ww), out=db_pad)
        da = self._dgrad3x3(blk.conv2, db_pad, n, hh, ww, st["a_pad"])
        c = None
        if cap is not None:
            cap[st["name"]] = c = dict(g=g, db_pad=db_pad.clone(), da=da)
        if wgrad and st["trainable"]:
            # the block's three / four weight gradients as ONE grouped launch on the side queue, issued when its last dY (da) exists
            wg = [self._wgrad_kw(blk.conv3, g, st["b"], rows), self._wgrad_kw(blk.conv2, db_pad, st["a_pad"], pp, ntaps=9, tap_w=ww + 2),
                  self._wgrad_kw(blk.conv1, da, st["xs"], rows)]
            if blk.has_shortcut:
                wg.append(self._wgrad_kw(blk.shortcut, g, st["xs"], rows))
            if ops.group_wgrad in (1, 2, 4):
                sq.run(lambda: ops.gemm_wgrad_group(wg), g, st["b"], db_pad, st["a_pad"], da, st["xs"])
            else:
                sq.run(lambda: [ops.gemm(**kw) for kw in wg], g, st["b"], db_pad, st["a_pad"], da, st["xs"])
        if not blk.has_shortcut:
            if not need_dx:
                return None
            gin = self._dgrad1x1(blk.conv1, da, rows, residual=g, aux=st["x_in"], mask=mask)
            if c is not None:
                c.update(gin=gin)
            return gin
        if bucket is not None:
            bucket()
        if not need_dx:
            return None
        dxs_sc = self._dgrad1x1(blk.shortcut, g, rows)
        dxs = self._dgrad1x1(blk.conv1, da, rows, residual=dxs_sc)
        if c is not None:
            c.update(dxs_sc=dxs_sc, dxs=dxs)
        if st["name"] == "res2.0":
            return dxs
        if blk.stride == 2:
            gin = torch.empty(n * st["h_in"] * st["w_in"], blk.cin, dtype=bf16, device=dev)
            ops.unsubsample2_mask(dxs, st["x_in"] if mask else None, gin, n, st["h_in"], st["w_in"], blk.cin)
        elif mask:
            gin = torch.empty(n * st["h_in"] * st["w_in"], blk.cin, dtype=bf16, device=dev)
            ops.relu_mask(dxs, st["x_in"], gin)
        else:
            gin = dxs
        if c is not None:
            c.update(gin=gin)
        return gin

    def _stem_backward(self, g, frames, n, cap=None):
        """The frame gradient, fp32 (n, 3, h, w), from g, the gradient at the stem's pooled output (compact): the pool (+ ReLU')
        to the conv output, then the transposed 7x7/s2 conv to the frames."""
        ho, wo = frames["ho"], frames["wo"]
        dc1 = torch.empty(n * ho * wo, 64, dtype=torch.bfloat16, device=g.device)
        ops.maxpool3x3s2_bwd(g, frames["c1"], dc1, n, ho, wo, 64, *frames["pitch"])
        dx = torch.empty(n, 3, frames["h"], frames["w"], dtype=torch.float32, device=g.device)
        ops.stem_dgrad(dc1, self._stem_w, dx, n, frames["h"], frames["w"])
        if cap is not None:
            cap["stem"] = dict(dpool=g, dc1=dc1, dx=dx)
        return dx
