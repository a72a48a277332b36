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
import math

import torch
from torch import nn

from . import ops
from .params import FlatGroup

RESNET50_STAGES = (("res2", 3, 64, 256, 1), ("res3", 4, 128, 512, 2), ("res4", 6, 256, 1024, 2), ("res5", 3, 512, 2048, 2))
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


class _Stem(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = ConvBN(3, 64, 7)


class _Backbone(nn.Module):
    def __init__(self):
        super().__init__()
        self.stem = _Stem()
        cin = 64
        for name, nblocks, mid, cout, stride in RESNET50_STAGES:
            blocks = []
            for b in range(nblocks):
                blocks.append(BottleneckBlock(cin, mid, cout, stride if b == 0 else 1, b == 0))
                cin = cout
            setattr(self, name, nn.Sequential(*blocks))


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
    def __init__(self, detectron2_model_cfg=None, config=None, input_format="BGR", freeze_at=2):
        super().__init__()
        assert input_format == "BGR", "detectron 2 image input format should be BGR"
        hidden = getattr(config, "hidden_size", 768) if config is not None else 768
        cin = getattr(config, "backbone_channel_in_size", 2048) if config is not None else 2048
        self.feature = _Feature()
        self.grid_encoder = nn.Sequential(_GridEncoderConv(cin, hidden))   # key: grid_encoder.0.weight
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
        if not (torch.is_grad_enabled() and (x.requires_grad or self._any_trainable())):
            return self._forward_impl(x, need_backward=False)[0]
        # a trainable parameter is passed only as an autograd anchor so that backward is scheduled; frames that require grad
        # (pixel attribution, attacks on the input) anchor the node themselves and receive d grid / d frames
        anchor = next((m.weight for _, m in self._convs() if m.weight.requires_grad), None)
        return _CnnFn.apply(self, x, anchor)

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
        block's activations (frozen blocks too) are kept."""
        dev = images.device
        bsz, n_frms, c, h, w = images.shape
        assert c == 3
        n = bsz * n_frms
        x = images.reshape(n, c, h, w)
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
        frames = dict(c1=c1, pitch=pitch, ho=ho, wo=wo, h=h, w=w) if need_backward and frames_grad else None
        del c1
        if self._capture is not None:
            self._capture["stem"] = cur.view(n, hh, ww, 64)
        # ---- res2..res5 ----
        blocks = []
        stage_names = [s[0] for s in RESNET50_STAGES]
        for si, name in enumerate(stage_names):
            stage = getattr(bb, name)
            for bi, blk in enumerate(stage):
                last = (si == len(stage_names) - 1) and (bi == len(stage) - 1)
                if self._inject is not None and ("%s.%d" % (name, bi)) in self._inject:
                    # test hook: this block starts from a given NHWC activation (layer-local parity: both implementations see the same input)
                    cur = self._inject["%s.%d" % (name, bi)].to(device=dev, dtype=bf16).reshape(n * hh * ww, -1).contiguous()
                x_in, h_in, w_in = cur, hh, ww
                if blk.stride == 2:
                    hh, ww = (hh - 1) // 2 + 1, (ww - 1) // 2 + 1
                    xs = torch.empty(n * hh * ww, blk.cin, dtype=bf16, device=dev)
                    ops.subsample2(x_in, xs, n, h_in, w_in, blk.cin)
                else:
                    xs = x_in
                rows = n * hh * ww
                sc = self._conv1x1(blk.shortcut, xs, rows, ops.ACT_NONE) if blk.has_shortcut else xs
                a_pad = self._pad_get(n, hh, ww, blk.mid, dev)
                self._conv1x1(blk.conv1, xs, rows, ops.ACT_RELU, rowmap=ops.ROWMAP_PAD, hw=(hh, ww), out=a_pad)
                b = self._conv3x3(blk.conv2, a_pad, n, hh, ww, ops.ACT_RELU)
                if last:
                    y = self._pad_get(n, hh, ww, blk.cout, dev)
                    self._conv1x1(blk.conv3, b, rows, ops.ACT_RELU, residual=sc, rowmap=ops.ROWMAP_PAD, hw=(hh, ww), out=y)
                else:
                    y = self._conv1x1(blk.conv3, b, rows, ops.ACT_RELU, residual=sc)
                if self._capture is not None:
                    # clones of the pooled buffers: the pool hands them to a later call
                    self._capture["%s.%d" % (name, bi)] = dict(xs=xs, sc=sc, a_pad=a_pad.clone(), b=b, y=y.clone() if last else y)
                trainable = blk.conv1.weight.requires_grad
                keep = need_backward and (trainable or frames is not None)     # a frozen block's dgrad chain leads to the frames
                if not keep:
                    self._pad_put(a_pad, n, hh, ww)     # consumed by conv2 above; stream order makes the reuse safe
                else:
                    blocks.append(dict(name="%s.%d" % (name, bi), blk=blk, x_in=x_in, xs=xs, a_pad=a_pad, b=b, y=y, h=hh, w=ww, h_in=h_in, w_in=w_in,
                                       trainable=trainable))
                cur = y
            if self._capture is not None:
                self._capture[name] = (cur.view(n, hh + 2, ww + 2, -1)[:, 1:-1, 1:-1] if name == "res5" else cur.view(n, hh, ww, -1))
        # ---- grid_encoder: conv3x3 (no norm) -> maxpool 2x2 -> ReLU ----
        ge = self.grid_encoder[0]
        gconv = self._conv3x3(ge, cur, n, hh, ww, ops.ACT_NONE)
        gh, gw = hh // 2, ww // 2
        grid = torch.empty(bsz, n_frms, gh, gw, ge.cout, dtype=bf16, device=dev)
        ops.maxpool2x2_relu_fwd(gconv, grid, n, hh, ww, ge.cout)
        if self._capture is not None:
            self._capture["gconv"] = gconv
        stash = None
        if not need_backward:
            self._pad_put(cur, n, hh, ww)           # res5 output (padded), consumed by the grid_encoder conv
        if need_backward:
            stash = dict(n=n, h=hh, w=ww, res5_pad=cur, gconv=gconv, blocks=blocks, frames=frames)
            if self._capture is not None:
                self._capture["stash"] = stash
        return grid, stash

    # ---- backward ---------------------------------------------------------------------------------
    def _wgrad_kw(self, m, dy, x, p, ntaps=1, tap_w=0):
        """dW[cout, t*cin + c] += scale[cout] * sum_p dy[p, cout] * x[p + shift_t, c]."""
        return dict(mode=ops.CB_GEMM_WGRAD, m=m.cout, n=m.cin, k=p, a=dy, a_rows=p, a_ld=m.cout, b=x, b_rows=p, b_ld=m.cin,
                    ntaps=ntaps, tap_w=tap_w, tap_sign=1, scale=m._scale, out=m._gw, out_ld=ntaps * m.cin, out_fp32=1)

    def _wgrad(self, m, dy, x, p, ntaps=1, tap_w=0):
        ops.gemm(**self._wgrad_kw(m, dy, x, p, ntaps, tap_w))

    def _dgrad1x1(self, m, dy, rows, residual=None, aux=None, rowmap=ops.ROWMAP_NONE, hw=None, out=None):
        """dx[rows, cin] = dy[rows, cout] @ w'[cout, cin]  (+residual) (* relu mask of aux)."""
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
        ops.gemm(**kw)
        return out

    def _dgrad3x3(self, m, dy_pad, n, h, w, aux_pad):
        p = n * (h + 2) * (w + 2)
        out = torch.empty(n * h * w, m.cin, dtype=torch.bfloat16, device=dy_pad.device)
        ops.gemm(mode=ops.CB_GEMM_NN, m=p, n=m.cin, k=m.cout, a=dy_pad, a_rows=p, a_ld=m.cout, b=m._w, b_rows=m.cout,
                 b_ld=9 * m.cin, ntaps=9, tap_w=w + 2, tap_sign=-1, aux=aux_pad, aux_ld=m.cin, aux_mode=ops.AUX_RELU_MASK,
                 out=out, out_ld=m.cin, rowmap=ops.ROWMAP_UNPAD, map_h=h, map_w=w)
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
        if ge.weight.requires_grad:
            sq.run(lambda: self._wgrad(ge, dg_pad, res5_pad, p, ntaps=9, tap_w=w + 2), dg_pad, res5_pad)
        blocks = stash["blocks"]
        frames = stash["frames"]
        if blocks:
            # grad w.r.t. the pre-ReLU output of the last block, compact
            g = self._dgrad3x3(ge, dg_pad, n, h, w, res5_pad)
        del dg_pad
        for st in reversed(blocks):
            blk, hh, ww = st["blk"], st["h"], st["w"]
            rows = n * hh * ww
            pp = n * (hh + 2) * (ww + 2)
            lowest = st is blocks[0]
            db_pad = self._pad_get(n, hh, ww, blk.mid, dev)
            recycle += [(db_pad, n, hh, ww), (st["a_pad"], n, hh, ww)]
            self._dgrad1x1(blk.conv3, g, rows, aux=st["b"], rowmap=ops.ROWMAP_PAD, hw=(hh, ww), out=db_pad)
            da = self._dgrad3x3(blk.conv2, db_pad, n, hh, ww, st["a_pad"])
            if cap is not None:
                cap[st["name"]] = c = dict(g=g, db_pad=db_pad.clone(), da=da)
            if st["trainable"]:
                # the block's three / four weight gradients as ONE grouped launch on the side queue, issued when its last dY (da) exists
                wg = [self._wgrad_kw(blk.conv3, g, st["b"], rows), self._wgrad_kw(blk.conv2, db_pad, st["a_pad"], pp, ntaps=9, tap_w=ww + 2),
                      self._wgrad_kw(blk.conv1, da, st["xs"], rows)]
                if blk.has_shortcut:
                    wg.append(self._wgrad_kw(blk.shortcut, g, st["xs"], rows))
                if ops.group_wgrad in (1, 2, 4):
                    sq.run(lambda: ops.gemm_wgrad_group(wg), g, st["b"], db_pad, st["a_pad"], da, st["xs"])
                else:
                    sq.run(lambda: [ops.gemm(**kw) for kw in wg], g, st["b"], db_pad, st["a_pad"], da, st["xs"])
            if blk.has_shortcut:
                if st["trainable"] and last and self._bucket_hook is not None and st["name"] == "res5.0":
                    # every weight gradient of res5 + grid_encoder (78 % of the CNN's trainable parameters, the tail of the
                    # flat buffer) has been enqueued: its exchange can overlap the res4 / res3 backward
                    self._bucket_hook(self._flat.grad, blk.shortcut._e["offset"], sq.side if sq.forked else None)
                if lowest and frames is None:
                    break                                     # d2 FREEZE_AT: no gradient below this block
                dxs_sc = self._dgrad1x1(blk.shortcut, g, rows)
                dxs = self._dgrad1x1(blk.conv1, da, rows, residual=dxs_sc)
                if lowest:
                    # res2.0 reads the stem's pooled output: dxs is the gradient at the pool output, whose backward applies the
                    # stem's ReLU' itself (a pooled value is > 0 exactly where the element it selects is)
                    g = dxs
                    if cap is not None:
                        c.update(dxs_sc=dxs_sc, dxs=dxs)
                    break
                g = torch.empty(n * st["h_in"] * st["w_in"], blk.cin, dtype=bf16, device=dev)
                if blk.stride == 2:
                    ops.unsubsample2_mask(dxs, st["x_in"], g, n, st["h_in"], st["w_in"], blk.cin)
                else:
                    ops.relu_mask(dxs, st["x_in"], g)
                if cap is not None:
                    c.update(dxs_sc=dxs_sc, dxs=dxs, gin=g)
            else:
                if lowest:
                    break
                g = self._dgrad1x1(blk.conv1, da, rows, residual=g, aux=st["x_in"])
                if cap is not None:
                    c.update(gin=g)
        dx = None
        if frames is not None:
            # stem backward: pool (+ ReLU') to the conv output, then the transposed 7x7/s2 conv to the frames
            ho, wo = frames["ho"], frames["wo"]
            dc1 = torch.empty(n * ho * wo, 64, dtype=bf16, device=dev)
            ops.maxpool3x3s2_bwd(g, frames["c1"], dc1, n, ho, wo, 64, *frames["pitch"])
            dx = torch.empty(n, 3, frames["h"], frames["w"], dtype=torch.float32, device=dev)
            ops.stem_dgrad(dc1, self._stem_w, dx, n, frames["h"], frames["w"])
            if cap is not None:
                cap["stem"] = dict(dpool=g, dc1=dc1, dx=dx)
        sq.join()
        for t, tn, th, tw in recycle:
            self._pad_put(t, tn, th, tw)
        if not self._optimizer_emits_packed and self._any_trainable():
            self._dirty = True   # an optimizer step normally follows: repack bf16 operands on the next forward
        return dx
