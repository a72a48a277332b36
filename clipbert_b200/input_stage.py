"""The frame pre-processing of the reference's data pipeline on the GPU (SURVEY.md §8 f3).

  reference (CPU tensors in the dataset worker, then the PrefetchLoader)          here
  ------------------------------------------------------------------------------  --------------------------------------------
  ImageResize(max_img_size, "bilinear")      src/datasets/data_utils.py:202-234   resize_pad(): one kernel, uint8 or fp32 in,
  ImagePad(max_img_size, max_img_size)       src/datasets/data_utils.py:136-160       fp32 (n, 3, S, S) out (cb_resize_pad);
                                                                                      differentiable (cb_resize_pad_bwd)
  ImageNorm(mean, std): (x - mean) / std     src/datasets/data_utils.py:256-276   fused into the stem: ``cnn.pixel_mean`` is
  x[:, [2, 1, 0]] BGR flip                   src/modeling/grid_feat.py:92-94          subtracted in the stem gather, ``cnn.pixel_std``
                                                                                      is folded into the stem conv weights

Host logic (``get_resize_size`` / ``get_padding``) follows the reference exactly: the longer side becomes ``max_size``, the
shorter ``int(max_size * short / long)``, the frame stays in the upper-left corner.
"""
import torch

from . import ops


def get_resize_size(height, width, max_size):
    """src/datasets/data_utils.py:166-198 for tensors (note its (h, w) order)."""
    if height >= width:
        new_height, new_width = max_size, max_size * (width * 1.0 / height)
    else:
        new_width, new_height = max_size, max_size * (height * 1.0 / width)
    return int(new_height), int(new_width)


def _require_cuda(t):
    assert t.is_cuda, "the input stage runs on CUDA only (no CPU fallback)"


def _resize_pad(frames, max_size):
    x = frames.contiguous()
    nh, nw = get_resize_size(x.shape[-2], x.shape[-1], max_size)
    out = torch.empty(tuple(x.shape[:-2]) + (max_size, max_size), dtype=torch.float32, device=x.device)
    ops.resize_pad(x, out, nh, nw)
    return out, (nh, nw)


class _ResizePad(torch.autograd.Function):
    """cb_resize_pad, with cb_resize_pad_bwd (its exact adjoint) as the backward: d loss / d frames at their decoded size."""

    @staticmethod
    def forward(ctx, frames, max_size):
        out, ctx.size = _resize_pad(frames, max_size)
        ctx.shape = frames.shape
        return out

    @staticmethod
    def backward(ctx, dy):
        dx = torch.empty(ctx.shape, dtype=torch.float32, device=dy.device)
        ops.resize_pad_bwd(dy.contiguous(), dx, *ctx.size)
        return dx, None


def resize_pad(frames, max_size):
    """``frames``: (..., 3, H, W) uint8 or fp32 CUDA tensor. Returns fp32 (..., 3, max_size, max_size): ImageResize(max_size)
    followed by ImagePad(max_size, max_size) - bilinear, align_corners=False, zeros at the bottom / right.

    Differentiable, as in the reference: when grad mode is on and fp32 ``frames`` require grad, the result carries an autograd
    node whose backward (cb_resize_pad_bwd) returns d loss / d frames in the frames' own (..., 3, H, W) shape, so gradients
    reach the decoded pixels (saliency at the original resolution, attacks clipped in raw pixel space). Otherwise this is the
    one forward launch and nothing else."""
    _require_cuda(frames)
    assert frames.dtype in (torch.uint8, torch.float32) and frames.dim() >= 3
    if torch.is_grad_enabled() and frames.requires_grad:
        return _ResizePad.apply(frames, max_size)
    return _resize_pad(frames, max_size)[0]


def set_image_norm(model_or_cnn, mean, std=(1.0, 1.0, 1.0), raw_float_inputs=True):
    """``ImageNorm(mean, std)`` fused into the backbone: the model then takes RAW RGB frames - uint8, and (``raw_float_inputs``)
    the fp32 0..255 frames ``resize_pad`` produces; with ``raw_float_inputs=False`` float frames keep meaning "already
    normalised", as in the reference. ``mean`` / ``std`` are the config's ``img_pixel_mean`` / ``img_pixel_std`` (0-255 scale in
    every shipped config)."""
    cnn = getattr(model_or_cnn, "cnn", model_or_cnn)
    cnn.pixel_mean = tuple(float(v) for v in mean)
    cnn.pixel_std = tuple(float(v) for v in std)
    cnn.raw_float_inputs = bool(raw_float_inputs)
    cnn.mark_weights_updated()
    return cnn
