"""Thin Python wrappers over the C ABI (include/clipbert_b200.h). Each function takes CUDA torch
tensors (used only as device buffers), validates the few things the C side cannot see (dtype,
contiguity, device) and enqueues the kernel on the current torch stream. No arithmetic happens in
Python or in torch on this path.
"""
import ctypes

import torch

from . import _lib as L
from ._lib import (ACT_GELU, ACT_GELU_STASH_GRAD, ACT_NONE, ACT_RELU, ACT_TANH, AUX_GELU_GRAD, AUX_MUL, AUX_NONE,  # noqa: F401
                   AUX_RELU_MASK, AUX_TANH_GRAD, CB_GEMM_TN, CB_GEMM_WGRAD, ROWMAP_NONE, ROWMAP_PAD, ROWMAP_UNPAD)

CB_GEMM_NN = 2
GEMM_FORCE_WIDE = 1 << 12   # cb_gemm_desc.reserved: TN / NN on 128 x 256 tiles (CB_GEMM_FORCE_WIDE)
GEMM_NO_WIDE = 1 << 13      # ... never on 128 x 256 tiles (CB_GEMM_NO_WIDE)
_c = ctypes
_vp, _i, _i64, _f, _u64 = _c.c_void_p, _c.c_int, _c.c_int64, _c.c_float, _c.c_uint64

_SIGS = {
    "cb_layernorm_fwd": [_vp, _vp, _vp, _vp, _vp, _i, _i, _f, _vp],
    "cb_layernorm_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _f, _u64, _vp],
    "cb_embed_text_fwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _f, _u64, _vp],
    "cb_embed_text_bwd": [_vp] * 12 + [_i, _i, _i, _i, _i, _f, _u64, _vp],
    "cb_embed_visual_fwd": [_vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _f, _f, _u64, _vp],
    "cb_embed_visual_bwd": [_vp, _vp, _vp, _vp, _i] + [_vp] * 12 + [_i, _i, _i, _i, _i, _i, _i, _i, _f, _u64, _vp],
    "cb_colsum": [_vp, _i64, _vp, _i, _i, _vp],
    "cb_dropout": [_vp, _vp, _i64, _f, _u64, _vp],
    "cb_dropout_offset_advance": [_vp, _vp, _vp],
    "cb_gelu_bwd": [_vp, _vp, _vp, _i64, _vp],
    "cb_pad_cast": [_vp, _i64, _vp, _i, _i, _i, _vp],
    "cb_cast_scale": [_vp, _vp, _i64, _vp, _i64, _vp],
    "cb_cast_bf16_f32": [_vp, _vp, _i64, _vp],
    "cb_cast_scale_segments": [_vp, _vp, _vp, _i, _vp, _vp],
    "cb_nvls_allreduce_f32": [_vp, _i64, _i, _i, _f, _i, _vp],
    "cb_clip_lse_loss": [_vp, _vp, _vp, _vp, _i, _i, _i, _f, _vp],
    "cb_clip_pool_ce_loss": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _vp],
    "cb_cross_entropy_fwd": [_vp, _i64, _vp, _vp, _vp, _i64, _i, _i64, _vp],
    "cb_cross_entropy_bwd": [_vp, _i64, _vp, _vp, _vp, _vp, _i64, _i64, _i, _i64, _vp],
    "cb_attention_fwd": [_vp, _i64, _vp, _vp, _i64, _vp, _i, _i, _i, _i, _i, _f, _u64, _vp],
    "cb_attention_bwd": [_vp, _i64, _vp, _vp, _vp, _i64, _vp, _vp, _i64, _i, _i, _i, _i, _i, _f, _u64, _vp],
    "cb_attention_probs": [_vp, _i64, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _u64, _vp],
    "cb_attention_probs_bwd": [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _i, _f, _u64, _vp],
    "cb_attention_dprobs": [_vp, _i64, _vp, _i64, _vp, _i, _i, _i, _i, _i, _vp],
    "cb_attention_probs_bwd_store": [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _i, _f, _u64, _vp],
    "cb_attention_bwd_dv": [_vp, _i64, _vp, _vp, _vp, _i64, _vp, _i64, _i, _i, _i, _i, _i, _f, _u64, _vp],
    "cb_stem_im2col": [_vp, _i, _vp, _i, _i, _i, _i, _f, _f, _f, _vp],
    "cb_maxpool3x3s2": [_vp, _vp, _i, _i, _i, _i, _vp],
    "cb_maxpool3x3s2_strided": [_vp, _vp, _i, _i, _i, _i, _i64, _i64, _vp],
    "cb_maxpool3x3s2_bwd": [_vp, _vp, _vp, _i, _i, _i, _i, _vp],
    "cb_maxpool3x3s2_bwd_strided": [_vp, _vp, _vp, _i, _i, _i, _i, _i64, _i64, _vp],
    "cb_stem_dgrad": [_vp, _vp, _i, _vp, _i, _i, _i, _vp],
    "cb_stem_s2d": [_vp, _i, _vp, _i, _i, _i, _i, _f, _f, _f, _vp],
    "cb_resize_pad": [_vp, _i, _vp, _i, _i, _i, _i, _i, _i, _vp],
    "cb_resize_pad_bwd": [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp],
    "cb_subsample2": [_vp, _vp, _i, _i, _i, _i, _vp],
    "cb_unsubsample2_mask": [_vp, _vp, _vp, _i, _i, _i, _i, _vp],
    "cb_maxpool2x2_relu_fwd": [_vp, _vp, _i, _i, _i, _i, _vp],
    "cb_maxpool2x2_relu_bwd": [_vp, _vp, _vp, _i, _i, _i, _i, _vp],
    "cb_relu_mask": [_vp, _vp, _vp, _i64, _vp],
    "cb_embed_text_fwd_vectors": [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _f, _u64, _vp],
    "cb_embed_text_bwd_vectors": [_vp, _vp, _i64] + [_vp] * 9 + [_i, _i, _i, _i, _f, _u64, _vp],
    "cb_embed_word_scatter": [_vp, _vp, _vp, _i, _i, _i, _vp],
    "cb_nhwc_intake": [_vp, _i, _i64, _i64, _i64, _i64, _i, _i, _i, _i, _vp, _i, _vp, _i, _vp],
    # deterministic variants: the arguments of the plain entry point, then (scratch, scratch_bytes) before the stream
    "cb_layernorm_bwd_det": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _f, _u64, _vp, _i64, _vp],
    "cb_embed_text_bwd_det": [_vp] * 12 + [_i, _i, _i, _i, _i, _f, _u64, _vp, _i64, _vp],
    "cb_embed_text_bwd_vectors_det": [_vp, _vp, _i64] + [_vp] * 9 + [_i, _i, _i, _i, _f, _u64, _vp, _i64, _vp],
    "cb_embed_visual_bwd_det": [_vp, _vp, _vp, _vp, _i] + [_vp] * 12 + [_i, _i, _i, _i, _i, _i, _i, _i, _f, _u64, _vp, _i64, _vp],
    "cb_colsum_det": [_vp, _i64, _vp, _i, _i, _vp, _i64, _vp],
    "cb_clip_lse_loss_det": [_vp, _vp, _vp, _vp, _i, _i, _i, _f, _vp, _i64, _vp],
    "cb_clip_pool_ce_loss_det": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _vp, _i64, _vp],
    "cb_sumsq_det": [_vp, _i64, _vp, _i, _vp, _vp, _i64, _vp],
    # scratch-size queries (int64 results)
    "cb_layernorm_bwd_scratch_bytes": [_i],
    "cb_embed_text_bwd_scratch_bytes": [_i, _i],
    "cb_embed_text_bwd_vectors_scratch_bytes": [_i, _i],
    "cb_embed_visual_bwd_scratch_bytes": [_i, _i, _i],
    "cb_colsum_scratch_bytes": [_i, _i],
    "cb_clip_loss_scratch_bytes": [_i],
    "cb_sumsq_scratch_bytes": [_i64, _vp, _i],
}
_bound = {}


def _fn(name):
    f = _bound.get(name)
    if f is None:
        f = getattr(L.lib(), name)
        f.argtypes = _SIGS[name]
        f.restype = _c.c_int64 if name.endswith("_scratch_bytes") else _c.c_int
        _bound[name] = f
    return f


def _p(t):
    return None if t is None else t.data_ptr()


def _s():
    return torch.cuda.current_stream().cuda_stream


_op_timing = None


def set_op_timing(events):
    """Profiling hook: when ``events`` is a list, EVERY kernel launch made through this module is bracketed by
    CUDA events on the launch stream and (label, start, end) is appended. None disables."""
    global _op_timing
    _op_timing = events


def _call(name, *args):
    if _op_timing is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    rc = _fn(name)(*args)
    if rc != 0:
        raise RuntimeError("%s failed (%d): %s" % (name, rc, L.lib().cb_last_error().decode()))
    if _op_timing is not None:
        e1.record()
        _op_timing.append((name, e0, e1))


def launch_count():
    return int(L.lib().cb_launch_count())


def set_attention_flash(on):
    """Forward attention of sequences longer than 64 tokens: 1 (default) = tensor-core online-softmax kernel, 0 = the
    CUDA-core kernel."""
    L.lib().cb_debug_attention_flash(int(bool(on)))


def set_attention_flash_pipe(on):
    """Long-sequence attention forward: 1 (default) = key / value tiles double-buffered through cp.async, 0 = synchronous loads (A/B)."""
    L.lib().cb_debug_attention_flash_pipe(int(bool(on)))


def set_attention_rows48(on):
    """Attention of sequences of up to 48 tokens (L = 41: every 224-px configuration): 1 (default) = 48-row tiles, three warps per
    (sequence, head); 0 = the 64-row / four-warp kernels (A/B)."""
    L.lib().cb_debug_attention_rows48(int(bool(on)))


def set_mn3d(on):
    """MN-major GEMM operands (B of the dgrad mode, both operands of the wgrad mode) through ONE 3-D TMA box per k-chunk
    (default) instead of BN/64 2-D boxes (the single producer lane issues 2 instead of 5-6 TMA instructions per chunk)."""
    L.lib().cb_debug_gemm_mn3d(int(bool(on)))


def set_occ2(mode, max_gflop=0.0):
    """Accepted for compatibility and ignored: every GEMM runs one CTA per SM. Weight gradients used to have a two-CTAs-per-SM
    instantiation (128 x 64 tiles); once their wgmma were pipelined it was slower than one CTA per SM on every weight-gradient
    shape of the training step, and it was removed."""
    f = L.lib().cb_debug_gemm_occ2
    f.argtypes = [ctypes.c_int, ctypes.c_double]
    f.restype = None
    f(int(mode), float(max_gflop))


# ------------------------------------------------------------------------------------------------
# dropout stream position on the device (fresh masks under CUDA-graph replay)
# ------------------------------------------------------------------------------------------------
def dropout_offset_bind(word):
    """Launches made after this call add the uint64 device word ``word`` (a 1-element int64 tensor; None unbinds), read when
    they RUN, into their dropout seed - see cb_dropout_offset_bind."""
    f = L.lib().cb_dropout_offset_bind
    f.argtypes = [_vp]
    f.restype = _c.c_int
    f(None if word is None else word.data_ptr())


def dropout_offset_advance(counter, snapshot=None):
    """++counter on the device (stream-ordered, graph-capturable); snapshot <- the new value."""
    _call("cb_dropout_offset_advance", _p(counter), _p(snapshot), _s())


def set_sm_limit(n):
    """Tuning hook: cap the persistent GEMM grid at ``n`` CTAs (0 = every SM): leaves SMs to a co-resident NCCL kernel so
    that the static tile schedule does not spill into a second wave while a gradient all-reduce overlaps the backward."""
    L.lib().cb_debug_gemm_sm_limit(int(n))


def set_pdl(enable):
    """Programmatic dependent launch between the library's kernels: 0 off (default), 1 every kernel, 2 every kernel except the
    persistent GEMMs. Returns the previous setting."""
    return int(L.lib().cb_set_pdl(2 if int(enable) == 2 else int(bool(enable))))


# ------------------------------------------------------------------------------------------------
# deterministic mode: torch.use_deterministic_algorithms(True) makes every accumulation run in a fixed order
# ------------------------------------------------------------------------------------------------
_lib_deterministic = False


def set_deterministic(on):
    """cb_set_deterministic: the library's mode (weight-gradient K-split plan and workspace; the atomic entry points refuse).
    Returns the previous setting. The wrappers below keep it equal to torch's flag; see ``deterministic``."""
    return bool(L.lib().cb_set_deterministic(int(bool(on))))


def deterministic():
    """torch.are_deterministic_algorithms_enabled(), mirrored into the library when it changes. Every wrapper that accumulates
    reads it when it issues its launches, so the flag in force while a pass (forward, backward, optimizer step, CUDA-graph
    capture) issues its launches decides how they accumulate."""
    global _lib_deterministic
    on = torch.are_deterministic_algorithms_enabled()
    if on != _lib_deterministic:
        set_deterministic(on)
        _lib_deterministic = on
    return on


def _scratch(nbytes, like):
    """fp32 scratch of at least nbytes from the caching allocator, on the current (launch) stream: when the caller drops it the
    allocator hands the block only to later work on that stream, which runs after the launches that use it."""
    return torch.empty(max(4, (int(nbytes) + 3) // 4), dtype=torch.float32, device=like.device)


def _scratch_args(nbytes, like):
    t = _scratch(nbytes, like)
    return t, t.numel() * 4


# ------------------------------------------------------------------------------------------------
# side queue: weight-gradient work off the backward critical path
# ------------------------------------------------------------------------------------------------
class SideQueue:
    """Runs launches that nothing downstream in the backward pass waits for (wgrad GEMMs, bias column sums) on a second
    CUDA stream, forked from / joined back into the current stream with events, so that they fill SMs the dgrad chain
    leaves idle (grids below one CTA per SM, tails, the LayerNorm / attention kernels between GEMMs). Works under CUDA-graph
    capture (fork/join become graph edges). Operands are kept referenced until ``join()`` so the caching allocator cannot
    hand their memory to a later launch on the main stream while the side stream still reads them."""
    _streams = {}

    def __init__(self, enabled=True):
        self.enabled = bool(enabled) and overlap_wgrad
        self.keep = []
        self.side = None
        self.forked = False

    def _side_stream(self):
        dev = torch.cuda.current_device()
        st = SideQueue._streams.get(dev)
        if st is None:
            st = SideQueue._streams[dev] = torch.cuda.Stream(device=dev)
        return st

    def run(self, fn, *keep):
        if not self.enabled:
            fn()
            return
        if self.side is None:
            self.side = self._side_stream()
        main = torch.cuda.current_stream()
        ev = torch.cuda.Event()
        ev.record(main)
        self.side.wait_event(ev)
        with torch.cuda.stream(self.side):
            fn()
        self.keep.extend(keep)
        self.forked = True

    def join(self):
        if self.forked:
            torch.cuda.current_stream().wait_stream(self.side)
            self.forked = False
        self.keep.clear()


overlap_wgrad = True      # module switch (bench --overlap_wgrad 0 / tests flip it)


# ------------------------------------------------------------------------------------------------
# tensor-core contraction
# ------------------------------------------------------------------------------------------------
_GEMM_PTR_FIELDS = ("a", "b", "scale", "shift", "residual", "aux", "out", "out2", "workspace")
_gemm_timing = None


def set_gemm_timing(events):
    """Profiling hook: when ``events`` is a list, every cb_gemm launch is bracketed by CUDA events
    recorded on the launch stream and the (start, end) pair is appended to it. None disables."""
    global _gemm_timing
    _gemm_timing = events


# Measured launch configurations (tools/autotune_gemm.py on the target GPU -> clipbert_b200/gemm_tuning.json, meant to be
# committed together with the GPU model it was measured on; absent by default): for each GEMM
# shape of the workload the fastest (tile width, wgrad K-split, k-chunks per stage). Shapes that are not in the table use
# the library's analytic model (choose_config in csrc/gemm.cu).
_tuning = None
_gemm_record = None


def gemm_key(kw):
    return "m%d n%d k%d mode%d t%d r%d a%d o%d f%d rm%d act%d" % (
        kw["m"], kw["n"], kw["k"], kw.get("mode", 0), kw.get("ntaps", 1), kw.get("residual") is not None, kw.get("aux") is not None,
        kw.get("out2") is not None, kw.get("out_fp32", 0), kw.get("rowmap", 0), kw.get("act", 0))


def _load_tuning():
    global _tuning
    import json
    import os
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "gemm_tuning.json")
    _tuning = {}
    if os.path.exists(path) and not os.environ.get("CB_NO_TUNING"):
        try:
            _tuning = json.load(open(path)).get("configs", {})
        except Exception:
            _tuning = {}


def _tuned(kw):
    """kw with the tuning table's launch configuration, when it has one for the shape and kw sets none. A TN / NN entry with
    block_n 256 is the 128 x 256 tile (an explicit block_n = 256 means 128 x 128 there)."""
    if _tuning is None:
        _load_tuning()
    if not _tuning or "block_n" in kw or "reserved" in kw:
        return kw
    t = _tuning.get(gemm_key(kw))
    if t is None:
        return kw
    bn, reserved = t[0], (t[2] << 8) | (32 if (len(t) > 3 and t[3]) else 0)
    if bn == 256 and kw.get("mode", CB_GEMM_TN) != CB_GEMM_WGRAD:
        bn, reserved = 0, reserved | GEMM_FORCE_WIDE
    return dict(kw, block_n=bn, split_k=t[1], reserved=reserved)


def _gemm_descs(kws):
    arr = (L.GemmDesc * len(kws))()
    for d, kw in zip(arr, kws):
        d.ntaps = 1
        d.tap_sign = 1
        d.split_k = 0
        for k, v in kw.items():
            if k in _GEMM_PTR_FIELDS:
                v = _p(v) if isinstance(v, torch.Tensor) else v
            setattr(d, k, v)
    return arr


def gemm_tile_width(kw):
    """cb_gemm_tile_width: the tile width cb_gemm runs the descriptor with (TN / NN 256: the 128 x 256 tile), after the tuning
    table as gemm() applies it."""
    return int(L.lib().cb_gemm_tile_width(_gemm_descs([_tuned(kw)])))


def gemm_workspace_bytes(kw):
    """cb_gemm_workspace_bytes: workspace a weight-gradient descriptor needs in deterministic mode (0: one K-split)."""
    return int(L.lib().cb_gemm_workspace_bytes(_gemm_descs([kw])))


def gemm_wgrad_group_plan(kws):
    """cb_gemm_wgrad_group_plan: (tile width, K-split) cb_gemm_wgrad_group runs the problems with, or None when it runs them as
    separate launches."""
    bn, split = _c.c_int(0), _c.c_int(0)
    if L.lib().cb_gemm_wgrad_group_plan(_gemm_descs(kws), len(kws), _c.byref(bn), _c.byref(split)) != 0:
        raise RuntimeError("cb_gemm_wgrad_group_plan failed: %s" % L.lib().cb_last_error().decode())
    return (bn.value, split.value) if bn.value else None


def gemm_wgrad_group_workspace_bytes(kws):
    """cb_gemm_wgrad_group_workspace_bytes: the whole group's workspace (carried by the first descriptor)."""
    return int(L.lib().cb_gemm_wgrad_group_workspace_bytes(_gemm_descs(kws), len(kws)))


def _with_workspace(kw, nbytes):
    if nbytes <= 0:
        return kw
    ws, nb = _scratch_args(nbytes, kw["out"])
    return dict(kw, workspace=ws, workspace_bytes=nb)


def _launch_gemm(name, kws):
    """cb_gemm (one descriptor) or cb_gemm_wgrad_group, with the profiling hooks."""
    arr = _gemm_descs(kws)
    timing = _gemm_timing is not None or _op_timing is not None
    if timing:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    if name == "cb_gemm":
        rc = L.lib().cb_gemm(arr, _s())
    else:
        rc = L.lib().cb_gemm_wgrad_group(arr, len(kws), _s())
    if rc != 0:
        raise RuntimeError("%s failed (%d): %s" % (name, rc, L.lib().cb_last_error().decode()))
    if timing:
        e1.record()
        if _gemm_timing is not None:
            _gemm_timing.append((e0, e1))
        if _op_timing is not None:
            d = arr[0]
            label = ("gemm mode=%d m=%d n=%d k=%d taps=%d res=%d aux=%d o2=%d f32=%d rm=%d" % (
                d.mode, d.m, d.n, d.k, d.ntaps, bool(d.residual), bool(d.aux), bool(d.out2), d.out_fp32, d.rowmap)
                if name == "cb_gemm" else "gemm wgrad group x%d" % len(kws))
            _op_timing.append((label, e0, e1))


def gemm(**kw):
    """cb_gemm with keyword fields of cb_gemm_desc; tensor-valued fields are converted to pointers. A weight gradient in
    deterministic mode gets its split workspace here."""
    if _tuning is None:
        _load_tuning()
    if _gemm_record is not None:
        _gemm_record.append(dict(kw))
    kw = _tuned(kw)
    if kw.get("mode", CB_GEMM_TN) == CB_GEMM_WGRAD and deterministic():
        kw = _with_workspace(kw, gemm_workspace_bytes(kw))
    _launch_gemm("cb_gemm", [kw])


# module switch (bench --group_wgrad): which weight-gradient GEMMs go out as grouped launches. 0 none; 1 BertLayer (4 in one) +
# bottleneck block; 2 bottleneck blocks only; 3 BertLayer only; 4 BertLayer as two pairs (FFN pair as soon as du exists, attention
# pair after dqkv) + bottleneck blocks
group_wgrad = 3


def gemm_wgrad_group(kws):
    """cb_gemm_wgrad_group: the CB_GEMM_WGRAD problems ``kws`` (keyword dicts as for ``gemm``) in one persistent launch."""
    if not kws:
        return
    if len(kws) == 1:
        for kw in kws:
            gemm(**kw)
        return
    if _gemm_record is not None:
        _gemm_record.append(dict(group=[dict(kw) for kw in kws]))
    kws = list(kws)
    if deterministic():
        kws[0] = _with_workspace(kws[0], gemm_wgrad_group_workspace_bytes(kws))
    _launch_gemm("cb_gemm_wgrad_group", kws)


# ------------------------------------------------------------------------------------------------
# BERT-side memory-bound ops
# ------------------------------------------------------------------------------------------------
def layernorm_fwd(x, gamma, beta, y, stats, eps):
    _call("cb_layernorm_fwd", _p(x), _p(gamma), _p(beta), _p(y), _p(stats), x.shape[0], x.shape[1], eps, _s())


def layernorm_bwd(dy, x, stats, gamma, dx, dx_drop, dgamma, dbeta, dbias_drop, p, seed):
    if (dgamma is not None or dbeta is not None or dbias_drop is not None) and deterministic():
        layernorm_bwd_det(dy, x, stats, gamma, dx, dx_drop, dgamma, dbeta, dbias_drop, p, seed,
                          _scratch(layernorm_bwd_scratch_bytes(x.shape[0]), x))
        return
    _call("cb_layernorm_bwd", _p(dy), _p(x), _p(stats), _p(gamma), _p(dx), _p(dx_drop), _p(dgamma), _p(dbeta),
          _p(dbias_drop), x.shape[0], x.shape[1], p, seed, _s())


def layernorm_bwd_scratch_bytes(m):
    return int(_fn("cb_layernorm_bwd_scratch_bytes")(m))


def layernorm_bwd_det(dy, x, stats, gamma, dx, dx_drop, dgamma, dbeta, dbias_drop, p, seed, scratch):
    """cb_layernorm_bwd_det: parameter gradients summed in block order through ``scratch`` (fp32)."""
    _call("cb_layernorm_bwd_det", _p(dy), _p(x), _p(stats), _p(gamma), _p(dx), _p(dx_drop), _p(dgamma), _p(dbeta),
          _p(dbias_drop), x.shape[0], x.shape[1], p, seed, _p(scratch), scratch.numel() * 4, _s())


def embed_text_fwd(ids, word, pos, type0, gamma, beta, out, stats, nseq, lt, l, eps, p, seed):
    _call("cb_embed_text_fwd", _p(ids), _p(word), _p(pos), _p(type0), _p(gamma), _p(beta), _p(out), _p(stats), nseq, lt, l,
          word.shape[0], word.shape[1], eps, p, seed, _s())


def embed_text_bwd(dh, ids, word, pos, type0, gamma, stats, dword, dpos, dtype0, dgamma, dbeta, nseq, lt, l, p, seed):
    if deterministic():
        embed_text_bwd_det(dh, ids, word, pos, type0, gamma, stats, dword, dpos, dtype0, dgamma, dbeta, nseq, lt, l, p, seed,
                           _scratch(embed_text_bwd_scratch_bytes(nseq, lt), dh))
        return
    _call("cb_embed_text_bwd", _p(dh), _p(ids), _p(word), _p(pos), _p(type0), _p(gamma), _p(stats), _p(dword), _p(dpos),
          _p(dtype0), _p(dgamma), _p(dbeta), nseq, lt, l, word.shape[0], word.shape[1], p, seed, _s())


def embed_text_bwd_scratch_bytes(nseq, lt):
    return int(_fn("cb_embed_text_bwd_scratch_bytes")(nseq, lt))


def embed_text_bwd_det(dh, ids, word, pos, type0, gamma, stats, dword, dpos, dtype0, dgamma, dbeta, nseq, lt, l, p, seed, scratch):
    """cb_embed_text_bwd_det: table gradients in block / row order through ``scratch`` (fp32)."""
    _call("cb_embed_text_bwd_det", _p(dh), _p(ids), _p(word), _p(pos), _p(type0), _p(gamma), _p(stats), _p(dword), _p(dpos),
          _p(dtype0), _p(dgamma), _p(dbeta), nseq, lt, l, word.shape[0], word.shape[1], p, seed, _p(scratch), scratch.numel() * 4,
          _s())


def embed_text_fwd_vectors(vec, pos, type0, gamma, beta, out, stats, nseq, lt, l, eps, p, seed):
    """cb_embed_text_fwd_vectors: the text embeddings from fp32 word vectors vec ([nseq * lt, 768] rows, any row pitch)."""
    _call("cb_embed_text_fwd_vectors", _p(vec), vec.stride(0), _p(pos), _p(type0), _p(gamma), _p(beta), _p(out), _p(stats), nseq, lt,
          l, vec.shape[1], eps, p, seed, _s())


def embed_text_bwd_vectors(dh, vec, pos, type0, gamma, stats, dvec, dpos, dtype0, dgamma, dbeta, nseq, lt, l, p, seed):
    """cb_embed_text_bwd_vectors (_det in deterministic mode): dvec[r] (fp32, contiguous) instead of a word-table scatter."""
    if deterministic():
        scratch = _scratch(int(_fn("cb_embed_text_bwd_vectors_scratch_bytes")(nseq, lt)), dh)
        _call("cb_embed_text_bwd_vectors_det", _p(dh), _p(vec), vec.stride(0), _p(pos), _p(type0), _p(gamma), _p(stats), _p(dvec),
              _p(dpos), _p(dtype0), _p(dgamma), _p(dbeta), nseq, lt, l, vec.shape[1], p, seed, _p(scratch), scratch.numel() * 4, _s())
        return
    _call("cb_embed_text_bwd_vectors", _p(dh), _p(vec), vec.stride(0), _p(pos), _p(type0), _p(gamma), _p(stats), _p(dvec), _p(dpos),
          _p(dtype0), _p(dgamma), _p(dbeta), nseq, lt, l, vec.shape[1], p, seed, _s())


def embed_word_scatter(ids, dvec, dword):
    """cb_embed_word_scatter: dword[ids[r]] += dvec[r], one writer and one order per table row."""
    _call("cb_embed_word_scatter", _p(ids), _p(dvec), _p(dword), ids.numel(), dword.shape[0], dword.shape[1], _s())


def embed_visual_fwd(grid, seq2vid, n_ex, rowemb, colemb, type0, gamma, beta, out, stats, nseq, t, gh, gw, lt, l, eps, p,
                     seed):
    _call("cb_embed_visual_fwd", _p(grid), _p(seq2vid), n_ex, _p(rowemb), _p(colemb), _p(type0), _p(gamma), _p(beta), _p(out),
          _p(stats), nseq, t, gh, gw, lt, l, rowemb.shape[1], eps, p, seed, _s())


def embed_visual_bwd(dh, grid, seq2vid, vid_start, n_ex, rowemb, colemb, type0, gamma, stats, dv_tmp, dgrid, drow, dcol,
                     dtype0, dgamma, dbeta, nseq, nvid, t, gh, gw, lt, l, p, seed):
    if deterministic():
        embed_visual_bwd_det(dh, grid, seq2vid, vid_start, n_ex, rowemb, colemb, type0, gamma, stats, dv_tmp, dgrid, drow, dcol,
                             dtype0, dgamma, dbeta, nseq, nvid, t, gh, gw, lt, l, p, seed,
                             _scratch(embed_visual_bwd_scratch_bytes(nseq, gh, gw), dh))
        return
    _call("cb_embed_visual_bwd", _p(dh), _p(grid), _p(seq2vid), _p(vid_start), n_ex, _p(rowemb), _p(colemb), _p(type0),
          _p(gamma), _p(stats), _p(dv_tmp), _p(dgrid), _p(drow), _p(dcol), _p(dtype0), _p(dgamma), _p(dbeta), nseq, nvid, t,
          gh, gw, lt, l, rowemb.shape[1], p, seed, _s())


def embed_visual_bwd_scratch_bytes(nseq, gh, gw):
    return int(_fn("cb_embed_visual_bwd_scratch_bytes")(nseq, gh, gw))


def embed_visual_bwd_det(dh, grid, seq2vid, vid_start, n_ex, rowemb, colemb, type0, gamma, stats, dv_tmp, dgrid, drow, dcol,
                         dtype0, dgamma, dbeta, nseq, nvid, t, gh, gw, lt, l, p, seed, scratch):
    """cb_embed_visual_bwd_det: table gradients in block order through ``scratch`` (fp32)."""
    _call("cb_embed_visual_bwd_det", _p(dh), _p(grid), _p(seq2vid), _p(vid_start), n_ex, _p(rowemb), _p(colemb), _p(type0),
          _p(gamma), _p(stats), _p(dv_tmp), _p(dgrid), _p(drow), _p(dcol), _p(dtype0), _p(dgamma), _p(dbeta), nseq, nvid, t,
          gh, gw, lt, l, rowemb.shape[1], p, seed, _p(scratch), scratch.numel() * 4, _s())


def nvls_allreduce(multicast_ptr, n, rank, world, scale, max_ctas=0):
    """All-reduce n fp32 elements at a multicast (symmetric-memory) address through the NVSwitch; see cb_nvls_allreduce_f32."""
    _call("cb_nvls_allreduce_f32", multicast_ptr, n, rank, world, scale, max_ctas, _s())


def clip_lse_loss(logits, labels, loss, dlogits, n_clips, nseq, ncls, grad_scale=1.0):
    if deterministic():
        clip_lse_loss_det(logits, labels, loss, dlogits, n_clips, nseq, ncls, grad_scale, _scratch(clip_loss_scratch_bytes(nseq), logits))
        return
    _call("cb_clip_lse_loss", _p(logits), _p(labels), _p(loss), _p(dlogits), n_clips, nseq, ncls, grad_scale, _s())


def clip_pool_ce_loss(logits, labels, loss, dlogits, n_clips, nseq, ncls, pool, grad_scale=1.0):
    """pool: 1 = mean, 2 = max over the clips, then cross entropy (cb_clip_pool_ce_loss)."""
    if deterministic():
        clip_pool_ce_loss_det(logits, labels, loss, dlogits, n_clips, nseq, ncls, pool, grad_scale,
                              _scratch(clip_loss_scratch_bytes(nseq), logits))
        return
    _call("cb_clip_pool_ce_loss", _p(logits), _p(labels), _p(loss), _p(dlogits), n_clips, nseq, ncls, pool, grad_scale, _s())


def clip_loss_scratch_bytes(nseq):
    return int(_fn("cb_clip_loss_scratch_bytes")(nseq))


def clip_lse_loss_det(logits, labels, loss, dlogits, n_clips, nseq, ncls, grad_scale, scratch):
    _call("cb_clip_lse_loss_det", _p(logits), _p(labels), _p(loss), _p(dlogits), n_clips, nseq, ncls, grad_scale, _p(scratch),
          scratch.numel() * 4, _s())


def clip_pool_ce_loss_det(logits, labels, loss, dlogits, n_clips, nseq, ncls, pool, grad_scale, scratch):
    _call("cb_clip_pool_ce_loss_det", _p(logits), _p(labels), _p(loss), _p(dlogits), n_clips, nseq, ncls, pool, grad_scale,
          _p(scratch), scratch.numel() * 4, _s())


def cross_entropy_fwd(logits, labels, loss, lse, ignore_index=-100):
    _call("cb_cross_entropy_fwd", _p(logits), logits.stride(0), _p(labels), _p(loss), _p(lse), logits.shape[0], logits.shape[1], ignore_index, _s())


def cross_entropy_bwd(logits, labels, lse, grad_loss, dlogits, ignore_index=-100):
    _call("cb_cross_entropy_bwd", _p(logits), logits.stride(0), _p(labels), _p(lse), _p(grad_loss), _p(dlogits), dlogits.stride(0), logits.shape[0],
          logits.shape[1], ignore_index, _s())


def colsum(x, out, m, n, ld=None):
    if deterministic():
        colsum_det(x, out, m, n, ld, _scratch(colsum_scratch_bytes(m, n), x))
        return
    _call("cb_colsum", _p(x), n if ld is None else ld, _p(out), m, n, _s())


def colsum_scratch_bytes(m, n):
    return int(_fn("cb_colsum_scratch_bytes")(m, n))


def colsum_det(x, out, m, n, ld, scratch):
    """cb_colsum_det: column sums added in slab order through ``scratch`` (fp32)."""
    _call("cb_colsum_det", _p(x), n if ld is None else ld, _p(out), m, n, _p(scratch), scratch.numel() * 4, _s())


def sumsq_scratch_bytes(n, chunks, nchunks):
    return int(_fn("cb_sumsq_scratch_bytes")(n, _p(chunks), nchunks))


def sumsq_det(x, n, chunks, nchunks, out, scratch):
    """cb_sumsq_det: out[0] += sum of x^2 (chunk table or x[0, n)), block partials added in a fixed order."""
    _call("cb_sumsq_det", _p(x), n, _p(chunks), nchunks, _p(out), _p(scratch), scratch.numel() * 4, _s())


def dropout(x, y, p, seed):
    _call("cb_dropout", _p(x), _p(y), x.numel(), p, seed, _s())


def gelu_bwd(dy, u, dx):
    _call("cb_gelu_bwd", _p(dy), _p(u), _p(dx), dy.numel(), _s())


def pad_cast(src, dst):
    _call("cb_pad_cast", _p(src), src.stride(0), _p(dst), src.shape[0], src.shape[1], dst.shape[1], _s())


def cast_scale(src, dst, rowscale=None, row_len=1):
    _call("cb_cast_scale", _p(src), _p(rowscale), row_len, _p(dst), src.numel(), _s())


def cast_bf16_f32(src, dst):
    _call("cb_cast_bf16_f32", _p(src), _p(dst), src.numel(), _s())


def cast_scale_segments(master, packed, segments, scales):
    _call("cb_cast_scale_segments", _p(master), _p(packed), _p(segments), segments.shape[0], _p(scales), _s())


def attention_fwd(qkv, text_mask, ctx, lse, nseq, l, lt, heads, p, seed):
    _call("cb_attention_fwd", _p(qkv), qkv.shape[1], _p(text_mask), _p(ctx), ctx.shape[1], _p(lse), nseq, l, lt, heads, 64, p,
          seed, _s())


def attention_bwd(qkv, text_mask, ctx, dctx, lse, dqkv, nseq, l, lt, heads, p, seed):
    _call("cb_attention_bwd", _p(qkv), qkv.shape[1], _p(text_mask), _p(ctx), _p(dctx), ctx.shape[1], _p(lse), _p(dqkv),
          dqkv.shape[1], nseq, l, lt, heads, 64, p, seed, _s())


def attention_probs(qkv, text_mask, lse, probs, nseq, l, lt, heads, p, seed):
    """probs: fp32 [nseq, heads, l, l] contiguous, from the lse cb_attention_fwd wrote for the same arguments."""
    assert probs.dtype == torch.float32 and probs.is_contiguous() and probs.numel() == nseq * heads * l * l
    _call("cb_attention_probs", _p(qkv), qkv.shape[1], _p(text_mask), _p(lse), _p(probs), nseq, l, lt, heads, 64, p, seed, _s())


def attention_probs_bwd(qkv, text_mask, lse, dprobs, drow, dqkv, nseq, l, lt, heads, p, seed):
    """Adds the gradient of a loss on the probabilities (dprobs: fp32 [nseq, heads, l, l] contiguous) into dqkv's Q and K
    blocks; drow: fp32 scratch of nseq * heads * l floats."""
    assert dprobs.dtype == torch.float32 and dprobs.is_contiguous() and dprobs.numel() == nseq * heads * l * l
    assert drow.dtype == torch.float32 and drow.numel() >= nseq * heads * l
    _call("cb_attention_probs_bwd", _p(qkv), qkv.shape[1], _p(text_mask), _p(lse), _p(dprobs), _p(drow), _p(dqkv), dqkv.shape[1],
          nseq, l, lt, heads, 64, p, seed, _s())


def attention_probs_bwd_store(qkv, text_mask, lse, dprobs, drow, dqkv, nseq, l, lt, heads, p, seed):
    """attention_probs_bwd with dQ / dK written to dqkv's Q and K blocks instead of added (their old contents are never read)."""
    assert dprobs.dtype == torch.float32 and dprobs.is_contiguous() and dprobs.numel() == nseq * heads * l * l
    assert drow.dtype == torch.float32 and drow.numel() >= nseq * heads * l
    _call("cb_attention_probs_bwd_store", _p(qkv), qkv.shape[1], _p(text_mask), _p(lse), _p(dprobs), _p(drow), _p(dqkv),
          dqkv.shape[1], nseq, l, lt, heads, 64, p, seed, _s())


def attention_bwd_dv(qkv, text_mask, lse, dctx, dqkv, nseq, l, lt, heads, p, seed):
    """dV = (P r)^T dO per head, written to dqkv's V block (Q and K blocks untouched), P rebuilt from qkv, the mask and lse."""
    _call("cb_attention_bwd_dv", _p(qkv), qkv.shape[1], _p(text_mask), _p(lse), _p(dctx), dctx.shape[1], _p(dqkv), dqkv.shape[1],
          nseq, l, lt, heads, 64, p, seed, _s())


def attention_dprobs(qkv, dctx, dprobs, accumulate, nseq, l, heads):
    """dprobs (fp32 [nseq, heads, l, l] contiguous) = (dprobs if accumulate else 0) + dO V^T per head: the gradient the returned
    attention probabilities receive from the context product, with dctx = d loss / d context and V from qkv."""
    assert dprobs.dtype == torch.float32 and dprobs.is_contiguous() and dprobs.numel() == nseq * heads * l * l
    _call("cb_attention_dprobs", _p(qkv), qkv.shape[1], _p(dctx), dctx.shape[1], _p(dprobs), int(bool(accumulate)), nseq, l, heads,
          64, _s())


# ------------------------------------------------------------------------------------------------
# CNN-side memory-bound ops (NHWC bf16)
# ------------------------------------------------------------------------------------------------
def stem_im2col(x, out, n, h, w, kp, mean=(0.0, 0.0, 0.0)):
    dt = 0 if x.dtype == torch.float32 else 1
    _call("cb_stem_im2col", _p(x), dt, _p(out), n, h, w, kp, mean[0], mean[1], mean[2], _s())


def stem_s2d(x, out, n, h, w, ld, mean=(0.0, 0.0, 0.0)):
    dt = 0 if x.dtype == torch.float32 else 1
    _call("cb_stem_s2d", _p(x), dt, _p(out), n, h, w, ld, mean[0], mean[1], mean[2], _s())


def resize_pad(x, y, new_h, new_w):
    """x: (..., h, w) uint8 / fp32 planes; y: (..., S, S) fp32 - bilinear (align_corners=False) resize to new_h x new_w, zero pad to S."""
    dt = 0 if x.dtype == torch.float32 else 1
    _call("cb_resize_pad", _p(x), dt, _p(y), x.numel() // (x.shape[-1] * x.shape[-2]), x.shape[-2], x.shape[-1], new_h, new_w, y.shape[-1], _s())


def resize_pad_bwd(dy, dx, new_h, new_w, accumulate=False):
    """dx: (..., h, w) fp32 = (dx if accumulate else 0) + the adjoint of resize_pad(x, y, new_h, new_w) applied to dy (..., S, S)
    fp32, the gradient of y: d loss / d x. Both contiguous; the pad region of dy contributes nothing."""
    assert dy.dtype == torch.float32 and dx.dtype == torch.float32 and dy.is_contiguous() and dx.is_contiguous()
    planes = dx.numel() // (dx.shape[-1] * dx.shape[-2])
    assert dy.shape[-1] == dy.shape[-2] and dy.numel() == planes * dy.shape[-1] * dy.shape[-2]
    _call("cb_resize_pad_bwd", _p(dy), _p(dx), planes, dx.shape[-2], dx.shape[-1], new_h, new_w, dy.shape[-1], int(bool(accumulate)), _s())


def maxpool3x3s2(x, y, n, h, w, c, row_pitch=None, img_pitch=None):
    if row_pitch is None:
        _call("cb_maxpool3x3s2", _p(x), _p(y), n, h, w, c, _s())
    else:
        _call("cb_maxpool3x3s2_strided", _p(x), _p(y), n, h, w, c, row_pitch, img_pitch, _s())


def maxpool3x3s2_bwd(dy, x, dx, n, h, w, c, row_pitch=None, img_pitch=None):
    """dx (compact [n*h*w, c]) = the pool's backward fused with the stem's ReLU'; x is the pool input on the pitches the forward
    read it with."""
    if row_pitch is None:
        _call("cb_maxpool3x3s2_bwd", _p(dy), _p(x), _p(dx), n, h, w, c, _s())
    else:
        _call("cb_maxpool3x3s2_bwd_strided", _p(dy), _p(x), _p(dx), n, h, w, c, row_pitch, img_pitch, _s())


def stem_dgrad(dc1, w, dx, n, h, wimg):
    """dx: fp32 NCHW RGB [n, 3, h, wimg] contiguous = the stem conv's input gradient from dc1 (bf16 [n*ho*wo, 64]) and the stem
    operand w (bf16 [64, >= 147], row pitch w.stride(0))."""
    assert dx.dtype == torch.float32 and dx.is_contiguous() and dx.numel() == n * 3 * h * wimg
    assert w.dtype == torch.bfloat16 and w.stride(1) == 1 and dc1.dtype == torch.bfloat16 and dc1.is_contiguous()
    _call("cb_stem_dgrad", _p(dc1), _p(w), w.stride(0), _p(dx), n, h, wimg, _s())


def subsample2(x, y, n, h, w, c):
    _call("cb_subsample2", _p(x), _p(y), n, h, w, c, _s())


def unsubsample2_mask(dsub, act, dx, n, h, w, c):
    """act None: the mask-free scatter (the gradient's mask is applied by the block that produced x)."""
    _call("cb_unsubsample2_mask", _p(dsub), _p(act), _p(dx), n, h, w, c, _s())


def maxpool2x2_relu_fwd(x, y, n, h, w, c):
    _call("cb_maxpool2x2_relu_fwd", _p(x), _p(y), n, h, w, c, _s())


def maxpool2x2_relu_bwd(dy, x, dx_pad, n, h, w, c):
    _call("cb_maxpool2x2_relu_bwd", _p(dy), _p(x), _p(dx_pad), n, h, w, c, _s())


def relu_mask(dy, act, dx):
    _call("cb_relu_mask", _p(dy), _p(act), _p(dx), dy.numel(), _s())


INTAKE_DTYPES = {torch.float32: 0, torch.bfloat16: 2, torch.float16: 3}


def nhwc_intake(x, out, act=None, out_bordered=False, act_bordered=False):
    """cb_nhwc_intake: x (n, c, h, w), any strides, fp32 / bf16 / fp16 -> out, bf16 NHWC compact [n*h*w, c] or (out_bordered) the
    interior of a zero-bordered [n*(h+2)*(w+2), c]; act (bf16 NHWC, compact or act_bordered): out = (act > 0) ? x : +0."""
    if x.dtype not in INTAKE_DTYPES:
        raise TypeError("nhwc_intake: dtype %s is not fp32, bf16 or fp16" % x.dtype)
    n, c, h, w = x.shape
    rows = n * (h + 2) * (w + 2) if out_bordered else n * h * w
    assert out.dtype == torch.bfloat16 and out.is_contiguous() and out.numel() == rows * c and x.device == out.device
    if act is not None:
        arows = n * (h + 2) * (w + 2) if act_bordered else n * h * w
        assert act.dtype == torch.bfloat16 and act.is_contiguous() and act.numel() == arows * c and act.device == out.device
    _call("cb_nhwc_intake", _p(x), INTAKE_DTYPES[x.dtype], *x.stride(), n, c, h, w, _p(act), int(bool(act_bordered)), _p(out),
          int(bool(out_bordered)), _s())
