"""CPU emulation of the C ABI's *contract* (include/clipbert_b200.h) in plain torch - TEST INFRASTRUCTURE ONLY.

Purpose: run the Python orchestration of clipbert_b200/modeling.py (buffer planning, stash, forward/backward call order,
epilogue flags, index bookkeeping) on a machine without a GPU and compare it with the oracle. It swaps the functions of
clipbert_b200.ops for torch code that does what the header says each entry point does (bf16 buffers in, fp32 arithmetic,
bf16 / fp32 out); nothing in the product imports this file, and the kernels themselves are only ever checked on an H100
(tests/test_gpu_*.py). Dropout must be off (the counter RNG of the kernels is not restated here).
"""
import contextlib
import math

import torch
import torch.nn.functional as F

F32 = torch.float32
IGNORE_DROPOUT = False      # emulated_ops(ignore_dropout=True): dropout arguments are accepted and treated as p = 0 (dry runs)


def _no_dropout(p):
    assert IGNORE_DROPOUT or not p, "emulator: dropout must be off"


def _mat(t, rows, cols, ld):
    """rows x cols window with row pitch ld starting at the first element of tensor t (a raw device pointer in the ABI)."""
    return torch.as_strided(t, (rows, cols), (ld, 1), t.storage_offset())


def _gelu(v):
    return 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))


def _gelu_grad(v):
    return 0.5 * (1.0 + torch.erf(v / math.sqrt(2.0))) + v * torch.exp(-0.5 * v * v) / math.sqrt(2.0 * math.pi)


def _shifted_rows(t, n_rows, cols, ld, m, shift):
    """[m, cols] fp32: row i = row (i + shift) of the [n_rows, cols] window (pitch ld) of t, zero when out of range - the
    zero fill TMA gives a box that leaves the tensor map. Rows may overlap (ld < cols: the space-to-depth stem)."""
    win = _mat(t, n_rows, cols, ld)
    idx = torch.arange(m) + shift
    ok = (idx >= 0) & (idx < n_rows)
    out = torch.zeros(m, cols, dtype=F32)
    out[ok] = win[idx[ok]].to(F32)
    return out


def _tap_shift(t, ntaps, tap_w, tap_sign):
    if ntaps == 9:
        return tap_sign * ((t // 3 - 1) * tap_w + (t % 3 - 1))
    return tap_sign * t * tap_w if ntaps > 1 else 0


def _out_rows(kw, m):
    """cb_rowmap: destination row of GEMM row i (-1 = dropped), and the number of destination rows."""
    rm = kw.get("rowmap", 0)
    i = torch.arange(m)
    if rm == 0:
        return i, m
    H, W = kw["map_h"], kw["map_w"]
    if rm == 1:                                          # compact -> zero-bordered
        img, r = i // (H * W), i % (H * W)
        y, x = r // W, r % W
        return (img * (H + 2) + y + 1) * (W + 2) + x + 1, (m // (H * W)) * (H + 2) * (W + 2)
    hp, wp = H + 2, W + 2                                # zero-bordered -> compact, border rows dropped
    img, r = i // (hp * wp), i % (hp * wp)
    y, x = r // wp, r % wp
    ok = (y >= 1) & (y <= H) & (x >= 1) & (x <= W)
    dst = (img * H + (y - 1)) * W + (x - 1)
    return torch.where(ok, dst, torch.full_like(dst, -1)), (m // (hp * wp)) * H * W


def gemm(**kw):
    mode, m, n, k = kw.get("mode", 0), kw["m"], kw["n"], kw["k"]
    ntaps, tap_w, tap_sign = kw.get("ntaps", 1), kw.get("tap_w", 0), kw.get("tap_sign", 1)
    _no_dropout(kw.get("dropout_p"))
    a, b, out = kw["a"], kw["b"], kw["out"]
    if mode == 1:                                       # WGRAD: out[m, t*N + n] += rowscale[m] * sum_p A[p, m] B[p + shift_t, n]
        A = _mat(a, k, m, kw["a_ld"]).to(F32)
        assert out.dtype == F32 and kw.get("out_fp32") == 1 and kw["a_rows"] == k and kw["b_rows"] == k
        O = _mat(out, m, ntaps * n, kw["out_ld"])
        for t in range(ntaps):
            g = (A.t().double() @ _shifted_rows(b, k, n, kw["b_ld"], k, _tap_shift(t, ntaps, tap_w, tap_sign)).double()).float()
            if kw.get("scale") is not None:
                g = g * kw["scale"][:m, None]
            O[:, t * n:(t + 1) * n] += g
        return
    # accumulate in float64: the result must not depend on how the CPU BLAS blocks a particular batch shape (the kernels'
    # per-element accumulation order is independent of M, and tests compare batched against per-clip runs)
    v = torch.zeros(m, n, dtype=torch.float64)
    for t in range(ntaps):
        At = _shifted_rows(a, kw["a_rows"], k, kw["a_ld"], m, _tap_shift(t, ntaps, tap_w, tap_sign)).double()
        if mode == 0:                                   # TN: B [n, ntaps*k]
            v += At @ _mat(b, n, ntaps * k, kw["b_ld"])[:, t * k:(t + 1) * k].double().t()
        else:                                           # NN: B [k, ntaps*n] (the forward weight read MN-major)
            v += At @ _mat(b, k, ntaps * n, kw["b_ld"])[:, t * n:(t + 1) * n].double()
    v = v.float()
    if kw.get("scale") is not None:
        v = v * kw["scale"][:n].to(F32)
    if kw.get("shift") is not None:
        v = v + kw["shift"][:n].to(F32)
    if kw.get("residual") is not None:
        v = v + _mat(kw["residual"], m, n, kw["res_ld"]).to(F32)
    act = kw.get("act", 0)
    dst, n_dst = _out_rows(kw, m)
    keep = dst >= 0
    if kw.get("out2") is not None:
        _mat(kw["out2"], n_dst, n, kw["out2_ld"])[dst[keep]] = (_gelu_grad(v) if act == 4 else v)[keep].to(kw["out2"].dtype)
    if act == 1:
        v = torch.relu(v)
    elif act in (2, 4):
        v = _gelu(v)
    elif act == 3:
        v = torch.tanh(v)
    if kw.get("aux") is not None:
        x = _mat(kw["aux"], m, n, kw["aux_ld"]).to(F32)
        am = kw.get("aux_mode", 0)
        if am == 1:
            v = v * (x > 0).to(F32)
        elif am == 2:
            v = v * _gelu_grad(x)
        elif am == 3:
            v = v * (1.0 - x * x)
        elif am == 4:
            v = v * x
    assert (out.dtype == F32) == bool(kw.get("out_fp32", 0))
    _mat(out, n_dst, n, kw["out_ld"])[dst[keep]] = v[keep].to(out.dtype)


def _ln_fwd(v, gamma, beta, eps):
    mean = v.mean(-1, keepdim=True)
    var = ((v - mean) ** 2).mean(-1, keepdim=True)
    rstd = torch.rsqrt(var + eps)
    return (v - mean) * rstd * gamma + beta, mean.squeeze(-1), rstd.squeeze(-1)


def _ln_bwd(dy, x, mean, rstd, gamma):
    xhat = (x - mean[:, None]) * rstd[:, None]
    g = dy * gamma
    dx = rstd[:, None] * (g - g.mean(-1, keepdim=True) - xhat * (g * xhat).mean(-1, keepdim=True))
    return dx, (dy * xhat).sum(0), dy.sum(0)


def layernorm_fwd(x, gamma, beta, y, stats, eps):
    o, mean, rstd = _ln_fwd(x.to(F32), gamma, beta, eps)
    y.copy_(o)
    stats[:, 0], stats[:, 1] = mean, rstd


def layernorm_bwd(dy, x, stats, gamma, dx, dx_drop, dgamma, dbeta, dbias_drop, p, seed):
    _no_dropout(p)
    d, dg, db = _ln_bwd(dy.to(F32), x.to(F32), stats[:, 0], stats[:, 1], gamma)
    dx.copy_(d)
    if dx_drop is not None:
        dx_drop.copy_(d)
    dgamma.add_(dg)
    dbeta.add_(db)
    if dbias_drop is not None:
        dbias_drop[: d.shape[1]].add_(dx.to(F32).sum(0))     # column sums of the bf16 tensor the dense's dgrad consumes


def embed_text_fwd(ids, word, pos, typ, gamma, beta, out, stats, nseq, lt, l, eps, p, seed):
    _no_dropout(p)
    v = word[ids] + pos[:lt][None] + typ[0][None, None]
    o, mean, rstd = _ln_fwd(v.reshape(nseq * lt, -1), gamma, beta, eps)
    out.view(nseq, l, -1)[:, :lt].copy_(o.view(nseq, lt, -1))
    stats[:, 0], stats[:, 1] = mean, rstd


def embed_text_bwd(dh, ids, word, pos, typ, gamma, stats, dword, dpos, dtyp, dgamma, dbeta, nseq, lt, l, p, seed):
    _no_dropout(p)
    h = word.shape[1]
    v = (word[ids] + pos[:lt][None] + typ[0][None, None]).reshape(nseq * lt, h)
    dy = dh.view(nseq, l, h)[:, :lt].reshape(nseq * lt, h).to(F32)
    d, dg, db = _ln_bwd(dy, v, stats[:, 0], stats[:, 1], gamma)
    dgamma.add_(dg)
    dbeta.add_(db)
    dword.index_add_(0, ids.reshape(-1), d)
    dpos[:lt].add_(d.view(nseq, lt, h).sum(0))
    dtyp[0].add_(d.sum(0))


def _visual_pre(grid, seq2vid, n_ex, rowemb, colemb, typ, nseq, t, gh, gw):
    h = grid.shape[-1]
    vid = seq2vid.long() if seq2vid is not None else torch.arange(nseq) // n_ex
    g = grid.reshape(-1, t, gh * gw, h).to(F32).sum(1) * (1.0 / t)            # [nvid, Lv, h]
    j = torch.arange(gh * gw)
    v = g[vid] + rowemb[j // gw][None] + colemb[j % gw][None] + typ[0][None, None]
    return v.reshape(nseq * gh * gw, h), vid, j


def embed_visual_fwd(grid, seq2vid, n_ex, rowemb, colemb, typ, gamma, beta, out, stats, nseq, t, gh, gw, lt, l, eps, p, seed):
    _no_dropout(p)
    v, _, _ = _visual_pre(grid, seq2vid, n_ex, rowemb, colemb, typ, nseq, t, gh, gw)
    o, mean, rstd = _ln_fwd(v, gamma, beta, eps)
    out.view(nseq, l, -1)[:, lt:].copy_(o.view(nseq, gh * gw, -1))
    stats[:, 0], stats[:, 1] = mean, rstd


def embed_visual_bwd(dh, grid, seq2vid, vid_start, n_ex, rowemb, colemb, typ, gamma, stats, dv_tmp, dgrid, drow, dcol, dtyp,
                     dgamma, dbeta, nseq, nvid, t, gh, gw, lt, l, p, seed):
    _no_dropout(p)
    h = grid.shape[-1]
    lv = gh * gw
    v, vid, j = _visual_pre(grid, seq2vid, n_ex, rowemb, colemb, typ, nseq, t, gh, gw)
    dy = dh.view(nseq, l, h)[:, lt:].reshape(nseq * lv, h).to(F32)
    d, dg, db = _ln_bwd(dy, v, stats[:, 0], stats[:, 1], gamma)
    dgamma.add_(dg)
    dbeta.add_(db)
    dv_tmp.copy_(d)
    d3 = d.view(nseq, lv, h)
    drow.index_add_(0, j // gw, d3.sum(0))
    dcol.index_add_(0, j % gw, d3.sum(0))
    dtyp[0].add_(d.sum(0))
    if dgrid is not None:
        per_vid = torch.zeros(nvid, lv, h).index_add_(0, vid, d3) * (1.0 / t)
        dgrid.view(nvid, t, lv, h).copy_(per_vid[:, None].expand(nvid, t, lv, h))


def _attention(qkv, text_mask, nseq, l, lt, heads):
    hd = qkv.shape[1] // (3 * heads)
    q, k, v = (x.reshape(nseq, l, heads, hd).permute(0, 2, 1, 3) for x in qkv.view(nseq, l, 3, heads * hd).unbind(2))
    mask = torch.cat([text_mask.to(qkv.dtype), torch.ones(nseq, l - lt, dtype=qkv.dtype)], dim=1)
    s = q @ k.transpose(-1, -2) / math.sqrt(hd) + ((1.0 - mask) * -10000.0)[:, None, None, :]
    pr = torch.softmax(s, dim=-1)
    return (pr @ v).permute(0, 2, 1, 3).reshape(nseq * l, heads * hd), torch.logsumexp(s, dim=-1)


def attention_fwd(qkv, text_mask, ctx, lse, nseq, l, lt, heads, p, seed):
    _no_dropout(p)
    o, ls = _attention(qkv.double(), text_mask, nseq, l, lt, heads)
    ctx.copy_(o)
    if lse is not None:
        lse.copy_(ls)


def attention_bwd(qkv, text_mask, ctx, dctx, lse, dqkv, nseq, l, lt, heads, p, seed):
    _no_dropout(p)
    x = qkv.to(F32).clone().requires_grad_(True)
    with torch.enable_grad():
        o, _ = _attention(x, text_mask, nseq, l, lt, heads)
        o.backward(dctx.to(F32))
    dqkv.copy_(x.grad)


def colsum(x, out, m, n, ld=None):
    out[:n].add_(_mat(x, m, n, n if ld is None else ld).to(F32).sum(0))


def dropout(x, y, p, seed):
    _no_dropout(p)
    y.copy_(x)


def gelu_bwd(dy, u, dx):
    dx.copy_(dy.to(F32) * _gelu_grad(u.to(F32)))


def pad_cast(src, dst):
    dst.zero_()
    dst[:, : src.shape[1]].copy_(src)


def cast_scale(src, dst, rowscale=None, row_len=1):
    v = src if rowscale is None else (src.view(-1, row_len) * rowscale[:, None]).reshape(-1)
    dst.copy_(v)


# ---------------------------------------------------------------------------------------------------
# CNN-side data movement (NHWC bf16)
# ---------------------------------------------------------------------------------------------------
def _bgr_frames(x, mean):
    """NCHW RGB (fp32 already mean-subtracted, or uint8 + ImageNorm mean) -> fp32 NCHW BGR, rounded to bf16 like the kernels."""
    v = x.to(F32) - torch.tensor(mean, dtype=F32).view(1, 3, 1, 1)
    return v[:, [2, 1, 0]].to(torch.bfloat16).to(F32)


def stem_im2col(x, out, n, h, w, kp, mean=(0.0, 0.0, 0.0)):
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    cols = F.unfold(_bgr_frames(x, mean), kernel_size=7, padding=3, stride=2)            # [n, (c, r, s), ho*wo]
    cols = cols.view(n, 3, 7, 7, ho * wo).permute(0, 4, 2, 3, 1).reshape(n * ho * wo, 147)
    out.zero_()
    out[:, :147].copy_(cols)


def stem_s2d(x, out, n, h, w, ld, mean=(0.0, 0.0, 0.0)):
    assert ld == 16, "emulator covers the overlapping-row layout"
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    hs, ws = ho + 3, wo + 3
    P = torch.zeros(n, 3, 2 * hs, 2 * ws, dtype=F32)
    P[:, :, 3:3 + h, 3:3 + w] = _bgr_frames(x, mean)
    S = torch.zeros(n, hs, ws, 2, 2, 4, dtype=F32)
    S[..., :3] = P.view(n, 3, hs, 2, ws, 2).permute(0, 2, 4, 3, 5, 1)
    out.view(-1)[: n * hs * ws * 16].copy_(S.reshape(-1))
    out.view(-1)[n * hs * ws * 16:].zero_()             # the slack the last windows run into (the kernel leaves it unwritten)


def resize_pad(x, y, new_h, new_w):
    lead = x.shape[:-2]
    r = F.interpolate(x.reshape(-1, 1, x.shape[-2], x.shape[-1]).float(), size=(new_h, new_w), mode="bilinear", align_corners=False)
    y.zero_()
    y.view(-1, y.shape[-2], y.shape[-1])[:, :new_h, :new_w] = r[:, 0]
    assert tuple(y.shape[:-2]) == tuple(lead)


def maxpool3x3s2(x, y, n, h, w, c, row_pitch=None, img_pitch=None):
    row_pitch = w if row_pitch is None else row_pitch
    img_pitch = h * w if img_pitch is None else img_pitch
    v = torch.as_strided(x, (n, h, w, c), (img_pitch * c, row_pitch * c, c, 1), x.storage_offset()).to(F32)
    o = F.max_pool2d(v.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    y.view(-1)[: o.numel()].copy_(o.reshape(-1))


def subsample2(x, y, n, h, w, c):
    y.view(-1).copy_(x.view(n, h, w, c)[:, ::2, ::2].reshape(-1))


def unsubsample2_mask(dsub, act, dx, n, h, w, c):
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    full = torch.zeros(n, h, w, c, dtype=F32)
    full[:, ::2, ::2] = dsub.view(n, ho, wo, c).to(F32)
    dx.view(-1).copy_((full * (act.view(n, h, w, c).to(F32) > 0)).reshape(-1))


def maxpool2x2_relu_fwd(x, y, n, h, w, c):
    o = F.max_pool2d(x.view(n, h, w, c).to(F32).permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
    y.view(-1).copy_(torch.relu(o).reshape(-1))


def maxpool2x2_relu_bwd(dy, x, dx_pad, n, h, w, c):
    xv = x.view(n, h, w, c).to(F32).permute(0, 3, 1, 2).clone().requires_grad_(True)
    with torch.enable_grad():
        torch.relu(F.max_pool2d(xv, 2, 2)).backward(dy.view(n, h // 2, w // 2, c).to(F32).permute(0, 3, 1, 2))
    pad = torch.zeros(n, h + 2, w + 2, c, dtype=F32)
    pad[:, 1:-1, 1:-1] = xv.grad.permute(0, 2, 3, 1)
    dx_pad.view(-1).copy_(pad.reshape(-1))


def relu_mask(dy, act, dx):
    dx.view(-1).copy_((dy.to(F32) * (act.to(F32) > 0)).reshape(-1))


def clip_lse_loss(logits, labels, loss, dlogits, n_clips, nseq, ncls, grad_scale=1.0):
    z = logits.detach().clone().requires_grad_(dlogits is not None)
    with torch.enable_grad():
        lg = z.permute(1, 0, 2)
        out = torch.logsumexp(lg.reshape(nseq, -1), dim=-1, keepdim=True) - torch.logsumexp(lg, dim=1)
        val = torch.gather(out, -1, labels.view(-1, 1)).mean()
        if dlogits is not None:
            val.backward()
            dlogits.copy_(z.grad * grad_scale)
    loss.copy_(val.detach().reshape(1))


NVLS_BUFFERS = {}       # data_ptr of a "symmetric" buffer -> tensor (registered by the test's stand-in for rendezvous())


def nvls_allreduce(multicast_ptr, n, rank, world, scale, max_ctas=0):
    """cb_nvls_allreduce_f32 over torch.distributed (gloo): the element range [ptr, ptr + n) of a registered buffer."""
    import torch.distributed as dist
    base, buf = next((b, t) for b, t in NVLS_BUFFERS.items() if b <= multicast_ptr < b + 4 * t.numel())
    off = (multicast_ptr - base) // 4
    assert (multicast_ptr - base) % 16 == 0 and n % 4 == 0 and off + n <= buf.numel()
    view = buf[off: off + n]
    dist.all_reduce(view, op=dist.ReduceOp.SUM)
    view.mul_(scale)


def cast_scale_segments(master, packed, segments, scales):
    for off, numel, row_len, soff in segments.tolist():
        v = master[off: off + numel].view(-1, row_len)
        if soff >= 0:
            v = v * scales[soff: soff + v.shape[0], None]
        packed[off: off + numel].copy_(v.reshape(-1))


# ---------------------------------------------------------------------------------------------------
# fused optimizer step (clipbert_b200/optim.py calls these with tensors)
# ---------------------------------------------------------------------------------------------------
def opt_sumsq(x, chunks, nchunks, out):
    acc = torch.zeros((), dtype=torch.float64)
    for off, n, *_ in chunks[:nchunks].tolist():
        acc += (x[off: off + n].double() ** 2).sum()
    out[0] += acc.float()


def opt_adamw_step(master, grad, exp_avg, exp_avg_sq, packed, chunks, nchunks, hyper, scales, grad_sumsq, max_norm, zero_grad):
    """cb_adamw_step (csrc/optim.cu): AdamW of src/optimization/adamw.py:40-103 per chunk-table row, clip coefficient from the
    total gradient norm, optional gradient zeroing and bf16 operand emission (FrozenBN row scale folded in)."""
    coef = 1.0
    if grad_sumsq is not None and max_norm > 0:
        coef = min(1.0, max_norm / (float(grad_sumsq.sqrt()) + 1e-6))
    for off, n, grp, row_len, soff, flags, elem0, _ in chunks[:nchunks].tolist():
        lr, step_size, wd, b1, b2, eps = (float(x) for x in hyper[grp][:6])
        sl = slice(off, off + n)
        g = grad[sl] * coef
        exp_avg[sl] = exp_avg[sl] * b1 + (1.0 - b1) * g
        exp_avg_sq[sl] = exp_avg_sq[sl] * b2 + (1.0 - b2) * g * g
        p = master[sl] - step_size * (exp_avg[sl] / (exp_avg_sq[sl].sqrt() + eps))
        if wd > 0:
            p = p - lr * wd * p
        master[sl] = p
        if zero_grad:
            grad[sl] = 0
        if (flags & 1) and packed is not None:
            if soff >= 0:
                rows = (elem0 + torch.arange(n)) // row_len
                p = p * scales[soff + rows]
            packed[sl] = p.to(packed.dtype)


def clip_pool_ce_loss(logits, labels, loss, dlogits, n_clips, nseq, ncls, pool, grad_scale=1.0):
    z = logits.detach().double().requires_grad_(True)
    pooled = z.mean(0) if pool == 1 else z.max(0)[0]
    v = torch.nn.functional.cross_entropy(pooled, labels, reduction="none").mean()
    v.backward()
    loss.copy_(v.detach().float().reshape(1))
    if dlogits is not None:
        dlogits.copy_((z.grad * grad_scale).float())


def cross_entropy_fwd(logits, labels, loss, lse, ignore_index=-100):
    z = logits.double()
    lse.copy_(torch.logsumexp(z, -1).float())
    loss.copy_(torch.nn.functional.cross_entropy(z, labels, reduction="none", ignore_index=ignore_index).float())


def cross_entropy_bwd(logits, labels, lse, grad_loss, dlogits, ignore_index=-100):
    z = logits.double()
    p = torch.exp(z - lse.double()[:, None])
    ok = (labels != ignore_index) & (labels >= 0) & (labels < z.shape[1])
    onehot = torch.zeros_like(p)
    onehot[ok, labels[ok]] = 1.0
    dlogits.copy_(((p - onehot) * (grad_loss.double() * ok.double())[:, None]).float())


def gemm_wgrad_group(kws):
    """cb_gemm_wgrad_group: n independent weight-gradient problems; the result is that of n cb_gemm launches."""
    from clipbert_b200 import ops as _ops
    for kw in kws:
        _ops.gemm(**kw)          # (the counted / recorded wrapper while the emulator is installed)


def cast_bf16_f32(src, dst):
    dst.copy_(src.float())


def dropout_offset_bind(word):
    """cb_dropout_offset_bind: process-wide device word folded into the dropout seeds (the emulator draws no masks)."""
    global BOUND_DROPOUT_WORD
    BOUND_DROPOUT_WORD = word


def dropout_offset_advance(counter, snapshot=None):
    """cb_dropout_offset_advance: ++*counter; *snapshot = *counter."""
    counter += 1
    if snapshot is not None:
        snapshot.copy_(counter)


BOUND_DROPOUT_WORD = None

_NAMES = ("gemm", "layernorm_fwd", "layernorm_bwd", "embed_text_fwd", "embed_text_bwd", "embed_visual_fwd", "embed_visual_bwd",
          "attention_fwd", "attention_bwd", "colsum", "dropout", "gelu_bwd", "pad_cast", "cast_scale", "stem_im2col", "stem_s2d",
          "maxpool3x3s2", "subsample2", "unsubsample2_mask", "maxpool2x2_relu_fwd", "maxpool2x2_relu_bwd", "relu_mask",
          "cast_scale_segments", "clip_lse_loss", "nvls_allreduce", "dropout_offset_bind", "dropout_offset_advance", "cast_bf16_f32",
          "clip_pool_ce_loss", "cross_entropy_fwd", "cross_entropy_bwd", "resize_pad", "gemm_wgrad_group")


@contextlib.contextmanager
def emulated_ops(ignore_dropout=False):
    """Swap the wrappers of clipbert_b200.ops (and the device checks of modeling.py / grid_feat.py) for the torch code above."""
    from clipbert_b200 import grid_feat, modeling, ops, optim
    saved = {n: getattr(ops, n) for n in _NAMES}
    saved_opt = (optim.sumsq, optim.adamw_step, optim._require_cuda)
    saved_overlap, saved_req, saved_req_cnn = ops.overlap_wgrad, modeling._require_cuda, grid_feat._require_cuda
    calls = {n: 0 for n in _NAMES}
    global IGNORE_DROPOUT
    saved_drop, IGNORE_DROPOUT = IGNORE_DROPOUT, bool(ignore_dropout)

    def counted(name, fn):
        def f(*a, **k):
            calls[name] += 1
            if name == "gemm" and ops._gemm_record is not None:     # the recording hook of ops.gemm (bench.py's roofline pass)
                ops._gemm_record.append(dict(k))
            return fn(*a, **k)
        return f
    try:
        for n in _NAMES:
            setattr(ops, n, counted(n, globals()[n]))
        ops.overlap_wgrad = False
        modeling._require_cuda = grid_feat._require_cuda = lambda t: None
        optim.sumsq, optim.adamw_step, optim._require_cuda = opt_sumsq, opt_adamw_step, (lambda dev: None)
        yield calls
    finally:
        for n, f in saved.items():
            setattr(ops, n, f)
        ops.overlap_wgrad, modeling._require_cuda, grid_feat._require_cuda = saved_overlap, saved_req, saved_req_cnn
        IGNORE_DROPOUT = saved_drop
        optim.sumsq, optim.adamw_step, optim._require_cuda = saved_opt


emulated_transformer_ops = emulated_ops
