"""Every dropout mask the training step draws, against the mask the generator defines (tests/dropout_ref.py).

Each consumer of the mask - cb_dropout, the GEMM epilogue (TN with a residual, the generic epilogue, the NN head backward),
cb_layernorm_bwd, the embeddings and every attention kernel family - is compared with a plain fp32 computation that applies
the restated mask explicitly, so a kernel that draws a shifted mask, reads the wrong index or seed, or applies the right mask
to the wrong term fails even when it agrees with the other kernels. The model-level test runs the transformer in train mode
with dropout on and compares it with fp32 autograd of the oracle with the same masks injected, which pins the seeds the model
hands to each launch.

Each comparison is shown to be sharp: the same reference built with the masks of seed + 1 must miss by far more than the
bound the right masks meet (both errors are printed; run with -s).
"""
import contextlib
import ctypes

import pytest
import torch

import dropout_ref as D
from util import TOL_BF16_OP, TOL_FP32_OP, TOL_GRAD, TOL_LOGITS, cosine, make_cfg, relerr

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
SEED = 0x5EED5
WORD = 2 ** 63 + 12345        # a bound device word with the top bit set (the word is unsigned)
MARGIN = 10                   # a reference with the wrong masks must miss by at least MARGIN x the asserted bound
# (p, bound word): the word is bound through ops.dropout_offset_bind on one case of every consumer
DROP_CASES = [(0.1, None), (0.5, WORD), (1.0, None)]
DROP_IDS = ["p0.1", "p0.5-word", "p1"]
SINGLE = 2                    # cb_gemm_desc.reserved bit with no meaning to the kernel: no tuning-table lookup


def _ops():
    from clipbert_b200 import ops
    return ops


def _rnd(g, *shape, scale=1.0, dev="cuda"):
    return (torch.randn(*shape, generator=g) * scale).to(dev).to(BF16)


def _mult(seed, idx, p, word=None, dev="cpu"):
    """fp32 tensor of the multipliers (0 or 1 / (1 - p)) a kernel must apply at the element indices idx."""
    return torch.from_numpy(D.multipliers(D.effective_seed(seed, word), idx, p)).to(dev)


@contextlib.contextmanager
def _bound(word, dev):
    """Bind `word` as the device-side dropout offset for the launches inside the block (None: leave it unbound)."""
    ops = _ops()
    if word is None:
        yield
        return
    w = torch.tensor([word - 2 ** 64 if word >= 2 ** 63 else word], dtype=torch.int64, device=dev)
    ops.dropout_offset_bind(w)
    try:
        yield
    finally:
        ops.dropout_offset_bind(None)
        torch.cuda.synchronize()


def _close(got, ref, tol, what):
    """relerr(got, ref) < tol; a reference that is exactly zero (p = 1 drops everything) must be met exactly."""
    got = got.detach().float()
    assert bool(torch.isfinite(got).all()), (what, "non-finite output")
    if float(ref.abs().max()) == 0.0:
        assert float(got.abs().max()) == 0.0, (what, "expected zeros", float(got.abs().max()))
        return 0.0
    e = relerr(got, ref)
    assert e < tol, (what, e)
    return e


def _sharp(got, ref, wrong, tol, what, p):
    """The right masks meet tol, the masks of seed + 1 miss it by MARGIN x. Returns the right-mask error."""
    e = _close(got, ref, tol, what)
    if p < 1.0:
        w = relerr(got, wrong)
        print("%s: error %.2e with the right masks, %.2e with the masks of seed + 1 (bound %.1e)" % (what, e, w, tol))
        assert w > MARGIN * tol, (what, "the comparison cannot tell the masks apart", e, w)
    return e


# ------------------------------------------------------------------------------------------------ cb_dropout
@pytest.mark.parametrize("p,word", DROP_CASES, ids=DROP_IDS)
def test_dropout_kernel_is_bit_exact(cuda, p, word):
    ops = _ops()
    n = (1 << 20) + 8
    g = torch.Generator().manual_seed(31)
    x = _rnd(g, n)
    x[::97] = 0.0                         # a kept zero times an infinite multiplier would be NaN
    y = torch.empty_like(x)
    with _bound(word, cuda):
        ops.dropout(x, y, p, SEED)
    want = (x.float() * _mult(SEED, D.flat_index(n), p, word, cuda)).to(BF16)
    assert bool(torch.isfinite(y.float()).all())
    assert torch.equal(y, want)
    if p < 1.0:
        wrong = (x.float() * _mult(SEED + 1, D.flat_index(n), p, word, cuda)).to(BF16)
        miss = float((y != wrong).float().mean())
        print("cb_dropout p=%g: mismatches 0 with the right mask, %.3f of the elements with the mask of seed + 1" % (p, miss))
        assert miss > 0.1 * p
        assert abs(float((y[x != 0] != 0).float().mean()) - (1 - p)) < 0.01


# ------------------------------------------------------------------------------------------------ GEMM epilogue
@pytest.mark.parametrize("p,word", DROP_CASES, ids=DROP_IDS)
@pytest.mark.parametrize("M,block_n", [(2624, 64), (2624, 128), (2624, 0), (20000, 64), (20000, 128), (20000, 0)])
def test_gemm_dropout_residual_epilogue(cuda, M, block_n, p, word):
    """EK_DROP_RES (BertSelfOutput / BertOutput dense): out = dropout(A B^T + shift) + residual, N = 768, bf16 out; block_n 0 =
    the launch configuration the library picks. 20000 rows put several tiles on every CTA of the ping-pong kernel."""
    ops = _ops()
    N, K = 768, 256
    g = torch.Generator().manual_seed(32)
    A, B, R = _rnd(g, M, K), _rnd(g, N, K, scale=0.1), _rnd(g, M, N)
    shift = torch.randn(N, generator=g).to(cuda)
    C = torch.empty(M, N, device=cuda, dtype=BF16)
    tiles = dict(block_n=block_n, reserved=SINGLE) if block_n else {}
    with _bound(word, cuda):
        ops.gemm(mode=ops.CB_GEMM_TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=N, b_ld=K, shift=shift, residual=R, res_ld=N,
                 dropout_p=p, dropout_seed=SEED, out=C, out_ld=N, **tiles)
    pre = A.float() @ B.float().t() + shift
    mult = _mult(SEED, D.gemm_index(M, N), p, word, cuda)
    dropped = mult == 0
    assert torch.equal(C[dropped], R[dropped])          # a dropped element is the residual, bit for bit
    wrong = pre * _mult(SEED + 1, D.gemm_index(M, N), p, word, cuda) + R.float()
    _sharp(C, pre * mult + R.float(), wrong, TOL_BF16_OP, "gemm drop+res M=%d block_n=%d p=%g" % (M, block_n, p), p)


def test_gemm_dropout_index_uses_n_not_the_output_pitch(cuda):
    """The mask of output element (row, col) is keyed by row * n + col also when rows are written with a wider pitch."""
    ops = _ops()
    M, N, K, LD = 2624, 768, 256, 832
    g = torch.Generator().manual_seed(33)
    A, B, R = _rnd(g, M, K), _rnd(g, N, K, scale=0.1), _rnd(g, M, N)
    C = torch.full((M, LD), 3.0, device=cuda, dtype=BF16)
    ops.gemm(mode=ops.CB_GEMM_TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=N, b_ld=K, residual=R, res_ld=N,
             dropout_p=0.1, dropout_seed=SEED, out=C, out_ld=LD)
    pre = A.float() @ B.float().t()
    mult = _mult(SEED, D.gemm_index(M, N), 0.1, None, cuda)
    assert torch.equal(C[:, :N][mult == 0], R[mult == 0])
    assert bool((C[:, N:] == 3.0).all())                # the pitch padding is not written
    wrong = pre * _mult(SEED, D.gemm_index(M, LD)[:, :N], 0.1, None, cuda) + R.float()     # keyed by the pitch instead
    _sharp(C[:, :N], pre * mult + R.float(), wrong, TOL_BF16_OP, "gemm drop+res out_ld=%d" % LD, 0.1)


@pytest.mark.parametrize("p,word", DROP_CASES, ids=DROP_IDS)
@pytest.mark.parametrize("M", [500, 3000])
def test_gemm_dropout_generic_epilogue(cuda, M, p, word):
    """The generic epilogue: N = 392 (guarded last columns), fp32 out, shift, dropout, residual, then ReLU."""
    ops = _ops()
    N, K = 392, 256
    g = torch.Generator().manual_seed(34)
    A, B, R = _rnd(g, M, K), _rnd(g, N, K, scale=0.1), _rnd(g, M, N)
    shift = torch.randn(N, generator=g).to(cuda)
    C = torch.empty(M, N, device=cuda)
    with _bound(word, cuda):
        ops.gemm(mode=ops.CB_GEMM_TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=N, b_ld=K, shift=shift, residual=R, res_ld=N,
                 act=ops.ACT_RELU, dropout_p=p, dropout_seed=SEED, out=C, out_ld=N, out_fp32=1, reserved=SINGLE)
    pre = A.float() @ B.float().t() + shift
    mult = _mult(SEED, D.gemm_index(M, N), p, word, cuda)
    dropped = mult == 0
    assert torch.equal(C[dropped], R.float().relu()[dropped])
    wrong = (pre * _mult(SEED + 1, D.gemm_index(M, N), p, word, cuda) + R.float()).relu()
    _sharp(C, (pre * mult + R.float()).relu(), wrong, TOL_FP32_OP, "gemm generic N=392 M=%d p=%g" % (M, p), p)


@pytest.mark.parametrize("p,word", DROP_CASES, ids=DROP_IDS)
@pytest.mark.parametrize("M", [6, 1000])
def test_gemm_dropout_nn_tanh_grad(cuda, M, p, word):
    """The classifier's backward (_mlp_head_backward): d pooled = (dC1 W0) * mask * (1 - pooled^2), NN form, bf16 out."""
    ops = _ops()
    N, K = 768, 1536
    g = torch.Generator().manual_seed(35)
    A, W = _rnd(g, M, K), _rnd(g, K, N, scale=0.05)
    aux = torch.tanh(torch.randn(M, N, generator=g)).to(cuda).to(BF16)
    C = torch.empty(M, N, device=cuda, dtype=BF16)
    with _bound(word, cuda):
        ops.gemm(mode=ops.CB_GEMM_NN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=W, b_rows=K, b_ld=N, out=C, out_ld=N, dropout_p=p,
                 dropout_seed=SEED, aux=aux, aux_ld=N, aux_mode=ops.AUX_TANH_GRAD)
    acc = A.float() @ W.float()
    tg = 1.0 - aux.float() ** 2
    mult = _mult(SEED, D.gemm_index(M, N), p, word, cuda)
    assert bool((C[mult == 0] == 0).all())
    wrong = acc * _mult(SEED + 1, D.gemm_index(M, N), p, word, cuda) * tg
    _sharp(C, acc * mult * tg, wrong, TOL_BF16_OP, "gemm NN tanh' M=%d p=%g" % (M, p), p)


# ------------------------------------------------------------------------------------------------ LayerNorm backward
def _bf16_ulp(x):
    """Spacing of bf16 numbers at |x| (8 significant bits)."""
    _, e = torch.frexp(x.abs())
    return torch.ldexp(torch.ones_like(x), e - 8)


@pytest.mark.parametrize("p,word", DROP_CASES, ids=DROP_IDS)
@pytest.mark.parametrize("M", [1, 5, 1312])
def test_layernorm_backward_dropout(cuda, M, p, word):
    ops = _ops()
    g = torch.Generator().manual_seed(36)
    x = _rnd(g, M, 768, scale=2.0)
    gam = (1 + 0.1 * torch.randn(768, generator=g)).to(cuda)
    bet = (0.1 * torch.randn(768, generator=g)).to(cuda)
    dy = _rnd(g, M, 768)
    y, stats = torch.empty_like(x), torch.empty(M, 2, device=cuda)
    ops.layernorm_fwd(x, gam, bet, y, stats, 1e-12)
    dx, dxd = torch.empty_like(x), torch.empty_like(x)
    dgam, dbet, dbias = (torch.zeros(768, device=cuda) for _ in range(3))
    with _bound(word, cuda):
        ops.layernorm_bwd(dy, x, stats, gam, dx, dxd, dgam, dbet, dbias, p, SEED)
    xr = x.float().requires_grad_(True)
    torch.nn.functional.layer_norm(xr, (768,), gam, bet, 1e-12).backward(dy.float())
    _close(dx, xr.grad, TOL_BF16_OP, "layernorm dx M=%d" % M)
    mult = _mult(SEED, D.layernorm_index(M), p, word, cuda)
    assert bool((dxd[mult == 0] == 0).all())
    kept = mult != 0
    ref = dx.float() * mult
    # dx_drop = bf16(dx_fp32 * m) and dx = bf16(dx_fp32): they differ by the rounding of the product (half an ulp) and the
    # rounding of dx carried through m (half an ulp of dx, times m)
    bound = 0.5 * _bf16_ulp(torch.maximum(ref.abs(), dxd.float().abs())) + 0.5 * _bf16_ulp(dx.float()) * mult
    assert bool(((dxd.float() - ref).abs() <= bound)[kept].all())
    # dbias_drop: column sums of exactly the tensor the dense layer's weight gradient reads
    _close(dbias, dxd.float().sum(0), 1e-5, "layernorm dbias_drop M=%d" % M)
    wrong = dx.float() * _mult(SEED + 1, D.layernorm_index(M), p, word, cuda)
    _sharp(dxd, ref, wrong, TOL_BF16_OP, "layernorm dx_drop M=%d p=%g" % (M, p), p)


# ------------------------------------------------------------------------------------------------ embeddings
@pytest.mark.parametrize("p,word", DROP_CASES, ids=DROP_IDS)
@pytest.mark.parametrize("gh,lt", [(3, 32), (7, 20), (12, 20)], ids=["224px", "448px", "768px"])
def test_embeddings_dropout(cuda, gh, lt, p, word):
    """Text and visual embeddings, forward and backward, against fp32 autograd of dropout(LN(.)) with the restated masks;
    uniform n_ex and ragged repeat counts (seq2vid / vid_start)."""
    ops = _ops()
    from oracle import clipbert_ref as R
    g = torch.Generator().manual_seed(37)
    nseq, T, gw = 6, 2, gh
    Lv, L = gh * gw, lt + gh * gw
    shapes = {"e.word_embeddings.weight": (500, 768), "e.position_embeddings.weight": (64, 768), "e.token_type_embeddings.weight": (2, 768),
              "v.row_position_embeddings.weight": (16, 768), "v.col_position_embeddings.weight": (16, 768),
              "v.token_type_embeddings.weight": (1, 768)}
    sd0 = {k: torch.randn(*s, generator=g) * 0.5 for k, s in shapes.items()}
    for pre in ("e.", "v."):
        sd0[pre + "LayerNorm.weight"] = 1 + 0.1 * torch.randn(768, generator=g)
        sd0[pre + "LayerNorm.bias"] = 0.1 * torch.randn(768, generator=g)
    ids = torch.randint(0, 500, (nseq, lt), generator=g)
    dh = _rnd(g, nseq, L, 768, dev="cpu")
    d = {k: v.to(cuda) for k, v in sd0.items()}
    mt = _mult(SEED + 1, D.embedding_index(nseq, L, range(lt)), p, word)
    mv = _mult(SEED + 2, D.embedding_index(nseq, L, range(lt, L)), p, word)
    mt_w = _mult(SEED + 2, D.embedding_index(nseq, L, range(lt)), p, word)
    mv_w = _mult(SEED + 3, D.embedding_index(nseq, L, range(lt, L)), p, word)
    for counts in ([2, 2, 2], [1, 3, 2]):
        nvid = len(counts)
        grid = _rnd(g, nvid, T, gh, gw, 768, dev="cpu").float()

        def reference(m_t, m_v):
            sd = {k: v.clone().requires_grad_(True) for k, v in sd0.items()}
            gr = grid.clone().requires_grad_(True)
            te = R.bert_embeddings(ids, sd, "e.", 1e-12) * m_t
            ve = R.visual_embeddings(R.repeat_tensor_rows(gr, counts), sd, "v.", 1e-12) * m_v
            out = torch.cat([te, ve], 1)
            out.backward(dh.float())
            return out.detach(), gr.grad, {k: v.grad for k, v in sd.items()}

        ref, dgrid_ref, gref = reference(mt, mv)
        wref, wdgrid, wg = reference(mt_w, mv_w)
        if counts[0] == counts[1] == counts[2]:
            s2v, starts, nx = None, None, counts[0]
        else:
            s2v = torch.tensor([i for i, r in enumerate(counts) for _ in range(r)], dtype=torch.int32, device=cuda)
            starts = torch.tensor([0, 1, 4, 6], dtype=torch.int32, device=cuda)
            nx = 0
        out = torch.zeros(nseq * L, 768, device=cuda, dtype=BF16)
        st_t, st_v = torch.empty(nseq * lt, 2, device=cuda), torch.empty(nseq * Lv, 2, device=cuda)
        gridc = grid.to(cuda).to(BF16)
        gz = {k: torch.zeros_like(v) for k, v in d.items()}
        dv_tmp = torch.empty(nseq * Lv, 768, device=cuda)
        dgrid = torch.empty(nvid, T, gh, gw, 768, device=cuda, dtype=BF16)
        dhc = dh.to(cuda).view(nseq * L, 768)
        with _bound(word, cuda):
            ops.embed_text_fwd(ids.to(cuda), d["e.word_embeddings.weight"], d["e.position_embeddings.weight"], d["e.token_type_embeddings.weight"],
                               d["e.LayerNorm.weight"], d["e.LayerNorm.bias"], out, st_t, nseq, lt, L, 1e-12, p, SEED + 1)
            ops.embed_visual_fwd(gridc, s2v, nx, d["v.row_position_embeddings.weight"], d["v.col_position_embeddings.weight"],
                                 d["v.token_type_embeddings.weight"], d["v.LayerNorm.weight"], d["v.LayerNorm.bias"], out, st_v, nseq, T, gh, gw,
                                 lt, L, 1e-12, p, SEED + 2)
            ops.embed_text_bwd(dhc, ids.to(cuda), d["e.word_embeddings.weight"], d["e.position_embeddings.weight"],
                               d["e.token_type_embeddings.weight"], d["e.LayerNorm.weight"], st_t, gz["e.word_embeddings.weight"],
                               gz["e.position_embeddings.weight"], gz["e.token_type_embeddings.weight"], gz["e.LayerNorm.weight"],
                               gz["e.LayerNorm.bias"], nseq, lt, L, p, SEED + 1)
            ops.embed_visual_bwd(dhc, gridc, s2v, starts, nx, d["v.row_position_embeddings.weight"], d["v.col_position_embeddings.weight"],
                                 d["v.token_type_embeddings.weight"], d["v.LayerNorm.weight"], st_v, dv_tmp, dgrid,
                                 gz["v.row_position_embeddings.weight"], gz["v.col_position_embeddings.weight"], gz["v.token_type_embeddings.weight"],
                                 gz["v.LayerNorm.weight"], gz["v.LayerNorm.bias"], nseq, nvid, T, gh, gw, lt, L, p, SEED + 2)
        o = out.view(nseq, L, 768).cpu()
        assert bool((o[:, :lt][mt == 0] == 0).all()) and bool((o[:, lt:][mv == 0] == 0).all())
        what = "embeddings %dx%d counts=%s p=%g" % (gh, gw, counts, p)
        _sharp(o, ref, wref, TOL_BF16_OP, what + " fwd", p)
        _sharp(dgrid.cpu(), dgrid_ref, wdgrid, TOL_BF16_OP, what + " dgrid", p)
        for k in sd0:
            _sharp(gz[k].cpu(), gref[k], wg[k], 2e-3, what + " d" + k, p)


# ------------------------------------------------------------------------------------------------ attention
def _attention_switch(path):
    """(set, restore) of the kernel-selection switch a path names."""
    from clipbert_b200 import _lib
    ops = _ops()
    general = lambda on: _lib.lib().cb_debug_attention_general(ctypes.c_int(on))      # noqa: E731
    return {"default": (lambda: None, lambda: None),
            "rows64": (lambda: ops.set_attention_rows48(0), lambda: ops.set_attention_rows48(1)),
            "cuda_core_fwd": (lambda: ops.set_attention_flash(0), lambda: ops.set_attention_flash(1)),
            "sync_loads": (lambda: ops.set_attention_flash_pipe(0), lambda: ops.set_attention_flash_pipe(1)),
            "general": (lambda: general(1), lambda: general(0))}[path]


_LENGTHS = [9, 41, 48, 49, 64, 65, 69, 149, 169, 521]
ATTN_CASES = ([("default", L, p, w) for L in _LENGTHS for p, w in DROP_CASES]
              + [("general", L, p, w) for L in _LENGTHS for p, w in DROP_CASES]
              + [("rows64", L, 0.1, None) for L in (9, 41, 48)]                 # the 64-row kernels for L <= 48
              + [("cuda_core_fwd", L, 0.1, None) for L in (65, 69, 149, 521)]   # CUDA-core forward beside the long tensor-core backward
              + [("sync_loads", L, 0.1, None) for L in (65, 169, 521)])         # flash forward without the cp.async double buffer


@pytest.mark.parametrize("path,L,p,word", ATTN_CASES,
                         ids=["%s-L%d-p%g%s" % (c[0], c[1], c[2], "-word" if c[3] else "") for c in ATTN_CASES])
def test_attention_dropout(cuda, path, L, p, word):
    """ctx and lse (taken before dropout) of the forward, dqkv of the backward, against fp32 autograd of softmax(S) * mask @ V."""
    ops = _ops()
    heads = 12
    nseq = 1 if L == 521 else 3
    lt = min(32, L - 1) if L < 521 else 512
    g = torch.Generator().manual_seed(38 + L)
    qkv = _rnd(g, nseq * L, 3 * 768)
    dctx = _rnd(g, nseq * L, 768)
    mask = torch.ones(nseq, lt, dtype=torch.int64)
    mask[0, lt - 3:] = 0                                   # masked text keys
    mask[-1, lt // 2:] = 0
    ctx = torch.empty(nseq * L, 768, device=cuda, dtype=BF16)
    lse = torch.empty(nseq, heads, L, device=cuda)
    dqkv = torch.empty_like(qkv)
    on, off = _attention_switch(path)
    try:
        on()
        with _bound(word, cuda):
            ops.attention_fwd(qkv, mask.to(cuda), ctx, lse, nseq, L, lt, heads, p, SEED)
            ops.attention_bwd(qkv, mask.to(cuda), ctx, dctx, lse, dqkv, nseq, L, lt, heads, p, SEED)
            torch.cuda.synchronize()
    finally:
        off()

    def reference(seed):
        x = qkv.float().cpu().view(nseq, L, 3, heads, 64).requires_grad_(True)
        q, k, v = (x[:, :, i].permute(0, 2, 1, 3) for i in range(3))
        full = torch.cat([mask, torch.ones(nseq, L - lt, dtype=torch.int64)], 1)
        s = q @ k.transpose(-1, -2) / 8.0 + (1.0 - full[:, None, None, :].float()) * -10000.0
        pr = torch.softmax(s, -1) * _mult(seed, D.attention_index(nseq, heads, L), p, word)
        o = (pr @ v).permute(0, 2, 1, 3).reshape(nseq * L, 768)
        o.backward(dctx.float().cpu())
        return o.detach(), torch.logsumexp(s, -1).detach(), x.grad.reshape(nseq * L, 3 * 768)

    ref_o, ref_lse, ref_d = reference(SEED)
    w_o, _, w_d = reference(SEED + 1)
    what = "attention %s L=%d p=%g" % (path, L, p)
    _close(lse.cpu(), ref_lse, 1e-4, what + " lse")
    _sharp(ctx.cpu(), ref_o, w_o, TOL_BF16_OP, what + " ctx", p)
    _sharp(dqkv.cpu(), ref_d, w_d, 2 * TOL_BF16_OP, what + " dqkv", p)


# ------------------------------------------------------------------------------------------------ model level
@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)


P_TRAIN = 0.1


def _model_drop(seed, word, nseq, l, lt, heads=12):
    """The oracle's dropout hook with the masks ClipBertForVideoTextRetrieval draws for the base seed `seed` and device word
    `word` (clipbert_b200/modeling.py):
      text / visual embeddings  seed + 1 / seed + 2                                     (_forward_body, :427-429, :620-634)
      encoder layer i           ls = seed + 16 (i + 1): attention probabilities ls + 1, attention-output dense ls + 2,
                                FFN-output dense ls + 3                                 (:434-458, backward :575, :598, :606)
      pooled, before the head   seed + 5                                                (:484, backward :526)"""
    def mult(s, idx):
        return torch.from_numpy(D.multipliers(D.effective_seed(s, word), idx, P_TRAIN))

    def drop(site, layer, x):
        if site == "text_emb":
            m = mult(seed + 1, D.embedding_index(nseq, l, range(lt)))
        elif site == "visual_emb":
            m = mult(seed + 2, D.embedding_index(nseq, l, range(lt, l)))
        elif site == "pooled":
            m = mult(seed + 5, D.flat_index(x.numel()))
        else:
            ls = seed + 16 * (layer + 1)
            if site == "attn_probs":
                m = mult(ls + 1, D.attention_index(nseq, heads, l))
            else:
                m = mult(ls + (2 if site == "attn_out" else 3), D.gemm_index(nseq * l, x.shape[-1]))
        return x * m.view(x.shape)
    return drop


MODEL_CASES = [(3, 32, [2, 2, 2]), (7, 20, [1, 3, 2])]


@pytest.mark.parametrize("case", MODEL_CASES, ids=["L41", "L69-ragged"])
def test_transformer_training_step_with_dropout(cuda, weights, case):
    """ClipBertForVideoTextRetrieval.transformer in train mode with hidden and attention dropout 0.1, forward and backward,
    against fp32 autograd of the oracle with the restated masks injected (tolerances and carve-outs of
    test_gpu_model.py::test_transformer_forward_backward). L = 41 runs the 48-row attention kernels, L = 69 the long-sequence
    kernels and the ragged seq2vid gather."""
    import clipbert_b200 as cb
    from oracle import clipbert_ref as R, synth
    gh, lt, counts = case
    nvid, T, nseq, L = len(counts), 2, sum(counts), lt + gh * gh
    cfg = make_cfg(hidden_dropout_prob=P_TRAIN, attention_probs_dropout_prob=P_TRAIN)
    model = cb.ClipBert(cfg, detectron2_model_cfg="R-50-grid.yaml", transformer_cls=cb.ClipBertForVideoTextRetrieval)
    assert not model.load_state_dict(weights).missing_keys
    model = model.to(cuda).train()
    tr = model.transformer
    g = torch.Generator().manual_seed(2)
    grid = (torch.randn(nvid, T, gh, gh, 768, generator=g).abs() * 2).to(BF16).float()
    ids, mask = synth.synth_text(nseq, lt, seed=3)
    labels = torch.randint(0, 2, (nseq,), generator=g)
    gc = grid.to(cuda).to(BF16).requires_grad_(True)
    tr._capture = {}
    out = tr(ids.to(cuda), gc, mask.to(cuda), labels=labels.to(cuda), sample_size=nvid, _repeat_counts=counts)
    cap, tr._capture = tr._capture, None
    # the base seed of this call (_next_seed, modeling.py:315-319) and the device word it advanced (:321-331, :416)
    seed = (tr._seed_base + tr._call_count * 1000003) & (2 ** 64 - 1)
    word = int(tr._drop_counter.item())
    out["loss"].mean().backward()

    def oracle(base_seed):
        sd = {k: (v.clone().requires_grad_(True) if k.startswith("transformer.") else v) for k, v in weights.items()}
        gr = grid.clone().requires_grad_(True)
        drop = _model_drop(base_seed, word, nseq, L, lt)
        _, pooled = R.clipbert_base_model(ids, R.repeat_tensor_rows(gr, counts), mask, sd, drop=drop)
        # the gradient is taken along the run's classifier ReLU pattern (see Rounding.relu_masks)
        hpat = R.Rounding(relu_masks={"transformer.classifier.relu": (cap["c1"] > 0).cpu()})
        logits = R.mlp_head(pooled, sd, rnd=hpat, drop=drop)
        loss = R.retrieval_loss(logits, labels).mean()
        loss.backward()
        return logits.detach(), float(loss.detach()), gr.grad, sd

    def errors(ref):
        logits, loss, dgrid, sd = ref
        grads = {}
        for name, p in tr.named_parameters():
            key = "transformer." + name
            r = sd[key].grad
            if r is None or float(r.abs().sum()) == 0.0 or name.endswith("attention.self.key.bias"):
                continue
            grads[key] = (relerr(p.grad, r), cosine(p.grad, r))
        return (relerr(out["logits"], logits), abs(float(out["loss"].mean()) - loss), relerr(gc.grad, dgrid), cosine(gc.grad, dgrid),
                grads)

    right = oracle(seed)
    e_logits, e_loss, e_dgrid, c_dgrid, grads = errors(right)
    w_logits, w_loss, w_dgrid, _, w_grads = errors(oracle(seed + 1))
    worst = max(e for e, _ in grads.values())
    w_median = sorted(e for e, _ in w_grads.values())[len(w_grads) // 2]
    print("transformer L=%d: logits %.2e / %.2e, loss %.2e / %.2e, dgrid %.2e / %.2e, parameter gradients worst %.2e / median %.2e "
          "(right masks / masks of seed + 1)" % (L, e_logits, w_logits, e_loss, w_loss, e_dgrid, w_dgrid, worst, w_median))
    assert e_logits < TOL_LOGITS and e_loss < 2e-3, (e_logits, e_loss)
    assert e_dgrid < TOL_GRAD and c_dgrid > 0.999, (e_dgrid, c_dgrid)
    bad = [(k, e, c) for k, (e, c) in grads.items() if not (e < TOL_GRAD and c > 0.999)]
    assert not bad, bad[:10]
    # carve-out of test_transformer_forward_backward: the key bias gradient is mathematically zero (rounding noise on both sides)
    for name, p in tr.named_parameters():
        if name.endswith("attention.self.key.bias"):
            qb = right[3]["transformer." + name.replace("key.bias", "query.bias")].grad
            assert float(p.grad.norm()) < 0.05 * float(qb.norm()), name
    assert len(grads) >= 180
    # the wrong masks miss by far: logits and dgrid by MARGIN x their bounds, half of the parameter gradients by 5 x
    assert w_logits > MARGIN * TOL_LOGITS and w_dgrid > MARGIN * TOL_GRAD and w_median > 5 * TOL_GRAD, (w_logits, w_dgrid, w_median)
