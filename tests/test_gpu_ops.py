"""Per-kernel parity: every C-ABI entry point against a plain PyTorch fp32 reference of the same op."""
import math

import pytest
import torch
import torch.nn.functional as F

from util import TOL_BF16_OP, TOL_FP32_OP, relerr

pytestmark = pytest.mark.gpu


def _ops():
    from clipbert_b200 import ops
    return ops


def _rnd(g, *shape, scale=1.0, dev="cuda"):
    return (torch.randn(*shape, generator=g) * scale).to(dev).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------ GEMM
# cb_gemm_desc.reserved values: SINGLE (bit 1, no meaning to the kernel) makes ops.gemm launch exactly the given descriptor
# (no tuning-table lookup); OCC2 (bit 5) asks for the two-CTAs-per-SM instantiation. NARROW is a test-side flag, not a reserved
# bit: the case runs on 128 x 64 tiles (block_n = 64) instead of the width the launch model picks.
SINGLE, NARROW, OCC2 = 2, 1, 32


def _tiles(flag):
    return dict(block_n=64) if flag & NARROW else {}


@pytest.mark.parametrize("cfg", [(64, SINGLE), (128, SINGLE), (256, SINGLE)])
@pytest.mark.parametrize("shape", [(128, 256, 64), (300, 512, 192), (1312, 768, 768), (77, 264, 1096), (40000, 256, 64)])
def test_gemm_tn_fp32_out(cuda, cfg, shape):
    """Every tile width, ragged M / N / K, several tiles per persistent CTA."""
    ops = _ops()
    M, N, K = shape
    bn, knob = cfg
    g = torch.Generator().manual_seed(1)
    A, B = _rnd(g, M, K), _rnd(g, N, K, scale=0.1)
    C = torch.full((M, N), 7.0, device=cuda)
    ops.gemm(mode=ops.CB_GEMM_TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=N, b_ld=K, out=C, out_ld=N, out_fp32=1, block_n=bn,
             reserved=knob)
    assert relerr(C, A.float() @ B.float().t()) < TOL_FP32_OP


@pytest.mark.parametrize("knob", [SINGLE])
@pytest.mark.parametrize("shape", [(500, 384, 256), (1312, 2304, 768), (64, 768, 3072)])
def test_gemm_nn_dgrad(cuda, shape, knob):
    ops = _ops()
    M, N, K = shape     # out [M, N] = A [M, K] @ B [K, N]
    g = torch.Generator().manual_seed(2)
    A, B = _rnd(g, M, K), _rnd(g, K, N, scale=0.1)
    C = torch.zeros(M, N, device=cuda)
    ops.gemm(mode=ops.CB_GEMM_NN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=K, b_ld=N, out=C, out_ld=N, out_fp32=1, reserved=knob)
    assert relerr(C, A.float() @ B.float()) < TOL_FP32_OP


@pytest.fixture(params=["tma_store", "two_ctas_per_sm"])
def epilogue_variant(request):
    """The GEMM in its two instantiations: one CTA per SM (id "tma_store", kept so that the test ids stay stable; the operands
    arrive by TMA, the epilogue runs in the consumer warpgroups), and two CTAs per SM (ops.set_occ2(2): every eligible launch
    on 128 x 64 tiles with <= 113 KB of shared memory)."""
    ops = _ops()
    ops.set_occ2(2 if request.param == "two_ctas_per_sm" else 0)
    yield request.param
    ops.set_occ2(1)


@pytest.mark.parametrize("narrow", [0, NARROW])
@pytest.mark.parametrize("shape", [(500, 384, 256), (20000, 512, 128), (3000, 64, 64), (500, 392, 256)])
def test_gemm_epilogues(cuda, narrow, shape, epilogue_variant):
    """Every epilogue kind on the width the launch model picks and on 128 x 64 tiles (narrow = NARROW), several tiles per
    persistent CTA; N = 392 (N % 16 == 8) takes the guarded epilogue with a ragged last column group in bf16."""
    ops = _ops()
    M, N, K = shape
    g = torch.Generator().manual_seed(3)
    A, B, R, AUX = _rnd(g, M, K), _rnd(g, N, K, scale=0.1), _rnd(g, M, N), _rnd(g, M, N)
    scale = (torch.rand(N, generator=g) + 0.5).to(cuda)
    shift = torch.randn(N, generator=g).to(cuda)
    acc = A.float() @ B.float().t()
    base = dict(mode=ops.CB_GEMM_TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=N, b_ld=K, out_ld=N, reserved=SINGLE)
    tiles = _tiles(narrow)
    C, C2 = torch.zeros(M, N, device=cuda, dtype=torch.bfloat16), torch.zeros(M, N, device=cuda, dtype=torch.bfloat16)
    ops.gemm(**base, **tiles, scale=scale, shift=shift, residual=R, res_ld=N, act=ops.ACT_RELU, out=C, out2=C2, out2_ld=N)
    pre = acc * scale + shift + R.float()
    assert relerr(C, pre.relu()) < TOL_BF16_OP and relerr(C2, pre) < TOL_BF16_OP
    ops.gemm(**base, **tiles, shift=shift, act=ops.ACT_GELU, out=C)
    assert relerr(C, F.gelu(acc + shift)) < TOL_BF16_OP
    ops.gemm(**base, **tiles, shift=shift, act=ops.ACT_TANH, out=C)
    assert relerr(C, torch.tanh(acc + shift)) < TOL_BF16_OP
    # gelu + stashed derivative from one erf (BertIntermediate forward), consumed by AUX_MUL in the backward
    u = acc + shift
    ops.gemm(**base, **tiles, shift=shift, act=ops.ACT_GELU_STASH_GRAD, out=C, out2=C2, out2_ld=N)
    dgelu = 0.5 * (1 + torch.erf(u / math.sqrt(2))) + u * torch.exp(-0.5 * u * u) / math.sqrt(2 * math.pi)
    assert relerr(C, F.gelu(u)) < TOL_BF16_OP and relerr(C2, dgelu) < TOL_BF16_OP
    a = AUX.float()
    ops.gemm(**base, **tiles, aux=AUX, aux_ld=N, aux_mode=ops.AUX_MUL, out=C)
    assert relerr(C, acc * a) < TOL_BF16_OP
    gelu_grad = 0.5 * (1 + torch.erf(a / math.sqrt(2))) + a * torch.exp(-0.5 * a * a) / math.sqrt(2 * math.pi)
    for mode, fac in [(ops.AUX_RELU_MASK, (a > 0).float()), (ops.AUX_GELU_GRAD, gelu_grad), (ops.AUX_TANH_GRAD, 1 - a * a)]:
        ops.gemm(**base, **tiles, residual=R, res_ld=N, aux=AUX, aux_ld=N, aux_mode=mode, out=C)
        assert relerr(C, (acc + R.float()) * fac) < TOL_BF16_OP
    # plain bf16 output, aux only, dropout + residual, every tile width
    for bn in (64, 128, 256):
        ops.gemm(**base, out=C, block_n=bn)
        assert relerr(C, acc) < TOL_BF16_OP
        ops.gemm(**base, aux=AUX, aux_ld=N, aux_mode=ops.AUX_RELU_MASK, out=C, block_n=bn)
        assert relerr(C, acc * (a > 0)) < TOL_BF16_OP
    ops.gemm(**base, **tiles, shift=shift, residual=R, res_ld=N, dropout_p=0.1, dropout_seed=5, out=C)
    ones = torch.ones(M, N, device=cuda, dtype=torch.bfloat16)
    msk = torch.empty_like(ones)
    ops.dropout(ones, msk, 0.1, 5)
    assert relerr(C, (acc + shift) * msk.float() + R.float()) < TOL_BF16_OP


@pytest.mark.parametrize("knob", [SINGLE, SINGLE | NARROW])
@pytest.mark.parametrize("dims", [(2, 7, 7, 64, 64), (3, 14, 14, 128, 128), (2, 28, 28, 64, 192), (1, 3, 5, 512, 64), (64, 14, 14, 256, 256)])
def test_conv3x3_fwd_and_dgrad(cuda, dims, knob, epilogue_variant):
    ops = _ops()
    NB, H, W, Cin, Cout = dims
    g = torch.Generator().manual_seed(4)
    x = _rnd(g, NB, H, W, Cin)
    w = _rnd(g, Cout, Cin, 3, 3, scale=0.05)
    xp = torch.zeros(NB, H + 2, W + 2, Cin, device=cuda, dtype=torch.bfloat16)
    xp[:, 1:-1, 1:-1] = x
    P = NB * (H + 2) * (W + 2)
    y = torch.zeros(NB * H * W, Cout, device=cuda, dtype=torch.bfloat16)
    wk = w.permute(0, 2, 3, 1).contiguous().view(Cout, 9 * Cin)
    ops.gemm(mode=ops.CB_GEMM_TN, m=P, n=Cout, k=Cin, a=xp, a_rows=P, a_ld=Cin, b=wk, b_rows=Cout, b_ld=9 * Cin, ntaps=9,
             tap_w=W + 2, tap_sign=1, out=y, out_ld=Cout, rowmap=ops.ROWMAP_UNPAD, map_h=H, map_w=W, reserved=SINGLE, **_tiles(knob))
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    assert relerr(y, ref) < TOL_BF16_OP
    # dgrad of a conv whose forward weight is wf [Cin(out), Cout(in), 3, 3] stored KRSC: x plays dY
    wf = _rnd(g, Cin, Cout, 3, 3, scale=0.05)
    wfk = wf.permute(0, 2, 3, 1).contiguous().view(Cin, 9 * Cout)         # [out_f, (r,s,in_f)] = forward layout
    ops.gemm(mode=ops.CB_GEMM_NN, m=P, n=Cout, k=Cin, a=xp, a_rows=P, a_ld=Cin, b=wfk, b_rows=Cin, b_ld=9 * Cout, ntaps=9,
             tap_w=W + 2, tap_sign=-1, out=y, out_ld=Cout, rowmap=ops.ROWMAP_UNPAD, map_h=H, map_w=W, reserved=SINGLE, **_tiles(knob))
    ref = F.conv_transpose2d(x.float().permute(0, 3, 1, 2), wf.float(), padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    assert relerr(y, ref) < TOL_BF16_OP


@pytest.mark.parametrize("knob", [0, NARROW])
@pytest.mark.parametrize("dims", [(3, 5, 6, 64, 64), (40, 28, 28, 256, 128)])
def test_rowmap_pad_keeps_border_zero(cuda, dims, knob, epilogue_variant):
    ops = _ops()
    NB, H, W, K, N = dims
    M = NB * H * W
    g = torch.Generator().manual_seed(5)
    A, B, AUX = _rnd(g, M, K), _rnd(g, N, K, scale=0.1), _rnd(g, M, N)
    yp = torch.zeros(NB, H + 2, W + 2, N, device=cuda, dtype=torch.bfloat16)
    ops.gemm(mode=ops.CB_GEMM_TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=N, b_ld=K, out=yp, out_ld=N,
             rowmap=ops.ROWMAP_PAD, map_h=H, map_w=W, aux=AUX, aux_ld=N, aux_mode=ops.AUX_RELU_MASK, reserved=SINGLE, **_tiles(knob))
    ref = ((A.float() @ B.float().t()) * (AUX.float() > 0)).view(NB, H, W, N)
    assert relerr(yp[:, 1:-1, 1:-1], ref) < TOL_BF16_OP
    border = yp.clone()
    border[:, 1:-1, 1:-1] = 0
    assert float(border.float().abs().max()) == 0.0


@pytest.mark.parametrize("case", [(64, 128, 64, 64, 1, SINGLE), (1312, 768, 768, 128, 1, SINGLE), (1000, 256, 192, 64, 1, SINGLE),
                                  (333, 136, 72, 64, 1, SINGLE), (5000, 256, 256, 128, 7, SINGLE), (640, 128, 128, 64, 100, SINGLE),
                                  (32, 8, 1536, 128, 1, SINGLE), (1312, 768, 3072, 256, 0, SINGLE), (5000, 512, 256, 128, 3, OCC2),
                                  (1312, 2304, 768, 0, 0, 0), (50176, 512, 128, 0, 0, 0)])
def test_wgrad(cuda, case):
    ops = _ops()
    P, Mo, No, bn, sk, knob = case
    g = torch.Generator().manual_seed(6)
    dY, X = _rnd(g, P, Mo), _rnd(g, P, No)
    rs = (torch.rand(Mo, generator=g) + 0.5).to(cuda)
    dW = torch.zeros(Mo, No, device=cuda)
    ops.gemm(mode=ops.CB_GEMM_WGRAD, m=Mo, n=No, k=P, a=dY, a_rows=P, a_ld=Mo, b=X, b_rows=P, b_ld=No, split_k=sk, scale=rs,
             out=dW, out_ld=No, out_fp32=1, block_n=bn, reserved=knob)
    assert relerr(dW, (dY.float().t() @ X.float()) * rs[:, None]) < TOL_FP32_OP
    # accumulation semantics: a second launch adds
    ops.gemm(mode=ops.CB_GEMM_WGRAD, m=Mo, n=No, k=P, a=dY, a_rows=P, a_ld=Mo, b=X, b_rows=P, b_ld=No, split_k=sk, scale=rs,
             out=dW, out_ld=No, out_fp32=1, block_n=bn, reserved=knob)
    assert relerr(dW, 2 * (dY.float().t() @ X.float()) * rs[:, None]) < TOL_FP32_OP


@pytest.mark.parametrize("dims", [(2, 7, 7, 64, 128, 1, SINGLE), (4, 14, 14, 128, 128, 3, SINGLE), (4, 14, 14, 256, 256, 0, OCC2)])
def test_wgrad_conv3x3(cuda, dims):
    ops = _ops()
    NB, H, W, Cin, Cout, sk, knob = dims
    g = torch.Generator().manual_seed(7)
    x, dy = _rnd(g, NB, H, W, Cin), _rnd(g, NB, H, W, Cout)
    xp = torch.zeros(NB, H + 2, W + 2, Cin, device=cuda, dtype=torch.bfloat16)
    dyp = torch.zeros(NB, H + 2, W + 2, Cout, device=cuda, dtype=torch.bfloat16)
    xp[:, 1:-1, 1:-1], dyp[:, 1:-1, 1:-1] = x, dy
    P = NB * (H + 2) * (W + 2)
    dW = torch.zeros(Cout, 9 * Cin, device=cuda)
    ops.gemm(mode=ops.CB_GEMM_WGRAD, m=Cout, n=Cin, k=P, a=dyp, a_rows=P, a_ld=Cout, b=xp, b_rows=P, b_ld=Cin, ntaps=9, tap_w=W + 2,
             tap_sign=1, split_k=sk, out=dW, out_ld=9 * Cin, out_fp32=1, reserved=knob)
    wz = torch.zeros(Cout, Cin, 3, 3, device=cuda, requires_grad=True)
    F.conv2d(x.float().permute(0, 3, 1, 2), wz, padding=1).backward(dy.float().permute(0, 3, 1, 2))
    assert relerr(dW, wz.grad.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin)) < TOL_FP32_OP


def test_gemm_dropout_is_a_pure_function_of_seed_and_index(cuda):
    ops = _ops()
    M, N, K = 512, 768, 64
    g = torch.Generator().manual_seed(8)
    A, B = _rnd(g, M, K), _rnd(g, N, K, scale=0.1)
    outs = []
    for bn in (64, 128):
        C = torch.zeros(M, N, device=cuda)
        ops.gemm(mode=ops.CB_GEMM_TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=N, b_ld=K, out=C, out_ld=N, out_fp32=1,
                 dropout_p=0.1, dropout_seed=99, block_n=bn)
        outs.append(C)
    assert torch.equal(outs[0], outs[1])            # same mask whatever the tiling
    keep = outs[0] != 0
    assert abs(float(keep.float().mean()) - 0.9) < 0.01
    ref = A.float() @ B.float().t()
    assert relerr(outs[0][keep], ref[keep] / 0.9) < TOL_FP32_OP
    # the standalone dropout kernel and the LayerNorm-backward mask use the same generator
    x = torch.ones(M, N, device=cuda, dtype=torch.bfloat16)
    y = torch.empty_like(x)
    ops.dropout(x, y, 0.1, 99)
    assert torch.equal(y != 0, keep)


def test_dropout_stream_advances_on_the_device_under_graph_replay(cuda):
    """The reference draws fresh masks at every call (transformers.py:170,222,295,375). Seeds are by-value kernel arguments,
    so a captured graph would replay the same masks; the stream position therefore lives in a device word that the graph
    advances (cb_dropout_offset_advance) and every mask consumer reads at run time (cb_dropout_offset_bind). Two replays must
    differ, and within one replay the 'backward' consumers (LayerNorm backward, a second launch) must regenerate the masks of
    the 'forward' consumers (GEMM epilogue, cb_dropout) - same word, same seed."""
    ops = _ops()
    M, N, K = 256, 768, 64
    g = torch.Generator().manual_seed(8)
    A, B = _rnd(g, M, K), _rnd(g, N, K, scale=0.1)
    ones = torch.ones(M, N, device=cuda, dtype=torch.bfloat16)
    gam = torch.ones(N, device=cuda)
    stats = torch.zeros(M, 2, device=cuda)
    stats[:, 1] = 1.0
    counter = torch.zeros(1, dtype=torch.int64, device=cuda)
    word = torch.zeros(1, dtype=torch.int64, device=cuda)
    C = torch.zeros(M, N, device=cuda)
    m_fwd, m_bwd, dx, dxd = (torch.empty_like(ones) for _ in range(4))

    def step():
        ops.dropout_offset_advance(counter, word)
        ops.dropout_offset_bind(word)
        ops.gemm(mode=ops.CB_GEMM_TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=N, b_ld=K, out=C, out_ld=N, out_fp32=1,
                 dropout_p=0.1, dropout_seed=99)
        ops.dropout(ones, m_fwd, 0.1, 99)
        ops.dropout(ones, m_bwd, 0.1, 99)                                       # a later launch of the same step: same mask
        ops.layernorm_bwd(ones, ones, stats, gam, dx, dxd, None, None, None, 0.1, 99)
        ops.dropout_offset_bind(None)

    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            step()
        masks = []
        for _ in range(3):
            graph.replay()
            torch.cuda.synchronize()
            keep = m_fwd != 0
            assert torch.equal(keep, m_bwd != 0)                 # regenerated identically within the step
            assert torch.equal(keep, C != 0)                     # GEMM epilogue: same (seed, word, index) -> same decision
            assert torch.equal(dxd != 0, (dx != 0) & keep)       # LayerNorm backward's dropped copy
            assert abs(float(keep.float().mean()) - 0.9) < 0.01
            masks.append(keep.clone())
        assert int(counter.item()) == 4                          # one eager warm-up step + three replays (capturing runs nothing)
    finally:
        ops.dropout_offset_bind(None)
    assert not torch.equal(masks[0], masks[1]) and not torch.equal(masks[1], masks[2])
    # two different positions are independent draws: they agree on ~0.9^2 + 0.1^2 of the elements
    agree = float((masks[0] == masks[1]).float().mean())
    assert abs(agree - 0.82) < 0.02
    # unbound launches are what they always were: a pure function of (seed, index)
    y0, y1 = torch.empty_like(ones), torch.empty_like(ones)
    ops.dropout(ones, y0, 0.1, 99)
    ops.dropout(ones, y1, 0.1, 99)
    assert torch.equal(y0, y1) and not torch.equal(y0 != 0, masks[0])


def test_gemm_rejects_bad_arguments(cuda):
    ops = _ops()
    A = torch.zeros(16, 12, device=cuda, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="multiple of 8"):
        ops.gemm(mode=ops.CB_GEMM_TN, m=16, n=12, k=12, a=A, a_rows=16, a_ld=12, b=A, b_rows=12, b_ld=12, out=A, out_ld=12)
    with pytest.raises(RuntimeError, match="null"):
        ops.gemm(mode=ops.CB_GEMM_TN, m=16, n=16, k=16, a=None, a_rows=16, a_ld=16, b=A, b_rows=16, b_ld=16, out=A, out_ld=16)


# ------------------------------------------------------------------------------------------------ LayerNorm
@pytest.mark.parametrize("M", [1, 5, 1312])
def test_layernorm_fwd_bwd(cuda, M):
    ops = _ops()
    g = torch.Generator().manual_seed(9)
    x = _rnd(g, M, 768, scale=2.0)
    gam = (1 + 0.1 * torch.randn(768, generator=g)).to(cuda)
    bet = (0.1 * torch.randn(768, generator=g)).to(cuda)
    dy = _rnd(g, M, 768)
    y = torch.empty_like(x)
    stats = torch.empty(M, 2, device=cuda)
    ops.layernorm_fwd(x, gam, bet, y, stats, 1e-12)
    xr = x.float().requires_grad_(True)
    gr, br = gam.clone().requires_grad_(True), bet.clone().requires_grad_(True)
    ref = F.layer_norm(xr, (768,), gr, br, 1e-12)
    assert relerr(y, ref) < TOL_BF16_OP
    ref.backward(dy.float())
    dx = torch.empty_like(x)
    dgam, dbet, dbias = torch.zeros(768, device=cuda), torch.zeros(768, device=cuda), torch.zeros(768, device=cuda)
    ops.layernorm_bwd(dy, x, stats, gam, dx, None, dgam, dbet, dbias, 0.0, 0)
    assert relerr(dx, xr.grad) < TOL_BF16_OP
    assert relerr(dgam, gr.grad) < 1e-4 and relerr(dbet, br.grad) < 1e-4
    assert relerr(dbias, dx.float().sum(0)) < 1e-4
    # dropped copy: same mask as the forward GEMM epilogue would have used for (row, col)
    dxd = torch.empty_like(x)
    ops.layernorm_bwd(dy, x, stats, gam, dx, dxd, None, None, None, 0.1, 1234)
    ones = torch.ones(M, 768, device=cuda, dtype=torch.bfloat16)
    msk = torch.empty_like(ones)
    ops.dropout(ones, msk, 0.1, 1234)
    assert relerr(dxd, dx.float() * msk.float()) < TOL_BF16_OP


# ------------------------------------------------------------------------------------------------ embeddings
def test_embed_text_and_visual(cuda):
    ops = _ops()
    from oracle import clipbert_ref as R
    g = torch.Generator().manual_seed(10)
    nseq, lt, T, gh, gw, n_ex = 6, 12, 2, 3, 3, 2
    nvid, Lv, L = nseq // n_ex, gh * gw, lt + gh * gw
    sd = {k: (torch.randn(*s, generator=g) * 0.5) for k, s in {
        "e.word_embeddings.weight": (500, 768), "e.position_embeddings.weight": (64, 768), "e.token_type_embeddings.weight": (2, 768),
        "v.row_position_embeddings.weight": (10, 768), "v.col_position_embeddings.weight": (10, 768),
        "v.token_type_embeddings.weight": (1, 768)}.items()}
    for p in ("e.", "v."):
        sd[p + "LayerNorm.weight"] = 1 + 0.1 * torch.randn(768, generator=g)
        sd[p + "LayerNorm.bias"] = 0.1 * torch.randn(768, generator=g)
    sd = {k: v.requires_grad_(True) for k, v in sd.items()}
    ids = torch.randint(0, 500, (nseq, lt), generator=g)
    grid = _rnd(g, nvid, T, gh, gw, 768, dev="cpu").float().requires_grad_(True)
    te = R.bert_embeddings(ids, sd, "e.", 1e-12)
    ve = R.visual_embeddings(R.repeat_tensor_rows(grid, [n_ex] * nvid), sd, "v.", 1e-12)
    ref = torch.cat([te, ve], 1)
    dh = _rnd(g, nseq, L, 768, dev="cpu")
    ref.backward(dh.float())

    d = {k: v.detach().to(cuda) for k, v in sd.items()}
    out = torch.zeros(nseq * L, 768, device=cuda, dtype=torch.bfloat16)
    st_t, st_v = torch.empty(nseq * lt, 2, device=cuda), torch.empty(nseq * Lv, 2, device=cuda)
    gridc = grid.detach().to(cuda).to(torch.bfloat16)
    ops.embed_text_fwd(ids.to(cuda), d["e.word_embeddings.weight"], d["e.position_embeddings.weight"], d["e.token_type_embeddings.weight"],
                       d["e.LayerNorm.weight"], d["e.LayerNorm.bias"], out, st_t, nseq, lt, L, 1e-12, 0.0, 0)
    for s2v, starts, nx in [(None, None, n_ex),
                            (torch.tensor([0, 0, 1, 1, 2, 2], dtype=torch.int32, device=cuda), torch.tensor([0, 2, 4, 6], dtype=torch.int32, device=cuda), 0)]:
        ops.embed_visual_fwd(gridc, s2v, nx, d["v.row_position_embeddings.weight"], d["v.col_position_embeddings.weight"],
                             d["v.token_type_embeddings.weight"], d["v.LayerNorm.weight"], d["v.LayerNorm.bias"], out, st_v, nseq, T, gh, gw,
                             lt, L, 1e-12, 0.0, 0)
        assert relerr(out.view(nseq, L, 768), ref) < TOL_BF16_OP
        gz = {k: torch.zeros_like(v) for k, v in d.items()}
        dhc = dh.to(cuda).view(nseq * L, 768)
        ops.embed_text_bwd(dhc, ids.to(cuda), d["e.word_embeddings.weight"], d["e.position_embeddings.weight"], d["e.token_type_embeddings.weight"],
                           d["e.LayerNorm.weight"], st_t, gz["e.word_embeddings.weight"], gz["e.position_embeddings.weight"],
                           gz["e.token_type_embeddings.weight"][0], gz["e.LayerNorm.weight"], gz["e.LayerNorm.bias"], nseq, lt, L, 0.0, 0)
        dv_tmp = torch.empty(nseq * Lv, 768, device=cuda)
        dgrid = torch.empty(nvid, T, gh, gw, 768, device=cuda, dtype=torch.bfloat16)
        ops.embed_visual_bwd(dhc, gridc, s2v, starts, nx, d["v.row_position_embeddings.weight"], d["v.col_position_embeddings.weight"],
                             d["v.token_type_embeddings.weight"], d["v.LayerNorm.weight"], st_v, dv_tmp, dgrid,
                             gz["v.row_position_embeddings.weight"], gz["v.col_position_embeddings.weight"], gz["v.token_type_embeddings.weight"],
                             gz["v.LayerNorm.weight"], gz["v.LayerNorm.bias"], nseq, nvid, T, gh, gw, lt, L, 0.0, 0)
        for k in sd:
            if sd[k].grad is None:
                continue
            assert relerr(gz[k], sd[k].grad) < 2e-3, k
        assert relerr(dgrid, grid.grad) < TOL_BF16_OP


# ------------------------------------------------------------------------------------------------ attention
def test_attention_tensor_core_path_matches_general_path(cuda):
    """L <= 64 runs on the mma.sync kernels, longer sequences on the general kernels: same results, same dropout stream."""
    import ctypes
    from clipbert_b200 import _lib
    ops = _ops()
    nseq, L, lt, heads = 4, 41, 32, 12
    g = torch.Generator().manual_seed(21)
    qkv, dctx = _rnd(g, nseq * L, 3 * 768), _rnd(g, nseq * L, 768)
    mask = torch.ones(nseq, lt, dtype=torch.int64, device=cuda)
    mask[1, 20:] = 0
    outs = []
    for general in (0, 1):
        _lib.lib().cb_debug_attention_general(ctypes.c_int(general))
        ctx = torch.empty(nseq * L, 768, device=cuda, dtype=torch.bfloat16)
        lse = torch.empty(nseq, heads, L, device=cuda)
        dqkv = torch.empty_like(qkv)
        for p, seed in ((0.0, 0), (0.1, 5)):
            ops.attention_fwd(qkv, mask, ctx, lse, nseq, L, lt, heads, p, seed)
            ops.attention_bwd(qkv, mask, ctx, dctx, lse, dqkv, nseq, L, lt, heads, p, seed)
            outs.append((ctx.clone(), lse.clone(), dqkv.clone()))
    _lib.lib().cb_debug_attention_general(ctypes.c_int(0))
    for a, b in ((outs[0], outs[2]), (outs[1], outs[3])):
        assert relerr(a[0], b[0]) < 2 * TOL_BF16_OP and relerr(a[1], b[1]) < 1e-4 and relerr(a[2], b[2]) < 3 * TOL_BF16_OP


def test_attention_dropout_consistency(cuda):
    """With p>0 the backward must regenerate the forward mask: check dV against a finite set of probes."""
    ops = _ops()
    nseq, L, lt, heads = 2, 41, 32, 12
    g = torch.Generator().manual_seed(12)
    qkv = _rnd(g, nseq * L, 3 * 768, scale=0.5)
    mask = torch.ones(nseq, lt, dtype=torch.int64, device=cuda)
    ctx = torch.empty(nseq * L, 768, device=cuda, dtype=torch.bfloat16)
    lse = torch.empty(nseq, heads, L, device=cuda)
    ops.attention_fwd(qkv, mask, ctx, lse, nseq, L, lt, heads, 0.1, 77)
    # recover the dropped probabilities through V = identity-like probes: P_drop = ctx when V = e_j; instead compare
    # against torch using the mask inferred from a second forward with V := ones (row sums of dropped P)
    x = qkv.float().view(nseq, L, 3, heads, 64)
    q, k, v = (x[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    p = torch.softmax(q @ k.transpose(-1, -2) / 8.0, -1)
    qkv1 = qkv.clone().view(nseq, L, 3, heads, 64)
    qkv1[:, :, 2] = 1.0
    ctx1 = torch.empty_like(ctx)
    ops.attention_fwd(qkv1.view(nseq * L, -1), mask, ctx1, None, nseq, L, lt, heads, 0.1, 77)
    rowsum = ctx1.float().view(nseq, L, heads, 64)[..., 0].permute(0, 2, 1)          # sum_j P_ij * keep_ij / 0.9
    assert abs(float(rowsum.mean()) - 1.0) < 0.02 and float(rowsum.std()) > 1e-3     # dropout really applied, unbiased
    # linearity in dO of the backward with the same seed (mask regenerated identically)
    d1, d2 = _rnd(g, nseq * L, 768), _rnd(g, nseq * L, 768)
    outs = []
    for d in (d1, d2, (d1.float() + d2.float()).to(torch.bfloat16)):
        dq = torch.empty_like(qkv)
        ops.attention_bwd(qkv, mask, ctx, d, lse, dq, nseq, L, lt, heads, 0.1, 77)
        outs.append(dq.float())
    assert relerr(outs[2], outs[0] + outs[1]) < 3 * TOL_BF16_OP


# ------------------------------------------------------------------------------------------------ small ops
def test_colsum_padcast_castscale(cuda):
    ops = _ops()
    g = torch.Generator().manual_seed(13)
    x = _rnd(g, 1000, 2304)
    out = torch.zeros(2304, device=cuda)
    ops.colsum(x, out, 1000, 2304)
    assert relerr(out, x.float().sum(0)) < 1e-5
    src = torch.randn(37, 2, generator=g).to(cuda)
    dst = torch.full((37, 8), 5.0, device=cuda, dtype=torch.bfloat16)
    ops.pad_cast(src, dst)
    assert torch.equal(dst[:, :2], src.to(torch.bfloat16)) and float(dst[:, 2:].abs().sum()) == 0.0
    w = torch.randn(64 * 147, generator=g).to(cuda)
    sc = (torch.rand(64, generator=g) + 0.5).to(cuda)
    o = torch.empty(64 * 147, device=cuda, dtype=torch.bfloat16)
    ops.cast_scale(w, o, sc, 147)
    assert torch.equal(o, (w.view(64, 147) * sc[:, None]).to(torch.bfloat16).view(-1))
    ops.cast_scale(w, o)
    assert torch.equal(o, w.to(torch.bfloat16))


# ------------------------------------------------------------------------------------------------ CNN aux ops
@pytest.mark.parametrize("hw", [(224, 224), (64, 96), (37, 53)])
def test_stem_im2col_matches_unfold_with_bgr_flip(cuda, hw):
    ops = _ops()
    H, W = hw
    g = torch.Generator().manual_seed(14)
    u8 = torch.randint(0, 256, (2, 3, H, W), generator=g, dtype=torch.uint8)
    mean = (123.675, 116.28, 103.53)
    xf = (u8.float() - torch.tensor(mean).view(1, 3, 1, 1)).to(cuda)
    ho, wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    col = torch.empty(2 * ho * wo, 152, device=cuda, dtype=torch.bfloat16)
    ops.stem_im2col(xf, col, 2, H, W, 152)
    bgr = xf[:, [2, 1, 0]]
    unf = F.unfold(bgr, kernel_size=7, padding=3, stride=2)                         # [N, 3*49, L] ordered (c, r, s)
    ref = unf.view(2, 3, 49, ho * wo).permute(0, 3, 2, 1).reshape(2 * ho * wo, 147)  # -> (r, s, c)
    assert torch.equal(col[:, :147], ref.to(torch.bfloat16)) and float(col[:, 147:].float().abs().sum()) == 0.0
    # uint8 input with fused mean subtraction (ImageNorm) gives the same bits
    col2 = torch.empty_like(col)
    ops.stem_im2col(u8.to(cuda), col2, 2, H, W, 152, mean)
    assert torch.equal(col, col2)


@pytest.mark.parametrize("ld", [16, 64])
@pytest.mark.parametrize("hw", [(224, 224), (64, 96), (38, 54)])
def test_stem_space_to_depth_conv_matches_conv2d(cuda, hw, ld):
    """The patch-matrix-free stem: cb_stem_s2d -> 4-row-tap cb_gemm over overlapping rows -> strided max pool, against
    F.conv2d(7, s2, p3) on the bf16-rounded BGR frame + F.max_pool2d, and bit-exact frame layout (index op)."""
    ops = _ops()
    H, W = hw
    N = 2
    g = torch.Generator().manual_seed(24)
    u8 = torch.randint(0, 256, (N, 3, H, W), generator=g, dtype=torch.uint8)
    mean = (123.675, 116.28, 103.53)
    xf = u8.float() - torch.tensor(mean).view(1, 3, 1, 1)
    ho, wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    hs, ws = ho + 3, wo + 3
    rows = N * hs * ws
    s2d = torch.zeros((rows + 4) * ld, device=cuda, dtype=torch.bfloat16)
    ops.stem_s2d(u8.to(cuda), s2d, N, H, W, ld, mean)
    # ---- layout, bit-exact: S[n, Y, X, (dy*2+dx)*4 + c] = padded_bgr[n, c, 2Y+dy, 2X+dx]
    pad = torch.zeros(N, 3, 2 * hs, 2 * ws)
    pad[:, :, 3:3 + H, 3:3 + W] = xf[:, [2, 1, 0]]
    ref = torch.zeros(N, hs, ws, 2, 2, 4)
    ref[..., :3] = pad.view(N, 3, hs, 2, ws, 2).permute(0, 2, 4, 3, 5, 1)
    ref = ref.reshape(rows, 16).to(torch.bfloat16)
    if ld == 16:
        assert torch.equal(s2d[: rows * 16].view(rows, 16).cpu(), ref)
    else:
        win = s2d[: rows * 64].view(N, hs, ws, 4, 16).cpu()
        r4 = ref.view(N, hs, ws, 16)
        for j in range(4):          # slot j of row (Y, X) = pixel (Y, X + j) wherever that pixel exists
            assert torch.equal(win[:, :, : ws - j, j], r4[:, :, j:])
    # ---- conv + BN shift + ReLU + pool through the tensor cores
    wt = (torch.randn(64, 3, 7, 7, generator=g) * 0.02)                 # BGR-order weights, as the model's
    shift = torch.randn(64, generator=g).to(cuda)
    w147 = wt.permute(0, 2, 3, 1).reshape(64, 147).to(torch.bfloat16)
    w8 = torch.zeros(64, 8, 8, 4, dtype=torch.bfloat16)
    w8[:, :7, :7, :3] = w147.view(64, 7, 7, 3)
    wp = w8.view(64, 4, 2, 4, 2, 4).permute(0, 1, 3, 2, 4, 5).reshape(64, 256).contiguous().to(cuda)
    c1 = torch.empty(rows, 64, device=cuda, dtype=torch.bfloat16)
    ops.gemm(mode=ops.CB_GEMM_TN, m=rows, n=64, k=64, a=s2d, a_rows=rows, a_ld=ld, b=wp, b_rows=64, b_ld=256, ntaps=4, tap_w=ws,
             tap_sign=1, shift=shift, act=ops.ACT_RELU, out=c1, out_ld=64)
    xb = xf[:, [2, 1, 0]].to(torch.bfloat16).float()
    conv = F.relu(F.conv2d(xb, w147.float().view(64, 7, 7, 3).permute(0, 3, 1, 2), stride=2, padding=3) + shift.cpu().view(1, 64, 1, 1))
    got = c1.view(N, hs, ws, 64)[:, :ho, :wo].float().cpu().permute(0, 3, 1, 2)
    assert relerr(got, conv) < TOL_BF16_OP
    hh, ww = (ho - 1) // 2 + 1, (wo - 1) // 2 + 1
    y = torch.empty(N, hh, ww, 64, device=cuda, dtype=torch.bfloat16)
    ops.maxpool3x3s2(c1, y, N, ho, wo, 64, row_pitch=ws, img_pitch=hs * ws)
    assert torch.equal(y.float().cpu(), F.max_pool2d(got, 3, 2, 1).permute(0, 2, 3, 1))


def test_pool_and_subsample_ops(cuda):
    ops = _ops()
    g = torch.Generator().manual_seed(15)
    N, H, W, C = 2, 13, 12, 64
    x = _rnd(g, N, H, W, C)
    nchw = x.float().permute(0, 3, 1, 2)
    ho, wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    y = torch.empty(N, ho, wo, C, device=cuda, dtype=torch.bfloat16)
    ops.maxpool3x3s2(x, y, N, H, W, C)
    assert torch.equal(y.float(), F.max_pool2d(nchw, 3, 2, 1).permute(0, 2, 3, 1))
    ops.subsample2(x, y, N, H, W, C)
    assert torch.equal(y, x[:, ::2, ::2])
    dsub, act = _rnd(g, N, ho, wo, C), _rnd(g, N, H, W, C)
    dx = torch.empty_like(x)
    ops.unsubsample2_mask(dsub, act, dx, N, H, W, C)
    ref = torch.zeros_like(x)
    ref[:, ::2, ::2] = dsub
    assert torch.equal(dx, ref * (act > 0))
    ops.relu_mask(x, act, dx)
    assert torch.equal(dx, x * (act > 0))
    # grid_encoder tail, 7x7 -> 3x3 (floor), backward into the padded layout
    H = W = 7
    xg = _rnd(g, N, H, W, C)
    xr = xg.float().permute(0, 3, 1, 2).requires_grad_(True)
    ref = F.relu(F.max_pool2d(xr, 2, 2))
    yg = torch.empty(N, 3, 3, C, device=cuda, dtype=torch.bfloat16)
    ops.maxpool2x2_relu_fwd(xg, yg, N, H, W, C)
    assert torch.equal(yg.float(), ref.permute(0, 2, 3, 1))
    dy = _rnd(g, N, 3, 3, C)
    ref.backward(dy.float().permute(0, 3, 1, 2))
    dxp = torch.full((N, H + 2, W + 2, C), 9.0, device=cuda, dtype=torch.bfloat16)
    ops.maxpool2x2_relu_bwd(dy, xg, dxp, N, H, W, C)
    assert torch.equal(dxp[:, 1:-1, 1:-1].float(), xr.grad.permute(0, 2, 3, 1))
    assert float(dxp.float().abs().sum() - dxp[:, 1:-1, 1:-1].float().abs().sum()) == 0.0


def test_grouped_wgrad_launch(cuda):
    """cb_gemm_wgrad_group: several independent dW = dY^T X problems in ONE persistent launch (the four Linear layers of a
    BertLayer; the 1x1 / 3x3 / 1x1 (+ shortcut) convs of a bottleneck block with its 9-tap conv and FrozenBN row scales) against
    fp32 torch and against the single launches; accumulation semantics (a second launch adds); the fall-backs (one problem,
    very different reduction lengths) give the same numbers."""
    ops = _ops()
    g = torch.Generator().manual_seed(12)

    def lin(P, Mo, No, scale=False):
        dY, X = _rnd(g, P, Mo), _rnd(g, P, No)
        rs = (torch.rand(Mo, generator=g) + 0.5).to(cuda) if scale else None
        dW = torch.zeros(Mo, No, device=cuda)
        kw = dict(mode=ops.CB_GEMM_WGRAD, m=Mo, n=No, k=P, a=dY, a_rows=P, a_ld=Mo, b=X, b_rows=P, b_ld=No, out=dW, out_ld=No, out_fp32=1)
        if scale:
            kw["scale"] = rs
        ref = dY.float().t() @ X.float()
        return kw, dW, (ref * rs[:, None] if scale else ref)

    def conv3x3(NB, H, W, Cin, Cout):
        x, dy = _rnd(g, NB, H, W, Cin), _rnd(g, NB, H, W, Cout)
        xp = torch.zeros(NB, H + 2, W + 2, Cin, device=cuda, dtype=torch.bfloat16)
        dyp = torch.zeros(NB, H + 2, W + 2, Cout, device=cuda, dtype=torch.bfloat16)
        xp[:, 1:-1, 1:-1], dyp[:, 1:-1, 1:-1] = x, dy
        P = NB * (H + 2) * (W + 2)
        dW = torch.zeros(Cout, 9 * Cin, device=cuda)
        kw = dict(mode=ops.CB_GEMM_WGRAD, m=Cout, n=Cin, k=P, a=dyp, a_rows=P, a_ld=Cout, b=xp, b_rows=P, b_ld=Cin, ntaps=9, tap_w=W + 2, tap_sign=1,
                  out=dW, out_ld=9 * Cin, out_fp32=1)
        wz = torch.zeros(Cout, Cin, 3, 3, device=cuda, requires_grad=True)
        F.conv2d(x.float().permute(0, 3, 1, 2), wz, padding=1).backward(dy.float().permute(0, 3, 1, 2))
        return kw, dW, wz.grad.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin)

    groups = {
        "bert layer": [lin(2624, 768, 3072), lin(2624, 3072, 768), lin(2624, 2304, 768), lin(2624, 768, 768)],
        "bottleneck block": [lin(4 * 14 * 14, 1024, 256, True), conv3x3(4, 14, 14, 256, 256), lin(4 * 14 * 14, 256, 1024, True), lin(4 * 14 * 14, 1024, 512, True)],
        "narrow + ragged": [lin(1000, 136, 72), lin(1100, 64, 264)],
        "single problem": [lin(640, 128, 128)],
        "different reduction lengths": [lin(5000, 256, 256), lin(640, 128, 128)],
    }
    for name, probs in groups.items():
        kws = [p[0] for p in probs]
        ops.gemm_wgrad_group(kws)
        for kw, dW, ref in probs:
            assert relerr(dW, ref) < TOL_FP32_OP, (name, kw["m"], kw["n"], relerr(dW, ref))
        ops.gemm_wgrad_group(kws)                                           # += semantics
        for kw, dW, ref in probs:
            assert relerr(dW, 2 * ref) < TOL_FP32_OP, (name, "second launch")
        singles = []
        for kw, dW, ref in probs:
            d1 = torch.zeros_like(dW)
            ops.gemm(**dict(kw, out=d1))
            singles.append(d1)
        for (kw, dW, ref), d1 in zip(probs, singles):
            assert relerr(dW, 2 * d1) < TOL_FP32_OP, (name, "vs single launches")
