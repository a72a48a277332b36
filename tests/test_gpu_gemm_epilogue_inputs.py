"""GEMM epilogue inputs (residual / aux, loaded by TMA into shared memory ahead of the epilogue) on the shapes of the HBM-bound
1x1 convolutions: a one-chunk K loop and many tiles per persistent CTA, so that the input buffers and the operand ring wrap their
barrier phases many times; strided residual / aux views; ragged M and N % 16 == 8; the PAD row map; the full grid and a
grid of three CTAs; long K loops, whose inputs share the operand ring; bit-identical repeats; and the alignment check on the
residual / aux bases."""
import pytest
import torch

from util import TOL_BF16_OP, relerr

pytestmark = pytest.mark.gpu

SINGLE = 2      # cb_gemm_desc.reserved bit 1: launch exactly this descriptor (no tuning-table lookup)


def _ops():
    from clipbert_b200 import ops
    return ops


def _rnd(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to("cuda").to(torch.bfloat16)


def _strided(g, M, N, pad):
    """A [M, N] bf16 view with row pitch N + pad + 8 that starts 8 columns (16 bytes) into its buffer."""
    ld = N + pad + 8
    return _rnd(g, M, ld)[:, 8:8 + N], ld


@pytest.fixture(params=["all_sms", "three_ctas"])
def grid(request):
    """The persistent grid on every SM, and capped at three CTAs (ops.set_sm_limit): hundreds of tiles per CTA, so that the
    input buffers and the operand ring wrap their phases many more times."""
    ops = _ops()
    ops.set_sm_limit(3 if request.param == "three_ctas" else 0)
    yield request.param
    ops.set_sm_limit(0)


# (M, N, K): 1x1-conv shapes with one or two k-chunks and ~7-30 tiles per CTA; M % 128 != 0 with N % 16 == 8; a short launch
SHAPES = [(60000, 256, 64), (60000, 512, 128), (30001, 392, 64), (777, 136, 256)]


@pytest.mark.parametrize("block_n", [0, 64, 128])
@pytest.mark.parametrize("shape", SHAPES)
def test_tn_shift_residual_relu(cuda, grid, shape, block_n):
    """conv + FrozenBN shift + shortcut + ReLU (a bottleneck's conv3), twice: same bits."""
    ops = _ops()
    M, N, K = shape
    g = torch.Generator().manual_seed(11)
    A, B, R = _rnd(g, M, K), _rnd(g, N, K, scale=0.1), _rnd(g, M, N)
    shift = torch.randn(N, generator=g).to(cuda)
    outs = []
    for _ in range(2):
        C = torch.full((M, N), 3.0, device=cuda, dtype=torch.bfloat16)
        ops.gemm(mode=ops.CB_GEMM_TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=N, b_ld=K, shift=shift, residual=R, res_ld=N,
                 act=ops.ACT_RELU, out=C, out_ld=N, block_n=block_n, reserved=SINGLE)
        outs.append(C)
    ref = (A.float() @ B.float().t() + shift + R.float()).relu()
    assert relerr(outs[0], ref) < TOL_BF16_OP
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("strided", [False, True])
@pytest.mark.parametrize("block_n", [0, 64])
@pytest.mark.parametrize("shape", SHAPES)
def test_nn_residual_relu_mask(cuda, grid, shape, block_n, strided):
    """dgrad of conv1 + shortcut gradient, through the block input's ReLU (residual and aux), and aux alone; residual / aux as
    strided views (res_ld, aux_ld > N) when asked; twice: same bits."""
    ops = _ops()
    M, N, K = shape
    g = torch.Generator().manual_seed(12)
    A, B = _rnd(g, M, K), _rnd(g, K, N, scale=0.1)
    if strided:
        (R, res_ld), (X, aux_ld) = _strided(g, M, N, 24), _strided(g, M, N, 56)
    else:
        (R, res_ld), (X, aux_ld) = (_rnd(g, M, N), N), (_rnd(g, M, N), N)
    base = dict(mode=ops.CB_GEMM_NN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=K, b_ld=N, out_ld=N, block_n=block_n,
                reserved=SINGLE)
    acc = A.float() @ B.float()
    outs = []
    for _ in range(2):
        C = torch.full((M, N), 3.0, device=cuda, dtype=torch.bfloat16)
        ops.gemm(**base, residual=R, res_ld=res_ld, aux=X, aux_ld=aux_ld, aux_mode=ops.AUX_RELU_MASK, out=C)
        outs.append(C)
    assert relerr(outs[0], (acc + R.float()) * (X.float() > 0)) < TOL_BF16_OP
    assert torch.equal(outs[0], outs[1])
    C = torch.full((M, N), 3.0, device=cuda, dtype=torch.bfloat16)
    ops.gemm(**base, aux=X, aux_ld=aux_ld, aux_mode=ops.AUX_MUL, out=C)
    assert relerr(C, acc * X.float()) < TOL_BF16_OP


@pytest.mark.parametrize("block_n", [0, 64])
@pytest.mark.parametrize("dims", [(40, 28, 28, 64, 256), (3, 5, 6, 128, 392)])
def test_rowmap_pad_residual_aux(cuda, grid, dims, block_n):
    """PAD row map (compact rows in, zero-bordered rows out): residual and aux are read at the compact row; the border stays zero."""
    ops = _ops()
    NB, H, W, K, N = dims
    M = NB * H * W
    g = torch.Generator().manual_seed(13)
    A, B, R, X = _rnd(g, M, K), _rnd(g, N, K, scale=0.1), _rnd(g, M, N), _rnd(g, M, N)
    shift = torch.randn(N, generator=g).to(cuda)
    acc = A.float() @ B.float().t()
    base = dict(mode=ops.CB_GEMM_TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=N, b_ld=K, out_ld=N, rowmap=ops.ROWMAP_PAD,
                map_h=H, map_w=W, block_n=block_n, reserved=SINGLE)
    for kw, ref in [(dict(shift=shift, residual=R, res_ld=N, act=ops.ACT_RELU), (acc + shift + R.float()).relu()),
                    (dict(residual=R, res_ld=N, aux=X, aux_ld=N, aux_mode=ops.AUX_RELU_MASK), (acc + R.float()) * (X.float() > 0))]:
        yp = torch.zeros(NB, H + 2, W + 2, N, device=cuda, dtype=torch.bfloat16)
        ops.gemm(**base, **kw, out=yp)
        assert relerr(yp[:, 1:-1, 1:-1], ref.view(NB, H, W, N)) < TOL_BF16_OP
        border = yp.clone()
        border[:, 1:-1, 1:-1] = 0
        assert float(border.float().abs().max()) == 0.0


@pytest.mark.parametrize("block_n", [0, 64, 128])
@pytest.mark.parametrize("shape", [(20000, 256, 1024), (3001, 392, 576), (2624, 768, 3072)])
def test_long_k_inputs(cuda, grid, shape, block_n):
    """K loops longer than four chunks (BERT dense layers, 3x3 dgrad): the inputs of a tile land in the ring stage after its
    operands where one stage holds them, in a dedicated buffer otherwise; several
    tiles per CTA on the first shape; twice: same bits."""
    ops = _ops()
    M, N, K = shape
    g = torch.Generator().manual_seed(15)
    A, Bt, Bn = _rnd(g, M, K), _rnd(g, N, K, scale=0.05), _rnd(g, K, N, scale=0.05)
    (R, res_ld), (X, aux_ld) = _strided(g, M, N, 8), (_rnd(g, M, N), N)
    shift = torch.randn(N, generator=g).to(cuda)
    tn = dict(mode=ops.CB_GEMM_TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=Bt, b_rows=N, b_ld=K, out_ld=N, block_n=block_n, reserved=SINGLE)
    nn = dict(mode=ops.CB_GEMM_NN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=Bn, b_rows=K, b_ld=N, out_ld=N, block_n=block_n, reserved=SINGLE)
    cases = [(tn, dict(shift=shift, residual=R, res_ld=res_ld, act=ops.ACT_RELU), (A.float() @ Bt.float().t() + shift + R.float()).relu()),
             (nn, dict(residual=R, res_ld=res_ld), A.float() @ Bn.float() + R.float()),
             (nn, dict(residual=R, res_ld=res_ld, aux=X, aux_ld=aux_ld, aux_mode=ops.AUX_RELU_MASK),
              (A.float() @ Bn.float() + R.float()) * (X.float() > 0))]
    for base, kw, ref in cases:
        outs = []
        for _ in range(2):
            C = torch.full((M, N), 3.0, device=cuda, dtype=torch.bfloat16)
            ops.gemm(**base, **kw, out=C)
            outs.append(C)
        assert relerr(outs[0], ref) < TOL_BF16_OP
        assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("mode", ["tn", "nn"])
@pytest.mark.parametrize("which", ["residual", "aux"])
def test_unaligned_epilogue_input_is_rejected(cuda, which, mode):
    """A residual / aux base that is not 16-byte aligned is refused by cb_gemm's own check, before anything is launched."""
    ops = _ops()
    M, N, K = 256, 128, 64
    g = torch.Generator().manual_seed(14)
    A = _rnd(g, M, K)
    if mode == "tn":
        B = _rnd(g, N, K, scale=0.1)
        base = dict(mode=ops.CB_GEMM_TN, b=B, b_rows=N, b_ld=K)
    else:
        B = _rnd(g, K, N, scale=0.1)
        base = dict(mode=ops.CB_GEMM_NN, b=B, b_rows=K, b_ld=N)
    X = _rnd(g, M * N + 8).view(-1)[1:1 + M * N].view(M, N)     # 2 bytes past a 16-byte boundary
    assert X.data_ptr() % 16 != 0
    C = torch.full((M, N), 3.0, device=cuda, dtype=torch.bfloat16)
    kw = dict(residual=X, res_ld=N) if which == "residual" else dict(aux=X, aux_ld=N, aux_mode=ops.AUX_RELU_MASK)
    with pytest.raises(RuntimeError, match="cb_gemm\\(TN\\): %s must be 16-byte aligned" % which):
        ops.gemm(**base, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, out=C, out_ld=N, reserved=SINGLE, **kw)
    torch.cuda.synchronize()
    assert bool((C == 3.0).all())
