"""TN / NN GEMMs on the ping-pong kernel (two consumer warpgroups that own alternate tiles of a CTA): tile counts below the grid,
exactly one tile per CTA, odd and even tile counts per CTA, ragged M, N % 16 == 8, a 9-tap K loop longer than the operand ring,
residual / aux through two, one or no dedicated input buffers, the PAD and UNPAD row maps, the dropout + residual and GELU-stash
epilogues on a BERT shape, and both tile widths. Every case is checked against torch and repeated for identical bits."""
import pytest
import torch
import torch.nn.functional as F

from util import TOL_BF16_OP, relerr

pytestmark = pytest.mark.gpu

SINGLE = 2      # cb_gemm_desc.reserved bit 1: launch exactly this descriptor (no tuning-table lookup)
N_SM = 132


def _ops():
    from clipbert_b200 import ops
    return ops


def _rnd(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to("cuda").to(torch.bfloat16)


def _twice(run):
    """run(out) twice into fresh outputs prefilled with 3.0: the results must be bit-identical."""
    outs = [run() for _ in range(2)]
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)
    return outs[0]


# (M, N, K, block_n): 2 tiles (< grid); 132 tiles (one per CTA); 133 tiles (one CTA with two); 782 tiles (5 or 6 per CTA,
# ragged M); N % 16 == 8 with ragged M on 64-wide tiles
SHAPES = [(256, 128, 64, 128), (66 * 128, 256, 64, 128), (133 * 128, 128, 128, 128), (50000, 256, 64, 128), (30001, 392, 64, 64),
          (50000, 256, 64, 64)]


@pytest.mark.parametrize("shape", SHAPES)
def test_tn_shift_residual_relu_tile_counts(cuda, shape):
    ops = _ops()
    M, N, K, bn = shape
    g = torch.Generator().manual_seed(21)
    A, B, R = _rnd(g, M, K), _rnd(g, N, K, scale=0.1), _rnd(g, M, N)
    shift = torch.randn(N, generator=g).to(cuda)

    def run():
        C = torch.full((M, N), 3.0, device=cuda, dtype=torch.bfloat16)
        ops.gemm(mode=ops.CB_GEMM_TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=N, b_ld=K, shift=shift, residual=R, res_ld=N,
                 act=ops.ACT_RELU, out=C, out_ld=N, block_n=bn, reserved=SINGLE)
        return [C]

    (C,) = _twice(run)
    assert relerr(C, (A.float() @ B.float().t() + shift + R.float()).relu()) < TOL_BF16_OP


@pytest.mark.parametrize("shape", SHAPES)
def test_nn_plain_tile_counts(cuda, shape):
    """No epilogue inputs: only the operand ring and the turn barriers."""
    ops = _ops()
    M, N, K, bn = shape
    g = torch.Generator().manual_seed(22)
    A, B = _rnd(g, M, K), _rnd(g, K, N, scale=0.1)

    def run():
        C = torch.full((M, N), 3.0, device=cuda, dtype=torch.bfloat16)
        ops.gemm(mode=ops.CB_GEMM_NN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=K, b_ld=N, out=C, out_ld=N, block_n=bn,
                 reserved=SINGLE)
        return [C]

    (C,) = _twice(run)
    assert relerr(C, A.float() @ B.float()) < TOL_BF16_OP


# residual + aux through (M, N, K, block_n): two input buffers (one-chunk K loop), one buffer (K = 256 on 128-wide tiles: the ring
# beside two buffers would not hold the K loop), the ring stage after the operands (K loop longer than four chunks)
@pytest.mark.parametrize("shape", [(20000, 512, 64, 128), (20000, 512, 256, 128), (9000, 256, 576, 128), (9000, 392, 576, 64)])
def test_nn_residual_relu_mask_input_buffers(cuda, shape):
    ops = _ops()
    M, N, K, bn = shape
    g = torch.Generator().manual_seed(23)
    A, B, R, X = _rnd(g, M, K), _rnd(g, K, N, scale=0.05), _rnd(g, M, N), _rnd(g, M, N)

    def run():
        C = torch.full((M, N), 3.0, device=cuda, dtype=torch.bfloat16)
        ops.gemm(mode=ops.CB_GEMM_NN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=K, b_ld=N, residual=R, res_ld=N, aux=X, aux_ld=N,
                 aux_mode=ops.AUX_RELU_MASK, out=C, out_ld=N, block_n=bn, reserved=SINGLE)
        return [C]

    (C,) = _twice(run)
    assert relerr(C, (A.float() @ B.float() + R.float()) * (X.float() > 0)) < TOL_BF16_OP


@pytest.mark.parametrize("block_n", [64, 128])
def test_conv3x3_nine_taps_unpad_and_pad_residual(cuda, block_n):
    """3x3 conv: a 9-tap K loop (18 chunks at Cin = 128, longer than the ring) written through the UNPAD row map; then a 1x1 conv
    whose output goes through the PAD row map with a residual."""
    ops = _ops()
    NB, H, W, Cin, Cout = 6, 14, 14, 128, 136
    g = torch.Generator().manual_seed(24)
    x = _rnd(g, NB, H, W, Cin)
    w = _rnd(g, Cout, Cin, 3, 3, scale=0.05)
    xp = torch.zeros(NB, H + 2, W + 2, Cin, device=cuda, dtype=torch.bfloat16)
    xp[:, 1:-1, 1:-1] = x
    P = NB * (H + 2) * (W + 2)
    wk = w.permute(0, 2, 3, 1).contiguous().view(Cout, 9 * Cin)

    def run3():
        y = torch.full((NB * H * W, Cout), 3.0, device=cuda, dtype=torch.bfloat16)
        ops.gemm(mode=ops.CB_GEMM_TN, m=P, n=Cout, k=Cin, a=xp, a_rows=P, a_ld=Cin, b=wk, b_rows=Cout, b_ld=9 * Cin, ntaps=9, tap_w=W + 2,
                 tap_sign=1, out=y, out_ld=Cout, rowmap=ops.ROWMAP_UNPAD, map_h=H, map_w=W, block_n=block_n, reserved=SINGLE)
        return [y]

    (y,) = _twice(run3)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    assert relerr(y, ref) < TOL_BF16_OP

    M = NB * H * W
    A, B, R = x.view(M, Cin), _rnd(g, Cout, Cin, scale=0.1), _rnd(g, M, Cout)

    def run1():
        yp = torch.zeros(NB, H + 2, W + 2, Cout, device=cuda, dtype=torch.bfloat16)
        ops.gemm(mode=ops.CB_GEMM_TN, m=M, n=Cout, k=Cin, a=A, a_rows=M, a_ld=Cin, b=B, b_rows=Cout, b_ld=Cin, residual=R, res_ld=Cout,
                 act=ops.ACT_RELU, out=yp, out_ld=Cout, rowmap=ops.ROWMAP_PAD, map_h=H, map_w=W, block_n=block_n, reserved=SINGLE)
        return [yp]

    (yp,) = _twice(run1)
    ref = (A.float() @ B.float().t() + R.float()).relu().view(NB, H, W, Cout)
    assert relerr(yp[:, 1:-1, 1:-1], ref) < TOL_BF16_OP
    border = yp.clone()
    border[:, 1:-1, 1:-1] = 0
    assert float(border.float().abs().max()) == 0.0


@pytest.mark.parametrize("block_n", [64, 128])
def test_bert_dropout_residual_and_gelu_stash(cuda, block_n):
    """BERT dense layers at M = 2624 (126 tiles of 128 x 128 on 132 SMs: CTAs with one tile and CTAs with none for consumer 1):
    dropout + residual (each output is either the residual alone or (acc + bias) / keep + residual), and GELU with its derivative
    stashed in out2."""
    ops = _ops()
    M, N, K, p = 2624, 768, 3072, 0.1
    g = torch.Generator().manual_seed(25)
    A, B, R = _rnd(g, M, K), _rnd(g, N, K, scale=0.02), _rnd(g, M, N)
    bias = torch.randn(N, generator=g).to(cuda)

    def run_drop():
        C = torch.full((M, N), 3.0, device=cuda, dtype=torch.bfloat16)
        ops.gemm(mode=ops.CB_GEMM_TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=N, b_ld=K, shift=bias, residual=R, res_ld=N,
                 dropout_p=p, dropout_seed=1234, out=C, out_ld=N, block_n=block_n, reserved=SINGLE)
        return [C]

    (C,) = _twice(run_drop)
    kept = (A.float() @ B.float().t() + bias) / (1.0 - p) + R.float()
    dropped = R.float()
    is_kept = (C.float() - kept).abs() <= (C.float() - dropped).abs()
    sel = torch.where(is_kept, kept, dropped)
    assert relerr(C, sel) < TOL_BF16_OP
    assert abs(1.0 - float(is_kept.float().mean()) - p) < 0.01

    K2, N2 = 768, 3072
    A2, B2 = _rnd(g, M, K2), _rnd(g, N2, K2, scale=0.05)
    b2 = torch.randn(N2, generator=g).to(cuda)

    def run_gelu():
        C = torch.full((M, N2), 3.0, device=cuda, dtype=torch.bfloat16)
        G = torch.full((M, N2), 3.0, device=cuda, dtype=torch.bfloat16)
        ops.gemm(mode=ops.CB_GEMM_TN, m=M, n=N2, k=K2, a=A2, a_rows=M, a_ld=K2, b=B2, b_rows=N2, b_ld=K2, shift=b2,
                 act=ops.ACT_GELU_STASH_GRAD, out=C, out_ld=N2, out2=G, out2_ld=N2, block_n=block_n, reserved=SINGLE)
        return [C, G]

    C, G = _twice(run_gelu)
    u = (A2.float() @ B2.float().t() + b2).requires_grad_(True)
    y = F.gelu(u)
    (dydu,) = torch.autograd.grad(y.sum(), u)
    assert relerr(C, y.detach()) < TOL_BF16_OP
    assert relerr(G, dydu) < TOL_BF16_OP


def test_explicit_block_n_256_runs_on_128_wide_tiles(cuda):
    """block_n = 256 for TN / NN (128 x 256 would not fit a consumer's registers) still computes the product."""
    ops = _ops()
    M, N, K = 3000, 512, 128
    g = torch.Generator().manual_seed(26)
    A, B, R = _rnd(g, M, K), _rnd(g, N, K, scale=0.1), _rnd(g, M, N)
    C = torch.full((M, N), 3.0, device=cuda, dtype=torch.bfloat16)
    ops.gemm(mode=ops.CB_GEMM_TN, m=M, n=N, k=K, a=A, a_rows=M, a_ld=K, b=B, b_rows=N, b_ld=K, residual=R, res_ld=N, out=C, out_ld=N,
             block_n=256, reserved=SINGLE)
    assert relerr(C, A.float() @ B.float().t() + R.float()) < TOL_BF16_OP
