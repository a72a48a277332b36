"""K loops longer than the operand ring keep at least three ring stages. On TN / NN 64-wide tiles and on weight gradients, the
automatic ring must give the same bits as the shallower ring used before (k-chunks per stage forced through cb_gemm_desc.reserved
bits 8-11). The ring shape only changes how chunks are grouped into barrier round trips, never the k order of an accumulator."""
import pytest
import torch
import torch.nn.functional as F

from util import TOL_BF16_OP, relerr

pytestmark = pytest.mark.gpu

SINGLE = 2      # cb_gemm_desc.reserved bit 1: launch exactly this descriptor (no tuning-table lookup)


def _rnd(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to("cuda").to(torch.bfloat16)


@pytest.mark.parametrize("mode", ["tn", "nn"])
def test_conv3x3_64_wide_ring_shape_does_not_change_bits(cuda, mode):
    """res2-like 3x3 conv at Cin = Cout = 64: nine one-chunk taps, more than the eight chunks a 64-wide ring holds."""
    from clipbert_b200 import ops
    NB, H, W, C = 8, 28, 28, 64
    g = torch.Generator().manual_seed(31)
    x = _rnd(g, NB, H, W, C)
    w = _rnd(g, C, C, 3, 3, scale=0.05)
    xp = torch.zeros(NB, H + 2, W + 2, C, device=cuda, dtype=torch.bfloat16)
    xp[:, 1:-1, 1:-1] = x
    P = NB * (H + 2) * (W + 2)
    b = w.permute(0, 2, 3, 1).contiguous().view(C, 9 * C)      # KRSC, the forward layout; NN reads it as the dgrad's B
    if mode == "tn":
        kw = dict(mode=ops.CB_GEMM_TN, tap_sign=1)
    else:
        kw = dict(mode=ops.CB_GEMM_NN, tap_sign=-1)
    outs = []
    for reserved in (SINGLE, SINGLE | (4 << 8)):
        y = torch.full((NB * H * W, C), 3.0, device=cuda, dtype=torch.bfloat16)
        ops.gemm(m=P, n=C, k=C, a=xp, a_rows=P, a_ld=C, b=b, b_rows=C, b_ld=9 * C, ntaps=9, tap_w=W + 2, out=y, out_ld=C,
                 rowmap=ops.ROWMAP_UNPAD, map_h=H, map_w=W, block_n=64, reserved=reserved, **kw)
        outs.append(y)
    assert torch.equal(outs[0], outs[1])
    conv = F.conv2d if mode == "tn" else F.conv_transpose2d
    ref = conv(x.float().permute(0, 3, 1, 2), w.float(), padding=1).permute(0, 2, 3, 1).reshape(-1, C)
    assert relerr(outs[0], ref) < TOL_BF16_OP


@pytest.mark.parametrize("block_n", [64, 256])
def test_wgrad_long_k_loop_ring_shape_does_not_change_bits(cuda, block_n):
    """Weight gradient over 20000 pixels (313 k-chunks, one split): 128 x 256 tiles now get four one-chunk stages instead of two
    of two, 128 x 64 tiles four stages of two instead of two of four. Each output is written by one tile, so the bits must match
    the old ring's."""
    from clipbert_b200 import ops
    P, M, N = 20000, 256, 512
    g = torch.Generator().manual_seed(32)
    dy, x = _rnd(g, P, M), _rnd(g, P, N)
    outs = []
    for kch in (0, 4 if block_n == 64 else 2):
        dW = torch.zeros(M, N, device=cuda)
        ops.gemm(mode=ops.CB_GEMM_WGRAD, m=M, n=N, k=P, a=dy, a_rows=P, a_ld=M, b=x, b_rows=P, b_ld=N, split_k=1, out=dW, out_ld=N,
                 out_fp32=1, block_n=block_n, reserved=SINGLE | (kch << 8))
        outs.append(dW)
    assert torch.equal(outs[0], outs[1])
    assert relerr(outs[0], dy.float().t() @ x.float()) < TOL_BF16_OP
