"""Weight-gradient main loop with one wgmma group in flight: every tile width, K-splits with a ragged last split and a ragged
last k-chunk, and many tiles per persistent CTA, so that the operand ring wraps across tiles while a stage's products are still
being waited for. Grouped launches at every tile width and with a forced K-split, and in deterministic mode the bits of a single
launch against the same problem inside a group."""
import pytest
import torch

from util import TOL_FP32_OP, relerr

pytestmark = pytest.mark.gpu

SINGLE = 2      # cb_gemm_desc.reserved bit 1: launch exactly this descriptor (no tuning-table lookup)


def _rnd(g, *shape):
    return torch.randn(*shape, generator=g).to("cuda").to(torch.bfloat16)


# P = 2373: 38 k-chunks, the last one 5 rows deep; five splits of 8 chunks leave a last split of 6
P, M, N = 2373, 2048, 1024


@pytest.fixture(scope="module")
def operands():
    g = torch.Generator().manual_seed(41)
    dy, x = _rnd(g, P, M), _rnd(g, P, N)
    return dy, x, dy.float().t() @ x.float()


@pytest.mark.parametrize("split", [1, 5])
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_wgrad_tile_widths_and_splits(cuda, operands, bn, split):
    from clipbert_b200 import ops
    dy, x, ref = operands
    dW = torch.zeros(M, N, device=cuda)
    ops.gemm(mode=ops.CB_GEMM_WGRAD, m=M, n=N, k=P, a=dy, a_rows=P, a_ld=M, b=x, b_rows=P, b_ld=N, split_k=split, out=dW, out_ld=N,
             out_fp32=1, block_n=bn, reserved=SINGLE)
    assert relerr(dW, ref) < TOL_FP32_OP


@pytest.mark.parametrize("bn", [64, 128, 256])
def test_wgrad_ring_shape_does_not_change_bits(cuda, operands, bn):
    """One split: every output is written by one tile in the same k order, whatever the k-chunks per ring stage."""
    from clipbert_b200 import ops
    dy, x, _ = operands
    outs = []
    for kch in (0, 1, 2):
        dW = torch.zeros(M, N, device=cuda)
        ops.gemm(mode=ops.CB_GEMM_WGRAD, m=M, n=N, k=P, a=dy, a_rows=P, a_ld=M, b=x, b_rows=P, b_ld=N, split_k=1, out=dW, out_ld=N,
                 out_fp32=1, block_n=bn, reserved=SINGLE | (kch << 8))
        outs.append(dW)
    for o in outs[1:]:
        assert torch.equal(outs[0], o)


@pytest.mark.parametrize("split", [1, 3])
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_grouped_wgrad_tile_widths_and_splits(cuda, bn, split):
    """block_n / split_k of the first descriptor fix the whole group's tile width and K-split."""
    from clipbert_b200 import ops
    g = torch.Generator().manual_seed(42)
    probs = []
    for mo, no, p in ((768, 1024, 2373), (1024, 768, 2373), (512, 256, 2400)):
        dy, x = _rnd(g, p, mo), _rnd(g, p, no)
        dW = torch.zeros(mo, no, device=cuda)
        probs.append((dict(mode=ops.CB_GEMM_WGRAD, m=mo, n=no, k=p, a=dy, a_rows=p, a_ld=mo, b=x, b_rows=p, b_ld=no, out=dW, out_ld=no,
                           out_fp32=1), dW, dy.float().t() @ x.float()))
    kws = [p[0] for p in probs]
    kws[0] = dict(kws[0], block_n=bn, split_k=split)
    ops.gemm_wgrad_group(kws)
    for kw, dW, ref in probs:
        assert relerr(dW, ref) < TOL_FP32_OP, (bn, split, kw["m"], kw["n"])


@pytest.mark.parametrize("split", [1, 3])
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_single_wgrad_gives_the_bits_of_its_group(cuda, bn, split):
    """Deterministic mode: a weight gradient launched alone and the same problem inside a group of three, at the same tile width
    and K-split, run the same tiles in the same k order and add their split planes in the same order."""
    from clipbert_b200 import ops
    g = torch.Generator().manual_seed(43)
    probs = []
    for mo, no, p in ((1024, 768, 2373), (768, 1024, 2373), (512, 256, 2400)):
        dy, x = _rnd(g, p, mo), _rnd(g, p, no)
        out0 = torch.randn(mo, no, generator=g).to(cuda)          # += semantics: the planes are added onto non-zero outputs
        probs.append((dict(mode=ops.CB_GEMM_WGRAD, m=mo, n=no, k=p, a=dy, a_rows=p, a_ld=mo, b=x, b_rows=p, b_ld=no, out_ld=no,
                           out_fp32=1), out0))
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        kw, out0 = probs[1]
        alone = out0.clone()
        ops.gemm(**kw, out=alone, block_n=bn, split_k=split, reserved=SINGLE)
        grouped = [o.clone() for _, o in probs]
        kws = [dict(k, out=o) for (k, _), o in zip(probs, grouped)]
        kws[0] = dict(kws[0], block_n=bn, split_k=split)
        ops.gemm_wgrad_group(kws)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert not torch.equal(alone, out0)
    assert torch.equal(alone, grouped[1])
