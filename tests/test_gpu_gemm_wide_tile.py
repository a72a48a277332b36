"""cb_gemm TN / NN on 128 x 256 tiles (gemm_coop_kernel: both consumer warpgroups on one tile, epilogue inputs streamed through
the operand ring), forced through cb_gemm_desc.reserved CB_GEMM_FORCE_WIDE, element by element against the float64 reference,
cases and bounds of tests/test_gpu_gemm_elementwise.py. Each case runs twice on the wide tile and once forced onto 128 x 128
tiles (CB_GEMM_NO_WIDE, block_n = 128): every accumulator sees its k steps in the same order on both kernels and the epilogue
is the same code, so all three must give the same bits.

The CPU tests check the tile the library picks (cb_gemm_tile_width, no launch): the reserved bits, the unchanged meaning of an
explicit block_n, and the model's picks for the convolution and BERT shapes of the training step on 132 SMs."""
import pytest
import torch

import test_gpu_gemm_elementwise as EW
from test_gpu_gemm_elementwise import NN, PAD, TN, UNPAD, _c

WIDE = 1 << 12      # CB_GEMM_FORCE_WIDE
NO_WIDE = 1 << 13   # CB_GEMM_NO_WIDE

CASES = [
    # ragged M and N, K tails, one tile per CTA and one CTA
    _c(TN, 1, 256, 64, shift=True, act="relu", sm=1),
    _c(TN, 127, 256, 200, shift=True, res=True, act="relu", pitch=16),
    _c(TN, 129, 392, 72, res=True),
    _c(TN, 333, 200, 200, scale=True, shift=True, fp32=True, act="tanh"),
    # NN: residual, aux, both; the 3-D box on and off, and N where it falls back to 2-D boxes
    _c(NN, 300, 256, 192, aux="mask"),
    _c(NN, 300, 256, 192, res=True, aux="mask"),
    _c(NN, 1000, 512, 256, res=True, aux="mask", sm=2, mn3d=0),
    _c(NN, 1000, 512, 256, aux="mask", sm=3),
    _c(NN, 333, 136, 72, aux="mask"),
    _c(NN, 1000, 392, 64, res=True, aux="mask", sm=3),
    # epilogue kinds
    _c(TN, 500, 768, 64, shift=True, res=True, p=0.1, sm=2),
    _c(TN, 500, 256, 128, shift=True, act="stash", out2=True, sm=2),
    _c(NN, 500, 256, 128, aux="mul"),
    _c(NN, 500, 256, 128, res=True, aux="mul", pitch=8),
    _c(TN, 300, 256, 192, scale=True, shift=True, res=True, out2=True, act="relu"),
    _c(TN, 300, 256, 192, shift=True, act="gelu"),
    _c(NN, 300, 256, 192, res=True, aux="gelu"),
    _c(NN, 300, 256, 192, res=True, aux="tanh"),
    _c(TN, 300, 256, 192, shift=True, p=0.1, res=True, out2=True, act="relu"),
    # many tiles per CTA (10 tiles on 1 / 2 / 3 CTAs: ring phases wrap many times), long K loops with inputs
    _c(TN, 1280, 256, 64, shift=True, res=True, act="relu", sm=1),
    _c(TN, 1280, 256, 64, shift=True, res=True, act="relu", sm=2),
    _c(TN, 1280, 256, 64, res=True, aux="mask", sm=3),
    _c(TN, 700, 512, 512, res=True),
    _c(NN, 700, 256, 3072, res=True, aux="mask", sm=3),
    _c(TN, 700, 512, 512, kch=2),
    # taps: 3x3 forward (+1) and dgrad (-1), K tails, row taps
    _c(TN, 0, 256, 72, ntaps=9, sign=1, img=(2, 7, 7), rowmap=UNPAD, res=True, sm=2),
    _c(TN, 0, 200, 200, ntaps=9, sign=-1, img=(1, 6, 9)),
    _c(NN, 0, 256, 72, ntaps=9, sign=-1, img=(2, 7, 7), rowmap=UNPAD, aux="mask", res=True),
    _c(NN, 0, 256, 64, ntaps=9, sign=-1, img=(2, 7, 7), rowmap=UNPAD, aux="mask", sm=2),
    _c(NN, 0, 256, 200, ntaps=9, sign=1, img=(1, 5, 6), p=0.1, shift=True, res=True, rowmap=UNPAD),
    _c(NN, 0, 256, 64, ntaps=9, sign=-1, img=(2, 5, 6), mn3d=0),
    _c(TN, 600, 256, 64, ntaps=4, sign=1, tap_w=9, shift=True, act="relu"),
    _c(TN, 600, 256, 64, ntaps=4, sign=-1, tap_w=13, res=True, sm=2),
    # row maps; dropout keyed by the mapped row, with a bound offset word
    _c(TN, 0, 256, 64, img=(3, 5, 6), rowmap=PAD, shift=True, res=True, act="relu", sm=2),
    _c(TN, 0, 256, 128, img=(2, 6, 7), rowmap=PAD, shift=True, p=0.1, word=True, res=True),
    _c(TN, 0, 256, 64, img=(2, 6, 7), rowmap=UNPAD, p=0.1, word=True, res=True),
    _c(NN, 0, 256, 128, img=(3, 5, 6), rowmap=UNPAD, res=True, aux="mask"),
    # NaN / inf
    _c(TN, 300, 256, 64, shift=True, act="relu", nan="nan_a_row"),
    _c(NN, 300, 256, 64, res=True, aux="mask", nan="inf"),
]


class _Forced(EW.Backend):
    """The device, with reserved bits (and a block_n) forced on every launch; records the tile width each launch ran with."""

    def __init__(self, bits, block_n=None):
        super().__init__("device")
        self.bits, self.block_n, self.widths = bits, block_n, set()

    def gemm(self, **kw):
        from clipbert_b200 import ops
        kw["reserved"] |= self.bits
        if self.block_n is not None:
            kw["block_n"] = self.block_n
        self.widths.add(ops.gemm_tile_width(kw))
        ops.gemm(**kw)


def _id(c):
    return c.id.replace("-bn64", "")


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_wide_tile_elementwise(case):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    c = case
    seed = 17 + c.M + 3 * c.N + c.K
    word = 0x5EED + c.M if c.word else None
    ins = EW._inputs(c, seed)
    wide, narrow = _Forced(WIDE), _Forced(NO_WIDE, 128)
    with EW._knobs(wide, c.sm, c.mn3d, word):
        out, out2 = EW._run(wide, c, ins, seed)
        out_b, out2_b = EW._run(wide, c, ins, seed)
        out_n, out2_n = EW._run(narrow, c, ins, seed)
    assert wide.widths == {256} and narrow.widths == {128}, (wide.widths, narrow.widths)
    for o, o_b, o_n, name in ((out, out_b, out_n, "out"), (out2, out2_b, out2_n, "out2")):
        if o is None:
            continue
        o.check("%s %s" % (c.id, name))
        EW._check_padded_border(c, o, name)
        assert torch.equal(EW._bits(o.t), EW._bits(o_b.t)), "%s: %s differs between two identical runs" % (c.id, name)
        assert torch.equal(EW._bits(o.t), EW._bits(o_n.t)), "%s: %s differs between 128 x 256 and 128 x 128 tiles" % (c.id, name)
    ins_d = {k: v.to(wide.dev) for k, v in ins.items()}
    for name, r in EW._compare(c, out, out2, EW.reference(c, ins_d, EW._mult(c, seed, word))).items():
        EW._record("wide", "%s-%s" % (_id(c), name), r)


# ------------------------------------------------------------------------------------------------ the tile the library picks
def _width(**kw):
    from clipbert_b200 import ops
    base = dict(mode=TN, a_rows=kw["m"], a_ld=kw["k"], b_rows=kw["n"], b_ld=kw["k"], out_ld=kw["n"], ntaps=1, tap_w=0)
    base.update(kw)
    return ops.gemm_tile_width(base)


def _sm132():
    """The picks below are for 132 SMs: the library's count without a device, or an H100 SXM's."""
    if torch.cuda.is_available() and torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("picks restated for 132 SMs")


def test_reserved_bits_and_explicit_block_n():
    _sm132()
    big = dict(m=32768, n=256, k=256, ntaps=9, tap_w=34)
    for mode in (TN, NN):
        assert _width(mode=mode, **big, reserved=WIDE) == 256
        assert _width(mode=mode, **big, reserved=WIDE, block_n=64) == 256
        assert _width(mode=mode, **big, reserved=NO_WIDE) in (64, 128)
        assert _width(mode=mode, **big, block_n=256) == 128          # an explicit 256 keeps meaning 128 x 128 on TN / NN
        assert _width(mode=mode, **big, block_n=128) == 128
        assert _width(mode=mode, **big, block_n=64) == 64
        assert _width(mode=mode, m=2624, n=64, k=768, reserved=WIDE) == 256
        assert _width(mode=mode, m=2624, n=128, k=768) != 256       # mostly padding
    # weight gradients ignore the bits
    wg = dict(mode=1, m=256, n=256, k=20000, a_rows=20000, a_ld=256, b_rows=20000, b_ld=256)
    assert _width(**wg, reserved=WIDE) == _width(**wg) == _width(**wg, reserved=NO_WIDE)


# (mode, m, n, k, ntaps, tap_w, expected pick), shapes of the training step: the grid-encoder and res4 3x3 convolutions, whose
# 128 x 256 wave count is about half the 128 x 128 one over a long K loop, take the wide tile; the BERT GEMMs (2624 tokens), the
# gelu'-stashing intermediate dense, the 16-chunk 1x1 convolutions and the HBM-bound ones do not
PICKS = [
    (TN, 10368, 768, 2048, 9, 26, 256),
    (NN, 10368, 2048, 768, 9, 26, 256),
    (TN, 32768, 256, 256, 9, 34, 256),
    (NN, 32768, 256, 256, 9, 34, 256),
    (TN, 6272, 512, 2048, 1, 0, 256),
    (TN, 2624, 768, 768, 1, 0, 128),
    (NN, 2624, 768, 3072, 1, 0, 128),
    (TN, 6272, 2048, 1024, 1, 0, 128),
    (NN, 25088, 512, 1024, 1, 0, 128),
    (TN, 401408, 256, 64, 1, 0, 128),
]


@pytest.mark.parametrize("mode,m,n,k,ntaps,tap_w,want", PICKS)
def test_model_picks(mode, m, n, k, ntaps, tap_w, want):
    _sm132()
    a_rows = m
    got = _width(mode=mode, m=m, n=n, k=k, ntaps=ntaps, tap_w=tap_w, a_rows=a_rows, a_ld=k,
                 b_rows=n if mode == TN else k, b_ld=k * ntaps if mode == TN else n * ntaps)
    assert (got == 256) == (want == 256), (got, want)


def test_gelu_stash_stays_off_the_wide_tile():
    _sm132()
    kw = dict(m=2624, n=3072, k=768)
    assert _width(**kw, out2=1) != 256      # (the out2 pointer only has to be non-null for the pick)
