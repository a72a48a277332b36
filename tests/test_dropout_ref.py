"""tests/dropout_ref.py (the NumPy restatement of the library's dropout mask) against a scalar one in Python integers.

The GPU tests trust dropout_ref to say which elements each kernel must keep; this pins the vectorised uint64 arithmetic
(wrap-around products, logical shifts, lane extraction) and the threshold / multiplier rules on the CPU.
"""
import numpy as np
import pytest

import dropout_ref as D

M64 = (1 << 64) - 1


def _py_keep_mult(seed, word, e, p):
    s = seed if word is None else (seed + word * 0xD1342543DE82EF95) & M64
    z = ((e >> 2) * 0x9E3779B97F4A7C15 + s) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    z ^= z >> 31
    lane = (z >> (16 * (e & 3))) & 0xFFFF
    p32 = float(np.float32(p))
    if p32 >= 1.0:
        th, mult = 65536, 0.0
    else:
        t = p32 * 65536.0 + 0.5
        th = max(1, 65535 if t >= 65535.0 else int(t))
        mult = float(np.float32(1.0) / (np.float32(1.0) - np.float32(p32)))
    return mult if lane >= th else 0.0


@pytest.mark.parametrize("p", [1e-6, 0.1, 0.5, 65535.6 / 65536, 1.0])
@pytest.mark.parametrize("seed,word", [(0, None), (12345, None), (2 ** 64 - 3, None), (99, 2 ** 63 - 1), (7, 2 ** 63),
                                       (2 ** 63 + 11, 2 ** 63 + 5), (1000003, 1)])
def test_multipliers_match_integer_restatement(p, seed, word):
    rng = np.random.default_rng(seed & 0xFFFF)
    idx = np.concatenate([np.arange(2000, dtype=np.uint64), rng.integers(0, 2 ** 40, 1000).astype(np.uint64),
                          np.array([2 ** 63 - 1, 2 ** 63, 2 ** 64 - 4, 2 ** 64 - 1], dtype=np.uint64)])
    got = D.multipliers(D.effective_seed(seed, word), idx, p)
    want = np.array([_py_keep_mult(seed, word, int(e), p) for e in idx], dtype=np.float32)
    assert got.dtype == np.float32 and np.array_equal(got, want)


def test_threshold_and_multiplier_rules():
    assert D.thresh(0.0) == 0 and D.inv_keep(0.0) == 1.0
    assert D.thresh(1e-9) == 1                          # any p > 0 drops something
    assert D.thresh(0.1) == 6554 and D.thresh(0.5) == 32768
    assert D.thresh(65535.6 / 65536) == 65535           # the largest threshold below p = 1
    assert D.thresh(1.0) == 65536 and D.thresh(3.0) == 65536
    assert D.inv_keep(1.0) == 0.0 and D.inv_keep(0.5) == np.float32(2.0)
    assert D.inv_keep(0.1) == np.float32(1.0) / np.float32(0.9)
    assert not D.multipliers(5, D.flat_index(1 << 18), 1.0).any()     # p = 1 drops everything
    keep = D.multipliers(5, D.flat_index(1 << 18), 0.1) != 0
    assert abs(float(keep.mean()) - 0.9) < 0.005


def test_index_layouts():
    assert np.array_equal(D.gemm_index(3, 5)[2], 10 + np.arange(5))
    assert np.array_equal(D.gemm_index(np.array([7]), 392)[0, :3], 7 * 392 + np.arange(3))
    assert np.array_equal(D.layernorm_index(2)[1, :2], [768, 769])
    e = D.embedding_index(2, 41, np.arange(32, 41))            # visual rows of a 32-token caption + 3x3 grid
    assert e.shape == (2, 9, 768) and int(e[1, 0, 0]) == (41 + 32) * 768
    a = D.attention_index(2, 12, 9)
    assert a.shape == (2, 12, 9, 9) and int(a[1, 3, 4, 5]) == ((1 * 12 + 3) * 9 + 4) * 9 + 5
    assert D.effective_seed(1, 2 ** 64 - 1) == (1 - 0xD1342543DE82EF95) % 2 ** 64
