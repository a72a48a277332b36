"""The library's dropout mask, restated in NumPy - TEST INFRASTRUCTURE ONLY.

Every mask consumer of the library (GEMM epilogue, LayerNorm backward, embeddings, attention probabilities, cb_dropout) keeps
or drops element e by one rule (csrc/common.cuh, csrc/drop_cfg.h, include/clipbert_b200.h):

    seed' = seed + word * 0xD1342543DE82EF95          (mod 2^64; word = the device word bound by cb_dropout_offset_bind)
    h     = splitmix64 finaliser of (e >> 2) * 0x9E3779B97F4A7C15 + seed'
    keep  = 16-bit lane (e & 3) of h  >=  thresh(p)
    y     = x * inv_keep(p) if keep else 0

What differs between consumers is only the element index e, so each family has its helper below. The tests compare each
kernel with a plain fp32 computation that multiplies by these masks.
"""
import numpy as np

HIDDEN = 768
WORD_MUL = 0xD1342543DE82EF95
_GOLDEN = np.uint64(0x9E3779B97F4A7C15)
_MIX1 = np.uint64(0xBF58476D1CE4E5B9)
_MIX2 = np.uint64(0x94D049BB133111EB)
_MASK64 = (1 << 64) - 1


def thresh(p):
    """make_drop: round(p * 65536) for a float32 p, at least 1 when p > 0, 65535 at most below p = 1; 65536 (drop everything)
    for p >= 1; 0 (no dropout) for p <= 0."""
    p = float(np.float32(p))
    if p >= 1.0:
        return 65536
    if not p > 0.0:
        return 0
    t = p * 65536.0 + 0.5
    return max(1, 65535 if t >= 65535.0 else int(t))


def inv_keep(p):
    """The multiplier of a kept element, 1 / (1 - p) in float32; 0 for p >= 1 (nothing is kept), 1 for p <= 0."""
    p = np.float32(p)
    if p >= 1:
        return np.float32(0.0)
    if not p > 0:
        return np.float32(1.0)
    return np.float32(1.0) / (np.float32(1.0) - p)


def effective_seed(seed, word=None):
    """The seed a kernel uses when `word` is bound (None: nothing bound, the seed as passed)."""
    seed = int(seed) & _MASK64
    return seed if word is None else (seed + (int(word) & _MASK64) * WORD_MUL) & _MASK64


def _hash(seed, group):
    with np.errstate(over="ignore"):
        z = group * _GOLDEN + np.uint64(seed)
        z = (z ^ (z >> np.uint64(30))) * _MIX1
        z = (z ^ (z >> np.uint64(27))) * _MIX2
        return z ^ (z >> np.uint64(31))


def multipliers(seed, idx, p):
    """float32 array shaped like idx: 0 where element idx is dropped, inv_keep(p) where it is kept. `seed` is the effective seed."""
    e = np.asarray(idx).astype(np.uint64)
    h = _hash(int(seed) & _MASK64, e >> np.uint64(2))
    lane = (h >> (np.uint64(16) * (e & np.uint64(3)))) & np.uint64(0xFFFF)
    keep = lane >= np.uint64(thresh(p))
    return np.where(keep, inv_keep(p), np.float32(0.0)).astype(np.float32)


# ---- element index of each consumer family ---------------------------------------------------------------------------------------
def flat_index(n):
    """cb_dropout: element i of the flat buffer."""
    return np.arange(n, dtype=np.uint64)


def gemm_index(rows, n):
    """cb_gemm epilogue: out_row * n + col, with n the descriptor's column count (not out_ld) and out_row the output row after
    the row map. `rows` is an int (rows 0 .. rows-1) or an array of output rows. Returns [len(rows), n]."""
    r = np.arange(rows, dtype=np.uint64) if np.isscalar(rows) else np.asarray(rows).astype(np.uint64)
    return r[:, None] * np.uint64(n) + np.arange(n, dtype=np.uint64)[None, :]


def layernorm_index(m):
    """cb_layernorm_bwd (dx_drop, dbias_drop): row * 768 + col. Returns [m, 768]."""
    return gemm_index(m, HIDDEN)


def embedding_index(nseq, l, pos):
    """cb_embed_*: (seq * l + pos) * 768 + col, for the positions `pos` of each sequence of length l (text rows: 0 .. lt-1,
    visual cell j: lt + j). Returns [nseq, len(pos), 768]."""
    pos = np.asarray(pos).astype(np.uint64)
    rows = np.arange(nseq, dtype=np.uint64)[:, None] * np.uint64(l) + pos[None, :]
    return rows[:, :, None] * np.uint64(HIDDEN) + np.arange(HIDDEN, dtype=np.uint64)[None, None, :]


def attention_index(nseq, heads, l):
    """cb_attention_* probabilities P[seq, h, i, j]: ((seq * heads + h) * l + i) * l + j. Returns [nseq, heads, l, l]."""
    return np.arange(nseq * heads * l * l, dtype=np.uint64).reshape(nseq, heads, l, l)
