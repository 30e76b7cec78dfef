"""The numpy rule of the binary search and the rescore (tests/_search_b1.py) agrees with itself, and the checks built on it reject
the wrong variants a kernel could implement: MSB-first packing, ties broken by the higher index, duplicates counted twice."""
import numpy as np

import _search_b1 as rule
from _util import fmaf_chain_dot


def test_hamming_score_is_the_signed_dot_product():
    rng = np.random.default_rng(1)
    for dim in (128, 768, 2048):
        q, x = rng.standard_normal((5, dim)).astype(np.float32), rng.standard_normal((300, dim)).astype(np.float32)
        qb, xb = rule.to_bits(q), rule.to_bits(x)
        want = rule.signs(qb, dim).astype(np.int64) @ rule.signs(xb, dim).astype(np.int64).T
        assert (rule.hamming_scores(qb, xb, dim) == want).all()
        assert (rule.signs(xb, dim) == np.where(x > 0, 1, -1)).all()


def test_packing_is_lsb_first_and_the_compare_is_ieee():
    x = np.zeros((1, 128), np.float32)
    x[0, 0] = 1.0                                                 # feature 0 -> byte 0, bit 0
    x[0, 9] = np.float32(1e-45)                                   # a subnormal above 0 -> 1
    x[0, 10] = -0.0                                               # -0 > 0 is false
    x[0, 11] = np.nan
    x[0, 127] = np.inf
    b = rule.to_bits(x)
    assert b.shape == (1, 16) and b[0, 0] == 1 and b[0, 1] == 2 and b[0, 15] == 0x80 and b.sum() == 1 + 2 + 0x80
    msb = np.packbits(x > 0, axis=1)                              # MSB first: the wrong variant
    assert (msb != b).any()
    c = np.full(128, 2.0, np.float32)
    assert rule.to_bits(x, c).sum() == 0x80                       # only +inf exceeds 2


def test_rank_breaks_ties_by_lower_index():
    s = np.array([[3, 5, 5, 1, 5]], np.int64)
    got_s, got_i = rule.rank(s, 3)
    assert got_i.tolist() == [[1, 2, 4]] and got_s.tolist() == [[5, 5, 5]]
    higher_first = np.argsort(-s[0] * 10 - np.arange(5))[:3]      # ties by higher index: the wrong variant
    assert higher_first.tolist() != got_i[0].tolist()


def test_rescore_dedupes_skips_and_pads():
    rng = np.random.default_rng(2)
    q, db = rng.standard_normal((3, 16)).astype(np.float32), rng.standard_normal((6, 16)).astype(np.float32)
    full = fmaf_chain_dot(q, db)
    cand = np.array([[4, 4, -1, 2, 2147483647, 4],                # duplicates and out-of-range entries
                     [6, -5, 7, 100, -1, -1],                     # nothing valid: all pads
                     [0, 1, 2, 3, 4, 5]], np.int32)
    S, I = rule.rescore(q, db, cand, 4)
    r0 = sorted([2, 4], key=lambda j: (-full[0, j], j))
    assert I[0].tolist() == r0 + [-1, -1] and S[0, :2].tolist() == [full[0, j] for j in r0] and np.isneginf(S[0, 2:]).all()
    assert I[1].tolist() == [-1] * 4 and np.isneginf(S[1]).all()
    r2 = sorted(range(6), key=lambda j: (-full[2, j], j))[:4]
    assert I[2].tolist() == r2 and (S[2].view(np.uint32) == full[2, r2].view(np.uint32)).all()
    twice = [j for j in cand[0] if 0 <= j < 6]                    # duplicates counted twice: the wrong variant
    assert len(twice) == 4 and sorted(twice, key=lambda j: (-full[0, j], j))[:4] != I[0].tolist()


def test_rescore_nan_ranks_last_among_valid():
    q = np.ones((1, 8), np.float32)
    db = np.ones((3, 8), np.float32)
    db[1, 3] = np.nan
    db[2] *= -1
    S, I = rule.rescore(q, db, np.array([[1, 2, 0]], np.int32), 3)
    assert I[0].tolist() == [0, 2, 1] and S[0, 2] == -rule.FLT_MAX
