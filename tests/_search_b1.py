"""The rule of clip_b200_rows_to_binary, clip_b200_topk_search_b1 and clip_b200_topk_rescore (include/clip_b200.h), in numpy.

- to_bits: bit i of a row is x_i > c_i (IEEE: NaN and -0 against 0 give 0), packed LSB first, numpy.packbits(..., "little").
- hamming_scores: s = dim - 2 popcount(q XOR x), exact int64.
- rank: the family's order, score descending, then lower index first; the best k.
- rescore: per query the distinct candidates in [0, n_db), scored by one fmaf chain (tests/_util.py), NaN as -FLT_MAX, ranked, the
  row padded with (-inf, -1)."""
import numpy as np

from _util import fmaf_chain_dot

FLT_MAX = np.float32(np.finfo(np.float32).max)
_POPC = np.array([bin(i).count("1") for i in range(256)], np.int64)


def to_bits(x, center=None):
    """float32 rows [n, dim] (centre [dim] or None) -> uint8 [n, dim / 8]"""
    x = np.asarray(x, np.float32)
    c = np.zeros(x.shape[1], np.float32) if center is None else np.asarray(center, np.float32)
    with np.errstate(invalid="ignore"):
        return np.packbits(x > c, axis=1, bitorder="little")


def signs(bits, dim):
    """uint8 [n, dim / 8] -> int8 [n, dim] of +-1 (bit 1 is +1)"""
    return (np.unpackbits(np.asarray(bits, np.uint8), axis=1, count=dim, bitorder="little").astype(np.int8) * 2 - 1)


def hamming_scores(qb, xb, dim):
    """uint8 [n_q, dim / 8] x [n_db, dim / 8] -> int64 [n_q, n_db], dim - 2 popcount(q XOR x)"""
    qb, xb = np.asarray(qb, np.uint8), np.asarray(xb, np.uint8)
    s = np.empty((len(qb), len(xb)), np.int64)
    for i in range(len(qb)):
        s[i] = dim - 2 * _POPC[qb[i][None, :] ^ xb].sum(1)
    return s


def rank(s, k):
    """scores [n_q, n] (no NaN) -> (scores, indices) [n_q, min(k, n)]: descending, ties by lower index"""
    n = s.shape[1]
    k = min(k, n)
    order = np.argsort(-np.asarray(s, np.float64), axis=1, kind="stable")[:, :k]
    return np.take_along_axis(s, order, 1), order.astype(np.int32)


def search_b1(qb, xb, dim, k):
    s, i = rank(hamming_scores(qb, xb, dim), k)
    return s.astype(np.float32), i


def rescore_lists(cand, n_db, scores_of):
    """cand [n_q, n_cand] -> per query the sorted distinct valid candidates and their float32 scores, scores_of(r, idx)"""
    out = []
    for r, row in enumerate(np.asarray(cand, np.int64)):
        idx = np.unique(row[(row >= 0) & (row < n_db)])
        s = np.asarray(scores_of(r, idx), np.float32) if len(idx) else np.empty(0, np.float32)
        out.append((idx, np.where(np.isnan(s), -FLT_MAX, s).astype(np.float32)))
    return out


def rescore_rank(lists, k):
    """lists of (distinct indices ascending, scores) -> (scores, indices) [n_q, k], padded with (-inf, -1)"""
    S = np.full((len(lists), k), -np.inf, np.float32)
    I = np.full((len(lists), k), -1, np.int32)
    for r, (idx, s) in enumerate(lists):
        order = np.argsort(-s.astype(np.float64), kind="stable")[:k]      # idx ascending, so stable ties go to the lower index
        S[r, :len(order)], I[r, :len(order)] = s[order], idx[order]
    return S, I


def rescore(q, db, cand, k):
    """float32 q [n_q, dim], db [n_db, dim], cand [n_q, n_cand] -> the rule's (scores, indices) [n_q, k], scores from fmaf chains"""
    q, db = np.asarray(q, np.float32), np.asarray(db, np.float32)
    return rescore_rank(rescore_lists(cand, len(db), lambda r, idx: fmaf_chain_dot(q[r:r + 1], db[idx])[0]), k)
