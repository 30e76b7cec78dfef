"""The rule of the inverted-file index with product-quantised residuals (clip_b200_ivfpq_*, include/clip_b200.h) in numpy.

Rows, queries and centroids are float32 values that are exact in the 16-bit type; codebooks are float32.  Every step is exact, so
these functions give the library's bits given the same inputs:
- the lists of the rows (the library's are clip_b200_topk_search_16(row, centroids, 1); `_search_ivf.exact_assign` equals them on
  exact data);
- for a search, the probes and their coarse scores (clip_b200_topk_search_16(q, centroids, nprobe)'s ids and values).
The fmaf chains use `_util.fmaf32`; the k-means sums follow `_search_ivf`'s chunk order (members in row order, chunks of 512,
chunk sums added in chunk order)."""
import numpy as np

from _search_ivf import layout
from _util import fmaf32

CHUNK = 512
FLT_MAX = np.finfo(np.float32).max


def residuals(x, cent, lists):
    """r = x - c[list] in fp32, rounded to nearest"""
    return np.asarray(x, np.float32) - np.asarray(cent, np.float32)[np.asarray(lists)]


def distances(r, book):
    """r [n, dsub], book [256, dsub] -> d [n, 256] f32: t = r_j - b_j in fp32, d = fmaf(t, t, d) in feature order from +0; NaN is +inf"""
    r, book = np.asarray(r, np.float32), np.asarray(book, np.float32)
    d = np.zeros((len(r), len(book)), np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for j in range(r.shape[1]):
            t = r[:, j:j + 1] - book[None, :, j]
            d = fmaf32(t, t, d)
    d[np.isnan(d)] = np.inf
    return d


def encode_residuals(r, books):
    """codes [n, m] uint8: per subspace the least distance, the lower index on ties (np.argmin takes the first)"""
    m, _, dsub = books.shape
    return np.stack([np.argmin(distances(r[:, s * dsub:(s + 1) * dsub], books[s]), axis=1) for s in range(m)], 1).astype(np.uint8)


def encode(x, cent, lists, books):
    return encode_residuals(residuals(x, cent, lists), books)


def seq_sum(v):
    """v [n, f] summed over rows in fp64 in row order, from +0 (cumsum is sequential; the leading zero makes -0 rows sum to +0)"""
    return np.cumsum(np.concatenate([np.zeros((1, v.shape[1])), np.asarray(v, np.float64)]), axis=0)[-1]


def update(r, codes, books):
    """each non-empty codeword -> fp32(fp64 mean of its members), members in row order, in chunks of 512 whose sums are added in
    chunk order; an empty codeword keeps its value"""
    books = np.array(books, np.float32)
    m, _, dsub = books.shape
    for s in range(m):
        rs = r[:, s * dsub:(s + 1) * dsub]
        for k in range(256):
            mem = np.flatnonzero(codes[:, s] == k)
            if len(mem) == 0:
                continue
            parts = np.stack([seq_sum(rs[mem[c0:c0 + CHUNK]]) for c0 in range(0, len(mem), CHUNK)])
            books[s, k] = (seq_sum(parts) / len(mem)).astype(np.float32)
    return books


def init(r, m):
    """codeword i of every subspace: the residual of training row floor(i n / 256)"""
    n, dim = r.shape
    return np.asarray(r, np.float32)[[i * n // 256 for i in range(256)]].reshape(256, m, dim // m).transpose(1, 0, 2).copy()


def train(x, cent, lists, m, n_iter):
    r = residuals(x, cent, lists)
    books = init(r, m)
    for _ in range(n_iter):
        books = update(r, encode_residuals(r, books), books)
    return books


def tables(q, books):
    """T [n_q, m, 256] f32: fmaf chain over subspace s's features of q_j * b_kj from +0, in order"""
    q = np.asarray(q, np.float32)
    m, _, dsub = books.shape
    t = np.zeros((len(q), m, 256), np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for s in range(m):
            for j in range(dsub):
                t[:, s] = fmaf32(q[:, s * dsub + j, None], books[s, None, :, j], t[:, s])
    return t


def adc(coarse, t, codes):
    """scores of stored rows for one query: v = coarse [n] f32, then v = v + T[s][c_s] in fp32 for s in order; NaN -> -FLT_MAX"""
    v = np.asarray(coarse, np.float32).copy()
    with np.errstate(invalid="ignore", over="ignore"):
        for s in range(codes.shape[1]):
            v = v + t[s, codes[:, s]]
    v[np.isnan(v)] = -FLT_MAX
    return v


def search(q, books, codes, lists, probe, coarse, top_k):
    """the best w = min(top_k, n_db) rows of each query's probed lists (probe [n_q, np] and their coarse scores [n_q, np]) by (score
    descending, original index ascending), padded with (-inf, -1): (scores f32 [n_q, w], indices [n_q, w])"""
    lists = np.asarray(lists)
    w = min(top_k, len(codes))
    t = tables(q, books)
    out_s, out_i = np.full((len(q), w), -np.inf, np.float32), np.full((len(q), w), -1, np.int64)
    for r in range(len(q)):
        sc = np.zeros(int(max(lists.max(initial=0), np.max(probe[r]))) + 1, np.float32)
        sc[np.asarray(probe[r])] = coarse[r]
        rows = np.flatnonzero(np.isin(lists, probe[r]))           # increasing original index
        v = adc(sc[lists[rows]], t[r], codes[rows])
        order = np.argsort(-v.astype(np.float64), kind="stable")[:w]
        out_s[r, :len(order)], out_i[r, :len(order)] = v[order], rows[order]
    return out_s, out_i


def build(lists, codes, n_lists):
    """(offsets, ids, stored codes): clip_b200_ivf_build_16's layout, the codes gathered"""
    off, ids = layout(lists, n_lists)
    return off, ids, np.asarray(codes)[ids]
