"""The rule of the inverted-file index (clip_b200_ivf_train_16 / _build_16 / _search_16, include/clip_b200.h) in numpy.

Rows and centroids are float values that are exact in the 16-bit type.  `assign` is a function (rows, centroids) -> the list of
each row; the library's is clip_b200_topk_search_16(row, centroids, 1), and `exact_assign` is the same ranking on fp64 scores,
which equals it on exact data (integers times 2^-3 at small dims, where every dot product is exact in any order).

The k-means update follows the library's summation order exactly (members in row order within chunks of 512, chunk sums added in
chunk order, the squares of the mean by the update kernel's fixed tree), so its centroids have the library's bits on any data,
given the same assignments."""
import numpy as np

CHUNK = 512


def rne_bf16(v):
    """fp64 -> bf16 value, rounded once to nearest even (no detour through f32)"""
    v = np.asarray(v, np.float64)
    m, e = np.frexp(v)                                 # v = m 2^e, 0.5 <= |m| < 1
    e = np.maximum(e, -125)                            # below the normal range the step stays 2^-133
    return np.ldexp(np.rint(np.ldexp(v, 8 - e)), e - 8)


def round16(v, bf):
    """fp64 -> the 16-bit type's value (as fp64), rounded once to nearest even"""
    return rne_bf16(v) if bf else np.asarray(v, np.float64).astype(np.float16).astype(np.float64)


def exact_assign(x, cent):
    """best centroid by fp64 score, the lower list index on ties (np.argmax takes the first maximum)"""
    return np.argmax(np.asarray(x, np.float64) @ np.asarray(cent, np.float64).T, axis=1)


def layout(lists, n_lists):
    """(offsets [n_lists + 1], ids [n]): list by list, rows within a list in increasing original index"""
    lists = np.asarray(lists, np.int64)
    off = np.zeros(n_lists + 1, np.int64)
    off[1:] = np.cumsum(np.bincount(lists, minlength=n_lists))
    return off, np.argsort(lists, kind="stable")


def _tree_sq(m):
    """sum of m^2 in the update kernel's order: 256 threads over features f = t, t + 256, ... in order, a warp butterfly, the
    eight warp sums in order"""
    t = np.zeros(256)
    for f in range(len(m)):
        t[f % 256] += m[f] * m[f]
    w = t.reshape(8, 32)
    for o in (16, 8, 4, 2, 1):
        w = w + w[:, np.arange(32) ^ o]
    tot = 0.0
    for v in w[:, 0]:
        tot += v
    return tot


def update(x, lists, cent, bf):
    """one k-means update: each non-empty list's centroid -> rne16(m / sqrt(sum m^2)), m the fp64 mean of its members; an empty
    list or a zero mean keeps its centroid"""
    x, cent = np.asarray(x, np.float64), np.array(cent, np.float64)
    off, ids = layout(lists, len(cent))
    for l in range(len(cent)):
        mem = ids[off[l]:off[l + 1]]
        if len(mem) == 0:
            continue
        s = np.zeros(x.shape[1])
        for c0 in range(0, len(mem), CHUNK):
            part = np.zeros(x.shape[1])
            for r in mem[c0:c0 + CHUNK]:
                part += x[r]
            s += part
        m = s / len(mem)
        tot = _tree_sq(m)
        if tot == 0.0:
            continue
        cent[l] = round16(m / np.sqrt(tot), bf)
    return cent


def init(x, n_lists):
    """the initial centroids: rows floor(i * n / n_lists)"""
    n = len(x)
    return np.array(x, np.float64)[[i * n // n_lists for i in range(n_lists)]]


def train(x, n_lists, n_iter, bf, assign=exact_assign):
    cent = init(x, n_lists)
    for _ in range(n_iter):
        cent = update(x, assign(x, cent), cent, bf)
    return cent


def probes(q, cent, nprobe):
    """each query's best min(nprobe, n_lists) lists: score descending, then the lower list index (exact scores)"""
    s = np.asarray(q, np.float64) @ np.asarray(cent, np.float64).T
    return np.argsort(-s, axis=1, kind="stable")[:, :min(nprobe, len(cent))]


def search(q, db, lists, probe, top_k):
    """the best w = min(top_k, n_db) of the rows whose list each query probes, by (exact score descending, original index
    ascending), padded with (-inf, -1): (scores fp64 [n_q, w], indices [n_q, w])"""
    q, db, lists = np.asarray(q, np.float64), np.asarray(db, np.float64), np.asarray(lists)
    w = min(top_k, len(db))
    out_s, out_i = np.full((len(q), w), -np.inf), np.full((len(q), w), -1, np.int64)
    for r in range(len(q)):
        rows = np.flatnonzero(np.isin(lists, probe[r]))          # increasing original index
        s = db[rows] @ q[r]
        order = np.argsort(-s, kind="stable")[:w]
        out_s[r, :len(order)], out_i[r, :len(order)] = s[order], rows[order]
    return out_s, out_i
