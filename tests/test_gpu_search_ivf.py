"""clip_b200_ivf_train_16 / _build_16 / _search_16 (K10's IVF instances, csrc/search.cu), called through prod.lib, against
clip_b200_topk_search_16 and the rule of tests/_search_ivf.py, byte for byte.

- K10's premise: a score's bits do not depend on the query's column in the query tile or on the tile's width.
- Build: the assignment is clip_b200_topk_search_16(row, centroids, 1); offsets, ids and rows are the rule's layout; edge cases and
  one build past 2^32 bytes.
- Train: the rule's centroids, given the library's own assignments, bit for bit; empty lists keep their centroid; a second call
  gives the same bits.
- Full probe equals clip_b200_topk_search_16 over the original database; partial probe equals it over the probed lists' rows.
- Recall on clustered rows; refusals in order, a malformed index refused, empty calls, output guards."""
import ctypes as C

import numpy as np
import pytest

import _search_ivf as rule
from _search_bound import bits16, unit_rows
from test_gpu_scoring_exact import GUARD, _Model, _assert_ranked
from test_gpu_search_16 import _dev, search16

pytestmark = pytest.mark.gpu
F16, BF16 = 1, 2
FP, IP = C.POINTER(C.c_float), C.POINTER(C.c_int)
FLT_MAX = np.finfo(np.float32).max


@pytest.fixture(scope="module")
def tiny(prod):
    m = _Model(prod, "tiny", "f16")
    yield m
    prod.free(m.ctx)


def _val16(bits, bf):
    """uint16 encodings -> float32 values"""
    return (bits.astype(np.uint32) << 16).view(np.float32) if bf else bits.view(np.float16).astype(np.float32)


def _host(m, p, shape, dtype):
    a = np.empty(shape, dtype)
    assert m.prod.lib.clip_b200_memcpy_d2h(m.ctx, a.ctypes.data, p, a.nbytes), m.prod.last_error()
    return a


def _free(m, *ps):
    for p in ps:
        m.prod.lib.clip_b200_device_free(m.ctx, p)


def train(m, x, n_lists, n_iter, in_type):
    bf = in_type == BF16
    d_x = _dev(m, bits16(x, bf))
    d_c = m.prod.lib.clip_b200_device_malloc(m.ctx, n_lists * x.shape[1] * 2)
    try:
        assert m.prod.lib.clip_b200_ivf_train_16(m.ctx, d_x, len(x), x.shape[1], in_type, n_lists, n_iter, d_c), m.prod.last_error()
        return _val16(_host(m, d_c, (n_lists, x.shape[1]), np.uint16), bf)
    finally:
        _free(m, d_x, d_c)


class Index:
    """an index built on the device from db rows and centroids (float values exact in in_type)"""

    def __init__(self, m, db, cent, in_type):
        self.m, self.bf, self.in_type, self.n, self.dim, self.L = m, in_type == BF16, in_type, len(db), db.shape[1], len(cent)
        L = m.prod.lib
        self.d_db, self.d_c = _dev(m, bits16(db, self.bf)), _dev(m, bits16(cent, self.bf))
        self.d_off = L.clip_b200_device_malloc(m.ctx, (self.L + 1) * 4)
        self.d_ids = L.clip_b200_device_malloc(m.ctx, max(self.n, 4) * 4)
        self.d_rows = L.clip_b200_device_malloc(m.ctx, max(self.n * self.dim * 2, 16))
        ok = L.clip_b200_ivf_build_16(m.ctx, self.d_db, self.n, self.dim, in_type, self.d_c, self.L, self.d_off, self.d_ids, self.d_rows)
        assert ok, m.prod.last_error()

    def layout(self, rows=True):
        off = _host(self.m, self.d_off, (self.L + 1,), np.int32)
        ids = _host(self.m, self.d_ids, (self.n,), np.int32)
        return off, ids, (_host(self.m, self.d_rows, (self.n, self.dim), np.uint16) if rows else None)

    def search(self, q, nprobe, top_k, expect_ok=True):
        nq, w = len(q), min(top_k, self.n)
        s = np.full(nq * w + GUARD, 7.0, np.float32)
        i = np.full(nq * w + GUARD, -7, np.int32)
        d_q = _dev(self.m, bits16(q, self.bf))
        try:
            ok = self.m.prod.lib.clip_b200_ivf_search_16(self.m.ctx, d_q, nq, self.dim, self.in_type, self.d_c, self.L, self.d_off,
                                                         self.d_ids, self.d_rows, self.n, nprobe, top_k, s.ctypes.data_as(FP),
                                                         i.ctypes.data_as(IP))
        finally:
            _free(self.m, d_q)
        assert ok == expect_ok, self.m.prod.last_error()
        assert (s[nq * w:] == 7.0).all() and (i[nq * w:] == -7).all(), "written past n_q * w"
        return s[:nq * w].reshape(nq, w), i[:nq * w].reshape(nq, w)

    def free(self):
        _free(self.m, self.d_db, self.d_c, self.d_off, self.d_ids, self.d_rows)


def _assign(m, x, cent, in_type):
    return search16(m, x, cent, 1, in_type)[1][:, 0]


# ---- 1. K10's premise ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("in_type", [F16, BF16])
def test_scores_do_not_depend_on_query_column_or_tile_width(tiny, in_type):
    rng = np.random.default_rng(11)
    bf = in_type == BF16
    q, db = unit_rows(rng, 1003, 256, bf), unit_rows(rng, 300, 256, bf)
    tracked = [0, 1, 2]

    def full(s, i):
        out = np.empty(s.shape, np.float32)
        np.put_along_axis(out, i, s, 1)
        return out
    alone = [full(*search16(tiny, q[t:t + 1], db, 300, in_type))[0] for t in tracked]
    for nq in (1, 7, 8, 9, 64, 65, 129, 1000):
        for pos in sorted({0, nq // 2, nq - 1}):
            qs = q[3:3 + nq].copy()
            for t in tracked:
                qs[pos] = q[t]
                got = full(*search16(tiny, qs, db, 300, in_type))[pos]
                assert np.array_equal(got.view(np.uint32), alone[t].view(np.uint32)), (nq, pos, t)


# ---- 2. build -----------------------------------------------------------------------------------------------------------------
def _check_build(m, db, cent, in_type):
    ix = Index(m, db, cent, in_type)
    try:
        lists = _assign(m, db, cent, in_type)
        off, ids, rows = ix.layout()
        want_off, want_ids = rule.layout(lists, len(cent))
        assert np.array_equal(off, want_off) and np.array_equal(ids, want_ids)
        assert np.array_equal(rows, bits16(db, in_type == BF16)[want_ids])
        return off
    finally:
        ix.free()


@pytest.mark.parametrize("in_type", [F16, BF16])
@pytest.mark.parametrize("case", ["random", "one_list", "empty_lists", "all_in_one", "ragged"])
def test_build_is_the_rule_layout(tiny, in_type, case):
    rng = np.random.default_rng(21)
    bf = in_type == BF16
    n = {"ragged": 1001}.get(case, 5000)
    db = unit_rows(rng, n, 64, bf)
    cent = unit_rows(rng, 1 if case == "one_list" else 40, 64, bf)
    if case == "empty_lists":
        cent[20:] = cent[:20]                            # duplicates: ties go to the lower list, so lists 20 .. 39 stay empty
    if case == "all_in_one":
        db[:, 0] = np.abs(db[:, 0]) + 4                  # every row leans on feature 0, and so does centroid 7 alone
        cent[:, 0] = -np.abs(cent[:, 0])
        cent[7] = 0
        cent[7, 0] = 1
    off = _check_build(tiny, db, cent, in_type)
    if case == "empty_lists":
        assert (np.diff(off)[20:] == 0).all()
    if case == "all_in_one":
        assert np.diff(off)[7] == n


def test_build_past_2_32_bytes(tiny):
    """2.9 M rows of 768 (4.45 GB): the database repeats 4096 rows, so row r's list is that of row r % 4096"""
    n, dim, P = 2_900_000, 768, 4096
    rng = np.random.default_rng(5)
    base = unit_rows(rng, P, dim, False)
    b16 = bits16(base, False)
    cent = unit_rows(rng, 64, dim, False)
    L = tiny.prod.lib
    d_db, d_rows = L.clip_b200_device_malloc(tiny.ctx, n * dim * 2), L.clip_b200_device_malloc(tiny.ctx, n * dim * 2)
    d_c, d_off, d_ids = _dev(tiny, bits16(cent, False)), L.clip_b200_device_malloc(tiny.ctx, 65 * 4), L.clip_b200_device_malloc(tiny.ctx, n * 4)
    try:
        assert d_db and d_rows and d_ids
        for r0 in range(0, n, P):
            c = min(P, n - r0)
            assert L.clip_b200_memcpy_h2d(tiny.ctx, C.c_void_p(d_db + r0 * dim * 2), b16.ctypes.data, c * dim * 2)
        assert L.clip_b200_ivf_build_16(tiny.ctx, d_db, n, dim, F16, d_c, 64, d_off, d_ids, d_rows), tiny.prod.last_error()
        lists = _assign(tiny, base, cent, F16)[np.arange(n) % P]
        want_off, want_ids = rule.layout(lists, 64)
        assert np.array_equal(_host(tiny, d_off, (65,), np.int32), want_off)
        ids = _host(tiny, d_ids, (n,), np.int32)
        assert np.array_equal(ids, want_ids)
        for p in (0, 1, n // 2, n - 2, n - 1, 2_796_202, 2_796_203):   # byte 2^32 lies inside stored row 2 796 202
            assert np.array_equal(_host_row(tiny, d_rows, p, dim), b16[ids[p] % P]), p
    finally:
        _free(tiny, d_db, d_rows, d_c, d_off, d_ids)


def _host_row(m, d, p, dim):
    a = np.empty(dim, np.uint16)
    assert m.prod.lib.clip_b200_memcpy_d2h(m.ctx, a.ctypes.data, C.c_void_p(d + p * dim * 2), a.nbytes), m.prod.last_error()
    return a


# ---- 3. train -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("in_type", [F16, BF16])
@pytest.mark.parametrize("data", ["exact", "unit"])
def test_train_is_the_rule(tiny, in_type, data):
    rng = np.random.default_rng(31 + in_type)
    bf = in_type == BF16
    x = (rng.integers(-4, 5, (3000, 16)) * 2.0 ** -3).astype(np.float32) if data == "exact" else unit_rows(rng, 3000, 128, bf)
    for n_iter in (1, 4):
        got = train(tiny, x, 24, n_iter, in_type)
        want = rule.train(x.astype(np.float64), 24, n_iter, bf, assign=lambda a, c: _assign(tiny, a, c, in_type))
        assert np.array_equal(got.view(np.uint32), want.astype(np.float32).view(np.uint32)), n_iter
        again = train(tiny, x, 24, n_iter, in_type)
        assert np.array_equal(got.view(np.uint32), again.view(np.uint32))
    if data == "unit":                                   # within one ulp of the fp64 normalised mean of the members
        prev = train(tiny, x, 24, 2, in_type)
        lists = _assign(tiny, x, prev, in_type)
        nxt = train(tiny, x, 24, 3, in_type)
        ulp = 2.0 ** -8 if bf else 2.0 ** -11
        for l in range(24):
            if (lists == l).any():
                m = x[lists == l].astype(np.float64).mean(0)
                assert (np.abs(nxt[l] - m / np.linalg.norm(m)) <= ulp).all(), l


def test_train_keeps_empty_lists(tiny):
    x = (np.random.default_rng(2).integers(-4, 5, (400, 16)) * 2.0 ** -3).astype(np.float32)
    x[[i * 400 // 8 for i in range(8)][4]] = x[0]        # initial centroid 4 duplicates centroid 0: list 4 stays empty
    got = train(tiny, x, 8, 1, F16)
    assert np.array_equal(got[4], x[0])


# ---- 4. full probe ------------------------------------------------------------------------------------------------------------
def _index(m, n, dim, L, in_type, seed, skew=False, empty=False):
    rng = np.random.default_rng(seed)
    bf = in_type == BF16
    db, cent = unit_rows(rng, n, dim, bf), unit_rows(rng, L, dim, bf)
    if skew:                                             # about 90 % of the rows lean towards centroid 0
        db[: n * 9 // 10] = unit_rows(rng, n * 9 // 10, dim, bf) * 0.3 + cent[0]
        db = np.asarray(bits16(db, bf), np.uint16)
        db = _val16(db, bf)
    if empty:
        cent[L // 2:] = cent[: L - L // 2]
    return rng, db, cent, Index(m, db, cent, in_type)


FULL = [(d, nq, k) for d in (8, 768, 2048) for nq in (1, 7, 129, 1000) for k in (1, 10, 1024)] + [(8, 40_000, 10), (768, 40_000, 1)]


@pytest.mark.parametrize("dim,nq,k", FULL)
def test_full_probe_is_the_flat_search(tiny, dim, nq, k):
    in_type = BF16 if (dim + nq + k) % 2 else F16
    rng, db, cent, ix = _index(tiny, 3000, dim, 16, in_type, dim + nq)
    try:
        q = unit_rows(rng, nq, dim, in_type == BF16)
        s, i = ix.search(q, 16, k)
        s16, i16 = search16(tiny, q, db, k, in_type)
        _assert_ranked(s, i, s16, i16, "full probe d=%d n_q=%d k=%d" % (dim, nq, k))
    finally:
        ix.free()


@pytest.mark.parametrize("kind", ["skew", "empty", "split"])
def test_full_probe_skewed_empty_and_split(tiny, kind):
    L = 32
    rng, db, cent, ix = _index(tiny, 20_000, 128, L, F16, 7, skew=kind == "skew", empty=kind == "empty")
    try:
        off, _, _ = ix.layout(rows=False)
        if kind == "skew":
            assert np.diff(off).max() >= 0.85 * 20_000
        if kind == "empty":
            assert (np.diff(off) == 0).sum() >= L // 2
        q = unit_rows(rng, 1000, 128, False)
        k = 1024 if kind == "split" else 10               # 1024: blocks of 2^24 / (1280 * 32) = 409 queries
        s, i = ix.search(q, 1024, k)
        s16, i16 = search16(tiny, q, db, k, F16)
        _assert_ranked(s, i, s16, i16, kind)
    finally:
        ix.free()


# ---- 5. partial probe ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("in_type", [F16, BF16])
@pytest.mark.parametrize("nprobe,k", [(1, 10), (3, 100), (5, 1024)])
def test_partial_probe_is_the_search_over_probed_lists(tiny, in_type, nprobe, k):
    rng, db, cent, ix = _index(tiny, 6000, 96, 40, in_type, 3 * nprobe + in_type, empty=nprobe == 3)
    db = db.copy()
    try:
        q = unit_rows(rng, 300, 96, in_type == BF16)
        s, i = ix.search(q, nprobe, k)
        lists = _assign(tiny, db, cent, in_type)
        probe = search16(tiny, q, cent, nprobe, in_type)[1]
        w = min(k, len(db))
        for r in range(0, 300, 15):
            rows = np.flatnonzero(np.isin(lists, probe[r]))
            ws, wi = np.full(w, -np.inf, np.float32), np.full(w, -1, np.int32)
            if len(rows):
                ss, si = search16(tiny, q[r:r + 1], db[rows], k, in_type)
                ws[:ss.shape[1]], wi[:ss.shape[1]] = ss[0], rows[si[0]]
            _assert_ranked(s[r:r + 1], i[r:r + 1], ws[None], wi[None], "query %d" % r)
    finally:
        ix.free()


def test_nan_rows_rank_last(tiny):
    rng = np.random.default_rng(9)
    db, cent = unit_rows(rng, 1000, 64, False), unit_rows(rng, 8, 64, False)
    db[[5, 700, 999], 3] = np.nan
    ix = Index(tiny, db, cent, F16)
    try:
        q = unit_rows(rng, 20, 64, False)
        s, i = ix.search(q, 8, 1000)
        s16, i16 = search16(tiny, q, db, 1000, F16)
        _assert_ranked(s, i, s16, i16, "NaN rows")
        assert (s[:, -3:] == -FLT_MAX).all()
    finally:
        ix.free()


# ---- 6. recall ----------------------------------------------------------------------------------------------------------------
def test_recall_on_clustered_rows(tiny):
    rng = np.random.default_rng(99)
    dim, C_, n = 64, 64, 20_000
    centers = unit_rows(rng, C_, dim, False)
    lab = rng.integers(0, C_, n)
    x = centers[lab] + 0.05 * rng.standard_normal((n, dim))
    x = (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)
    cent = train(tiny, x[rng.permutation(n)[:5000]], 64, 10, F16)
    ix = Index(tiny, x, cent, F16)
    try:
        q = x[rng.choice(n, 200, replace=False)] + 0.02 * rng.standard_normal((200, dim)).astype(np.float32)
        _, i = ix.search(q, 8, 10)
        _, i16 = search16(tiny, q, x, 10, F16)
        recall = np.mean([len(np.intersect1d(a, b)) / 10 for a, b in zip(i, i16)])
        assert recall >= 0.9, recall
    finally:
        ix.free()


# ---- 7. contract --------------------------------------------------------------------------------------------------------------
def test_refusals_in_order_and_empty_calls(tiny):
    L = tiny.prod.lib
    ctx = tiny.ctx
    rng = np.random.default_rng(1)
    db = unit_rows(rng, 300, 32, False)
    cent = db[:4].copy()
    ix = Index(tiny, db, cent, F16)
    s, i = np.zeros(64, np.float32), np.zeros(64, np.int32)
    sp, ip = s.ctypes.data_as(FP), i.ctypes.data_as(IP)
    err = lambda: tiny.prod.last_error()
    try:
        d_q = ix.d_db

        def srch(**kw):
            a = dict(ctx=ctx, q=d_q, nq=2, dim=32, t=F16, c=ix.d_c, L=4, off=ix.d_off, ids=ix.d_ids, rows=ix.d_rows, n=300, npr=2, k=5,
                     s=sp, i=ip)
            a.update(kw)
            return L.clip_b200_ivf_search_16(a["ctx"], a["q"], a["nq"], a["dim"], a["t"], a["c"], a["L"], a["off"], a["ids"], a["rows"],
                                             a["n"], a["npr"], a["k"], a["s"], a["i"])
        steps = [(dict(ctx=None), "null context"), (dict(t=0), "in_type"), (dict(dim=12), "dim"), (dict(L=0), "n_lists"),
                 (dict(npr=1025), "nprobe"), (dict(k=0), "top_k"), (dict(nq=1 << 31), "2^31"), (dict(rows=ix.d_rows + 8), "aligned"),
                 (dict(off=ix.d_off + 2), "4-byte"), (dict(s=None), "null output")]
        for j, (kw, msg) in enumerate(steps):
            bad = {}
            for kw2, _ in steps[j:]:
                bad.update(kw2)                           # this fault and every later one: the first is reported
            assert not srch(**bad)
            assert err().startswith("clip_b200_ivf_search_16") and msg in err(), (msg, err())
        assert srch(nq=0, q=None, s=None) and srch(n=0, rows=None, i=None)
        # a malformed index is refused before any device work
        good = _host(tiny, ix.d_off, (5,), np.int32)
        for bad_off in ([1, 2, 3, 4, 300], [0, 5, 3, 200, 300], [0, 1, 2, 3, 299], [0, 1, 2, 3, 1 << 30]):
            tiny.prod.lib.clip_b200_memcpy_h2d(ctx, ix.d_off, np.array(bad_off, np.int32).ctypes.data, 20)
            assert not srch() and "d_offsets" in err(), bad_off
        tiny.prod.lib.clip_b200_memcpy_h2d(ctx, ix.d_off, good.ctypes.data, 20)
        assert srch()
        # train and build: their own steps
        assert not L.clip_b200_ivf_train_16(ctx, d_q, 300, 32, F16, 4, 0, ix.d_c) and "n_iter" in err()
        assert not L.clip_b200_ivf_train_16(ctx, d_q, 3, 32, F16, 4, 1, ix.d_c) and "n_lists" in err()
        assert not L.clip_b200_ivf_train_16(ctx, d_q, 300, 32, F16, 65537, 1, ix.d_c) and "n_lists" in err()
        assert not L.clip_b200_ivf_train_16(ctx, d_q, 300, 32, F16, 4, 1, None) and "aligned" in err()
        assert not L.clip_b200_ivf_build_16(ctx, d_q, 300, 32, F16, ix.d_c, 4, ix.d_off, None, ix.d_rows) and "d_ids" in err()
        assert err().startswith("clip_b200_ivf_build_16")
        zeros = np.full(6, -7, np.int32)
        d_o = _dev(tiny, zeros)
        assert L.clip_b200_ivf_build_16(ctx, None, 0, 32, F16, None, 5, d_o, None, None), err()
        assert np.array_equal(_host(tiny, d_o, (6,), np.int32), [0] * 6)
        _free(tiny, d_o)
    finally:
        ix.free()
