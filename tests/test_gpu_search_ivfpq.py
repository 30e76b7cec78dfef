"""clip_b200_ivfpq_train_16 / _encode_16 / _build / _search_16 (K13 and its kernels, csrc/search.cu), called through prod.lib,
against the rule of tests/_search_ivfpq.py and the library's own IVF and flat searches, byte for byte.

- Train: the rule's codebooks given the library's lists, at m 16, 48 and 96, f16 and bf16, with empty codewords; a second call gives
  the same bits.
- Encode: lists are clip_b200_topk_search_16(row, centroids, 1); codes are the rule's; NaN / Inf rows give code 0 where they touch;
  two chunks give the bytes of one call.
- Build: clip_b200_ivf_build_16's layout for the same rows, codes gathered; n_db == 0; a list out of range refused; codes past 2^32 B.
- Search: the rule, fed the coarse scores clip_b200_topk_search_16 returns, at every table-slice boundary, dims 64 to 2048, nprobe
  1 to >= n_lists, top_k 1 to 1024 with padding, skewed and empty lists, query counts across the query block, ties and NaN.
- Recall on clustered rows, with an exact rescore; refusals in order, empty calls, output guards."""
import ctypes as C

import numpy as np
import pytest

import _search_ivf as ivf_rule
import _search_ivfpq as rule
from _search_bound import bits16, unit_rows
from test_gpu_scoring_exact import GUARD, _assert_ranked
from test_gpu_search_16 import _dev, search16
from test_gpu_search_ivf import BF16, F16, Index, _free, _host, _val16, tiny  # noqa: F401  (tiny: the model fixture)

pytestmark = pytest.mark.gpu
FP, IP = C.POINTER(C.c_float), C.POINTER(C.c_int)
FLT_MAX = np.finfo(np.float32).max


def _assign(m, x, cent, in_type):
    return search16(m, x, cent, 1, in_type)[1][:, 0]


def _val(x, bf):
    """float32 values rounded to the 16-bit type, with NaN and Inf kept"""
    return _val16(bits16(x, bf), bf)


def pq_train(m, x, cent, M, n_iter, in_type):
    dim = x.shape[1]
    d_x, d_c = _dev(m, bits16(x, in_type == BF16)), _dev(m, bits16(cent, in_type == BF16))
    d_b = m.prod.lib.clip_b200_device_malloc(m.ctx, M * 256 * (dim // M) * 4)
    try:
        ok = m.prod.lib.clip_b200_ivfpq_train_16(m.ctx, d_x, len(x), dim, in_type, d_c, len(cent), M, n_iter, d_b)
        assert ok, m.prod.last_error()
        return _host(m, d_b, (M, 256, dim // M), np.float32)
    finally:
        _free(m, d_x, d_c, d_b)


def pq_encode(m, x, cent, books, in_type):
    M, dim = books.shape[0], x.shape[1]
    d_x, d_c, d_b = _dev(m, bits16(x, in_type == BF16)), _dev(m, bits16(cent, in_type == BF16)), _dev(m, np.ascontiguousarray(books))
    d_l, d_k = m.prod.lib.clip_b200_device_malloc(m.ctx, len(x) * 4 + 16), m.prod.lib.clip_b200_device_malloc(m.ctx, len(x) * M + 16)
    try:
        ok = m.prod.lib.clip_b200_ivfpq_encode_16(m.ctx, d_x, len(x), dim, in_type, d_c, len(cent), d_b, M, d_l, d_k)
        assert ok, m.prod.last_error()
        return _host(m, d_l, (len(x),), np.int32), _host(m, d_k, (len(x), M), np.uint8)
    finally:
        _free(m, d_x, d_c, d_b, d_l, d_k)


class PqIndex:
    """an IVF-PQ index built on the device from rows, centroids and codebooks (the encode and build calls)"""

    def __init__(self, m, db, cent, books, in_type):
        self.m, self.in_type, self.bf, self.n, self.dim, self.L, self.M = m, in_type, in_type == BF16, len(db), db.shape[1], len(cent), len(books)
        self.books = books
        self.lists, self.codes = pq_encode(m, db, cent, books, in_type)
        L = m.prod.lib
        self.d_c, self.d_b = _dev(m, bits16(cent, self.bf)), _dev(m, np.ascontiguousarray(books))
        d_l, d_k = _dev(m, self.lists), _dev(m, self.codes)
        self.d_off = L.clip_b200_device_malloc(m.ctx, (self.L + 1) * 4)
        self.d_ids = L.clip_b200_device_malloc(m.ctx, max(self.n, 4) * 4)
        self.d_codes = L.clip_b200_device_malloc(m.ctx, max(self.n * self.M, 16))
        try:
            assert L.clip_b200_ivfpq_build(m.ctx, d_l, d_k, self.n, self.L, self.M, self.d_off, self.d_ids, self.d_codes), m.prod.last_error()
        finally:
            _free(m, d_l, d_k)

    def layout(self):
        return (_host(self.m, self.d_off, (self.L + 1,), np.int32), _host(self.m, self.d_ids, (self.n,), np.int32),
                _host(self.m, self.d_codes, (self.n, self.M), np.uint8))

    def search(self, q, nprobe, top_k):
        nq, w = len(q), min(top_k, self.n)
        s, i = np.full(nq * w + GUARD, 7.0, np.float32), np.full(nq * w + GUARD, -7, np.int32)
        d_q = _dev(self.m, bits16(q, self.bf))
        try:
            ok = self.m.prod.lib.clip_b200_ivfpq_search_16(self.m.ctx, d_q, nq, self.dim, self.in_type, self.d_c, self.L, self.d_b, self.M,
                                                           self.d_off, self.d_ids, self.d_codes, self.n, nprobe, top_k,
                                                           s.ctypes.data_as(FP), i.ctypes.data_as(IP))
        finally:
            _free(self.m, d_q)
        assert ok, self.m.prod.last_error()
        assert (s[nq * w:] == 7.0).all() and (i[nq * w:] == -7).all(), "written past n_q * w"
        return s[:nq * w].reshape(nq, w), i[:nq * w].reshape(nq, w)

    def free(self):
        _free(self.m, self.d_c, self.d_b, self.d_off, self.d_ids, self.d_codes)


def _books(rng, M, dim, scale=0.1):
    return (rng.standard_normal((M, 256, dim // M)) * scale).astype(np.float32)


# ---- 1. train ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("in_type", [F16, BF16])
@pytest.mark.parametrize("M,data", [(16, "unit"), (48, "unit"), (96, "unit"), (16, "dup"), (96, "dup")])
def test_train_is_the_rule(tiny, in_type, M, data):
    rng = np.random.default_rng(M + in_type)
    bf, dim, L = in_type == BF16, 96, 8
    x = unit_rows(rng, 1200, dim, bf)
    if data == "dup":                                    # 40 distinct rows: duplicate initial codewords, the later ones stay empty
        x = x[rng.integers(0, 40, 1200)]
    cent = unit_rows(rng, L, dim, bf)
    lists = _assign(tiny, x, cent, in_type)
    for n_iter in (1, 3):
        got = pq_train(tiny, x, cent, M, n_iter, in_type)
        want = rule.train(x, cent, lists, M, n_iter)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), n_iter
        again = pq_train(tiny, x, cent, M, n_iter, in_type)
        assert np.array_equal(got.view(np.uint32), again.view(np.uint32))
    if data == "dup":
        r = rule.residuals(x, cent, lists)
        codes = rule.encode_residuals(r, rule.train(x, cent, lists, M, 2))
        assert len(np.unique(codes[:, 0])) < 256, "some codewords are empty"


# ---- 2. encode -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("in_type", [F16, BF16])
@pytest.mark.parametrize("M,dim", [(16, 64), (48, 768), (256, 256)])
def test_encode_is_the_rule(tiny, in_type, M, dim):
    rng = np.random.default_rng(dim + M)
    bf = in_type == BF16
    x, cent = unit_rows(rng, 2000, dim, bf), unit_rows(rng, 12, dim, bf)
    x[7, 3], x[8, dim - 1], x[9, :] = np.nan, np.inf, -np.inf
    books = _books(rng, M, dim)
    lists, codes = pq_encode(tiny, x, cent, books, in_type)
    assert np.array_equal(lists, _assign(tiny, x, cent, in_type))
    assert np.array_equal(codes, rule.encode(x, cent, lists, books))
    dsub = dim // M
    assert codes[7, 3 // dsub] == 0 and codes[8, (dim - 1) // dsub] == 0 and (codes[9] == 0).all()
    l1, c1 = pq_encode(tiny, x[:777], cent, books, in_type)
    l2, c2 = pq_encode(tiny, x[777:], cent, books, in_type)
    assert np.array_equal(np.concatenate([l1, l2]), lists) and np.array_equal(np.concatenate([c1, c2]), codes)


# ---- 3. build ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("in_type", [F16, BF16])
def test_build_is_the_ivf_layout(tiny, in_type):
    rng = np.random.default_rng(3 + in_type)
    bf = in_type == BF16
    db, cent = unit_rows(rng, 5000, 64, bf), unit_rows(rng, 40, 64, bf)
    cent[20:] = cent[:20]                                # lists 20 .. 39 stay empty
    ix, flat = PqIndex(tiny, db, cent, _books(rng, 16, 64), in_type), Index(tiny, db, cent, in_type)
    try:
        off, ids, codes = ix.layout()
        off16, ids16, _ = flat.layout(rows=False)
        assert np.array_equal(off, off16) and np.array_equal(ids, ids16)
        assert np.array_equal(codes, ix.codes[ids])
        assert (np.diff(off)[20:] == 0).all()
    finally:
        ix.free(), flat.free()


def test_build_edges(tiny):
    L = tiny.prod.lib
    ctx = tiny.ctx
    d_o = _dev(tiny, np.full(6, -7, np.int32))
    assert L.clip_b200_ivfpq_build(ctx, None, None, 0, 5, 16, d_o, None, None), tiny.prod.last_error()
    assert np.array_equal(_host(tiny, d_o, (6,), np.int32), [0] * 6)
    # a list out of range: refused, nothing written
    codes = np.arange(40 * 16, dtype=np.uint8).reshape(40, 16)
    for bad in (5, -1):
        lists = np.zeros(40, np.int32)
        lists[17] = bad
        d_l, d_k = _dev(tiny, lists), _dev(tiny, codes)
        d_ids, d_out = _dev(tiny, np.full(40, -7, np.int32)), _dev(tiny, np.full((40, 16), 9, np.uint8))
        d_o2 = _dev(tiny, np.full(6, -7, np.int32))
        try:
            assert not L.clip_b200_ivfpq_build(ctx, d_l, d_k, 40, 5, 16, d_o2, d_ids, d_out)
            assert tiny.prod.last_error().startswith("clip_b200_ivfpq_build") and "d_lists" in tiny.prod.last_error()
            assert (_host(tiny, d_o2, (6,), np.int32) == -7).all() and (_host(tiny, d_ids, (40,), np.int32) == -7).all()
            assert (_host(tiny, d_out, (40, 16), np.uint8) == 9).all()
        finally:
            _free(tiny, d_l, d_k, d_ids, d_out, d_o2)
    _free(tiny, d_o)


def test_build_past_2_32_bytes(tiny):
    """16.78 M rows of 256 codes (4.3 GB): the codes repeat a block of 4096 rows, row r's list is (r * 7) % 64"""
    M, P, Lc = 256, 4096, 64
    n = (1 << 32) // M + 5000
    L = tiny.prod.lib
    block = np.random.default_rng(8).integers(0, 256, (P, M), dtype=np.uint8)
    lists = ((np.arange(n, dtype=np.int64) * 7) % Lc).astype(np.int32)
    d_k, d_out = L.clip_b200_device_malloc(tiny.ctx, n * M), L.clip_b200_device_malloc(tiny.ctx, n * M)
    d_l, d_off, d_ids = _dev(tiny, lists), L.clip_b200_device_malloc(tiny.ctx, (Lc + 1) * 4), L.clip_b200_device_malloc(tiny.ctx, n * 4)
    try:
        assert d_k and d_out and d_ids
        for r0 in range(0, n, P):
            c = min(P, n - r0)
            assert L.clip_b200_memcpy_h2d(tiny.ctx, C.c_void_p(d_k + r0 * M), block.ctypes.data, c * M)
        assert L.clip_b200_ivfpq_build(tiny.ctx, d_l, d_k, n, Lc, M, d_off, d_ids, d_out), tiny.prod.last_error()
        want_off, want_ids = ivf_rule.layout(lists, Lc)
        assert np.array_equal(_host(tiny, d_off, (Lc + 1,), np.int32), want_off)
        ids = _host(tiny, d_ids, (n,), np.int32)
        assert np.array_equal(ids, want_ids)
        for p in (0, 1, n // 2, n - 2, n - 1, (1 << 32) // M - 1, (1 << 32) // M):    # byte 2^32 starts stored row 2^24
            a = np.empty(M, np.uint8)
            assert L.clip_b200_memcpy_d2h(tiny.ctx, a.ctypes.data, C.c_void_p(d_out + p * M), M)
            assert np.array_equal(a, block[ids[p] % P]), p
    finally:
        _free(tiny, d_k, d_out, d_l, d_off, d_ids)


# ---- 4. search against the rule ------------------------------------------------------------------------------------------------
def _check_search(m, ix, q, nprobe, k, rows=None, what=""):
    s, i = ix.search(q, nprobe, k)
    rows = np.arange(len(q)) if rows is None else rows
    cs, ci = search16(m, q[rows], _val(_cent_of(ix), ix.bf), nprobe, ix.in_type)
    ws, wi = rule.search(q[rows], ix.books, ix.codes, ix.lists, ci, cs, k)
    _assert_ranked(s[rows], i[rows], ws, wi.astype(np.int32), what)
    return s, i


def _cent_of(ix):
    return _val16(_host(ix.m, ix.d_c, (ix.L, ix.dim), np.uint16), ix.bf)


SEARCH = [  # M, dim, n_q, nprobe, top_k, in_type
    (16, 64, 100, 4, 10, F16), (32, 256, 8, 1, 1, BF16), (48, 768, 100, 8, 10, F16), (96, 768, 8, 64, 1024, BF16),
    (96, 768, 1, 1, 1024, F16), (128, 512, 20, 3, 100, BF16), (144, 1152, 8, 5, 10, F16), (160, 1280, 8, 3, 100, F16),
    (256, 2048, 1, 2, 10, BF16), (256, 256, 100, 16, 10, F16), (16, 2048, 8, 1000, 1, BF16)]


@pytest.mark.parametrize("M,dim,nq,nprobe,k,in_type", SEARCH)
def test_search_is_the_rule(tiny, M, dim, nq, nprobe, k, in_type):
    rng = np.random.default_rng(M * 7 + dim)
    bf = in_type == BF16
    db, cent = unit_rows(rng, 3000, dim, bf), unit_rows(rng, 24, dim, bf)
    ix = PqIndex(tiny, db, cent, _books(rng, M, dim, 0.05), in_type)
    try:
        s, _ = _check_search(tiny, ix, unit_rows(rng, nq, dim, bf), nprobe, k, what="M=%d dim=%d" % (M, dim))
        if nprobe == 1 and k == 1024:
            assert (s[:, -1] == -np.inf).all(), "the probed rows are fewer than w: padding"
    finally:
        ix.free()


@pytest.mark.parametrize("M,dim", [(96, 192), (160, 320), (256, 256)])
def test_search_units_span_tiles_and_compact(tiny, M, dim):
    """10^5 rows in 4 lists, 200 queries probing all of them: K13's units run thousands of rows, so a unit walks many 256-row tiles
    (m = 96: the table staged once per pair and reused; m = 160, 256: every slice re-staged each tile, the sums carried across) and its
    buffer is compacted, at top_k 1 and 10 after every tile and at 1024 once it passes 1152 entries.  The plan's row range R is
    asserted from the offsets: R = max(128, 128 * ceil(ceil(work / (4 * #SMs)) / 128)), work = sum over lists of ceil(pairs_l / 8) *
    rows_l (8 pairs a K13 unit), and with at most 132 SMs R is at least that value at 132."""
    rng = np.random.default_rng(M + dim)
    n, L, nq = 100_000, 4, 200
    db, cent = unit_rows(rng, n, dim, False), unit_rows(rng, L, dim, False)
    ix = PqIndex(tiny, db, cent, _books(rng, M, dim, 0.05), F16)
    try:
        sizes = np.diff(ix.layout()[0])
        work = int(sum(-(-nq // 8) * sz for sz in sizes if sz > 0))
        R = max(128, -(-(-(-work // (4 * 132))) // 128) * 128)
        assert R > 1152 + 256 and (sizes > R).all(), (R, sizes)
        q = unit_rows(rng, nq, dim, False)
        rows = np.arange(0, nq, 10)
        cs, ci = search16(tiny, q[rows], cent, L, F16)
        ws, wi = rule.search(q[rows], ix.books, ix.codes, ix.lists, ci, cs, 1024)    # the best 1024; a smaller top_k is its prefix
        for k in (1, 10, 1024):
            s, i = ix.search(q, L, k)
            _assert_ranked(s[rows], i[rows], ws[:, :k], wi[:, :k].astype(np.int32), "M=%d k=%d" % (M, k))
    finally:
        ix.free()


@pytest.mark.parametrize("M,nq", [(16, 3000), (256, 2500)])
def test_search_across_query_blocks(tiny, M, nq):
    """m = 256: blocks of 2^18 / 256 = 1024 queries; m = 16: one block (2^24 / (266 * 4) = 15 768)"""
    rng = np.random.default_rng(nq)
    db, cent = unit_rows(rng, 4000, 256, False), unit_rows(rng, 16, 256, False)
    ix = PqIndex(tiny, db, cent, _books(rng, M, 256, 0.05), F16)
    try:
        _check_search(tiny, ix, unit_rows(rng, nq, 256, False), 4, 10, rows=np.arange(0, nq, 37), what="n_q=%d" % nq)
    finally:
        ix.free()


@pytest.mark.parametrize("kind", ["skew", "empty", "dup", "nan"])
def test_search_skew_empty_ties_nan(tiny, kind):
    rng = np.random.default_rng(17)
    dim, L, M = 128, 32, 32
    db, cent = unit_rows(rng, 20_000, dim, False), unit_rows(rng, L, dim, False)
    if kind == "skew":                                   # about 90 % of the rows in one list: its row range is split
        db[:18_000] = _val(unit_rows(rng, 18_000, dim, False) * 0.3 + cent[0], False)
    if kind == "empty":
        cent[L // 2:] = cent[:L - L // 2]
    if kind == "dup":                                    # 200 distinct rows: equal codes and scores, ties by original index
        db = db[rng.integers(0, 200, len(db))]
    q = unit_rows(rng, 40, dim, False)
    if kind == "nan":
        db[[5, 700, 19_999], 3] = np.nan
        q[[2, 30], 100] = np.nan
    ix = PqIndex(tiny, db, cent, _books(rng, M, dim, 0.05), F16)
    try:
        off = ix.layout()[0]
        if kind == "skew":
            assert np.diff(off).max() >= 0.85 * len(db)
        for nprobe, k in ((L, 10), (3, 1024), (1, 100)):
            s, i = _check_search(tiny, ix, q, nprobe, k, what="%s nprobe=%d" % (kind, nprobe))
            if kind == "nan":
                assert (s[[2, 30]][s[[2, 30]] != -np.inf] == -FLT_MAX).all()
            if kind == "dup":
                tie = s[:, 1:] == s[:, :-1]
                assert tie.any() and (i[:, 1:][tie & (i[:, 1:] >= 0)] > i[:, :-1][tie & (i[:, 1:] >= 0)]).all()
    finally:
        ix.free()


# ---- 5. recall -----------------------------------------------------------------------------------------------------------------
def test_recall_with_rescore(tiny, capsys):
    """10^5 non-repeated rows of tools/bench_ivf.py's clustered data at dim 768, m = 96, n_lists = 256, nprobe = n_lists: recall@10
    of the PQ search's top 100 rescored exactly, against clip_b200_topk_search_16.  The floor is a sanity check set from the first
    H100 run, which measured 1.000 with the rescore (0.567 for PQ alone); the values are printed."""
    rng = np.random.default_rng(7)
    dim, L, M, n = 768, 256, 96, 100_000
    c = rng.standard_normal((4096, dim)).astype(np.float32)
    centres = c / np.linalg.norm(c, axis=1, keepdims=True)

    def clustered(k):
        v = centres[rng.integers(0, 4096, k)] + rng.standard_normal((k, dim)).astype(np.float32) * (0.6 / np.sqrt(dim))
        return _val((v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32), False)
    x, q = clustered(n), clustered(200)
    lib = tiny.prod.lib
    d_x = _dev(tiny, bits16(x, False))
    d_c = lib.clip_b200_device_malloc(tiny.ctx, L * dim * 2)
    try:
        assert lib.clip_b200_ivf_train_16(tiny.ctx, d_x, 20_000, dim, F16, L, 10, d_c), tiny.prod.last_error()
        cent = _val16(_host(tiny, d_c, (L, dim), np.uint16), False)
        books = pq_train(tiny, x[:20_000], cent, M, 10, F16)
        ix = PqIndex(tiny, x, cent, books, F16)
        try:
            _, i100 = ix.search(q, L, 100)
            _, truth = search16(tiny, q, x, 10, F16)
            s, i = np.zeros(200 * 10, np.float32), np.zeros(200 * 10, np.int32)
            d_q = _dev(tiny, bits16(q, False))
            cand = np.ascontiguousarray(i100, np.int32)
            ok = lib.clip_b200_topk_rescore(tiny.ctx, d_q, 200, d_x, n, dim, F16, cand.ctypes.data_as(IP), 100, 10, s.ctypes.data_as(FP),
                                            i.ctypes.data_as(IP))
            _free(tiny, d_q)
            assert ok, tiny.prod.last_error()
            i = i.reshape(200, 10)
            pq = np.mean([len(np.intersect1d(a, b)) / 10 for a, b in zip(i100[:, :10], truth)])
            rs = np.mean([len(np.intersect1d(a, b)) / 10 for a, b in zip(i, truth)])
            with capsys.disabled():
                print("\nIVF-PQ recall@10 (m = 96, nprobe = n_lists): PQ alone %.4f, PQ + rescore of 100 %.4f" % (pq, rs))
            assert rs >= 0.95, rs
        finally:
            ix.free()
    finally:
        _free(tiny, d_x, d_c)


# ---- 6. contract ---------------------------------------------------------------------------------------------------------------
def test_refusals_in_order_and_empty_calls(tiny):
    L = tiny.prod.lib
    ctx = tiny.ctx
    rng = np.random.default_rng(1)
    db = unit_rows(rng, 300, 32, False)
    ix = PqIndex(tiny, db, db[:4].copy(), _books(rng, 16, 32), F16)
    s, i = np.zeros(64, np.float32), np.zeros(64, np.int32)
    sp, ip = s.ctypes.data_as(FP), i.ctypes.data_as(IP)
    err = lambda: tiny.prod.last_error()
    d_q = _dev(tiny, bits16(db, False))
    try:
        def srch(**kw):
            a = dict(ctx=ctx, q=d_q, nq=2, dim=32, t=F16, c=ix.d_c, L=4, b=ix.d_b, m=16, off=ix.d_off, ids=ix.d_ids, k_=ix.d_codes, n=300,
                     npr=2, k=5, s=sp, i=ip)
            a.update(kw)
            return L.clip_b200_ivfpq_search_16(a["ctx"], a["q"], a["nq"], a["dim"], a["t"], a["c"], a["L"], a["b"], a["m"], a["off"],
                                               a["ids"], a["k_"], a["n"], a["npr"], a["k"], a["s"], a["i"])
        steps = [(dict(ctx=None), "null context"), (dict(t=0), "in_type"), (dict(dim=12), "dim"), (dict(m=24), "m must"),
                 (dict(L=0), "n_lists"), (dict(npr=1025), "nprobe"), (dict(k=0), "top_k"), (dict(nq=1 << 31), "2^31"),
                 (dict(k_=ix.d_codes + 8), "16-byte"), (dict(off=ix.d_off + 2), "4-byte"), (dict(s=None), "null output")]
        for j, (kw, msg) in enumerate(steps):
            bad = {}
            for kw2, _ in steps[j:]:
                bad.update(kw2)                          # this fault and every later one: the first is reported
            assert not srch(**bad)
            assert err().startswith("clip_b200_ivfpq_search_16") and msg in err(), (msg, err())
        assert not srch(m=48) and "divides dim" in err()
        assert not srch(m=272) and "m must" in err()
        assert srch(nq=0, q=None, s=None) and srch(n=0, k_=None, i=None)
        good = _host(tiny, ix.d_off, (5,), np.int32)
        L.clip_b200_memcpy_h2d(ctx, ix.d_off, np.array([0, 5, 3, 200, 300], np.int32).ctypes.data, 20)
        assert not srch() and "d_offsets" in err()
        L.clip_b200_memcpy_h2d(ctx, ix.d_off, good.ctypes.data, 20)
        assert srch()
        # train: its own steps
        tr = lambda **kw: L.clip_b200_ivfpq_train_16(*[dict(dict(ctx=ctx, x=d_q, n=300, dim=32, t=F16, c=ix.d_c, L=4, m=16, it=2, b=ix.d_b), **kw)[k]
                                                       for k in ("ctx", "x", "n", "dim", "t", "c", "L", "m", "it", "b")])
        for kw, msg in ((dict(t=3, m=5), "in_type"), (dict(m=5, L=0), "m must"), (dict(L=0, it=0), "n_lists"), (dict(it=0), "n_iter"),
                        (dict(n=1 << 31, b=None), "n_train must be below"), (dict(n=255, b=None), "at least 256"), (dict(b=None), "16-byte")):
            assert not tr(**kw) and err().startswith("clip_b200_ivfpq_train_16") and msg in err(), (msg, err())
        # encode and build
        d_l, d_k = L.clip_b200_device_malloc(ctx, 300 * 4), L.clip_b200_device_malloc(ctx, 300 * 16)
        assert not L.clip_b200_ivfpq_encode_16(ctx, d_q, 300, 32, F16, ix.d_c, 4, ix.d_b, 16, None, d_k) and "4-byte" in err()
        assert err().startswith("clip_b200_ivfpq_encode_16")
        assert L.clip_b200_ivfpq_encode_16(ctx, None, 0, 32, F16, None, 4, None, 16, None, None), err()
        assert not L.clip_b200_ivfpq_build(ctx, d_l, d_k, 300, 4, 8, ix.d_off, ix.d_ids, ix.d_codes) and "m must" in err()
        assert not L.clip_b200_ivfpq_build(ctx, d_l, d_k, 300, 4, 16, ix.d_off, None, ix.d_codes) and "4-byte" in err()
        assert err().startswith("clip_b200_ivfpq_build")
        _free(tiny, d_l, d_k)
    finally:
        _free(tiny, d_q)
        ix.free()
