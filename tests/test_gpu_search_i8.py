"""clip_b200_rows_to_int8 and clip_b200_topk_search_i8 (K10's s8 instance, csrc/search.cu), called through prod.lib, against the
rule of tests/_search_i8.py.

- rows_to_int8 equals the numpy quantiser bit for bit, codes and scales, including a call with n * dim > 2^32.
- Exact data: _tie_ints' integers taken as codes with every scale 2^-3 make every score acc * 2^-6, exact, so the search must return
  _tie_case's ranking and what clip_b200_topk_search returns on the same values, byte for byte.
- Random unit rows quantised on the GPU: scores and indices equal the numpy emulation and ranking bit for bit; every score lies
  within the bound of the f32 dot product, and no row left out could beat a returned one.
- Scores depend on the query and the row alone; non-finite rows and queries rank last; refusals, empty calls and output guards
  (the refusals through the table of tests/test_gpu_search_forms.py); a database past 2^32 bytes."""
import ctypes as C

import numpy as np
import pytest

from _search_i8 import FLT_MAX, bound, emulate, exact, quantize, rank, unit_rows
from test_gpu_scoring_exact import GUARD, _Model, _assert_ranked, _tie_case, _tie_ints
from test_gpu_search_16 import EXACT_CASES, _dev
import test_gpu_search_forms as forms


@pytest.fixture(scope="module")
def tiny(prod):
    m = _Model(prod, "tiny", "f16")                    # projection dim 128: the fp32 path's d
    yield m
    prod.free(m.ctx)


def _free(m, *ps):
    for p in ps:
        m.prod.lib.clip_b200_device_free(m.ctx, p)


def search_i8(m, qc, qs, xc, xs, top_k, expect_ok=True):
    """codes and scales of the queries [n_q, dim], [n_q] and of the database [n_db, dim], [n_db] -> (scores, indices) [n_q, w],
    w = min(top_k, n_db).  The output runs GUARD entries further, and those must come back untouched."""
    qc, xc = np.ascontiguousarray(qc, np.int8), np.ascontiguousarray(xc, np.int8)
    qs, xs = np.ascontiguousarray(qs, np.float32), np.ascontiguousarray(xs, np.float32)
    nq, n, dim = len(qc), len(xc), qc.shape[1]
    w = min(top_k, n)
    scores = np.full(nq * w + GUARD, 7.0, np.float32)
    idx = np.full(nq * w + GUARD, -7, np.int32)
    L = m.prod.lib
    ptrs = [_dev(m, a) for a in (qc, qs, xc, xs)]
    try:
        ok = L.clip_b200_topk_search_i8(m.ctx, ptrs[0], ptrs[1], nq, ptrs[2], ptrs[3], n, dim, top_k,
                                        scores.ctypes.data_as(C.POINTER(C.c_float)), idx.ctypes.data_as(C.POINTER(C.c_int)))
    finally:
        _free(m, *ptrs)
    assert ok == expect_ok, m.prod.last_error()
    assert (scores[nq * w:] == 7.0).all() and (idx[nq * w:] == -7).all(), "written past n_q * top_k"
    return scores[:nq * w].reshape(nq, w), idx[:nq * w].reshape(nq, w)


def q8(m, x):
    """clip_b200_rows_to_int8 of float32 rows [n, dim] -> (codes, scales) on the host"""
    x = np.ascontiguousarray(x, np.float32)
    n, dim = x.shape
    L = m.prod.lib
    d_x = _dev(m, x)
    d_c, d_s = L.clip_b200_device_malloc(m.ctx, max(n * dim, 16)), L.clip_b200_device_malloc(m.ctx, max(4 * n, 16))
    try:
        assert L.clip_b200_rows_to_int8(m.ctx, d_x, n, dim, d_c, d_s), m.prod.last_error()
        c, s = np.empty((n, dim), np.int8), np.empty(n, np.float32)
        assert L.clip_b200_memcpy_d2h(m.ctx, c.ctypes.data, d_c, c.nbytes) and L.clip_b200_memcpy_d2h(m.ctx, s.ctypes.data, d_s, s.nbytes)
    finally:
        _free(m, d_x, d_c, d_s)
    return c, s


def _assert_q8(got, want, what):
    (gc, gs), (wc, ws) = got, want
    bad = np.nonzero((gc != wc).any(1) | (gs.view(np.uint32) != ws.view(np.uint32)))[0]
    assert not len(bad), "%s: %d rows differ, first %d: scale %r / %r" % (what, len(bad), bad[0], gs[bad[0]], ws[bad[0]])


# ---- 1. rows_to_int8 bit for bit ----------------------------------------------------------------------------------------------
def _hard_rows(rng, n, dim):
    """magnitudes over 2^+-30, exact half-way quotients, zero rows, subnormal maxima, NaN / +Inf / -Inf rows"""
    x = (rng.standard_normal((n, dim)) * 2.0 ** rng.integers(-30, 31, (n, 1)) * 2.0 ** rng.integers(-6, 1, (n, dim))).astype(np.float32)
    h = n // 8                                           # rows h .. 2h: every quotient a tie (s = 2^e exactly)
    e = rng.integers(-30, 30, h)
    x[h:2 * h] = ((rng.integers(-127, 127, (h, dim)) + 0.5) * 2.0 ** e[:, None]).astype(np.float32)
    x[h:2 * h, 0] = (127 * 2.0 ** e).astype(np.float32)
    x[2 * h:2 * h + 3] = 0
    e = rng.integers(-149, -117, h)                     # rows 3h .. 4h: maxima 2^-149 .. 2^-118, s subnormal or 0
    x[3 * h:4 * h] = (rng.uniform(-1, 1, (h, dim)) * 2.0 ** e[:, None]).astype(np.float32)
    x[3 * h + np.arange(h), rng.integers(0, dim, h)] = (2.0 ** e).astype(np.float32)
    for j, v in enumerate((np.nan, np.inf, -np.inf, np.nan)):
        x[5 * h + j, rng.integers(0, dim)] = v
    x[5 * h + 3, :] = np.nan
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [16, 48, 144, 768, 2032, 2048])
def test_rows_to_int8_matches_rule(tiny, dim):
    rng = np.random.default_rng(dim)
    x = _hard_rows(rng, 400, dim)
    want = quantize(x)
    assert (want[1] == 0).sum() >= 3 and np.isnan(want[1]).sum() == 4 and (want[1][150:200] < np.finfo(np.float32).tiny).any()
    _assert_q8(q8(tiny, x), want, "dim %d" % dim)
    for n in (1, 7, 9):                                  # partial blocks of eight rows
        _assert_q8(q8(tiny, x[:n]), quantize(x[:n]), "dim %d n %d" % (dim, n))


@pytest.mark.gpu
def test_rows_to_int8_refusals(prod):
    """refusals, their order and empty calls: the table of the search forms (tests/test_gpu_search_forms.py) for this form"""
    forms.check_form(prod, "clip_b200_rows_to_int8")


@pytest.mark.gpu
def test_rows_to_int8_past_2_32_elements(tiny):
    """2^21 + 3 rows of 2048: 4.3e9 elements, the rows from 2^21 on lie past element 2^32"""
    L, ctx = tiny.prod.lib, tiny.ctx
    dim, n = 2048, (1 << 21) + 3
    rng = np.random.default_rng(1)
    blk = (rng.standard_normal((8192, dim)) * 2.0 ** rng.integers(-8, 8, (8192, 1))).astype(np.float32)
    src = L.clip_b200_device_malloc(ctx, n * dim * 4)
    codes = L.clip_b200_device_malloc(ctx, n * dim)
    scales = L.clip_b200_device_malloc(ctx, n * 4)
    assert src and codes and scales, tiny.prod.last_error()
    try:
        for r0 in range(0, n, len(blk)):
            r = min(len(blk), n - r0)
            assert L.clip_b200_memcpy_h2d(ctx, src + r0 * dim * 4, blk.ctypes.data, r * dim * 4)
        assert L.clip_b200_rows_to_int8(ctx, src, n, dim, codes, scales), tiny.prod.last_error()
        for r0 in (0, (1 << 21) - 2, n - 5):
            c, s = np.empty((5, dim), np.int8), np.empty(5, np.float32)
            assert L.clip_b200_memcpy_d2h(ctx, c.ctypes.data, codes + r0 * dim, c.nbytes)
            assert L.clip_b200_memcpy_d2h(ctx, s.ctypes.data, scales + r0 * 4, s.nbytes)
            _assert_q8((c, s), quantize(blk[[(r0 + j) % len(blk) for j in range(5)]]), "rows from %d" % r0)
    finally:
        _free(tiny, src, codes, scales)


# ---- 2. exact data against the 16-bit and fp32 searches --------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("nq,ndb", EXACT_CASES)
def test_exact_data_matches_fp32_search(tiny, nq, ndb):
    q, db, want_s, want_i = _tie_case(nq, ndb, tiny.d)
    qi, dbi = _tie_ints(nq, ndb, tiny.d)
    qs, xs = np.full(nq, 2.0 ** -3, np.float32), np.full(ndb, 2.0 ** -3, np.float32)
    for k in (1, 7, 100, 1024):
        s, i = search_i8(tiny, qi, qs, dbi, xs, k)
        w = min(k, ndb)
        _assert_ranked(s, i, want_s[:, :w], want_i[:, :w], "int8 top-%d of %d x %d" % (k, nq, ndb))
        if ndb <= 8193 or k in (7, 1024):              # the fp32 path itself, byte for byte
            s32, i32 = tiny.run("search", q, db, k)
            _assert_ranked(s, i, s32, i32.astype(np.int32), "against clip_b200_topk_search, k=%d" % k)


# ---- 3. random rows: the emulation bit for bit ------------------------------------------------------------------------------
def _random_case(seed, nq, ndb, dim):
    rng = np.random.default_rng(seed)
    q, db = unit_rows(rng, nq, dim), unit_rows(rng, ndb, dim)
    db[100:104] = q[:4]                                # a few near-1 scores among near-0 ones
    db[ndb - 40:ndb - 20] = db[10:30]                  # exact ties, settled by the index
    return q, db


def _check_emulation(m, q, db, ks):
    qc, qs = q8(m, q)
    xc, xs = q8(m, db)
    _assert_q8((qc, qs), quantize(q), "queries")
    _assert_q8((xc, xs), quantize(db), "rows")
    em = emulate(qc, qs, xc, xs)
    for k in ks:
        s, i = search_i8(m, qc, qs, xc, xs, k)
        ws, wi = rank(em, min(k, len(db)))
        _assert_ranked(s, i, ws, wi, "top-%d of %d x %d, dim %d" % (k, len(q), len(db), q.shape[1]))
    return qc, qs, xc, xs


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [16, 48, 128, 768, 2048])
def test_random_rows_match_emulation(tiny, dim):
    q, db = _random_case(dim, 129, 3000, dim)
    _check_emulation(tiny, q, db, (1, 100, 1024))


@pytest.mark.gpu
@pytest.mark.parametrize("nq", [1, 7, 8, 9, 127, 128, 129, 257, 40_000])
def test_query_counts_match_emulation(tiny, nq):
    q, db = _random_case(nq, nq, 700, 48)
    _check_emulation(tiny, q, db, (5, 700, 1024))      # 1024 > n_db means n_db


# ---- 4. bound and recall ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dim", [16, 128, 768, 2048])
def test_random_rows_within_bound(tiny, dim):
    q, db = _random_case(dim + 1, 9, 3000, dim)
    qc, qs = q8(tiny, q)
    xc, xs = q8(tiny, db)
    k = 100
    s, i = search_i8(tiny, qc, qs, xc, xs, k)
    ex = exact(q, db)
    b = bound(q, qs, db, xs, emulate(qc, qs, xc, xs))
    rows = np.arange(len(q))[:, None]
    err = np.abs(s.astype(np.float64) - ex[rows, i])
    assert (err <= b[rows, i]).all(), "max error / bound %.3f" % (err / b[rows, i]).max()
    for r in range(len(q)):
        out = np.setdiff1d(np.arange(len(db)), i[r])
        worst_in = (ex[r, i[r]] + b[r, i[r]]).min()
        best_out = (ex[r, out] - b[r, out]).max()
        assert best_out <= worst_in, (r, best_out, worst_in)


# ---- 5. determinism ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_scores_depend_on_query_and_row_only(tiny):
    q, db = _random_case(17, 5, 1000, 768)
    qc, qs = q8(tiny, q)
    xc, xs = q8(tiny, db)
    a = search_i8(tiny, qc, qs, xc, xs, 1000)
    b = search_i8(tiny, qc, qs, xc, xs, 1000)
    assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1])
    assert (np.sort(a[1], 1) == np.arange(1000)).all()
    full = np.empty((5, 1000), np.float32)
    np.put_along_axis(full, a[1], a[0], 1)
    for s0 in (1, 63, 64, 65, 127):
        s, i = search_i8(tiny, qc, qs, xc[s0:], xs[s0:], 1000)
        got = np.empty((5, 1000 - s0), np.float32)
        np.put_along_axis(got, i, s, 1)
        assert np.array_equal(got.view(np.uint32), full[:, s0:].view(np.uint32)), s0


# ---- 6. non-finite rows and queries -----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_non_finite_rows_and_queries_rank_last(tiny):
    q, db = _random_case(23, 4, 5000, 128)
    bad_rows = {17: np.nan, 2500: np.inf, 4095: -np.inf, 4096: np.nan, 4999: np.inf}
    for r, v in bad_rows.items():
        db[r, 5] = v
    q[3, 7] = -np.inf                                   # every score of query 3 is NaN
    qc, qs = q8(tiny, q)
    xc, xs = q8(tiny, db)
    assert np.isnan(xs[list(bad_rows)]).all() and np.isnan(qs[3])
    s, i = search_i8(tiny, qc, qs, xc, xs, 1024)
    ws, wi = rank(emulate(qc, qs, xc, xs), 1024)
    _assert_ranked(s, i, ws, wi, "non-finite rows")
    assert (s[3] == -FLT_MAX).all() and np.array_equal(i[3], np.arange(1024))
    s, i = search_i8(tiny, qc[:1], qs[:1], xc[15:20], xs[15:20], 5)   # row 2 (17) is NaN and comes last as -FLT_MAX
    assert i[0, -1] == 2 and s[0, -1] == -FLT_MAX
    s, i = search_i8(tiny, qc[:3], qs[:3], xc[4094:4098], xs[4094:4098], 4)
    assert (i[:, 2:] == [1, 2]).all() and (s[:, 2:] == -FLT_MAX).all()


# ---- 7. refusals, empty calls, guards ---------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refusals_and_empty_calls(prod):
    """refusals, their order and empty calls: the table of the search forms (tests/test_gpu_search_forms.py) for this form"""
    forms.check_form(prod, "clip_b200_topk_search_i8")


# ---- 8. a database past 2^32 bytes ------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_database_past_2_32_bytes(tiny):
    """2^22 + 5 rows of 1024: codes past byte 2^32 from row 2^22 on.  Queries 0, 1 and 2 are planted at rows 2^22 - 1, 2^22 and
    the last row; everything else repeats a block of 8192 random unit rows."""
    L, ctx = tiny.prod.lib, tiny.ctx
    dim, n, B = 1024, (1 << 22) + 5, 8192
    rng = np.random.default_rng(9)
    blk = unit_rows(rng, B, dim)
    q = unit_rows(rng, 3, dim)
    plant = [(1 << 22) - 1, 1 << 22, n - 1]
    d_blk = _dev(tiny, blk)
    codes, scales = L.clip_b200_device_malloc(ctx, n * dim), L.clip_b200_device_malloc(ctx, n * 4)
    assert codes and scales, tiny.prod.last_error()
    try:
        for r0 in range(0, n, B):
            assert L.clip_b200_rows_to_int8(ctx, d_blk, min(B, n - r0), dim, codes + r0 * dim, scales + r0 * 4), tiny.prod.last_error()
        qc, qs = quantize(q)
        for j, r in enumerate(plant):
            assert L.clip_b200_memcpy_h2d(ctx, codes + r * dim, qc[j].ctypes.data, dim)
            assert L.clip_b200_memcpy_h2d(ctx, scales + r * 4, qs[j:j + 1].ctypes.data, 4)
        d_qc, d_qs = _dev(tiny, qc), _dev(tiny, qs)
        k = 4
        sc, ix = np.full(3 * k + GUARD, 7.0, np.float32), np.full(3 * k + GUARD, -7, np.int32)
        try:
            assert L.clip_b200_topk_search_i8(ctx, d_qc, d_qs, 3, codes, scales, n, dim, k, sc.ctypes.data_as(C.POINTER(C.c_float)),
                                              ix.ctypes.data_as(C.POINTER(C.c_int))), tiny.prod.last_error()
        finally:
            _free(tiny, d_qc, d_qs)
        assert (sc[3 * k:] == 7.0).all() and (ix[3 * k:] == -7).all()
        sc, ix = sc[:3 * k].reshape(3, k), ix[:3 * k].reshape(3, k)
        bc, bs = quantize(blk)
        eb = emulate(qc, qs, bc, bs)                    # the block's rows, each repeated every B rows from row 0
        eq = emulate(qc, qs, qc, qs)                    # query j against the planted rows
        for j in range(3):
            best = int(np.argmax(eb[j]))
            assert (eb[j] == eb[j, best]).sum() == 1 and eb[j, best] > np.delete(eq[j], j).max()
            assert ix[j, 0] == plant[j] and sc[j, 0].view(np.uint32) == eq[j, j].view(np.uint32), (j, ix[j], sc[j])
            assert list(ix[j, 1:]) == [best, best + B, best + 2 * B] and (sc[j, 1:] == eb[j, best]).all(), (j, ix[j], sc[j])
    finally:
        _free(tiny, d_blk, codes, scales)
