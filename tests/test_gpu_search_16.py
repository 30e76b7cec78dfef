"""clip_b200_topk_search_16 (K10, csrc/search.cu) and clip_b200_rows_to_16bit, called through prod.lib.

- Exact data: _tie_case's integer inputs scaled by 2^-3 are exact in f16 and bf16 and every dot product is exact in any order,
  so the 16-bit search must return what clip_b200_topk_search returns on the same values, byte for byte, across K10's tile (128
  rows), partition and candidate-buffer edges and the fp32 path's slice edges.
- Random unit rows: every score within the bound of tests/_search_bound.py, and no row left out that could beat a returned one.
- Scores depend on the query and the row alone; the contract's edges and guards; refusals and empty calls through the table of
  tests/test_gpu_search_forms.py.
- rows_to_16bit equals numpy's round-to-nearest-even, including a call with n * dim > 2^32."""
import ctypes as C
import functools

import numpy as np
import pytest

from _search_bound import bits16, bound, exact, unit_rows
from test_gpu_scoring_exact import GUARD, _Model, _assert_ranked, _tie_case, _tie_ints
import test_gpu_search_forms as forms

FLT_MAX = np.finfo(np.float32).max
F16, BF16 = 1, 2


@pytest.fixture(scope="module")
def tiny(prod):
    m = _Model(prod, "tiny", "f16")                    # projection dim 128: the fp32 path's d
    yield m
    prod.free(m.ctx)


def _dev(m, a):
    p = m.prod.lib.clip_b200_device_malloc(m.ctx, max(a.nbytes, 16))
    assert p and m.prod.lib.clip_b200_memcpy_h2d(m.ctx, p, a.ctypes.data, a.nbytes), m.prod.last_error()
    return p


def search16(m, q, db, top_k, in_type=F16, expect_ok=True):
    """q [n_q, dim], db [n_db, dim] float32 values (rounded to in_type on the host) -> (scores, indices) [n_q, w], w = min(top_k,
    n_db).  The output runs GUARD entries further, and those must come back untouched."""
    bf = in_type == BF16
    q16, db16 = bits16(q, bf), bits16(db, bf)
    nq, n, dim = len(q), len(db), q.shape[1]
    w = min(top_k, n)
    scores = np.full(nq * w + GUARD, 7.0, np.float32)
    idx = np.full(nq * w + GUARD, -7, np.int32)
    L = m.prod.lib
    d_q, d_db = _dev(m, q16), _dev(m, db16)
    try:
        ok = L.clip_b200_topk_search_16(m.ctx, d_q, nq, d_db, n, dim, in_type, top_k, scores.ctypes.data_as(C.POINTER(C.c_float)),
                                        idx.ctypes.data_as(C.POINTER(C.c_int)))
    finally:
        L.clip_b200_device_free(m.ctx, d_q)
        L.clip_b200_device_free(m.ctx, d_db)
    assert ok == expect_ok, m.prod.last_error()
    assert (scores[nq * w:] == 7.0).all() and (idx[nq * w:] == -7).all(), "written past n_q * top_k"
    return scores[:nq * w].reshape(nq, w), idx[:nq * w].reshape(nq, w)


# ---- a. byte-identical to the fp32 path on exact data -----------------------------------------------------------------------
# n_q = 1: 132 partitions of whole 128-row tiles; 3: 132 for one query tile of 8; 300: three tiles of 128, 44 partitions each.  n_db
# covers one ragged tile, one tile, one row past it, several tiles in few partitions, and the fp32 path's 4096 / 8192 / 131 072
# edges.  k = 1024 over 140 000 rows runs through the candidate-buffer compaction many times.
EXACT_CASES = ([(1, n) for n in (1, 127, 128, 129, 1000, 16_897, 140_000)] + [(3, n) for n in (4096, 4097, 8192, 8193)]
               + [(300, 140_000)])


@pytest.mark.gpu
@pytest.mark.parametrize("nq,ndb", EXACT_CASES)
@pytest.mark.parametrize("in_type", [F16, BF16])
def test_exact_data_matches_fp32_search(tiny, nq, ndb, in_type):
    q, db, want_s, want_i = _tie_case(nq, ndb, tiny.d)
    for k in (1, 7, 100, 1024):
        s, i = search16(tiny, q, db, k, in_type)
        w = min(k, ndb)
        _assert_ranked(s, i, want_s[:, :w], want_i[:, :w], "16-bit top-%d of %d x %d" % (k, nq, ndb))
        if ndb <= 8193 or k in (7, 1024):              # the fp32 path itself, byte for byte
            s32, i32 = tiny.run("search", q, db, k)
            _assert_ranked(s, i, s32, i32.astype(np.int32), "against clip_b200_topk_search, k=%d" % k)


# ---- b. random unit rows: bound and ranking ---------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dim", [8, 40, 128, 768, 2048])
@pytest.mark.parametrize("in_type", [F16, BF16])
def test_random_rows_within_bound(tiny, dim, in_type):
    bf = in_type == BF16
    rng = np.random.default_rng(dim * 3 + in_type)
    q, db = unit_rows(rng, 9, dim, bf), unit_rows(rng, 3000, dim, bf)
    db[100:104] = q[:4]                                # a few near-1 scores among near-0 ones
    ex, b = exact(q, db), bound(q, db)
    k = 100
    s, i = search16(tiny, q, db, k, in_type)
    rows = np.arange(len(q))[:, None]
    err = np.abs(s.astype(np.float64) - ex[rows, i])
    assert (err <= b[rows, i]).all(), "max error / bound %.3f" % (err / b[rows, i]).max()
    for r in range(len(q)):
        out = np.setdiff1d(np.arange(len(db)), i[r])
        worst_in = (ex[r, i[r]] + b[r, i[r]]).min()
        best_out = (ex[r, out] - b[r, out]).max()
        assert best_out <= worst_in, (r, best_out, worst_in)
        assert (np.diff(s[r]) <= 0).all()
        tie = s[r, 1:] == s[r, :-1]
        assert (i[r, 1:][tie] > i[r, :-1][tie]).all()


# ---- c. determinism ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("in_type", [F16, BF16])
def test_scores_depend_on_query_and_row_only(tiny, in_type):
    rng = np.random.default_rng(17)
    bf = in_type == BF16
    q, db = unit_rows(rng, 5, 768, bf), unit_rows(rng, 1000, 768, bf)
    a = search16(tiny, q, db, 1000, in_type)
    b = search16(tiny, q, db, 1000, in_type)
    assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1])
    full = np.empty((5, 1000), np.float32)
    np.put_along_axis(full, a[1], a[0], 1)
    assert (np.sort(a[1], 1) == np.arange(1000)).all()
    for s0 in (1, 63, 64, 65, 127):
        s, i = search16(tiny, q, db[s0:], 1000, in_type)
        got = np.empty((5, 1000 - s0), np.float32)
        np.put_along_axis(got, i, s, 1)
        assert np.array_equal(got.view(np.uint32), full[:, s0:].view(np.uint32)), s0


# ---- d. contract edges ------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _edge_case(nq, ndb, d):
    qi, dbi = _tie_ints(nq, ndb, d, seed=nq)
    return (qi * 2.0 ** -3).astype(np.float32), (dbi * 2.0 ** -3).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("nq", [1, 7, 8, 9, 127, 128, 129, 255, 256, 257, 40_000])
def test_query_counts_match_fp32_search(tiny, nq):
    q, db = _edge_case(nq, 700, tiny.d)
    for k in (5, 700, 1024):                           # 1024 > n_db means n_db
        s, i = search16(tiny, q, db, k)
        s32, i32 = tiny.run("search", q, db, min(k, 700))
        _assert_ranked(s, i, s32, i32.astype(np.int32), "n_q=%d top-%d" % (nq, k))


@pytest.mark.gpu
def test_nan_ranks_last_as_minus_flt_max(tiny):
    q, db = _edge_case(4, 5000, tiny.d)
    db = db.copy()
    nan_rows = [17, 2500, 4095, 4096, 4999]
    db[nan_rows, 5] = np.nan
    s, i = search16(tiny, q, db, 1024)
    ex = exact(q, np.nan_to_num(db, nan=0.0))
    ex[:, nan_rows] = -np.inf
    order = np.argsort(-ex, axis=1, kind="stable")[:, :1024]
    want = np.take_along_axis(ex, order, 1)
    want[np.isinf(want)] = -FLT_MAX
    _assert_ranked(s, i, want.astype(np.float32), order.astype(np.int32), "NaN rows")
    s, i = search16(tiny, q[:1], db[15:20], 5)          # every row returned: row 2 (17) is NaN and comes last as -FLT_MAX
    assert i[0, -1] == 2 and s[0, -1] == -FLT_MAX


@pytest.mark.gpu
def test_refusals_and_empty_calls(prod):
    """refusals, their order and empty calls: the table of the search forms (tests/test_gpu_search_forms.py) for this form"""
    forms.check_form(prod, "clip_b200_topk_search_16")


# ---- e. rows_to_16bit -------------------------------------------------------------------------------------------------------
def _rows16(m, x, out_type):
    n, dim = x.shape
    d_x = _dev(m, np.ascontiguousarray(x, np.float32))
    d_o = m.prod.lib.clip_b200_device_malloc(m.ctx, n * dim * 2)
    try:
        assert m.prod.lib.clip_b200_rows_to_16bit(m.ctx, d_x, n, dim, out_type, d_o), m.prod.last_error()
        out = np.empty((n, dim), np.uint16)
        assert m.prod.lib.clip_b200_memcpy_d2h(m.ctx, out.ctypes.data, d_o, out.nbytes)
    finally:
        m.prod.lib.clip_b200_device_free(m.ctx, d_x)
        m.prod.lib.clip_b200_device_free(m.ctx, d_o)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("out_type", [F16, BF16])
def test_rows_to_16bit_is_rne(tiny, out_type):
    rng = np.random.default_rng(out_type)
    x = (rng.standard_normal((333, 768)) * 2.0 ** rng.integers(-30, 30, (333, 768))).astype(np.float32)
    # values on and next to a rounding tie of either type
    t = rng.integers(0, 1 << 20, 5000).astype(np.uint32)
    ties = np.array([0x3F808000, 0x3F818000, 0x3F801000, 0x3F803000], np.uint32)
    x.reshape(-1)[:5004] = np.concatenate([np.uint32(0x3F800000) | (t << np.uint32(3)), ties]).view(np.float32)
    got = _rows16(tiny, x, out_type)
    assert np.array_equal(got, bits16(x, out_type == BF16))


@pytest.mark.gpu
def test_rows_to_16bit_past_2_32_elements(tiny):
    """2^21 + 3 rows of 2048: 4.3e9 elements, the last rows lie past element 2^32"""
    L, ctx = tiny.prod.lib, tiny.ctx
    dim, n = 2048, (1 << 21) + 3
    rng = np.random.default_rng(1)
    blk = rng.standard_normal((8192, dim)).astype(np.float32)          # 64 MB, copied over the whole source
    src = L.clip_b200_device_malloc(ctx, n * dim * 4)
    dst = L.clip_b200_device_malloc(ctx, n * dim * 2)
    assert src and dst, tiny.prod.last_error()
    try:
        for r0 in range(0, n, len(blk)):
            r = min(len(blk), n - r0)
            assert L.clip_b200_memcpy_h2d(ctx, src + r0 * dim * 4, blk.ctypes.data, r * dim * 4)
        for out_type in (F16, BF16):
            assert L.clip_b200_rows_to_16bit(ctx, src, n, dim, out_type, dst), tiny.prod.last_error()
            for r0 in (0, (1 << 21) - 2, n - 5):
                got = np.empty((5, dim), np.uint16)
                assert L.clip_b200_memcpy_d2h(ctx, got.ctypes.data, dst + r0 * dim * 2, got.nbytes)
                want = bits16(blk[[(r0 + j) % len(blk) for j in range(5)]], out_type == BF16)
                assert np.array_equal(got, want), (out_type, r0)
    finally:
        L.clip_b200_device_free(ctx, src)
        L.clip_b200_device_free(ctx, dst)
