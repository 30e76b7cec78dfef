"""clip_b200_rows_to_binary, clip_b200_topk_search_b1 (K11) and clip_b200_topk_rescore (K12), called through prod.lib, against the
rule of tests/_search_b1.py, byte for byte, no tolerance.

- rows_to_binary at every dim from 128 to 2048, with and without a centre, on zeros, -0, subnormals, NaN and +-Inf; one call past
  2^32 source elements.
- search_b1 on random, low-entropy and all-identical databases at tile and partition edges, n_q from 1 to 32 769, top_k from 1 to
  1024 and above n_db; the same answer as clip_b200_topk_search on the +-1 rows in f32; a score depends on its pair alone; a
  database past 2^32 bytes.
- rescore: every row as candidates equals clip_b200_topk_search; random subsets equal the rule; 16-bit rows equal the f32 call on
  the widened rows; duplicates, -1, INT_MAX, short lists, NaN rows and output guards.
- The binary search then the rescore equals the exact search wherever the shortlist holds the exact top 10.
- Refusals in the documented order, two faults reporting the first, empty calls."""
import ctypes as C

import numpy as np
import pytest

import _search_b1 as rule
from test_gpu_scoring_exact import GUARD, _Model, _assert_ranked
from test_gpu_search_16 import _dev

pytestmark = pytest.mark.gpu
F32, F16, BF16 = 0, 1, 2
FP, IP = C.POINTER(C.c_float), C.POINTER(C.c_int)
INT_MAX = 2147483647


@pytest.fixture(scope="module")
def tiny(prod):
    m = _Model(prod, "tiny", "f16")                    # projection dim 128: clip_b200_topk_search's d
    yield m
    prod.free(m.ctx)


def _free(m, *ps):
    for p in ps:
        m.prod.lib.clip_b200_device_free(m.ctx, p)


def _host(m, p, shape, dtype):
    a = np.empty(shape, dtype)
    assert m.prod.lib.clip_b200_memcpy_d2h(m.ctx, a.ctypes.data, p, a.nbytes), m.prod.last_error()
    return a


def to_bits(m, x, center=None):
    x = np.ascontiguousarray(x, np.float32)
    n, dim = x.shape
    d_x = _dev(m, x)
    d_c = _dev(m, np.ascontiguousarray(center, np.float32)) if center is not None else None
    d_b = m.prod.lib.clip_b200_device_malloc(m.ctx, max(n * dim // 8, 16))
    try:
        assert m.prod.lib.clip_b200_rows_to_binary(m.ctx, d_x, n, dim, d_c, d_b), m.prod.last_error()
        return _host(m, d_b, (n, dim // 8), np.uint8)
    finally:
        _free(m, d_x, d_b, *([d_c] if d_c else []))


def _out(nq, w):
    return np.full(nq * w + GUARD, 7.0, np.float32), np.full(nq * w + GUARD, -7, np.int32)


def _unguard(s, i, nq, w):
    assert (s[nq * w:] == 7.0).all() and (i[nq * w:] == -7).all(), "written past n_q * top_k"
    return s[:nq * w].reshape(nq, w), i[:nq * w].reshape(nq, w)


def search_b1_dev(m, d_q, nq, d_x, n, dim, top_k):
    w = min(top_k, n)
    s, i = _out(nq, w)
    assert m.prod.lib.clip_b200_topk_search_b1(m.ctx, d_q, nq, d_x, n, dim, top_k, s.ctypes.data_as(FP), i.ctypes.data_as(IP)), \
        m.prod.last_error()
    return _unguard(s, i, nq, w)


def search_b1(m, qb, xb, dim, top_k):
    qb, xb = np.ascontiguousarray(qb, np.uint8), np.ascontiguousarray(xb, np.uint8)
    d_q, d_x = _dev(m, qb), _dev(m, xb)
    try:
        return search_b1_dev(m, d_q, len(qb), d_x, len(xb), dim, top_k)
    finally:
        _free(m, d_q, d_x)


def rescore(m, q, db, cand, top_k, in_type=F32):
    """q, db as arrays of the element type (float32, or uint16 bit patterns for 16-bit) -> (scores, indices) [n_q, top_k]"""
    q, db, cand = np.ascontiguousarray(q), np.ascontiguousarray(db), np.ascontiguousarray(cand, np.int32)
    nq, n, dim = len(q), len(db), q.shape[1]
    s, i = _out(nq, top_k)
    d_q, d_x = _dev(m, q), _dev(m, db)
    try:
        assert m.prod.lib.clip_b200_topk_rescore(m.ctx, d_q, nq, d_x, n, dim, in_type, cand.ctypes.data_as(IP), cand.shape[1], top_k,
                                                 s.ctypes.data_as(FP), i.ctypes.data_as(IP)), m.prod.last_error()
    finally:
        _free(m, d_q, d_x)
    return _unguard(s, i, nq, top_k)


def want_b1(qb, xb, dim, k):
    """the rule's ranking, scores as the exact +-1 dot products (equal to dim - 2 hamming: tests/test_search_b1_rule.py)"""
    sq, sx = rule.signs(qb, dim).astype(np.float32), rule.signs(xb, dim).astype(np.float32)
    S = np.empty((len(qb), min(k, len(xb))), np.float32)
    I = np.empty(S.shape, np.int32)
    for r0 in range(0, len(qb), 1024):
        S[r0:r0 + 1024], I[r0:r0 + 1024] = rule.rank(sq[r0:r0 + 1024] @ sx.T, k)
    return S, I


# ---- 1. rows_to_binary ----------------------------------------------------------------------------------------------------------
def _special_rows(rng, n, dim):
    x = (rng.standard_normal((n, dim)) * 2.0 ** rng.integers(-20, 21, (n, dim))).astype(np.float32)
    specials = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-39, np.nan, np.inf, -np.inf], np.float32)
    mask = rng.random((n, dim)) < 0.2
    x[mask] = rng.choice(specials, mask.sum())
    return x


@pytest.mark.parametrize("dim", range(128, 2049, 128))
def test_rows_to_binary_every_dim(tiny, dim):
    rng = np.random.default_rng(dim)
    x = _special_rows(rng, 37, dim)
    for center in (None, _special_rows(rng, 1, dim)[0], np.zeros(dim, np.float32), np.full(dim, -0.0, np.float32)):
        got = to_bits(tiny, x, center)
        assert (got == rule.to_bits(x, center)).all(), "dim %d, centre %s" % (dim, "none" if center is None else "given")


def test_rows_to_binary_past_2_32_elements(tiny):
    """dim 2048, 2^21 + 5 rows: the last rows start past 2^32 floats (about 17 GB of source)"""
    m, L = tiny, tiny.prod.lib
    dim, blk = 2048, 65536
    n = (1 << 21) + 5
    rng = np.random.default_rng(5)
    block = _special_rows(rng, blk, dim)
    tail = _special_rows(rng, 5, dim)
    center = rng.standard_normal(dim).astype(np.float32)
    d_x = L.clip_b200_device_malloc(m.ctx, n * dim * 4)
    d_b = L.clip_b200_device_malloc(m.ctx, n * dim // 8)
    d_c = _dev(m, center)
    assert d_x and d_b, m.prod.last_error()
    try:
        for r0 in range(0, 1 << 21, blk):
            assert L.clip_b200_memcpy_h2d(m.ctx, d_x + r0 * dim * 4, block.ctypes.data, block.nbytes)
        assert L.clip_b200_memcpy_h2d(m.ctx, d_x + (1 << 21) * dim * 4, tail.ctypes.data, tail.nbytes)
        assert L.clip_b200_rows_to_binary(m.ctx, d_x, n, dim, d_c, d_b), m.prod.last_error()
        last = _host(m, d_b + (n - blk - 5) * dim // 8, (blk + 5, dim // 8), np.uint8)
    finally:
        _free(m, d_x, d_b, d_c)
    assert (last == rule.to_bits(np.concatenate([block, tail]), center)).all()


# ---- 2. search_b1 against the rule --------------------------------------------------------------------------------------------
def _db(kind, rng, n, dim):
    if kind == "random":
        return rng.integers(0, 256, (n, dim // 8), dtype=np.uint8)
    if kind == "identical":
        return np.repeat(rng.integers(0, 256, (1, dim // 8), dtype=np.uint8), n, 0)
    pats = rng.integers(0, 256, (3, dim // 8), dtype=np.uint8)          # low entropy: three patterns, rare single-bit flips
    x = pats[rng.integers(0, 3, n)]
    flip = rng.random(n) < 0.05
    cols = rng.integers(0, dim // 8, n)
    x[flip, cols[flip]] ^= (1 << rng.integers(0, 8, flip.sum())).astype(np.uint8)
    return x


PLAN_EDGE = 2 * 132 * 128                               # one query: 2 x #SMs partitions of one tile each (H100 SXM, 132 SMs)
SEARCH_CASES = [
    # n_q, n_db, dim, top_k, kinds
    (1, 1, 128, 1), (1, 127, 768, 10), (1, 128, 2048, 100), (1, 129, 768, 1024), (7, 255, 128, 10), (8, 256, 1024, 300),
    (9, 257, 640, 10), (1, PLAN_EDGE - 1, 768, 10), (1, PLAN_EDGE, 768, 100), (1, PLAN_EDGE + 1, 768, 1024),
    (127, 4097, 1280, 10), (128, 20000, 768, 100), (129, 20001, 128, 1024), (1000, 33793, 768, 10), (32769, 129, 128, 10),
    (3, 50, 256, 1024),
]


@pytest.mark.parametrize("kind", ["random", "lowent", "identical"])
@pytest.mark.parametrize("nq,n,dim,k", SEARCH_CASES, ids=["q%d-n%d-d%d-k%d" % c for c in SEARCH_CASES])
def test_search_b1_equals_rule(tiny, kind, nq, n, dim, k):
    rng = np.random.default_rng(nq * 7 + n + dim + k)
    xb = _db(kind, rng, n, dim)
    qb = _db("random", rng, nq, dim) if kind == "random" else xb[rng.integers(0, n, nq)]
    gs, gi = search_b1(tiny, qb, xb, dim, k)
    ws, wi = want_b1(qb, xb, dim, k)
    _assert_ranked(gs, gi, ws, wi, "search_b1 %s" % kind)
    if kind == "identical":
        assert (gi == np.arange(min(k, n))[None, :]).all()


def test_search_b1_equals_fp32_search_on_signs(tiny):
    """the +-1 rows in f32 through clip_b200_topk_search: a chain of +-1 products is exact, so both rankings are the same"""
    rng = np.random.default_rng(3)
    dim = tiny.d
    assert dim % 128 == 0
    for nq, n, k in ((1, 5000, 1024), (100, 3000, 10), (64, 777, 777)):
        xb = _db("lowent", rng, n, dim)
        qb = _db("random", rng, nq, dim)
        gs, gi = search_b1(tiny, qb, xb, dim, k)
        fs, fi = tiny.run("search", rule.signs(qb, dim).astype(np.float32), rule.signs(xb, dim).astype(np.float32), k)
        _assert_ranked(gs, gi, fs, fi, "search_b1 vs clip_b200_topk_search")


def test_search_b1_score_depends_on_its_pair_alone(tiny):
    rng = np.random.default_rng(4)
    dim = 768
    q = _db("random", rng, 1, dim)
    row = q ^ np.uint8(0x11)                                       # 2 bits a byte flipped: s = 768 - 4 * 96
    want = float(dim - 2 * 2 * (dim // 8))
    for n, pos in ((1, 0), (300, 299), (40000, 12345), (PLAN_EDGE + 7, PLAN_EDGE + 3)):
        xb = np.zeros((n, dim // 8), np.uint8)
        xb[:] = q ^ np.uint8(0xff)                                  # every other row scores -dim
        xb[pos] = row
        s, i = search_b1(tiny, q, xb, dim, 1)
        assert i[0, 0] == pos and s[0, 0] == want


def test_search_b1_database_past_2_32_bytes(tiny):
    """dim 2048 (256 bytes a row), 2^24 + 1000 rows: the planted best row starts past byte 2^32"""
    m, L = tiny, tiny.prod.lib
    dim, blk = 2048, 1 << 16
    n = (1 << 24) + 1000
    rng = np.random.default_rng(6)
    block = rng.integers(0, 256, (blk, dim // 8), dtype=np.uint8)
    q = rng.integers(0, 256, (1, dim // 8), dtype=np.uint8)
    d_x = L.clip_b200_device_malloc(m.ctx, n * dim // 8)
    d_q = _dev(m, q)
    assert d_x, m.prod.last_error()
    try:
        for r0 in range(0, n, blk):
            r = min(blk, n - r0)
            assert L.clip_b200_memcpy_h2d(m.ctx, d_x + r0 * dim // 8, block.ctypes.data, r * dim // 8)
        plant = (1 << 24) + 500
        assert L.clip_b200_memcpy_h2d(m.ctx, d_x + plant * dim // 8, q.ctypes.data, dim // 8)     # query 0 itself
        s, i = search_b1_dev(m, d_q, 1, d_x, n, dim, 10)
    finally:
        _free(m, d_x, d_q)
    assert i[0, 0] == plant and s[0, 0] == dim
    bs, bi = want_b1(q, block[:4096], dim, 9)                        # the rest: the best rows of the block's first copy
    assert s[0, 1] >= bs[0, 0] and (i[0, 1:] < (1 << 24)).all()


# ---- 3. rescore -----------------------------------------------------------------------------------------------------------------
def _unit(rng, n, dim):
    v = rng.standard_normal((n, dim)).astype(np.float32)
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def test_rescore_every_row_equals_fp32_search(tiny):
    rng = np.random.default_rng(7)
    dim = tiny.d
    for nq, n, k in ((1, 2048, 2048), (50, 1000, 100), (300, 7, 3)):
        q, db = _unit(rng, nq, dim), _unit(rng, n, dim)
        cand = np.tile(rng.permutation(n).astype(np.int32), (nq, 1))
        gs, gi = rescore(tiny, q, db, cand, k)
        ws, wi = tiny.run("search", q, db, k)
        _assert_ranked(gs, gi, ws, wi, "rescore every row")


def test_rescore_subsets_equal_rule(tiny):
    rng = np.random.default_rng(8)
    dim, nq, n = tiny.d, 40, 1500
    q, db = _unit(rng, nq, dim), _unit(rng, n, dim)
    fs, fi = tiny.run("search", q, db, n)                       # every score of every pair, from clip_b200_topk_search
    full = np.empty((nq, n), np.float32)
    np.put_along_axis(full, fi.astype(np.int64), fs, 1)
    for n_cand, k in ((1, 1), (100, 10), (2048, 2048), (333, 200)):
        cand = rng.integers(-3, n + 3, (nq, n_cand)).astype(np.int32)
        cand[:, ::7] = cand[:, :1]                               # duplicates
        cand[rng.random(cand.shape) < 0.05] = INT_MAX
        gs, gi = rescore(tiny, q, db, cand, k)
        ws, wi = rule.rescore_rank(rule.rescore_lists(cand, n, lambda r, idx: full[r, idx]), k)
        _assert_ranked(gs, gi, ws, wi, "rescore n_cand %d" % n_cand)


def test_rescore_16bit_equals_f32_on_widened_rows(tiny):
    import torch
    rng = np.random.default_rng(9)
    for dim in (8, 136, 768, 2048):
        q, db = _unit(rng, 20, dim), _unit(rng, 900, dim)
        cand = rng.integers(-1, 900, (20, 300)).astype(np.int32)
        for t, tt in ((F16, torch.float16), (BF16, torch.bfloat16)):
            q16, db16 = torch.from_numpy(q).to(tt), torch.from_numpy(db).to(tt)
            gs, gi = rescore(tiny, q16.view(torch.int16).numpy(), db16.view(torch.int16).numpy(), cand, 50, t)
            ws, wi = rescore(tiny, q16.float().numpy(), db16.float().numpy(), cand, 50, F32)
            _assert_ranked(gs, gi, ws, wi, "rescore in_type %d dim %d" % (t, dim))
        ws, wi = rule.rescore(q[:3], db, cand[:3], 50)                      # and the f32 call on the fmaf rule
        gs, gi = rescore(tiny, q[:3], db, cand[:3], 50)
        _assert_ranked(gs, gi, ws, wi, "rescore rule dim %d" % dim)


def test_rescore_edge_cases(tiny):
    rng = np.random.default_rng(10)
    dim, n = 64, 12
    q, db = _unit(rng, 4, dim), _unit(rng, n, dim)
    db[3, 5] = np.nan
    q[:, 0] = np.abs(q[:, 0]) + 0.1
    db[7, :] = 0.0
    db[7, 0] = -np.inf                                           # fmaf(q_0 > 0, -inf, +0) = -inf, and fmaf(q_i, 0, -inf) stays -inf
    cand = np.array([[3, 3, 3, -1, INT_MAX, 5],                  # NaN row, duplicates, skips: two valid, k = 4 pads two
                     [-1, -1, -1, -1, -1, -1],                   # nothing valid
                     [7, 0, 7, 12, -2, 1],                       # a -inf score ranks before the pads, 12 is out of range
                     [11, 10, 9, 8, 7, 6]], np.int32)
    gs, gi = rescore(tiny, q, db, cand, 4)
    ws, wi = rule.rescore(q, db, cand, 4)
    _assert_ranked(gs, gi, ws, wi, "rescore edges")
    assert gi[0].tolist()[1:] == [3, -1, -1] and gs[0, 1] == -rule.FLT_MAX and gi[1].tolist() == [-1] * 4
    assert gi[2, 2] == 7 and np.isneginf(gs[2, 2]) and gi[2, 3] == -1


# ---- 4. pipeline: binary shortlist, then exact rescoring -----------------------------------------------------------------------
def test_binary_then_rescore_equals_exact_search(tiny):
    rng = np.random.default_rng(11)
    dim, n, nq = tiny.d, 20000, 200
    db = _unit(rng, n, dim)
    src = rng.integers(0, n, nq)
    for j in range(nq):                                          # near-duplicates of each query's source row
        db[rng.integers(0, n, 12)] = db[src[j]] + 0.05 * rng.standard_normal((12, dim)).astype(np.float32)
    q = db[src] + 0.02 * rng.standard_normal((nq, dim)).astype(np.float32)
    center = db[:2000].mean(0)
    qb, xb = to_bits(tiny, q, center), to_bits(tiny, db, center)
    _, short = search_b1(tiny, qb, xb, dim, 100)
    gs, gi = rescore(tiny, q, db, short, 10)
    ws, wi = tiny.run("search", q, db, 10)
    held = np.array([set(wi[r]) <= set(short[r]) for r in range(nq)])
    assert held.sum() >= nq // 2, held.sum()
    _assert_ranked(gs[held], gi[held], ws[held], wi[held], "binary + rescore")


# ---- 5. argument checks ---------------------------------------------------------------------------------------------------------
class _Args:
    def __init__(self, m):
        self.m, L = m, m.prod.lib
        self.buf = [L.clip_b200_device_malloc(m.ctx, 1 << 20) for _ in range(3)]
        self.cand = np.zeros(64, np.int32)
        self.s, self.i = _out(0, 0)

    def call(self, form, **kw):
        L, b = self.m.prod.lib, self.buf
        a = dict(ctx=self.m.ctx, nq=2, ndb=2, dim=128, top_k=1, t=F32, n_cand=2, p0=b[0], p1=b[1], p2=None, cand=True, out=True)
        a.update(kw)
        s, i = (self.s.ctypes.data_as(FP), self.i.ctypes.data_as(IP)) if a["out"] else (None, None)
        if form == "rows_to_binary":
            return L.clip_b200_rows_to_binary(a["ctx"], a["p0"], a["nq"], a["dim"], a["p2"], a["p1"])
        if form == "search_b1":
            return L.clip_b200_topk_search_b1(a["ctx"], a["p0"], a["nq"], a["p1"], a["ndb"], a["dim"], a["top_k"], s, i)
        cand = self.cand.ctypes.data_as(IP) if a["cand"] else None
        return L.clip_b200_topk_rescore(a["ctx"], a["p0"], a["nq"], a["p1"], a["ndb"], a["dim"], a["t"], cand, a["n_cand"], a["top_k"], s, i)

    def refused(self, form, word, **kw):
        assert not self.call(form, **kw), (form, kw)
        e = self.m.prod.last_error()
        assert e.startswith("clip_b200_" + ("topk_" if form != "rows_to_binary" else "") + form) and word in e, (form, kw, e)


FAULTS = {   # form -> [(keyword in the message, arguments)] in the documented order
    "rows_to_binary": [("null context", dict(ctx=None)), ("dim", dict(dim=64)), ("dim", dict(dim=2176)), ("dim", dict(dim=200)),
                       ("2^31", dict(nq=1 << 31)), ("pointer", dict(p0=None)), ("pointer", dict(p1=None)),
                       ("pointer", dict(p2="odd"))],
    "search_b1": [("null context", dict(ctx=None)), ("dim", dict(dim=0)), ("dim", dict(dim=136)), ("top_k", dict(top_k=0)),
                  ("top_k", dict(top_k=1025)), ("2^31", dict(ndb=1 << 31)), ("pointer", dict(p0=None)), ("pointer", dict(p1="odd")),
                  ("output", dict(out=False))],
    "rescore": [("null context", dict(ctx=None)), ("in_type", dict(t=3)), ("dim", dict(dim=12)), ("dim", dict(dim=2056)),
                ("n_cand", dict(n_cand=0)), ("n_cand", dict(n_cand=2049)), ("top_k", dict(top_k=0)), ("top_k", dict(top_k=3)),
                ("2^31", dict(nq=1 << 31)), ("pointer", dict(p1=None)), ("pointer", dict(p0="odd")), ("null cand", dict(cand=False)),
                ("output", dict(out=False))],
}


@pytest.mark.parametrize("form", sorted(FAULTS))
def test_refusals_and_empty_calls(tiny, form):
    a = _Args(tiny)
    try:
        fix = lambda kw: {k: (a.buf[2] + 4 if v == "odd" else v) for k, v in kw.items()}
        assert a.call(form), tiny.prod.last_error()
        faults = FAULTS[form]
        for word, kw in faults:
            a.refused(form, word, **fix(kw))
        for j in range(len(faults) - 1):                          # two faults: the first is reported
            word, kw = faults[j]
            later = [f for f in faults[j + 1:] if not set(f[1]) & set(kw)]
            if later:
                a.refused(form, word, **fix({**later[-1][1], **kw}))
        # empty calls return true and write nothing, even with null pointers and outputs
        s, i = a.s.copy(), a.i.copy()
        assert a.call(form, nq=0, p0=None, p1=None, cand=False, out=False)
        if form != "rows_to_binary":
            assert a.call(form, ndb=0, p0=None, p1=None, cand=False, out=False)
        assert (a.s.view(np.uint32) == s.view(np.uint32)).all() and (a.i == i).all()
    finally:
        _free(tiny, *a.buf)
