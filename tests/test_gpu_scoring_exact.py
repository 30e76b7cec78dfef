"""Device scoring checked exactly: csrc/search.cu (similarity, softmax_with_sorting arithmetic, bitonic top-k) as
search_locked in csrc/api.cu drives it, through clip_b200_topk_search and clip_b200_zero_shot_batch.

- Similarity: each entry is one sequential fmaf chain over the features, bit for bit (_util.fmaf_chain_dot, whose fmaf is pinned
  to libm's below).  topk_search with top_k = n_db <= 4096 sorts the whole row in one device slice, so it returns every entry.
- Top-k: integer-valued inputs make every similarity exact in any summation order, so the expected ranking (value descending,
  ties by ascending index) is known exactly and compared with no tolerance, across every slice, column-chunk, row-pass and
  merge-stage boundary the driver has.
- Softmax: p within 1 float32 ulp of the reference arithmetic, and the ranking exact.
- NaN ranks last, ordered by index, and reads -FLT_MAX, on the device-selected (top_k <= 1024) and host-ranked paths alike.
- top_k <= 0 or top_k > n means all n, and rows are packed at that stride.

How search_locked splits the work of these two forms, for the cases below (SL = 4096 columns per sort slice):
  column chunk  CH = min(n_db, max(2^25 / min(n_q, 256), SL)); whole rows for softmax and for top_k > 1024
  row pass      RB = min(n_q, 2^25 / CH + 1, 32768)
  selection     on the device when the chunks hold one slice in all or top_k <= 1024 (one stage per slice, then merge stages
                until one slice is left); otherwise each whole row is ranked on the host.

The C functions are called through prod.lib: the Python wrappers clamp top_k themselves, which would hide the C contract."""
import ctypes as C
import ctypes.util
import functools

import numpy as np
import pytest

from _util import fmaf32, fmaf_chain_dot, model_file, softmax_sorted, ulp_dist

FLT_MAX = np.finfo(np.float32).max
GUARD = 64                                    # output entries past n_q * top_k that a call must leave alone


# ---- fmaf emulation against libm --------------------------------------------------------------------------------------------
def _fma_cases(rng):
    """name -> (a, b, c) float32 triples: random alignments, results on or next to a float32 tie, cancellation, subnormals"""
    f32 = np.float32
    n = 100_000
    a = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 21, n)).astype(f32)
    b = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 21, n)).astype(f32)
    c = (rng.standard_normal(n) * np.abs(a * b.astype(np.float64)) * 2.0 ** rng.integers(-40, 41, n)).astype(f32)
    cases = {"random": (a, b, c)}
    # a * b = +-h * m, h half an ulp of c: m = 1 is an exact tie; 1 - 2^-46 and 1 + 2^-22 + 2^-46 lie just beside one, where an
    # fp64 sum rounds onto the tie (or not) and a second rounding to float32 can go the wrong way
    m = 2000
    c = (rng.uniform(1, 2, m) * 2.0 ** rng.integers(-20, 21, m) * rng.choice([-1, 1], m)).astype(f32)
    h = (np.spacing(np.abs(c)) / 2).astype(f32)
    one_up, one_dn = f32(1 + 2.0 ** -23), f32(1 - 2.0 ** -23)
    ta, tb, tc = [], [], []
    for hm, bm in ((h, f32(1)), (h * one_up, one_dn), (h * one_up, one_up)):
        for sign in (1, -1):
            ta.append(hm.astype(f32))
            tb.append((sign * np.sign(c) * bm).astype(f32))
            tc.append(c)
    cases["ties"] = tuple(np.concatenate(x) for x in (ta, tb, tc))
    # c = -rn(a * b) (and a neighbour of it): the result is the product's own rounding error, or close to it
    a = rng.standard_normal(m).astype(f32)
    b = rng.standard_normal(m).astype(f32)
    p = (a.astype(np.float64) * b).astype(f32)
    cases["cancel"] = (np.concatenate([a, a, a]), np.concatenate([b, b, b]),
                       np.concatenate([-p, -p * one_up, -p * one_dn]).astype(f32))
    # products and sums at and below the float32 normal range (2^-126), down past the smallest subnormal (2^-149)
    a = (rng.uniform(1, 2, m) * 2.0 ** rng.integers(-80, -60, m)).astype(f32)
    b = (rng.uniform(1, 2, m) * 2.0 ** rng.integers(-90, -60, m) * rng.choice([-1, 1], m)).astype(f32)
    sub = rng.integers(1, 1 << 23, m).astype(np.uint32).view(f32) * rng.choice([-1, 1], m).astype(f32)
    cases["subnormal"] = (np.concatenate([a, a, a]), np.concatenate([b, b, b]),
                          np.concatenate([np.zeros(m, f32), sub, np.full(m, np.finfo(f32).tiny, f32)]))
    return cases


def test_fmaf_emulation_matches_libm():
    """_util.fmaf32 (the reference of every similarity below) bit for bit against the C library's fmaf on this CPU"""
    fmaf = C.CDLL(ctypes.util.find_library("m")).fmaf
    fmaf.restype, fmaf.argtypes = C.c_float, [C.c_float] * 3
    for name, (a, b, c) in _fma_cases(np.random.default_rng(11)).items():
        want = np.array([fmaf(x, y, z) for x, y, z in zip(a.tolist(), b.tolist(), c.tolist())], np.float32)
        got = fmaf32(a, b, c)
        bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
        assert not len(bad), (name, len(bad), [(a[i], b[i], c[i], got[i], want[i]) for i in bad[:3]])
        if name == "ties":      # the cases do reach the double-rounding hazard: one plain fp64 sum gets some of them wrong
            naive = (a.astype(np.float64) * b + c).astype(np.float32)
            assert (naive != want).any()
    # the chain: acc = fmaf(a[k], b[k], acc) for k ascending from +0
    rng = np.random.default_rng(12)
    a, b = rng.standard_normal((3, 40)).astype(np.float32), rng.standard_normal((5, 40)).astype(np.float32)
    a[:, ::3] *= 1e4
    want = np.zeros((3, 5), np.float32)
    for i in range(3):
        for j in range(5):
            acc = 0.0
            for k in range(40):
                acc = fmaf(float(a[i, k]), float(b[j, k]), acc)
            want[i, j] = acc
    assert np.array_equal(fmaf_chain_dot(a, b).view(np.uint32), want.view(np.uint32))


# ---- calling the library ----------------------------------------------------------------------------------------------------
class _Model:
    def __init__(self, prod, geom, ftype):
        self.prod = prod
        self.ctx = prod.load(model_file(geom, ftype, prod), 0)
        assert self.ctx, prod.last_error()
        self.d = prod.vision_hparams(self.ctx).projection_dim

    def _dev(self, a):
        p = self.prod.lib.clip_b200_device_malloc(self.ctx, a.nbytes)
        assert p and self.prod.lib.clip_b200_memcpy_h2d(self.ctx, p, a.ctypes.data, a.nbytes), self.prod.last_error()
        return p

    def run(self, entry, q, db, top_k):
        """entry "search" (clip_b200_topk_search) or "zero_shot" (clip_b200_zero_shot_batch) of q [n_q, d] against db [n, d] ->
        (scores, indices) [n_q, w], w = n when top_k <= 0 or top_k > n, else top_k.  The output buffers run GUARD entries
        further, and those must come back untouched."""
        q, db = np.ascontiguousarray(q, np.float32), np.ascontiguousarray(db, np.float32)
        nq, n = len(q), len(db)
        w = n if top_k <= 0 or top_k > n else top_k
        scores = np.full(nq * w + GUARD, 7.0, np.float32)
        idx = np.full(nq * w + GUARD, -7, np.int32)
        sp, ip = scores.ctypes.data_as(C.POINTER(C.c_float)), idx.ctypes.data_as(C.POINTER(C.c_int))
        L = self.prod.lib
        d_q, d_db = self._dev(q), self._dev(db)
        try:
            if entry == "search":
                ok = L.clip_b200_topk_search(self.ctx, d_q, nq, d_db, n, top_k, sp, ip)
            else:
                ok = L.clip_b200_zero_shot_batch(self.ctx, d_q, nq, d_db, n, sp, ip, top_k)
            assert ok, self.prod.last_error()
        finally:
            L.clip_b200_device_free(self.ctx, d_q)
            L.clip_b200_device_free(self.ctx, d_db)
        assert (scores[nq * w:] == 7.0).all() and (idx[nq * w:] == -7).all(), "written past n_q * top_k"
        return scores[:nq * w].reshape(nq, w), idx[:nq * w].reshape(nq, w)


def _model(prod, geom, ftype):
    m = _Model(prod, geom, ftype)
    yield m
    prod.free(m.ctx)


@pytest.fixture(scope="module")
def tiny(prod):
    yield from _model(prod, "tiny", "f16")              # projection dim 128


@pytest.fixture(scope="module")
def wide(prod):
    yield from _model(prod, "wide-h1280", "q4_0")       # projection dim 1024


def _assert_ranked(got_s, got_i, want_s, want_i, what):
    """indices identical and scores bit-identical; on failure, name the first differing row and rank"""
    bad = (got_i != want_i) | (got_s.view(np.uint32) != want_s.view(np.uint32))
    if bad.any():
        r, j = map(int, np.argwhere(bad)[0])
        raise AssertionError("%s: %d of %d entries differ; first at row %d rank %d: got (%r, %d), want (%r, %d)" % (
            what, bad.sum(), bad.size, r, j, got_s[r, j], got_i[r, j], want_s[r, j], want_i[r, j]))


# ---- a. similarity: one sequential fmaf chain -------------------------------------------------------------------------------
SIM_NQ = (1, 63, 64, 65, 130)                 # ragged against the 64 x 64 output tile
SIM_NDB = (1, 63, 64, 65, 4095, 4096)


@functools.lru_cache(maxsize=None)
def _sim_case(d, kind):
    """queries [130, d] and database [4096, d] (each shape below takes leading rows) and the emulated similarity matrix.
    kind "mixed": every row mixes entries near 1e4 and 1e-4, so any other summation order changes the bits."""
    rng = np.random.default_rng(d * 10 + (kind == "mixed"))

    def rows(n):
        x = rng.standard_normal((n, d))
        if kind == "mixed":
            x = np.where(rng.random((n, d)) < 0.5, 1e4, 1e-4) * np.sign(x) * rng.uniform(1, 2, (n, d))
        return x.astype(np.float32)
    q, db = rows(max(SIM_NQ)), rows(max(SIM_NDB))
    return q, db, fmaf_chain_dot(q, db)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["normal", "mixed"])
@pytest.mark.parametrize("model", ["tiny", "wide"])
def test_similarity_is_one_fmaf_chain(request, model, kind):
    m = request.getfixturevalue(model)
    q, db, sim = _sim_case(m.d, kind)
    for nq in SIM_NQ:
        for ndb in SIM_NDB:
            s, i = m.run("search", q[:nq], db[:ndb], ndb)
            assert (np.sort(i, 1) == np.arange(ndb)).all(), (nq, ndb, "indices are not a permutation")
            want = sim[:nq, :ndb]
            got = np.empty_like(s)
            np.put_along_axis(got, i, s, 1)
            bad = got.view(np.uint32) != want.view(np.uint32)
            assert not bad.any(), (nq, ndb, "%d of %d similarities differ from the fmaf chain" % (bad.sum(), bad.size))
            order = np.argsort(-want, axis=1, kind="stable")
            _assert_ranked(s, i, np.take_along_axis(want, order, 1), order, "ranking n_q=%d n_db=%d" % (nq, ndb))


# ---- b. top-k with ties everywhere ------------------------------------------------------------------------------------------
EDGES = (4096, 8192, 131072)                  # slice edges, and the column-chunk edge of the 300-query cases


def _ints(rng, shape):
    """integers in [-4, 4], half of them 0 (sparse rows make equal scores common)"""
    x = rng.integers(-4, 5, shape)
    x[rng.random(shape) < 0.5] = 0
    return x


def _tie_ints(nq, ndb, d, seed=7):
    """integer queries [nq, d] and database rows [ndb, d] with exact ties planted across every edge:
    - every third query carries one pattern on its first 32 features.  Hub row m has 4 * sign(pattern) on the first 32 - 6m of
      them and 0 elsewhere, so for those queries hubs 0 and 1 outscore every random row and hubs 2 and 3 fall among the best
      random rows.  Hub m is copied to both sides of every edge (e - 1 - m, e + m) and to rows m and ndb - 1 - m.
    - random rows are duplicated across every edge too: row e - 1 - o is copied to e + o for o = 4 .. 11."""
    rng = np.random.default_rng(seed)
    q, db = _ints(rng, (nq, d)), _ints(rng, (ndb, d))
    pattern = rng.integers(1, 5, 32) * rng.choice([-1, 1], 32)
    q[::3, :32] = pattern
    for e in EDGES:
        for o in range(4, 12):
            if e + o < ndb:
                db[e + o] = db[e - 1 - o]
    for m in range(4):
        hub = np.zeros(d, np.int64)
        hub[:32 - 6 * m] = 4 * np.sign(pattern[:32 - 6 * m])
        for r in [m, ndb - 1 - m] + [x for e in EDGES for x in (e - 1 - m, e + m)]:
            if 0 <= r < ndb:
                db[r] = hub
    return q, db


@functools.lru_cache(maxsize=None)
def _tie_case(nq, ndb, d):
    """float32 inputs (the integers scaled by 2^-3: every similarity is a multiple of 2^-6 below 2^11, exact in fp32 in any
    order) and the expected best min(ndb, 9000) per row, by (value descending, index ascending)."""
    qi, dbi = _tie_ints(nq, ndb, d)
    q, db = (qi * 2.0 ** -3).astype(np.float32), (dbi * 2.0 ** -3).astype(np.float32)
    kmax = min(ndb, 9000)
    want_s, want_i = np.empty((nq, kmax), np.float32), np.empty((nq, kmax), np.int64)
    dbt = dbi.T.astype(np.float64)
    for r0 in range(0, nq, 64):                                    # integers below 2^53: the fp64 product is exact too
        s = qi[r0:r0 + 64].astype(np.float64) @ dbt
        order = np.argsort(-s, axis=1, kind="stable")[:, :kmax]
        want_i[r0:r0 + 64] = order
        want_s[r0:r0 + 64] = np.take_along_axis(s, order, 1) * 2.0 ** -6
    return q, db, want_s, want_i


# n_q, n_db, top_k.  n_q = 3: one chunk, one row pass; n_db = 4096 is one slice, 4097 / 8192 two, 8193 three (one merge stage).
# n_q = 300, n_db = 140 000: CH = 131 072, so two column chunks, the second 8 928 wide and numbered from idx_base = 131 072;
# RB = 257, so two row passes; 35 slices, so at top_k = 1024 three merge stages.  top_k > 1024 ranks whole rows on the host
# (9000 is wider than the last column chunk).  n_q = 40 000: RB is capped at 32 768, so two row passes.
TOPK_CASES = ([(3, n, k) for n in (4096, 4097, 8192, 8193) for k in (1, 7, 1024)]
              + [(300, 140_000, k) for k in (10, 1024, 1025, 2000, 9000)] + [(40_000, 100, 5)])


@pytest.mark.gpu
@pytest.mark.parametrize("nq,ndb,k", TOPK_CASES)
def test_topk_search_exact_with_ties(tiny, nq, ndb, k):
    q, db, want_s, want_i = _tie_case(nq, ndb, tiny.d)
    s, i = tiny.run("search", q, db, k)
    _assert_ranked(s, i, want_s[:, :k], want_i[:, :k], "top-%d of %d x %d" % (k, nq, ndb))


@pytest.mark.gpu
def test_topk_search_device_1024_is_prefix_of_host_1025(tiny):
    q, db, _, _ = _tie_case(300, 140_000, tiny.d)
    s0, i0 = tiny.run("search", q, db, 1024)
    s1, i1 = tiny.run("search", q, db, 1025)
    _assert_ranked(s1[:, :1024], i1[:, :1024], s0, i0, "top-1025 prefix against top-1024")


# ---- c. softmax arithmetic and ranking of zero_shot_batch -------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _softmax_case(n_img, n_txt, d):
    """image rows [n_img, d] and label rows [n_txt, d] whose logits are exact fp32 values, and the reference (p sorted, order).
    - Entries are integers in [-4, 4] times 2^-3, and each image row is scaled by its own power of two 2^t, t <= 0, the largest
      that keeps |logit| <= 24.  Every logit is then exact, and distinct logits of a row differ by at least 2^-7.  Over
      [-24, 24] that moves e = exp(s) + 1e-9 by more than 2 000 float32 ulps, so distinct probabilities are thousands of ulps
      apart, while equal logits give bit-equal probabilities.  The ranking is therefore fixed by the logits alone.
    - Row 1 is the floor row: -4 on features 0-7 scaled by 2^7, against labels whose features 0-7 are all in [1, 4].  Its
      logits are <= -64, every e is exactly float32(1e-9), and its ranking is pure index order.
    - Labels n_txt - 1 and n_txt // 2 duplicate labels 0 and 1."""
    rng = np.random.default_rng(n_img * 7 + n_txt)
    img, txt = _ints(rng, (n_img, d)), _ints(rng, (n_txt, d))
    txt[:, :8] = rng.integers(1, 5, (n_txt, 8))
    if n_txt >= 4:
        txt[n_txt - 1], txt[n_txt // 2] = txt[0], txt[1]
    t = np.zeros(n_img)
    if n_img > 1:
        img[1] = 0
        img[1, :8] = -4
        t[1] = 7
    logits = np.empty((n_img, n_txt), np.float32)
    for r in range(n_img):
        s = img[r].astype(np.float64) @ txt.T.astype(np.float64)
        if r != 1:
            top = np.abs(s).max()
            t[r] = 0 if top == 0 else min(0, np.floor(np.log2(24 * 64 / top)))
        logits[r] = s * 2.0 ** (t[r] - 6)
    p, order = softmax_sorted(logits)
    if n_img > 1:
        assert (order[1] == np.arange(n_txt)).all() and (p[1] == p[1, 0]).all()
    return (img * 2.0 ** (t[:, None] - 3)).astype(np.float32), (txt * 2.0 ** -3).astype(np.float32), p, order


# n_txt = 1: p is exactly 1.  5 000 and 9 000: rows longer than the kernel's 256 threads, two and three slices.  337 x 100 000:
# RB = 336, two row passes.  top_k 1024 selects on the device, 1025 and n_txt rank on the host once a row spans two slices.
SOFTMAX_CASES = [(n_img, n_txt, k) for n_img, n_txt in ((3, 1), (5, 5000), (4, 9000), (337, 100_000))
                 for k in (5, 1024, 1025, n_txt)]


@pytest.mark.gpu
@pytest.mark.parametrize("n_img,n_txt,k", SOFTMAX_CASES)
def test_zero_shot_batch_softmax_exact(tiny, n_img, n_txt, k):
    img, txt, p, order = _softmax_case(n_img, n_txt, tiny.d)
    s, i = tiny.run("zero_shot", img, txt, k)
    w = s.shape[1]
    assert np.array_equal(i, order[:, :w]), "ranking differs in %d of %d entries" % ((i != order[:, :w]).sum(), i.size)
    du = ulp_dist(s, p[:, :w])
    print("%d x %d top-%d: %d of %d probabilities 1 ulp from the reference" % (n_img, n_txt, k, (du == 1).sum(), du.size))
    assert du.max() <= 1
    assert (du == 1).sum() <= 8
    if n_txt == 1:
        assert (s == 1.0).all()


@pytest.mark.gpu
def test_zero_shot_batch_device_1024_is_prefix_of_host_1025(tiny):
    img, txt, _, _ = _softmax_case(337, 100_000, tiny.d)
    s0, i0 = tiny.run("zero_shot", img, txt, 1024)
    s1, i1 = tiny.run("zero_shot", img, txt, 1025)
    _assert_ranked(s1[:, :1024], i1[:, :1024], s0, i0, "top-1025 prefix against top-1024")


# ---- d. NaN ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_nan_ranks_last_as_minus_flt_max(tiny):
    """a NaN feature makes a database row's every similarity NaN.  top_k = 1024 over 5 000 rows selects on the device,
    top_k = 5 000 ranks on the host, and 4 096 rows with top_k = 4 096 sort on the device in one slice: all rank NaN last, by
    index, as -FLT_MAX."""
    qi, dbi = _tie_ints(4, 5000, tiny.d)
    q, db = (qi * 2.0 ** -3).astype(np.float32), (dbi * 2.0 ** -3).astype(np.float32)
    nan_rows = [17, 2500, 4095, 4096, 4999]
    db[nan_rows, 5] = np.nan
    runs = {}
    for n, k in ((5000, 1024), (5000, 5000), (4096, 4096)):
        s = (qi.astype(np.float64) @ dbi[:n].T.astype(np.float64)) * 2.0 ** -6
        s[:, [r for r in nan_rows if r < n]] = -np.inf
        order = np.argsort(-s, axis=1, kind="stable")[:, :k]
        want = np.take_along_axis(s, order, 1)
        want[np.isinf(want)] = -FLT_MAX
        runs[n, k] = tiny.run("search", q, db[:n], k)
        _assert_ranked(*runs[n, k], want.astype(np.float32), order, "top-%d of %d with NaN rows" % (k, n))
    _assert_ranked(*(x[:, :1024] for x in runs[5000, 5000]), *runs[5000, 1024], "host ranking prefix against device top-1024")


# ---- e. the top_k contract --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["search", "zero_shot"])
def test_top_k_out_of_range_means_all(tiny, entry):
    """top_k <= 0 and top_k > n both return all n per row, rows packed at stride n (run() checks the stride's end)"""
    if entry == "search":
        q, db, want_s, want_i = _tie_case(5, 300, tiny.d)
    else:
        q, db, want_s, want_i = _softmax_case(5, 300, tiny.d)
    for k in (0, -1, 301, 1 << 30):
        s, i = tiny.run(entry, q, db, k)
        assert s.shape == (5, 300)
        assert np.array_equal(i, want_i), k
        if entry == "search":
            _assert_ranked(s, i, want_s, want_i, "top_k=%d" % k)
        else:
            assert ulp_dist(s, want_s).max() <= 1, k
