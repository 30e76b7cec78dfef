"""The IVF-PQ rule of tests/_search_ivfpq.py checked against fp64 on exact data, and shown to tell apart the mistakes a kernel could
plausibly make: pairwise table sums, a table built in fp64, the coarse score added last, ties broken by stored position, NaN
distances not ranked last, and an unchunked fp64 mean."""
import numpy as np

import _search_ivf as ivf_rule
import _search_ivfpq as rule


def _exact(rng, shape, step=2.0 ** -3):
    """small integers times a power of two: exact in f16 and bf16, every sum of products exact in fp32 at these sizes"""
    return (rng.integers(-4, 5, shape) * step).astype(np.float32)


def test_scores_on_exact_data_are_fp64():
    rng = np.random.default_rng(1)
    dim, M, L = 32, 16, 6
    db, cent, q = _exact(rng, (500, dim)), _exact(rng, (L, dim)), _exact(rng, (20, dim))
    books = _exact(rng, (M, 256, dim // M), 2.0 ** -4)
    lists = ivf_rule.exact_assign(db, cent)
    codes = rule.encode(db, cent, lists, books)
    probe = ivf_rule.probes(q, cent, 3)
    coarse = np.take_along_axis(q.astype(np.float64) @ cent.T.astype(np.float64), probe, 1).astype(np.float32)
    s, i = rule.search(q, books, codes, lists, probe, coarse, 50)
    recon = books[np.arange(M)[None, :], codes.astype(np.int64)].reshape(len(db), dim).astype(np.float64)   # r^ of each row
    for r in range(len(q)):
        n_in = np.isin(lists, probe[r]).sum()
        want = q[r].astype(np.float64) @ cent[lists[i[r, :min(50, n_in)]]].T.astype(np.float64) + recon[i[r, :min(50, n_in)]] @ q[r]
        assert np.array_equal(s[r, :len(want)].astype(np.float64), want)
        full = q[r].astype(np.float64) @ cent[lists].T + recon @ q[r]
        rows = np.flatnonzero(np.isin(lists, probe[r]))
        order = rows[np.argsort(-full[rows], kind="stable")][:50]
        assert np.array_equal(i[r, :len(order)], order)


def test_encode_is_the_least_distance_with_lower_index_ties():
    r = np.array([[0.5, 0.25], [1.0, 1.0]], np.float32)
    books = np.zeros((1, 256, 2), np.float32)
    books[0, :, 0] = 8.0
    books[0, 3], books[0, 9] = [0.5, 0.0], [0.5, 0.5]              # row 0: codewords 3 and 9 are equally far (0.25 ** 2)
    books[0, 200] = [1.0, 1.0]
    assert list(rule.encode_residuals(r, books)[:, 0]) == [3, 200]


def test_sequential_table_sums_not_pairwise():
    t = np.zeros((4, 256), np.float32)
    t[:, 1] = [1.0, 2.0 ** -24, 2.0 ** -24, 2.0 ** -24]
    codes = np.ones((1, 4), np.uint8)
    v = rule.adc(np.zeros(1, np.float32), t, codes)[0]
    pairwise = np.float32(np.float32(1.0 + np.float32(2.0 ** -24)) + np.float32(np.float32(2.0 ** -24) + np.float32(2.0 ** -24)))
    assert v == np.float32(1.0) and pairwise != v


def test_table_in_fp32_fmaf_chain_not_fp64():
    q = np.array([[1.0, 2.0 ** -24, 2.0 ** -24]], np.float32)
    books = np.zeros((1, 256, 3), np.float32)
    books[0, 0] = [1.0, 1.0, 1.0]
    t = rule.tables(q, books)[0, 0, 0]
    fp64 = np.float32(1.0 + 2.0 ** -24 + 2.0 ** -24)
    assert t == np.float32(1.0) and fp64 != t


def test_coarse_score_added_first():
    t = np.zeros((2, 256), np.float32)
    t[:, 1] = [2.0 ** -24, 2.0 ** -24]
    codes = np.ones((1, 2), np.uint8)
    v = rule.adc(np.ones(1, np.float32), t, codes)[0]
    last = np.float32(np.float32(2.0 ** -24 + 2.0 ** -24) + np.float32(1.0))
    assert v == np.float32(1.0) and last != v


def test_ties_by_original_index_not_stored_position():
    # rows 0 and 1 score alike; row 0 is in list 1 and row 1 in list 0, so stored position puts row 1 first
    books = np.zeros((16, 256, 1), np.float32)
    codes = np.zeros((3, 16), np.uint8)
    lists = np.array([1, 0, 0])
    probe, coarse = np.array([[0, 1]]), np.array([[0.5, 0.5]], np.float32)
    s, i = rule.search(np.zeros((1, 16), np.float32), books, codes, lists, probe, coarse, 2)
    assert list(i[0]) == [0, 1] and s[0, 0] == s[0, 1]
    off, ids, _ = rule.build(lists, codes, 2)
    assert list(ids[:2]) == [1, 2], "the stored-position order would put row 1 first"


def test_nan_distances_rank_last():
    r = np.array([[np.nan, 0.0], [0.0, 0.0]], np.float32)
    books = np.zeros((1, 256, 2), np.float32)
    books[0, :, 0] = np.arange(256, dtype=np.float32)
    codes = rule.encode_residuals(r, books)
    assert list(codes[:, 0]) == [0, 0]
    d = rule.distances(r[1:], books[0])
    d[0, 0] = np.nan                                  # a kernel that does not read NaN as +inf: argmin lands on the NaN
    assert np.argmin(d[0]) == 0 and np.nanargmin(np.where(np.isnan(d[0]), np.inf, d[0])) == 1
    # and a NaN score of a search ranks last, reported as -FLT_MAX
    v = rule.adc(np.array([np.nan, 1.0], np.float32), np.zeros((1, 256), np.float32), np.zeros((2, 1), np.uint8))
    assert v[0] == -rule.FLT_MAX and v[1] == 1.0


def test_chunked_mean_not_unchunked():
    n = 1024
    r = np.zeros((n, 16), np.float32)
    r[0, 0], r[1:512, 0] = 2.0 ** 60, 1.0               # each chunk loses its ones to +-2^60; one unchunked sum keeps chunk 2's
    r[512, 0], r[513:, 0] = -(2.0 ** 60), 1.0
    codes = np.zeros((n, 16), np.uint8)
    books = rule.update(r, codes, np.full((16, 256, 1), 7.0, np.float32))
    unchunked = np.float32(rule.seq_sum(r[:, :1].astype(np.float64))[0] / n)
    assert books[0, 0, 0] == 0.0 and unchunked == np.float32(511.0 / n)
    assert (books[:, 1:] == 7.0).all(), "empty codewords keep their value"


def test_train_is_deterministic():
    rng = np.random.default_rng(4)
    x, cent = _exact(rng, (600, 32)), _exact(rng, (4, 32))
    lists = ivf_rule.exact_assign(x, cent)
    a, b = rule.train(x, cent, lists, 16, 2), rule.train(x, cent, lists, 16, 2)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert np.array_equal(rule.init(rule.residuals(x, cent, lists), 16)[3, 5], rule.residuals(x, cent, lists)[5 * 600 // 256, 6:8])
