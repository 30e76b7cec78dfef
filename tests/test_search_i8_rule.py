"""The int8 search's rule on the CPU (tests/_search_i8.py): the numpy quantiser keeps every code in [-127, 127] and rounds half-way
quotients to even, and the bound holds between the emulated scores and the fp64 dot products of the f32 rows, on random unit
rows at every dim from 16 to 2048 and on the rows where quantisation is worst: one dominant element, subnormal maxima, and
values exactly on a code boundary."""
import numpy as np
import pytest

from _search_i8 import FLT_MAX, bound, emulate, exact, quantize, rank, unit_rows


def _check_bound(q, x):
    qc, qs = quantize(q)
    xc, xs = quantize(x)
    for c in (qc, xc):
        assert c.dtype == np.int8 and (c != -128).all() and (np.abs(c.astype(np.int32)) <= 127).all()
    s = emulate(qc, qs, xc, xs)
    ok = np.isfinite(s)
    err = np.abs(s.astype(np.float64) - exact(q, x))
    b = bound(q, qs, x, xs, s)
    assert (err[ok] <= b[ok]).all(), "max error / bound %.4f" % (err[ok] / b[ok]).max()
    return err[ok] / b[ok]


@pytest.mark.parametrize("dim", [16, 32, 48, 128, 512, 768, 1024, 2032, 2048])
def test_bound_on_unit_rows(dim):
    rng = np.random.default_rng(dim)
    q, x = unit_rows(rng, 17, dim), unit_rows(rng, 300, dim)
    x[:4] = q[:4]
    r = _check_bound(q, x)
    assert r.max() > 0.02                             # the bound is not vacuous: some errors come within sight of it


def test_bound_on_dominant_elements():
    """one element carries the row: every other code is 0 or +-1, so their relative error is the largest the rule allows"""
    rng = np.random.default_rng(3)
    dim = 768
    q, x = rng.standard_normal((9, dim)).astype(np.float32) * 1e-3, rng.standard_normal((400, dim)).astype(np.float32) * 1e-3
    q[np.arange(9), rng.integers(0, dim, 9)] = 1.0
    x[np.arange(400), rng.integers(0, dim, 400)] = rng.uniform(0.5, 2, 400).astype(np.float32)
    _check_bound(q, x)


def test_bound_on_subnormal_scales():
    """maxima from 2^-149 up to 2^-118: s = RN(m / 127) is subnormal or 0, codes clamp, and some products underflow"""
    rng = np.random.default_rng(5)
    dim = 64
    e = rng.integers(-149, -117, 200)
    x = (rng.uniform(-1, 1, (200, dim)) * 2.0 ** e[:, None]).astype(np.float32)
    x[np.arange(200), rng.integers(0, dim, 200)] = (2.0 ** e).astype(np.float32)
    xc, xs = quantize(x)
    sub = (xs > 0) & (xs < np.finfo(np.float32).tiny)
    assert sub.sum() > 50 and (xs == 0).sum() > 5
    assert (np.abs(xc[sub].astype(np.int32)) == 127).any()
    q = np.vstack([unit_rows(rng, 5, dim), x[:5] * np.float32(2.0 ** 120)])
    _check_bound(q, x)
    _check_bound(x[:20], x)


def _halfway_rows(rng, n, dim):
    """rows whose scale is exactly 2^e (m = 127 * 2^e) and whose other elements are (k + 1/2) 2^e: every quotient is a tie"""
    e = rng.integers(-20, 20, n)
    k = rng.integers(-127, 127, (n, dim))
    x = ((k + 0.5) * 2.0 ** e[:, None]).astype(np.float32)
    x[:, 0] = (127 * 2.0 ** e).astype(np.float32)
    return x, k, e


def test_halfway_quotients_round_to_even():
    rng = np.random.default_rng(7)
    x, k, e = _halfway_rows(rng, 50, 128)
    c, s = quantize(x)
    assert np.array_equal(s, (2.0 ** e).astype(np.float32))
    want = np.clip(np.where(k % 2 == 0, k, k + 1), -127, 127)          # k + 1/2 to the even neighbour
    want[:, 0] = 127
    assert np.array_equal(c.astype(np.int64), want)
    assert (c[:, 1:] % 2 == 0).all()
    _check_bound(x[:10], x)


def test_zero_and_non_finite_rows():
    x = np.zeros((5, 32), np.float32)
    x[1, 3] = 2.0 ** -149                                                # m / 127 underflows to 0
    x[2, 4] = np.nan
    x[3, 5] = np.inf
    x[4, 6] = -np.inf
    x[2:, 0] = 1.0
    c, s = quantize(x)
    assert (c == 0).all()
    assert s[0] == 0 and s[1] == 0 and np.isnan(s[2:]).all()
    q = np.ones((1, 32), np.float32)
    sc, ix = rank(emulate(*quantize(q), c, s), 5)
    assert np.array_equal(ix[0], [0, 1, 2, 3, 4]) and (sc[0, 2:] == -FLT_MAX).all() and (sc[0, :2] == 0).all()


def test_ranking_order():
    s = np.array([[1.0, np.nan, 2.0, 1.0, -np.inf, 2.0]], np.float32)
    v, i = rank(s, 6)
    assert np.array_equal(i[0], [2, 5, 0, 3, 1, 4]) and v[0, 4] == -FLT_MAX and v[0, 5] == -np.inf
