"""The int8 search (clip_b200_rows_to_int8 and clip_b200_topk_search_i8, K10's s8 instance in csrc/search.cu): the quantisation
rule and the score rule in numpy, the ranking, and the bound between a score and the exact dot product of the f32 rows.  Shared by
the CPU test of the rule (tests/test_search_i8_rule.py) and the GPU test (tests/test_gpu_search_i8.py).

The bound.  Let s be a row's scale, m its max |x_i|, c_i its codes, and u = 2^-24.
1. One element.  When c_i is not clamped, c_i = rint(r) with r = RN(x_i / s), and rint(r) <= 127 means r <= 127.5, so
   |r - x_i / s| <= 127.5 u (or 2^-150 where the quotient is subnormal).  Then |c_i - x_i / s| <= 1/2 + 127.5 u + 2^-150, and
   |x_i - c_i s| <= d = s (1/2 + 2^-16).  When c_i is clamped to +-127, r > 127.5, so |x_i| > 127 s and |x_i - c_i s| <= m - 127 s.
   A row whose s is 0 has zero codes and |x_i| <= m = m - 127 s.  So every element is within
       d = max(s (1/2 + 2^-16), m - 127 s)
   of c_i s.  For a normal s the second term is below the first: s = RN(m / 127) >= m / 127 (1 - u), so m - 127 s <= m u.
2. The dot product of the dequantised rows q^ = c_q s_q, x^ = c_x s_x: with q^ = q - a, x^ = x - b (|a_i| <= d_q, |b_i| <= d_x),
   q.x - q^.x^ = q.b + a.x - a.b, so |q.x - q^.x^| <= d_x sum|q_i| + d_q sum|x_i| + dim d_q d_x.
3. The arithmetic: acc is exact and Q = q^.x^ = acc s_q s_x exactly.  score = RN(RN(RN(acc) s_q) s_x): three roundings of
   relative error <= u each while nothing underflows, so |score - Q| <= ((1 + u)^3 - 1) |Q| <= 4u |score|.  An underflowing
   product adds at most half the subnormal spacing, 2^-150, and the first product's is then scaled by s_x: 2^-149 (1 + s_x)
   covers both.
So, for finite scores:
    |score - q.x| <= d_x sum_i |q_i| + d_q sum_i |x_i| + dim d_q d_x + 2^-22 |score| + 2^-149 (1 + s_x).
With normal scales that is sum_i (|q_i| s_x + |x_i| s_q) / 2 + dim s_q s_x / 4 and a few ulps of |score|, widened by 2^-15
relative."""
import numpy as np

FLT_MAX = np.finfo(np.float32).max
U = 2.0 ** -24


def quantize(x):
    """float32 rows [n, dim] -> (codes int8 [n, dim], scales float32 [n]) by the rule: s = RN(m / 127) in float32, c =
    clamp(rint(x / s), -127, 127) with float32 division and half-to-even rint; s == 0 rows get zero codes, rows holding a NaN or
    an Inf get s = NaN and zero codes."""
    x = np.ascontiguousarray(x, np.float32)
    fin = np.isfinite(x).all(axis=1)
    with np.errstate(all="ignore"):
        m = np.abs(np.where(np.isfinite(x), x, np.float32(0))).max(axis=1)
        s = (m / np.float32(127)).astype(np.float32)
        c = np.clip(np.rint(x / s[:, None]), -127, 127)
    zero = ~fin | (s == 0)
    c[zero] = 0
    s = np.where(fin, s, np.float32(np.nan)).astype(np.float32)
    return c.astype(np.int8), s


def acc(qc, xc):
    """exact int32 dot products of the codes [n_q, n_db] (fp64: every partial sum is an integer below 2^31, exact in any order)"""
    return np.asarray(qc, np.float64) @ np.asarray(xc, np.float64).T


def emulate(qc, qs, xc, xs):
    """the kernel's scores, bit for bit: fp32(fp32(float_rn(acc) * s_q) * s_x), two float32 products rounded to nearest"""
    a = acc(qc, xc).astype(np.float32)                           # an integer below 2^31: one rounding to float32
    with np.errstate(all="ignore"):
        t = (a * np.asarray(qs, np.float32)[:, None]).astype(np.float32)
        return (t * np.asarray(xs, np.float32)[None, :]).astype(np.float32)


def rank(scores, k):
    """the best k per row: score descending, then lower index; NaN ranks last as -FLT_MAX -> (scores, indices int32)"""
    s = np.where(np.isnan(scores), -FLT_MAX, scores).astype(np.float32)
    order = np.argsort(-s, axis=1, kind="stable")[:, :k]
    return np.take_along_axis(s, order, 1), order.astype(np.int32)


def delta(x, s):
    """per row: how far any c_i s may lie from x_i (step 1 of the module docstring)"""
    x, s = np.asarray(x, np.float64), np.asarray(s, np.float64)
    m = np.abs(x).max(axis=1)
    return np.maximum(s * (0.5 + 2.0 ** -16), m - 127 * s)


def bound(q, qs, x, xs, scores):
    """the bound of the module docstring [n_q, n_db] for f32 rows q, x, their scales and the scores"""
    q, x = np.asarray(q, np.float64), np.asarray(x, np.float64)
    dq, dx = delta(q, qs), delta(x, xs)
    xs64 = np.asarray(xs, np.float64)
    return (np.abs(q).sum(1)[:, None] * dx[None, :] + dq[:, None] * np.abs(x).sum(1)[None, :] + q.shape[1] * dq[:, None] * dx[None, :]
            + 4 * U * np.abs(np.asarray(scores, np.float64)) + 2.0 ** -149 * (1 + xs64[None, :]))


def exact(q, x):
    """fp64 dot products of the f32 rows [n_q, n_db]"""
    return np.asarray(q, np.float64) @ np.asarray(x, np.float64).T


def unit_rows(rng, n, dim):
    """seeded unit-norm float32 rows"""
    v = rng.standard_normal((n, dim))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    return v.astype(np.float32)
