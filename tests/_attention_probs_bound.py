"""K9's attention probabilities (csrc/attention_tc.cu, attention_probs_kernel): an fp64 reference, an element-wise bound on how far the
kernel's output may be from it, derived from the kernel's rounding points, and a numpy emulation of the kernel's arithmetic.  Shared by
the GPU test (tests/test_gpu_attention_probs.py) and by the CPU test that checks the bound against the emulation and against two wrong
results (tests/test_attention_probs_bound.py).

Notation as in tests/_attention_bound.py: u = 2^-24, q and k the 16-bit operands (exact in fp64), s_j = q.k_j, m = max_j s_j over the
keys the row sees, w_j = e^(s_j - m), l = sum_j w_j >= 1, pi_j = w_j / l the exact probability; nb the 128-key blocks the row's group
visits.  K9 computes p_j = ex2(fl(s'_j log2e) - fl(m' log2e)) * fl(1 / l'), with l' summed block by block exactly as K3 sums it.

Its errors, in the order they happen:
  1-4. _attention_bound.py's steps 1-4: the scores on the tensor cores (D per key), the exponent argument (6 u S_max), ex2.approx
     (2^-22) and, for l' only, the running-max rescales (nb 2^-22 + 6 u S_max).  The numerator uses the final m' directly, the
     denominator the rescaled block sums: both carry the same factor e^(m - m'), which cancels.  So every w_j reaches the numerator
     and l' multiplied by (1 + e_j), |e_j| <= E = expm1(D) + 12 u S_max + (1 + nb) 2^-22, and
     |w'_j / sum_k w'_k - pi_j| <= 2 E / (1 - E) pi_j.
  5. The sum l': per thread and block a pair and up to 15 chained adds, one multiply and one add per block, 2 shuffles:
     (19 + 2 nb) u relative.
  6. 1 / l' (correctly rounded) and the product: 2 u relative.
  7. ex2.approx.ftz flushes a weight below 2^-126 to +0: an absolute error below 2^-126 (l' >= 1).
  8. The output type: f32 as it is; a 16-bit output is the RNE of the f32 value, u16 relative, and fp16 outputs below 2^-14 lose
     up to half the subnormal spacing, 2^-25.
The bound is the sum, with 1 % on top for second-order products."""
import numpy as np

from _attention_bound import AK, EX2, U, kend_of_rows, round16

LOG2E = np.float32(1.4426950408889634)
OUT_U = {0: 0.0, 1: 2.0 ** -11, 2: 2.0 ** -8}             # out_type -> unit roundoff of the output
OUT_TINY = {0: 2.0 ** -150, 1: 2.0 ** -25, 2: 2.0 ** -134}


def reference_probs(q, k, causal, bf, out_type=0, rows=None):
    """fp64 softmax of rows `rows` (default all) of one (sequence, head) and the bound of the module docstring.  q, k: [T, dh] of
    values exact in the 16-bit operand type (bf), Q already scaled.  Returns (pi [R, T], bound [R, T]); masked keys have pi = 0 and
    bound 0 (the kernel writes exactly +0 there)."""
    T, dh = k.shape
    rows = np.arange(T) if rows is None else np.asarray(rows)
    q = np.asarray(q, np.float64)[rows]
    k = np.asarray(k, np.float64)
    s = q @ k.T
    vis = np.ones_like(s, bool) if not causal else np.arange(T)[None, :] <= rows[:, None]
    s = np.where(vis, s, -np.inf)
    m = s.max(-1, keepdims=True)
    w = np.exp(s - m)
    pi = w / w.sum(-1, keepdims=True)
    d = (2 * dh / 16 + 4) * U * np.where(vis, np.abs(q) @ np.abs(k).T, 0.0).max(-1, keepdims=True)
    smax = np.where(vis, np.abs(s), 0.0).max(-1, keepdims=True) + d
    nb = np.ceil(kend_of_rows(rows, T, causal)[:, None] / AK)
    e = np.expm1(d) + 12 * U * smax + EX2 * (1 + nb)
    b32 = pi * (2 * e / (1 - e) + (19 + 2 * nb + 2) * U) + 2.0 ** -126
    bound = 1.01 * (b32 + OUT_U[out_type] * (pi + b32) + (OUT_TINY[out_type] if out_type else 0.0))
    return pi, np.where(vis, bound, 0.0)


# ---- the kernel's arithmetic in numpy ------------------------------------------------------------------------------------------
def _ex2(x):
    """2^x of float32 arguments, correctly rounded to float32 and flushed to zero below 2^-126 (ex2.approx.ftz is within 2 ulp of it)"""
    r = np.exp2(np.asarray(x, np.float64)).astype(np.float32)
    return np.where(r < np.float32(2.0 ** -126), np.float32(0.0), r)


def emulate_scores(q, k):
    """S = Q.K^T as the tensor cores form it: exact products, each k16 step rounded to fp32 and added to an fp32 accumulator"""
    q = np.asarray(q, np.float64)
    k = np.asarray(k, np.float64)
    acc = np.zeros((q.shape[0], k.shape[0]), np.float32)
    for c in range(0, q.shape[1], 16):
        acc = (acc + (q[:, c:c + 16] @ k[:, c:c + 16].T).astype(np.float32)).astype(np.float32)
    return acc


def emulate(q, k, causal):
    """K9's fp32 output [T, T] for one (sequence, head): pass 1's running max and per-thread sums over 128-key blocks (a quad of
    threads per row, thread t holding columns 8j + 2t + {0, 1}), the quad reduction, 1 / l, then pass 2's products"""
    T = k.shape[0]
    s = emulate_scores(q, k)
    rows = np.arange(T)
    vis = np.ones((T, T), bool) if not causal else np.arange(T)[None, :] <= rows[:, None]
    s = np.where(vis, s, np.float32(-np.inf)).astype(np.float32)
    kend = kend_of_rows(rows, T, causal)
    m_run = np.full(T, -np.inf, np.float32)
    l_run = np.zeros((T, 4), np.float32)
    with np.errstate(invalid="ignore"):
        for key0 in range(0, int(kend.max()), AK):
            live = kend > key0                                   # the rows whose group visits this block
            blk = s[:, key0:key0 + AK]
            if blk.shape[1] < AK:
                blk = np.concatenate([blk, np.full((T, AK - blk.shape[1]), -np.inf, np.float32)], 1)
            m_new = np.maximum(m_run, blk.max(1))
            alpha = _ex2(((m_run - m_new).astype(np.float32) * LOG2E).astype(np.float32))
            mb = (m_new * LOG2E).astype(np.float32)
            p = _ex2(((blk * LOG2E).astype(np.float32) - mb[:, None]).astype(np.float32))
            for t in range(4):
                rs = np.zeros(T, np.float32)
                for j in range(AK // 8):
                    rs = (rs + (p[:, 8 * j + 2 * t] + p[:, 8 * j + 2 * t + 1]).astype(np.float32)).astype(np.float32)
                l_new = ((l_run[:, t] * alpha).astype(np.float32) + rs).astype(np.float32)
                l_run[:, t] = np.where(live, l_new, l_run[:, t])
            m_run = np.where(live, m_new, m_run)
    l = ((l_run[:, 0] + l_run[:, 1]).astype(np.float32) + (l_run[:, 2] + l_run[:, 3]).astype(np.float32)).astype(np.float32)
    inv = (np.float32(1.0) / l).astype(np.float32)
    mb = (m_run * LOG2E).astype(np.float32)
    p = _ex2(((s * LOG2E).astype(np.float32) - mb[:, None]).astype(np.float32))
    return np.where(vis, (p * inv[:, None]).astype(np.float32), np.float32(0.0))


def to_out(p32, out_type):
    """the kernel's output values of fp32 probabilities: f32 as they are, or the RNE 16-bit value (as float32)"""
    if out_type == 0:
        return np.asarray(p32, np.float32)
    return round16(p32, out_type == 2)


def exceed(got, want, bound):
    """max over elements of |got - want| / bound, where bound 0 demands equality (<= 1 passes)"""
    err = np.abs(np.asarray(got, np.float64) - want)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))
    return float(r.max())
