"""K3's attention at long T: test inputs, a high-precision reference on sampled query rows, and an element-wise bound on how
far the kernel's output may be from it, derived from the kernel's rounding points (csrc/attention_tc.cu).  Shared by the GPU test
(tests/test_gpu_attention_long.py) and by the CPU test that checks the bound against a numpy emulation of the kernel's arithmetic
and against emulated faults (tests/test_attention_long_bound.py).

Notation: u = 2^-24 (fp32), u16 the unit roundoff of the 16-bit operand type (2^-8 for bf16: 8 significant bits; 2^-11 for
fp16: 11 bits).  q, k, v are the 16-bit operands (exact in fp64), s_j = q.k_j the exact score, m = max_j s_j over the keys the
row sees, pi_j = e^(s_j - m) / l with l = sum_j e^(s_j - m) >= 1, O = sum_j pi_j v_j, A = sum_j pi_j |v_j| >= |O|.  nb is the
number of key blocks the row's group visits -- blocks of the instance's width, keys_per_block(dh): 128 keys at head_dim 64 and 80,
64 at 104 -- and kend the keys it visits.  dh is the width the kernel multiplies: at head_dim 104 the operands padded with zeros to
112 columns, so S takes 7 k16 steps.

Every error of the kernel is one of these, in the order it happens:
  1. S = Q.K^T on the tensor cores: products exact in fp32, dh/16 k16 steps accumulated in fp32.  As in test_gpu_gemm.py, with
     2u per step (test_gpu_tokens.py's allowance for the tensor cores' accumulation): |ds_j| <= D_j = (2 dh/16 + 4) u sum_i |q_i k_ji|.
  2. The exponent argument fl(s LOG2E - fl(m LOG2E)), LOG2E itself rounded: the constant (2 uses), the products (2, if not fused)
     and the difference (1, at most 2 S_max) give |dx| <= 6 u S_max log2(e), S_max = max |s| + D.  As a relative error of 2^x:
     ln 2 |dx| <= 6 u S_max.
  3. ex2.approx.ftz.f32: 2 ulp, 2^-22 relative (the CUDA programming guide's bound for exp2f, which is this instruction).
  4. The running-max rescale alpha = ex2(fl((m_old - m_new) LOG2E)): per visited block 2^-22 (ex2) plus 3 u |m_old - m_new|
     (difference, constant, product); the |m_old - m_new| of one row add up to at most 2 S_max.  alpha multiplies O and l alike, so
     this is a common factor on a block's keys in both; it is counted as a per-key weight error all the same.
  Together: every weight w_j = e^(s_j - m) reaches both the numerator and l multiplied by (1 + e_j), |e_j| <= E with
     E = expm1(D) + 6 u S_max + 2^-22 + nb 2^-22 + 6 u S_max.
  5. P is rounded to 16 bits for P.V but not for l: a relative u16 on each numerator weight, and where the weight is below the
     format's smallest normal (2^-14 for fp16; 2^-126 for bf16, where ex2.ftz already flushes) an absolute error of at most
     min(half the subnormal spacing, the weight itself) -- 2^-25 for fp16, 2^-126 for bf16.  Rescales (alpha <= 1) only shrink it
     and a weight that is subnormal when rounded is subnormal at the final max as well, so in final-max units:
     P_abs = sum over keys with w_j < min normal of min(tiny, w_j) |v_j|.
  With numerator N' = sum w_j (1 + e_j + r_j) v_j (+ P_abs) and denominator l' = sum w_j (1 + e'_j):
     |N'/l' - O| <= ((2 E + u16) A + P_abs / l) / (1 - E).
  6. The sums.  O: per block one rescale rounding and a k16 step of P.V per 16 keys into fp32, i.e. (2 kend/16 + 4 + nb) u
     sum |p v| (<= 1.01 A l).  l: per thread and block 32 keys summed in sequence at 128-key blocks (17 roundings deep: one pair,
     16 chained adds; 16 keys and 9 deep at 64-key blocks, which the 17-deep term covers), then one multiply and one add per block,
     then 2 shuffles: (19 + 2 nb) u relative.
  7. 1/l (correctly rounded; 2^-23 even for an approximate reciprocal) and o * (1/l): 3 u |O'|.
  8. The final 16-bit rounding: u16 |O'| (fp16 outputs below 2^-14: + 2^-25).
The bound is the sum of 5-8, with O' = |O| + the error before step 8, and 1 % on top for second-order products (every term is far
below 1, so their products are far below 1 % of the sum)."""
import numpy as np

U = 2.0 ** -24
U16 = {1: 2.0 ** -8, 0: 2.0 ** -11}             # operand_bf16 -> unit roundoff
MIN_NORMAL = {1: 2.0 ** -126, 0: 2.0 ** -14}
TINY = {1: 2.0 ** -126, 0: 2.0 ** -25}
EX2 = 2.0 ** -22
AG, AK = 64, 128                                # query rows per group, keys per block (csrc/attention_tc.cu)


def keys_per_block(dh):
    """K3's key block at head_dim dh: 64 keys at 104 (a three-stage ring of 64-key blocks), 128 otherwise"""
    return 64 if dh == 104 else AK


def bf16(x):
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(np.uint32).view(np.float32)


def round16(x, bf):
    """float32 values rounded once (to nearest even) to the 16-bit type, returned as float32"""
    x = np.asarray(x, np.float32)
    return bf16(x) if bf else x.astype(np.float16).astype(np.float32)


def kend_of_rows(rows, T, causal):
    """the keys a row's 64-row group visits: T, or up to the end of the group's diagonal block"""
    rows = np.asarray(rows)
    return np.minimum(T, (rows // AG + 1) * AG) if causal else np.full(rows.shape, T)


def reference_rows(q, k, v, rows, causal, bf, kb=AK):
    """fp64 attention of query rows `rows` over every key they see, and the element-wise bound of the module docstring for a
    kernel of kb-key blocks.  q, k: [T, dh] and v: [T, dv] of values exact in the 16-bit type (Q already scaled); dh counts the
    k16 steps of S, so at head_dim 104 q and k come padded to 112 columns and v does not.  Returns (O [R, dv], bound [R, dv])."""
    rows = np.asarray(rows)
    if len(rows) > 128:                         # keeps the [rows, T] fp64 intermediates to a few hundred MB at T = 85 265
        parts = [reference_rows(q, k, v, rows[i:i + 128], causal, bf, kb) for i in range(0, len(rows), 128)]
        return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
    T, dh = k.shape
    q = np.asarray(q, np.float64)[rows]
    k = np.asarray(k, np.float64)
    v = np.asarray(v, np.float64)
    s = q @ k.T
    vis = np.ones_like(s, bool) if not causal else np.arange(T)[None, :] <= rows[:, None]
    s = np.where(vis, s, -np.inf)
    m = s.max(-1, keepdims=True)
    w = np.exp(s - m)
    l = w.sum(-1, keepdims=True)
    pi = w / l
    o = pi @ v
    a = pi @ np.abs(v)
    d = (2 * dh / 16 + 4) * U * np.where(vis, np.abs(q) @ np.abs(k).T, 0.0).max(-1, keepdims=True)
    smax = np.where(vis, np.abs(s), 0.0).max(-1, keepdims=True) + d
    kend = kend_of_rows(rows, T, causal)[:, None].astype(np.float64)
    nb = np.ceil(kend / kb)
    e = np.expm1(d) + 12 * U * smax + EX2 * (1 + nb)
    u16 = U16[bf]
    small = w * np.exp(2 * d) < MIN_NORMAL[bf]
    p_abs = np.where(small, np.minimum(TINY[bf], w * np.exp(2 * d)), 0.0) @ np.abs(v)
    pre = ((2 * e + u16) * a + p_abs / l) / (1 - e)
    pre += (2 * np.ceil(kend / 16) + 4 + nb) * U * 1.01 * a + (19 + 2 * nb + 3) * U * (np.abs(o) + pre)
    out_abs = TINY[0] if not bf else 0.0
    bound = 1.01 * (pre + u16 * (np.abs(o) + pre) + out_abs)
    return o, bound


# ---- inputs --------------------------------------------------------------------------------------------------------------------
PATTERNS = ("random", "needle", "ramp", "late_spike", "early_spike")


def needle_key(T, causal):
    """the key each row's query points at: thousands of positions away once T is in the thousands (behind the row when causal)"""
    t = np.arange(T)
    return (t * 7) // 13 if causal else (t + T // 2 + 37 * (t % 11)) % T


def pattern_head(pattern, T, dh, causal, rng):
    """(q, k, v) [T, dh] float32 for one (sequence, head), Q already scaled:
      random       scores of a few units, so a handful of keys carry each row
      needle       q_t = alpha k_pi(t): one key thousands of positions away dominates (score ~ 24 against a max of ~ 13 elsewhere)
      ramp         the score grows by 0.25 per key block of K3 at this head_dim (keys_per_block; exactly, through two integer
                   columns), so every block raises the running maximum and rescales O and l; half a unit more across each block
      late_spike   a score of 60 at key T - 3 (in the last block), small noise elsewhere
      early_spike  a score of 60 at key 2
    """
    sc = 1.0 / np.sqrt(dh)
    v = rng.standard_normal((T, dh)).astype(np.float32)
    if pattern == "random":
        q = rng.standard_normal((T, dh)) * 2.0 * sc
        k = rng.standard_normal((T, dh))
    elif pattern == "needle":
        k = rng.standard_normal((T, dh))
        q = (24.0 / dh) * k[needle_key(T, causal)]
    else:
        q = rng.standard_normal((T, dh)) * 0.05
        k = rng.standard_normal((T, dh)) * 0.05
        j = np.arange(T)
        if pattern == "ramp":
            w = keys_per_block(dh)
            kb = j // w
            q[:, 0], q[:, 1], q[:, 2] = 26 * 0.25, 0.25, 0.5          # powers of two times small integers: exact in 16 bits
            k[:, 0], k[:, 1], k[:, 2] = kb // 26, kb % 26, (j % w) / w
        else:
            q[:, 0] = 1.0
            k[:, 0] = np.where(j == (T - 3 if pattern == "late_spike" else 2), 60.0, 0.0)
    return q.astype(np.float32), k.astype(np.float32), v


def sampled_rows(T, causal, rng, n_random=256):
    """0, T - 1, the 64 / 128 boundaries of the last 1024 rows, group edges (the diagonal blocks when causal) spread over the
    sequence, and random rows"""
    near_end = [b + d for b in range(max(0, T - 1024) // AG * AG, T + 1, AG) for d in (-1, 0)]
    spread = [g * AG + d for g in np.linspace(0, (T - 1) // AG, 48).astype(int) for d in (0, 1, 31, 62, 63)]
    rows = np.array([0, T - 1] + near_end + spread + list(rng.integers(0, T, n_random)))
    return np.unique(rows[(rows >= 0) & (rows < T)])


def exceed(got, want, bound):
    """max over elements of |got - want| / bound (<= 1 passes)"""
    return float((np.abs(np.asarray(got, np.float64) - want) / bound).max())
