"""K3 (csrc/attention_tc.cu) at the sequence lengths any-resolution images and long text contexts reach, through the test hook
clip_b200_debug_attention_hd: T up to 85 265 (a 4088 x 4088 image at patch 14), causal T up to 4096 (the longest context_length
the loader takes), at head_dim 64, 80 and 104.  Hundreds of key blocks per group -- 128 keys in a two-stage ring at 64 and 80, 64
keys in a three-stage ring at 104 -- run the ring stages, the running max and the fp32 sums of l and O far past anything the
224 / 336 models reach, with TMA row coordinates far from 0.  nseq = 2 and H = 3 throughout, so that with an odd number of 64-row
groups per head the warpgroup pairs straddle heads.

  1. Counting: Q = 0 and V in {-1, 0, +1}, so every score is exactly 0 and every p exactly 1 (ex2.approx(0) = 1).  O is then an
     exact integer sum and l an exact key count, both below 2^24 and so exact in the fp32 accumulators whatever the summation
     order.  The kernel's output is round16(fl(c fl(1 / l))): two fp32 roundings, each at most 2^-24 relative (the division is
     correctly rounded; even an approximate reciprocal's 1 ulp would give at most 2^-23 + 2^-24), so the fp32 value lies within
     2^-23 (1 + 2^-24) < 2^-22 of c / l, and the one 16-bit rounding of it is round16 of some point of c / l (1 +- 2^-22).  Every
     output row t must lie between round16 of those two ends (c_t the sum of V over the keys row t sees, l_t = t + 1 causal, T
     otherwise); the ends are the same 16-bit value except where c / l is within 2^-22 of a rounding midpoint.  The V columns are
     chosen so that each fault moves outputs by far more than a 16-bit ulp -- see count_v.  Every row, every column.
  2. Scores that matter: random, needle, ramp and spike patterns (tests/_attention_bound.py), one per (sequence, head), against
     fp64 on sampled query rows, at the element-wise bound derived in tests/_attention_bound.py (checked on the CPU against an
     emulation of the kernel and against emulated faults by tests/test_attention_long_bound.py)."""
import numpy as np
import pytest

from _attention_bound import PATTERNS, exceed, keys_per_block, pattern_head, reference_rows, round16, sampled_rows
from test_gpu_attention_hd80 import run
from test_gpu_attention_probs_hd104 import padded

pytestmark = pytest.mark.gpu

NSEQ, H = 2, 3
LONG = [(1025, 0), (2305, 0), (4097, 0), (16385, 0), (65537, 0), (85265, 0), (78, 1), (248, 1), (1000, 1), (2049, 1), (4096, 1)]
# Column kinds: alternating +-1 (prefix sums 0 / +-1, so a causal off-by-one turns 0 into +-1 / (t + 1)); +-1 square waves whose
# periods divide neither 64 nor 128 (a dropped, doubled or misplaced key block changes c_t); a random walk over {-1, 0, +1}; and a
# constant +1 column, whose output must be exactly 1.  Each (sequence, head) draws its own columns, so at head_dim 104 a store of
# the 8 pad columns over the next head's columns 0-7, or a block read from another head's ring slot, shows.
KINDS = ("alt", 3, 5, 7, 127, 129, 1000, "walk", "one")


def count_v(T, dh, seq, head, bf):
    """V [T, dh] of one (sequence, head), seeded by (sequence, head) and with each column's kind and phase its own, so that a
    read across heads or sequences shows"""
    rng = np.random.default_rng((T, dh, seq, head, bf))
    j = np.arange(T)
    v = np.empty((T, dh), np.float32)
    for c in range(dh):
        kind = KINDS[(c + 4 * seq + 7 * head) % len(KINDS)]
        ph = int(rng.integers(0, 1000))
        if kind == "alt":
            v[:, c] = np.where((j + ph) % 2, 1, -1)
        elif kind == "walk":
            v[:, c] = rng.integers(-1, 2, T)
        elif kind == "one":
            v[:, c] = 1
        else:
            v[:, c] = np.where((j + ph) % kind < (kind + 1) // 2, 1, -1)
    return v


def rounding_interval(c, l, bf):
    """the 16-bit values round16 takes on c / l (1 +- 2^-22), as (low, high)"""
    y = c.astype(np.float64) / l.astype(np.float64)
    a = round16((y * (1 - 2.0 ** -22)).astype(np.float32), bf)
    b = round16((y * (1 + 2.0 ** -22)).astype(np.float32), bf)
    return np.minimum(a, b), np.maximum(a, b), round16(y.astype(np.float32), bf)


@pytest.mark.parametrize("T,causal", LONG)
@pytest.mark.parametrize("dh", [64, 80, 104])
@pytest.mark.parametrize("bf", [1, 0])
def test_counting_every_row(prod, T, causal, dh, bf):
    rng = np.random.default_rng(T + dh)
    qkv = np.zeros((NSEQ, T, 3, H, dh), np.float32)
    qkv[:, :, 1] = rng.standard_normal((NSEQ, T, H, dh))          # K does not matter: every score is 0 * k
    for s in range(NSEQ):
        for h in range(H):
            qkv[s, :, 2, h] = count_v(T, dh, s, h, bf)
    got = run(prod, qkv.reshape(NSEQ * T, -1), NSEQ, T, H, causal, bf, dh=dh).reshape(NSEQ, T, H, dh)
    v = qkv[:, :, 2].astype(np.int64)
    c = np.cumsum(v, axis=1) if causal else np.broadcast_to(v.sum(1, keepdims=True), v.shape)
    l = (np.arange(1, T + 1) if causal else np.full(T, T))[None, :, None, None]
    lo, hi, near = rounding_interval(c, np.broadcast_to(l, c.shape), bf)
    bad = ~((got >= lo) & (got <= hi))
    if bad.any():
        s, t, h, d = (int(x[0]) for x in np.nonzero(bad))
        raise AssertionError("%d of %d outputs off; first at sequence %d row %d head %d column %d: %r, want %r (c = %d, l = %d)" %
                             (bad.sum(), bad.size, s, t, h, d, got[s, t, h, d], near[s, t, h, d], c[s, t, h, d], l.ravel()[t]))
    ones = [c_ for c_ in range(dh) if KINDS[(c_ + 4 * 0 + 7 * 0) % len(KINDS)] == "one"]
    assert (got[0, :, 0, ones] == 1.0).all()
    print("T=%d causal=%d dh=%d bf=%d: all %d outputs exact, %d of them on a rounding edge" %
          (T, causal, dh, bf, got.size, int((lo != hi).sum())))


@pytest.mark.parametrize("T,causal", LONG)
@pytest.mark.parametrize("dh", [64, 80, 104])
@pytest.mark.parametrize("bf", [1, 0])
def test_sampled_rows_against_fp64(prod, T, causal, dh, bf):
    rng = np.random.default_rng(3 * T + dh + bf)
    slots = PATTERNS + ("random",)                               # one pattern per (sequence, head)
    qkv = np.empty((NSEQ, T, 3, H, dh), np.float32)
    for i, pattern in enumerate(slots):
        for j, x in enumerate(pattern_head(pattern, T, dh, causal, rng)):
            qkv[i // H, :, j, i % H] = round16(x, bf)
    got = run(prod, qkv.reshape(NSEQ * T, -1), NSEQ, T, H, causal, bf, dh=dh).reshape(NSEQ, T, H, dh)
    assert np.isfinite(got).all()
    rows = sampled_rows(T, causal, rng, 256 if T <= 16385 else 64)       # the fp64 rows cost O(T) each
    # the bound at the instance's key blocks, of the Q and K that S multiplies (head_dim 104: padded to 112 columns, 7 k16 steps)
    pad = padded if dh == 104 else (lambda x: x)
    for i, pattern in enumerate(slots):
        s, h = i // H, i % H
        want, bound = reference_rows(pad(qkv[s, :, 0, h]), pad(qkv[s, :, 1, h]), qkv[s, :, 2, h], rows, causal, bf,
                                     keys_per_block(dh))
        r = exceed(got[s, rows, h], want, bound)
        print("T=%d causal=%d dh=%d bf=%d %-11s %d rows  err/bound %.3f" % (T, causal, dh, bf, pattern, len(rows), r))
        assert r <= 1.0, (pattern, r)
