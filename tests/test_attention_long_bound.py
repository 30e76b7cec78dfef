"""The element-wise bound of tests/_attention_bound.py, checked without a GPU: a numpy emulation of K3's arithmetic
(csrc/attention_tc.cu: key blocks in order -- 128 keys at head_dim 64 and 80, 64 at 104 --, fp32 scores, the running max and its
rescale of O and l, fp32 exp2, P rounded to 16 bits for P.V and kept in fp32 for l, O / l rounded once to 16 bits) must stay within
it at T up to a few thousand, and the same emulation with one fault each -- a key block dropped or counted twice, the causal
diagonal one key off, one block's rescale skipped, the 16-column tail of an 80-wide head read from the next head, and at head_dim
104 a block handed the K / V of three blocks before (the stale stage of a three-stage ring whose parity is wrong) or columns
64-95 or 96-103 read from the next head -- must break it on the inputs that fault shows on."""
import numpy as np
import pytest

from _attention_bound import AK, PATTERNS, exceed, kend_of_rows, keys_per_block, pattern_head, reference_rows, round16, sampled_rows

DHP = {64: 64, 80: 80, 104: 112}                 # the columns S multiplies: head_dim 104 is padded with zeros to 112
# the columns that come from the next head under each "neighbour" fault
NEIGHBOUR = {"tail80": (64, 80), "mid": (64, 96), "tail": (96, 104)}


def padded(x, dh):
    return np.concatenate([x, np.zeros((x.shape[0], DHP[dh] - x.shape[1]), x.dtype)], 1)

LOG2E = np.float32(1.4426950408889634)


def emulate(q, k, v, causal, bf, fault=None, fault_block=None, kb_keys=AK):
    """K3 on one (sequence, head), every row, in blocks of kb_keys keys: q, k, v [T, dh] exact in the 16-bit type.  fault: None,
    "drop", "double", "diagonal" (a row sees one key past itself), "rescale" (block fault_block does not rescale O and l), "stale"
    (block fault_block multiplies the K and V of block fault_block - 3, its keys' positions and masks its own)."""
    T, dh = k.shape
    s_all = (q.astype(np.float64) @ k.T.astype(np.float64)).astype(np.float32)
    rows = np.arange(T)
    nkb = -(-kend_of_rows(rows, T, causal) // kb_keys)
    o = np.zeros((T, dh), np.float32)
    l = np.zeros(T, np.float32)
    m = np.full(T, -np.inf, np.float32)
    fb = fault_block if fault_block is not None else (nkb.max() - 1) // 2
    seen = 1 if fault == "diagonal" else 0
    for kb in range(nkb.max()):
        for rep in range(2 if fault == "double" and kb == fb else 1):
            if fault == "drop" and kb == fb:
                continue
            live = nkb > kb
            keys = np.arange(kb * kb_keys, min(T, (kb + 1) * kb_keys))
            src = keys - 3 * kb_keys if fault == "stale" and kb == fb else keys
            s = s_all[np.ix_(live, src)]
            if causal:
                s = np.where(keys[None, :] <= rows[live, None] + seen, s, np.float32(-np.inf))
            m_new = np.maximum(m[live], s.max(-1))
            with np.errstate(invalid="ignore"):
                alpha = np.exp2(((m[live] - m_new) * LOG2E).astype(np.float32)).astype(np.float32)
            if fault == "rescale" and kb == fb:
                alpha = np.ones_like(alpha)
            mb = (m_new * LOG2E).astype(np.float32)
            p = np.exp2((s * LOG2E).astype(np.float32) - mb[:, None]).astype(np.float32)
            l[live] = (l[live] * alpha).astype(np.float32) + p.sum(-1, dtype=np.float32)
            pv = (round16(p, bf).astype(np.float64) @ v[src].astype(np.float64)).astype(np.float32)
            o[live] = (o[live] * alpha[:, None]).astype(np.float32) + pv
            m[live] = m_new
    inv = (np.float32(1.0) / l).astype(np.float32)
    return round16(o * inv[:, None], bf)


def check(T, dh, causal, bf, pattern, fault=None, neighbour=None, seed=0):
    """the emulation's worst |err| / bound over every row of two heads (head 1 reads columns NEIGHBOUR[neighbour] of K and V
    from head 0 if neighbour is given); the bound is taken at the instance's block width and of the operands S multiplies"""
    rng = np.random.default_rng(seed)
    heads = [pattern_head(pattern, T, dh, causal, rng) for _ in range(2)]
    heads = [tuple(round16(x, bf) for x in h) for h in heads]
    kb = keys_per_block(dh)
    worst = 0.0
    for hh, (q, k, v) in enumerate(heads):
        if neighbour and hh == 1:
            a, b = NEIGHBOUR[neighbour]
            k, v = k.copy(), v.copy()
            k[:, a:b], v[:, a:b] = heads[0][1][:, a:b], heads[0][2][:, a:b]
        got = emulate(q, k, v, causal, bf, fault, kb_keys=kb)
        rows = np.arange(T) if T <= 1024 else sampled_rows(T, causal, rng)
        q0, k0, v0 = heads[hh]
        want, bound = reference_rows(padded(q0, dh), padded(k0, dh), v0, rows, causal, bf, kb)
        worst = max(worst, exceed(got[rows], want, bound))
    return worst


CASES = [(1025, 0), (2305, 0), (248, 1), (1000, 1), (2049, 1)]


@pytest.mark.parametrize("T,causal", CASES)
@pytest.mark.parametrize("dh", [64, 80, 104])
@pytest.mark.parametrize("bf", [1, 0])
@pytest.mark.parametrize("pattern", PATTERNS)
def test_emulated_kernel_meets_the_bound(T, causal, dh, bf, pattern):
    r = check(T, dh, causal, bf, pattern, seed=T + dh + bf)
    print("T=%d causal=%d dh=%d bf=%d %s  err/bound %.3f" % (T, causal, dh, bf, pattern, r))
    assert r <= 1.0, r


# each fault and an input it must show on
FAULTS = [("drop", "random", 0, 1025), ("drop", "needle", 1, 1000), ("double", "random", 0, 1025), ("double", "ramp", 1, 2049),
          ("diagonal", "random", 1, 248), ("diagonal", "needle", 1, 1000), ("rescale", "ramp", 0, 1025), ("rescale", "ramp", 1, 1000),
          ("neighbour", "random", 0, 1025), ("neighbour", "random", 1, 248)]
# head_dim 104: 64-key blocks in a three-stage ring, columns in three pieces.  The diagonal fault is paired with random scores
# only: at 64-key blocks the needle input moves too little under it.
FAULTS_104 = [("stale", "random", 0, 1025), ("stale", "random", 1, 1000), ("stale", "needle", 1, 1000), ("stale", "ramp", 0, 1025),
              ("mid", "random", 0, 1025), ("mid", "random", 1, 248), ("tail", "random", 0, 1025), ("tail", "random", 1, 248),
              ("drop", "random", 0, 1025), ("drop", "needle", 1, 1000), ("double", "random", 0, 1025), ("double", "ramp", 1, 2049),
              ("diagonal", "random", 1, 248), ("rescale", "ramp", 0, 1025), ("rescale", "ramp", 1, 1000)]


def fault_check(fault, pattern, causal, T, bf, dh):
    neighbour = {"neighbour": "tail80", "mid": "mid", "tail": "tail"}.get(fault)
    r = check(T, dh, causal, bf, pattern, None if neighbour else fault, neighbour, seed=T + dh + bf)
    print("%s on %s T=%d causal=%d dh=%d bf=%d  err/bound %.1f" % (fault, pattern, T, causal, dh, bf, r))
    return r


@pytest.mark.parametrize("fault,pattern,causal,T", FAULTS)
@pytest.mark.parametrize("bf", [1, 0])
def test_emulated_faults_break_the_bound(fault, pattern, causal, T, bf):
    r = fault_check(fault, pattern, causal, T, bf, 80 if fault == "neighbour" else 64)
    assert r > 1.0, r


@pytest.mark.parametrize("fault,pattern,causal,T", FAULTS_104)
@pytest.mark.parametrize("bf", [1, 0])
def test_emulated_faults_break_the_bound_at_head_dim_104(fault, pattern, causal, T, bf):
    r = fault_check(fault, pattern, causal, T, bf, 104)
    assert r > 1.0, r


def test_the_bound_is_tight_enough_to_matter():
    """On random scores the bound is a few 16-bit ulps of the row's weighted |v|, not a blanket tolerance: below 2.5 u16 A
    in bf16 at T = 2305 (u16 A from P's rounding, u16 |O| from the output's, the rest far smaller)."""
    rng = np.random.default_rng(1)
    q, k, v = (round16(x, 1) for x in pattern_head("random", 2305, 64, 0, rng))
    rows = sampled_rows(2305, 0, rng)
    o, bound = reference_rows(q, k, v, rows, 0, 1)
    s = q.astype(np.float64)[rows] @ k.T.astype(np.float64)
    p = np.exp(s - s.max(-1, keepdims=True))
    a = (p / p.sum(-1, keepdims=True)) @ np.abs(v.astype(np.float64))
    assert (bound <= 2.5 * 2.0 ** -8 * a).all()
