"""K9, the attention-probability kernel behind CLIP_B200_TOKENS_ATTENTION, through the C-ABI test hook clip_b200_debug_attention_probs:
against an fp64 softmax of the 16-bit-rounded Q and K within the bound derived in tests/_attention_probs_bound.py, at sequence lengths
that end a 64-row group or a 128-key block early, exactly or one past it, several sequences per launch (so groups end mid-sequence),
one to sixteen heads, head_dim 64 and 80, both operand types.  Rows sum to 1 within the bound, causal entries above the diagonal are
+0 bit for bit, the 16-bit outputs are the RNE of the f32 output bit for bit, the CLS row equals row 0 of the full map bit for bit,
and the guard bytes after the output stay untouched (the hook returns 5 otherwise).

At the lengths any-resolution images and long text contexts reach (full maps at T = 2049 causal and 4097, CLS rows up to
T = 85 265, where one (sequence, head) runs hundreds of 128-key blocks twice), at head_dim 64, 80 and 104:
  1. Counting: Q = 0, so every score is exactly 0, every weight ex2(0) = 1 and l an exact key count (below 2^24, so exact in fp32
     whatever the order of the sums).  Every visible entry of row t is then fl(1 / l) bit for bit, l = T (t + 1 when causal), every
     masked entry +0, and the 16-bit outputs the RNE of that.  Every element of every row.
  2. The score patterns of tests/_attention_bound.py, one per (sequence, head), against fp64 on sampled rows of the full maps
     and on the CLS row, within the bound of tests/_attention_probs_bound.py."""
import ctypes as C

import numpy as np
import pytest

from _attention_bound import PATTERNS, pattern_head, sampled_rows
from _attention_probs_bound import exceed, reference_probs, round16

pytestmark = pytest.mark.gpu

CASES = [(1, 0), (2, 0), (17, 0), (50, 0), (64, 0), (65, 0), (77, 1), (128, 0), (129, 0), (257, 0), (577, 0), (1025, 0), (129, 1), (257, 1)]
HEADS = (1, 3, 16)


def run(prod, qkv, bf, nseq, T, H, dh, causal, cls_row, out_type):
    qkv = np.ascontiguousarray(qkv, np.float32)
    out = np.empty((nseq, H, 1 if cls_row else T, T), np.float32 if out_type == 0 else np.uint16)
    rc = prod.lib.clip_b200_debug_attention_probs(bf, nseq, T, H, dh, causal, cls_row, out_type, qkv.ctypes.data_as(C.POINTER(C.c_float)),
                                                  out.ctypes.data)
    assert rc == 0, (rc, prod.last_error())
    return out


def rne16(p32, out_type):
    """the 16-bit patterns (uint16) that round p32 to nearest even in fp16 (1) or bf16 (2)"""
    r = round16(p32, out_type == 2)
    return r.astype(np.float16).view(np.uint16) if out_type == 1 else (r.view(np.uint32) >> 16).astype(np.uint16)


@pytest.mark.parametrize("T,causal", CASES)
@pytest.mark.parametrize("dh", [64, 80])
@pytest.mark.parametrize("bf", [1, 0])
def test_probabilities(prod, T, causal, dh, bf):
    i = CASES.index((T, causal))
    H = HEADS[i % 3] if T < 1025 else 16
    nseq = 1 if T >= 577 else 3
    rng = np.random.default_rng(1000 * T + 10 * dh + bf + causal)
    qkv = rng.standard_normal((nseq * T, 3 * H * dh)).astype(np.float32)
    qkv[:, :H * dh] *= 3.0 / np.sqrt(dh)                    # scaled queries, scores of a few units
    p32 = run(prod, qkv, bf, nseq, T, H, dh, causal, 0, 0)
    x = round16(qkv, bf).reshape(nseq, T, 3, H, dh)
    worst = 0.0
    for s in range(nseq):
        for h in range(H):
            pi, bound = reference_probs(x[s, :, 0, h], x[s, :, 1, h], causal, bf)
            worst = max(worst, exceed(p32[s, h], pi, bound))
            assert abs(p32[s, h].astype(np.float64).sum(-1) - 1.0).max() <= bound.sum(-1).max(), (s, h)
    print("T=%d causal=%d dh=%d bf=%d H=%d: worst |p - pi| / bound = %.3g" % (T, causal, dh, bf, H, worst))
    assert worst <= 1.0
    assert np.isfinite(p32).all()
    if causal:
        above = np.triu(np.ones((T, T), bool), 1)
        assert (p32.view(np.uint32)[:, :, above] == 0).all()
    for ot in (1, 2):
        p16 = run(prod, qkv, bf, nseq, T, H, dh, causal, 0, ot)
        assert np.array_equal(p16, rne16(p32, ot)), ot
    for ot in (0, 1, 2):
        full = p32 if ot == 0 else rne16(p32, ot)
        cls = run(prod, qkv, bf, nseq, T, H, dh, causal, 1, ot)
        assert np.array_equal(cls.view(np.uint8), np.ascontiguousarray(full[:, :, :1]).view(np.uint8)), ot


def test_bad_arguments(prod):
    qkv = np.zeros((5, 3 * 2 * 64), np.float32)
    out = np.zeros(1024, np.float32)
    fp = C.POINTER(C.c_float)
    L = prod.lib
    assert L.clip_b200_debug_attention_probs(1, 1, 5, 2, 88, 0, 0, 0, qkv.ctypes.data_as(fp), out.ctypes.data) == 2
    assert "64 or 80" in prod.last_error()
    assert L.clip_b200_debug_attention_probs(1, 1, 5, 2, 64, 0, 0, 3, qkv.ctypes.data_as(fp), out.ctypes.data) == 2
    assert L.clip_b200_debug_attention_probs(1, 0, 5, 2, 64, 0, 0, 0, qkv.ctypes.data_as(fp), out.ctypes.data) == 2


# ---- long sequences --------------------------------------------------------------------------------------------------------------
NSEQ_L, H_L = 2, 3
LONG_FULL = [(2049, 1), (4097, 0)]
LONG_CLS = [(4097, 0), (16385, 0), (65537, 0), (85265, 0), (4096, 1)]


def kernel_operand(x, dh):
    """Q or K as the kernel multiplies it: at head_dim 104 padded with zeros to 112 columns (7 k16 steps of S)"""
    from test_gpu_attention_probs_hd104 import padded       # imported here: that module imports this one
    return padded(x) if dh == 104 else x


def as_f32(out, out_type):
    """the kernel's output as float32 values: f32 as it is, fp16 or bf16 bit patterns widened"""
    if out_type == 0:
        return out
    return out.view(np.float16).astype(np.float32) if out_type == 1 else (out.astype(np.uint32) << 16).view(np.float32)


@pytest.mark.parametrize("T,causal,cls_row", [(T, c, 0) for T, c in LONG_FULL] + [(T, c, 1) for T, c in LONG_CLS])
@pytest.mark.parametrize("dh", [64, 80, 104])
@pytest.mark.parametrize("bf", [1, 0])
def test_counting_every_element(prod, T, causal, cls_row, dh, bf):
    rng = np.random.default_rng(T + dh + bf)
    qkv = np.zeros((NSEQ_L * T, 3, H_L, dh), np.float32)
    qkv[:, 1] = rng.standard_normal((NSEQ_L * T, H_L, dh))          # K does not matter: every score is 0 * k
    qkv = qkv.reshape(NSEQ_L * T, -1)
    rows = np.arange(1 if cls_row else T)
    l = (rows + 1 if causal else np.full(len(rows), T)).astype(np.float32)
    vis = np.arange(T)[None, :] <= rows[:, None] if causal else np.ones((1, T), bool)
    want = np.where(vis, (np.float32(1) / l)[:, None], np.float32(0)).astype(np.float32)
    for out_type in (0, 1, 2):
        got = run(prod, qkv, bf, NSEQ_L, T, H_L, dh, causal, cls_row, out_type)
        w = want.view(np.uint32) if out_type == 0 else rne16(want, out_type)
        bad = got.view(w.dtype) != w[None, None]
        if bad.any():
            s, h, r, j = (int(x[0]) for x in np.nonzero(bad))
            raise AssertionError("out_type %d: %d of %d entries off; first at sequence %d head %d row %d key %d: %r, want %r (l = %d)" %
                                 (out_type, bad.sum(), bad.size, s, h, r, j, as_f32(got, out_type)[s, h, r, j],
                                  as_f32(want if out_type == 0 else w, out_type)[r, j], l[r]))
    print("T=%d causal=%d cls=%d dh=%d bf=%d: all %d entries exact in every output type" % (T, causal, cls_row, dh, bf, got.size))


def pattern_qkv(T, dh, causal, bf, rng):
    """qkv [NSEQ_L * T, 3 H_L dh] with one pattern of tests/_attention_bound.py per (sequence, head), exact in the operand type"""
    slots = PATTERNS + ("random",)
    qkv = np.zeros((NSEQ_L, T, 3, H_L, dh), np.float32)
    for i, pattern in enumerate(slots):
        q, k, _ = pattern_head(pattern, T, dh, causal, rng)
        qkv[i // H_L, :, 0, i % H_L], qkv[i // H_L, :, 1, i % H_L] = round16(q, bf), round16(k, bf)
    return slots, qkv


@pytest.mark.parametrize("T,causal", LONG_FULL)
@pytest.mark.parametrize("dh", [64, 80, 104])
@pytest.mark.parametrize("bf", [1, 0])
def test_long_maps_against_fp64(prod, T, causal, dh, bf):
    rng = np.random.default_rng(5 * T + dh + bf)
    slots, qkv = pattern_qkv(T, dh, causal, bf, rng)
    flat = qkv.reshape(NSEQ_L * T, -1)
    p32 = run(prod, flat, bf, NSEQ_L, T, H_L, dh, causal, 0, 0)
    assert np.isfinite(p32).all()
    rows = sampled_rows(T, causal, rng)
    for i, pattern in enumerate(slots):
        s, h = i // H_L, i % H_L
        pi, bound = reference_probs(kernel_operand(qkv[s, :, 0, h], dh), kernel_operand(qkv[s, :, 1, h], dh), causal, bf, rows=rows)
        r = exceed(p32[s, h, rows], pi, bound)
        print("T=%d causal=%d dh=%d bf=%d %-11s %d rows  err/bound %.3f" % (T, causal, dh, bf, pattern, len(rows), r))
        assert r <= 1.0, (pattern, r)
    for out_type in (0, 1, 2):
        full = p32 if out_type == 0 else run(prod, flat, bf, NSEQ_L, T, H_L, dh, causal, 0, out_type)
        if out_type:
            assert np.array_equal(full, rne16(p32, out_type)), out_type
        cls = run(prod, flat, bf, NSEQ_L, T, H_L, dh, causal, 1, out_type)
        assert np.array_equal(cls.view(np.uint8), np.ascontiguousarray(full[:, :, :1]).view(np.uint8)), out_type


@pytest.mark.parametrize("T,causal", LONG_CLS)
@pytest.mark.parametrize("dh", [64, 80, 104])
@pytest.mark.parametrize("bf", [1, 0])
def test_long_cls_row_against_fp64(prod, T, causal, dh, bf):
    rng = np.random.default_rng(7 * T + dh + bf)
    slots, qkv = pattern_qkv(T, dh, causal, bf, rng)
    flat = qkv.reshape(NSEQ_L * T, -1)
    cls32 = run(prod, flat, bf, NSEQ_L, T, H_L, dh, causal, 1, 0)
    for out_type in (0, 1, 2):
        cls = cls32 if out_type == 0 else run(prod, flat, bf, NSEQ_L, T, H_L, dh, causal, 1, out_type)
        if out_type:
            assert np.array_equal(cls, rne16(cls32, out_type)), out_type
        for i, pattern in enumerate(slots):
            s, h = i // H_L, i % H_L
            pi, bound = reference_probs(kernel_operand(qkv[s, :, 0, h], dh), kernel_operand(qkv[s, :, 1, h], dh), causal, bf,
                                        out_type, rows=[0])
            r = exceed(as_f32(cls[s, h], out_type), pi, bound)
            print("T=%d causal=%d dh=%d bf=%d out_type=%d %-11s CLS row  err/bound %.3f" % (T, causal, dh, bf, out_type, pattern, r))
            assert r <= 1.0, (pattern, out_type, r)
