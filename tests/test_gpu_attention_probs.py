"""K9, the attention-probability kernel behind CLIP_B200_TOKENS_ATTENTION, through the C-ABI test hook clip_b200_debug_attention_probs:
against an fp64 softmax of the 16-bit-rounded Q and K within the bound derived in tests/_attention_probs_bound.py, at sequence lengths
that end a 64-row group or a 128-key block early, exactly or one past it, several sequences per launch (so groups end mid-sequence),
one to sixteen heads, head_dim 64 and 80, both operand types.  Rows sum to 1 within the bound, causal entries above the diagonal are
+0 bit for bit, the 16-bit outputs are the RNE of the f32 output bit for bit, the CLS row equals row 0 of the full map bit for bit,
and the guard bytes after the output stay untouched (the hook returns 5 otherwise)."""
import ctypes as C

import numpy as np
import pytest

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
