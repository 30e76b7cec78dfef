"""K9 (the attention-probability kernel) at head_dim 104 through clip_b200_debug_attention_probs, which lays the unpadded input out as
the loader does (each head padded to 112 columns, the last 8 zero): Q and K reach shared memory as three pieces, columns 0-63, 64-95
and 96-111.  Checked as tests/test_gpu_attention_probs.py checks 64 and 80, within the bound of tests/_attention_probs_bound.py.  The
bound is taken of the operands padded to 112 columns with zeros, which is what the kernel multiplies: its scores take 7 k16 steps."""
import numpy as np
import pytest

from _attention_probs_bound import exceed, reference_probs, round16
from test_gpu_attention_probs import rne16, run

pytestmark = pytest.mark.gpu

DH, DHP = 104, 112
CASES = [(1, 0), (17, 0), (64, 0), (65, 0), (77, 1), (128, 0), (129, 0), (257, 0), (577, 0), (129, 1), (257, 1)]


def padded(x):
    return np.concatenate([x, np.zeros(x.shape[:-1] + (DHP - DH,), x.dtype)], -1)


@pytest.mark.parametrize("T,causal", CASES)
@pytest.mark.parametrize("bf", [1, 0])
def test_probabilities(prod, T, causal, bf):
    H = 16 if T == 257 else 3
    nseq = 1 if T >= 257 else 3
    rng = np.random.default_rng(1000 * T + bf + causal)
    qkv = rng.standard_normal((nseq * T, 3 * H * DH)).astype(np.float32)
    qkv[:, :H * DH] *= 3.0 / np.sqrt(DH)                    # scaled queries, scores of a few units
    p32 = run(prod, qkv, bf, nseq, T, H, DH, causal, 0, 0)
    x = round16(qkv, bf).reshape(nseq, T, 3, H, DH)
    worst = 0.0
    for s in range(nseq):
        for h in range(H):
            pi, bound = reference_probs(padded(x[s, :, 0, h]), padded(x[s, :, 1, h]), causal, bf)
            worst = max(worst, exceed(p32[s, h], pi, bound))
            assert abs(p32[s, h].astype(np.float64).sum(-1) - 1.0).max() <= bound.sum(-1).max(), (s, h)
    print("T=%d causal=%d bf=%d H=%d: worst |p - pi| / bound = %.3g" % (T, causal, bf, H, worst))
    assert worst <= 1.0
    assert np.isfinite(p32).all()
    if causal:
        above = np.triu(np.ones((T, T), bool), 1)
        assert (p32.view(np.uint32)[:, :, above] == 0).all()
    for ot in (1, 2):
        assert np.array_equal(run(prod, qkv, bf, nseq, T, H, DH, causal, 0, ot), rne16(p32, ot)), ot
    for ot in (0, 1, 2):
        full = p32 if ot == 0 else rne16(p32, ot)
        cls = run(prod, qkv, bf, nseq, T, H, DH, causal, 1, ot)
        assert np.array_equal(cls.view(np.uint8), np.ascontiguousarray(full[:, :, :1]).view(np.uint8)), ot


@pytest.mark.parametrize("col", [80, 100])
def test_scores_from_one_piece(prod, col):
    """scores carried by one column of the 64-95 piece or of the 96-103 piece alone, the rest small noise"""
    rng = np.random.default_rng(col)
    nseq, T, H = 2, 257, 2
    qkv = (rng.standard_normal((nseq * T, 3 * H * DH)) * 0.05).astype(np.float32)
    x = qkv.reshape(nseq, T, 3, H, DH)
    x[:, :, 0, :, col] += 1.0
    x[:, :, 1, :, col] += (0.05 * np.arange(T, dtype=np.float32))[None, :, None]
    p32 = run(prod, qkv, 1, nseq, T, H, DH, 0, 0, 0)
    xr = round16(qkv, 1).reshape(nseq, T, 3, H, DH)
    for s in range(nseq):
        for h in range(H):
            pi, bound = reference_probs(padded(xr[s, :, 0, h]), padded(xr[s, :, 1, h]), 0, 1)
            assert exceed(p32[s, h], pi, bound) <= 1.0, (s, h)
