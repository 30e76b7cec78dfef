"""K1's epilogues against each other, bit for bit: the residual add must be exactly x0 + (the fp32 store's value), one fp32
round-to-nearest add with subnormals kept, and the 16-bit store exactly the fp32 store's value times the column scale, rounded once to
the operand type.  Token counts end on partial 192-row tiles, and one spans more than 132 token tiles (CTAs walk several tiles)."""
import numpy as np
import pytest

import oracle as orc
from test_gpu_gemm import EPI_REDADD32, EPI_STORE16, EPI_STORE32, QT, make_weight, round16, run_gemm

pytestmark = pytest.mark.gpu

N, K = 256, 128
MS = [77, 300, 1000, 134 * 192 - 37]
TYPES = [("q4_0", True), ("q8_0", True), ("f16", False)]
# features with all-zero weights and zero bias: their value v = acc + 0 is exactly +0, so x0 + v must give back every x0 bit for bit
# (subnormals kept, -0 turned into +0) -- an add that flushes subnormals to zero fails there.  Both consumer groups, rows f and f + 8.
ZERO_FEATURES = [3, 13, 70, 200]


def weight_with_zero_features(qt, rng):
    w = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
    w[ZERO_FEATURES] = 0.0
    return w.astype(np.float16).tobytes() if qt == "f16" else orc.quantize_rows(QT[qt], w)


def residual(rng, M):
    """mixed magnitudes: ordinary values, subnormals of both signs, signed zeros, and values large enough that x + v rounds"""
    x = rng.standard_normal((M, N)).astype(np.float32)
    kind = rng.integers(0, 5, (M, N))
    sub = (rng.uniform(-1, 1, (M, N)) * 2.0 ** -127).astype(np.float32)       # |sub| < 2^-126: subnormal fp32
    x = np.where(kind == 1, sub, x)
    x = np.where(kind == 2, np.where(rng.integers(0, 2, (M, N)) == 1, np.float32(-0.0), np.float32(0.0)), x)
    x = np.where(kind == 3, (rng.standard_normal((M, N)) * 3e3).astype(np.float32), x)
    x = np.where(kind == 4, (rng.standard_normal((M, N)) * 1e8).astype(np.float32), x)
    x = x.astype(np.float32)
    assert np.count_nonzero((x != 0) & (np.abs(x) < np.finfo(np.float32).tiny)) > 0
    return x


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a, np.float32).view(np.uint32), np.ascontiguousarray(b, np.float32).view(np.uint32))


@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("qt,bf16", TYPES)
def test_redadd_is_one_add_of_store32(prod, qt, bf16, M):
    rng = np.random.default_rng(M + 7)
    raw = weight_with_zero_features(qt, rng)
    x = rng.standard_normal((M, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    bias[ZERO_FEATURES] = 0.0
    x0 = residual(rng, M)
    v, _ = run_gemm(prod, qt, bf16, M, N, K, EPI_STORE32, x, raw, bias)
    y, _ = run_gemm(prod, qt, bf16, M, N, K, EPI_REDADD32, x, raw, bias, x0)
    zc = x0[:, ZERO_FEATURES]
    assert same_bits(v[:, ZERO_FEATURES], np.zeros_like(zc))                             # v == +0 exactly there
    assert np.count_nonzero((zc != 0) & (np.abs(zc) < np.finfo(np.float32).tiny)) > 0   # ... and those x0 hold subnormals
    assert np.count_nonzero(np.signbit(zc) & (zc == 0)) > 0                             # ... and -0
    want = x0 + v                       # numpy: fp32 round-to-nearest, subnormals kept
    bad = np.flatnonzero(y.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, (qt, M, bad.size, bad[:4], y.ravel()[bad[:4]], want.ravel()[bad[:4]])


@pytest.mark.parametrize("M", MS[:3])
@pytest.mark.parametrize("qt,bf16", TYPES)
def test_store16_is_scaled_store32_rounded(prod, qt, bf16, M):
    rng = np.random.default_rng(M + 11)
    raw, _ = make_weight(qt, N, K, rng)
    x = rng.standard_normal((M, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    v, _ = run_gemm(prod, qt, bf16, M, N, K, EPI_STORE32, x, raw, bias)
    y, _ = run_gemm(prod, qt, bf16, M, N, K, EPI_STORE16, x, raw, bias)
    v[:, :N // 2] *= np.float32(0.125)  # the hook's Q scale on the first N/2 features: a power of two, exact
    assert same_bits(y, round16(v, bf16)), (qt, M)
