"""K1's staged epilogue: values go through a ring of shared-memory slots (32 tokens of 16-bit or 16 tokens of fp32 per chunk) and
leave by bulk tensor stores that clip at row M.  Token counts end at, just before and just after chunk boundaries; N of 768 and 1280
(6 and 10 feature tiles); the two tightest shared-memory plans (q8_0, f16) next to q4_0; 40 token tiles or more, so every CTA walks
several tiles and reuses each slot many times.  The hook fills one token tile past row M of its output with 0xFF and fails (rc 5) if
any of it changes, so every call here also checks that rows past M are never written.

STORE32 is checked against an fp64 restatement; the other epilogues against STORE32 from the same call site: the residual add bit for
bit as x0 + v, the 16-bit store bit for bit as v times the column scale rounded once, the GELUs by the rule of
tests/_epilogue_rule.py at v (one 16-bit ulp where the result is normal)."""
import numpy as np
import pytest

import _epilogue_rule as rule

from test_gpu_gemm import (EPI_GELU16, EPI_QGELU16, EPI_REDADD32, EPI_STORE16, EPI_STORE32, expected, make_weight, round16,
                           run_gemm)

pytestmark = pytest.mark.gpu

K = 128
TAILS = [1, 15, 16, 17, 33, 63, 64, 65, 127, 129, 191, 192]
TYPES = [("q4_0", True), ("q8_0", True), ("q8_0", False), ("f16", False)]


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a, np.float32).view(np.uint32), np.ascontiguousarray(b, np.float32).view(np.uint32))


@pytest.mark.parametrize("tail", TAILS)
@pytest.mark.parametrize("N", [768, 1280])
@pytest.mark.parametrize("qt,bf16", TYPES)
def test_staged_epilogues(prod, qt, bf16, N, tail):
    M = 192 * 39 + tail
    rng = np.random.default_rng(N + tail)
    raw, deq = make_weight(qt, N, K, rng)
    x = rng.standard_normal((M, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    x0 = rng.standard_normal((M, N)).astype(np.float32)

    v, _ = run_gemm(prod, qt, bf16, M, N, K, EPI_STORE32, x, raw, bias)
    ref = expected(x, deq, bias, bf16, EPI_STORE32, None, N)
    assert np.abs(v - ref).max() <= 2e-3 * max(1.0, np.abs(ref).max()), (qt, N, M)

    y, _ = run_gemm(prod, qt, bf16, M, N, K, EPI_REDADD32, x, raw, bias, x0)
    assert same_bits(y, x0 + v), (qt, N, M)

    y, _ = run_gemm(prod, qt, bf16, M, N, K, EPI_STORE16, x, raw, bias)
    s = v.copy()
    s[:, :N // 2] *= np.float32(0.125)   # the hook's Q scale on the first N/2 features: a power of two, exact
    assert same_bits(y, round16(s, bf16)), (qt, N, M)

    for fn, epi in (("gelu", EPI_GELU16), ("qgelu", EPI_QGELU16)):
        y, _ = run_gemm(prod, qt, bf16, M, N, K, epi, x, raw, bias)
        rule.check(y, v, fn, bf16, (qt, N, M))
