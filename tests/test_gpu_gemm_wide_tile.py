"""K1's 128-feature x 256-token tile at its edges: token counts around the 256-row tile and its 128-row half, feature counts of
one and several feature tiles, single and deep k-blocks, every weight type, both operand types and every epilogue, against
test_gpu_gemm.py's numpy restatement and tolerances.  Non-finite activations stay in their own rows, and the hook's guard rows past
M stay intact (the hook fails the call otherwise)."""
import numpy as np
import pytest

from test_gpu_gemm import EPI_GELU16, EPI_QGELU16, EPI_REDADD32, EPI_STORE16, EPI_STORE32, check_gelu, expected, make_weight, run_gemm

pytestmark = pytest.mark.gpu

EPIS = [EPI_STORE16, EPI_GELU16, EPI_QGELU16, EPI_REDADD32, EPI_STORE32]


def tol(epi):
    return 2e-2 if epi in (EPI_STORE16, EPI_GELU16, EPI_QGELU16) else 2e-3     # one 16-bit output ulp at |v|~2


def check(prod, qt, bf16, M, N, K, epi, seed):
    rng = np.random.default_rng(seed)
    raw, deq = make_weight(qt, N, K, rng)
    x = rng.standard_normal((M, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    resid = rng.standard_normal((M, N)).astype(np.float32) if epi == EPI_REDADD32 else None
    y, _ = run_gemm(prod, qt, bf16, M, N, K, epi, x, raw, bias, resid)
    if epi in (EPI_GELU16, EPI_QGELU16):
        check_gelu(prod, qt, bf16, M, N, K, epi, x, raw, bias, y)
    ref = expected(x, deq, bias, bf16, epi, resid, N)
    err = np.abs(y - ref).max()
    assert err <= tol(epi) * max(1.0, np.abs(ref).max()), (qt, bf16, M, N, K, epi, err)


# 40 * 256 + 5 rows = 41 token tiles x 5 feature tiles (N = 640) = 205 tiles: CTAs walk one or two tiles, and since 132 % 5 = 2 the
# tiles of one CTA fall in different feature tiles
@pytest.mark.parametrize("M", [1, 127, 128, 129, 255, 256, 257, 511, 513, 40 * 256 + 5])
@pytest.mark.parametrize("epi", [EPI_STORE16, EPI_REDADD32, EPI_STORE32])
def test_wide_tile_token_edges(prod, M, epi):
    check(prod, "q4_0", True, M, 640, 128, epi, M + epi)


@pytest.mark.parametrize("K", [64, 128, 4096])
@pytest.mark.parametrize("N", [128, 384, 1664])
def test_wide_tile_feature_and_depth_edges(prod, N, K):
    """N = 128: one feature tile; 384 and 1664 (ViT-bigG/14's width): an odd count.  K = 64 is one k-block, K = 4096 wraps every ring
    many times inside a tile."""
    check(prod, "q4_0", True, 257, N, K, EPI_STORE32, N + K)


@pytest.mark.parametrize("qt,bf16", [(qt, bf) for qt in ("q4_0", "q4_1", "q5_0", "q5_1", "q8_0") for bf in (True, False)]
                         + [("f16", False)])
def test_wide_tile_all_types(prod, qt, bf16):
    """every weight type over more tiles than SMs (3 feature x 53 token tiles), 3 k-blocks, a ragged last token tile"""
    check(prod, qt, bf16, 52 * 256 + 77, 384, 192, EPI_STORE32, 7)


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("qt,bf16", [("q4_0", True), ("q4_0", False), ("q8_0", True), ("f16", False)])
def test_wide_tile_epilogues(prod, qt, bf16, epi):
    """every epilogue on a full and a ragged token tile; the residual add has more x chunks per tile than staging slots"""
    check(prod, qt, bf16, 513, 384, 128, epi, 11 + epi)


@pytest.mark.parametrize("qt,bf16", [("q4_0", True), ("q8_0", False), ("f16", False)])
def test_wide_tile_nonfinite_rows(prod, qt, bf16):
    """Row 3 carries +Inf at k = 5 and row 7 NaN at k = 9.  The outputs are the restatement's: row 7 NaN, row 3 sign(w[n, 5]) Inf
    (NaN where w[n, 5] = 0), the other rows finite and within tolerance."""
    rng = np.random.default_rng(384)
    M, N, K = 200, 384, 128
    raw, deq = make_weight(qt, N, K, rng)
    x = rng.standard_normal((M, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    x[3, 5], x[7, 9] = np.inf, np.nan
    y, _ = run_gemm(prod, qt, bf16, M, N, K, EPI_STORE32, x, raw, bias)
    assert np.isnan(y[7]).all()
    w5 = expected(np.eye(K, dtype=np.float32)[5:6], deq, None, bf16, EPI_STORE32, None, N)[0]   # the operand-type w[:, 5]
    want3 = np.where(w5 > 0, np.inf, np.where(w5 < 0, -np.inf, np.nan))
    assert np.array_equal(y[3], want3, equal_nan=True)
    live = np.ones(M, bool)
    live[[3, 7]] = False
    xf = x.copy()
    xf[~live] = 0
    ref = expected(xf, deq, bias, bf16, EPI_STORE32, None, N)
    assert np.isfinite(y[live]).all()
    assert np.abs(y[live] - ref[live]).max() <= 2e-3 * max(1.0, np.abs(ref[live]).max())
