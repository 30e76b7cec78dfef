"""K1 in isolation: the fused block-dequant wgmma GEMM through the C-ABI test hook, against a numpy restatement
built on the ORACLE's dequantizer (ggml.c:1496-1606 semantics).  The comparison emulates the kernel's declared
rounding points exactly -- operands rounded to fp16/bf16, fp32 accumulation -- so the tolerance can be tight."""
import ctypes as C

import numpy as np
import pytest

import _epilogue_rule as rule
import oracle as orc

pytestmark = pytest.mark.gpu

QT = {"f16": 1, "q4_0": 2, "q4_1": 3, "q5_0": 6, "q5_1": 7, "q8_0": 8}
EPI_STORE16, EPI_GELU16, EPI_QGELU16, EPI_REDADD32, EPI_STORE32 = range(5)


def round16(a, bf16):
    a = np.asarray(a, np.float32)
    if not bf16:
        return a.astype(np.float16).astype(np.float32)
    u = a.view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) >> 16 << 16
    return u.astype(np.uint32).view(np.float32)


def decode_blocks(qt, raw, N, K):
    """Independent numpy decoder of the ggml block formats (ggml.c:866-911): returns integer quants q [N,K] (with the
    zero point already subtracted for q4_0/q5_0), per-element d and m (fp32 values of the stored fp16 scale / min)."""
    bs = {"q4_0": 18, "q4_1": 20, "q5_0": 22, "q5_1": 24, "q8_0": 34}[qt]
    b = np.frombuffer(raw, np.uint8).reshape(N, K // 32, bs)
    d = b[:, :, 0:2].copy().view(np.float16)[..., 0].astype(np.float32)
    m = np.zeros_like(d)
    o = 2
    if qt in ("q4_1", "q5_1"):
        m = b[:, :, 2:4].copy().view(np.float16)[..., 0].astype(np.float32)
        o = 4
    if qt == "q8_0":
        q = b[:, :, 2:34].copy().view(np.int8).astype(np.int32)
    else:
        qh = np.zeros(d.shape, np.uint32)
        if qt in ("q5_0", "q5_1"):
            qh = b[:, :, o:o + 4].copy().view(np.uint32)[..., 0]
            o += 4
        qs = b[:, :, o:o + 16].astype(np.int32)
        lo, hi = qs & 15, qs >> 4
        j = np.arange(16)
        if qt in ("q5_0", "q5_1"):
            lo = lo | (((qh[..., None] >> j) & 1).astype(np.int32) << 4)
            hi = hi | (((qh[..., None] >> (j + 16)) & 1).astype(np.int32) << 4)
        q = np.concatenate([lo, hi], axis=-1)
        if qt == "q4_0":
            q = q - 8
        if qt == "q5_0":
            q = q - 16
    rep = lambda a: np.repeat(a, 32, axis=1)
    return q.reshape(N, K), rep(d), rep(m)


def make_weight(qt, N, K, rng):
    """returns (raw ggml bytes, decoded (q, d, m) or the fp16 matrix)."""
    w = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
    if qt == "f16":
        return w.astype(np.float16).tobytes(), w.astype(np.float16).astype(np.float32)
    raw = orc.quantize_rows(QT[qt], w)
    q, d, m = decode_blocks(qt, raw, N, K)
    # cross-check the numpy decoder against the oracle's dequantizer (bit-exact)
    deq = np.empty((N, K), np.float32)
    buf = np.frombuffer(raw, np.uint8)
    rs = len(raw) // N
    for r in range(0, N, 17):
        orc.lib().orc_dequantize_row(QT[qt], buf.ctypes.data + r * rs, deq[r].ctypes.data_as(C.POINTER(C.c_float)), K)
        assert np.array_equal(deq[r], (q[r].astype(np.float32) * d[r] + m[r]).astype(np.float32))
    return raw, (q, d, m)


def unpacked(wdesc, bf16):
    """The operand-type weight exactly as the unpack warps build it: scale (and min) converted to the operand type,
    integer part exact, ONE rounding of q*d (+m) to the operand type."""
    if not isinstance(wdesc, tuple):
        return wdesc
    q, d, m = wdesc
    d16, m16 = round16(d, bf16).astype(np.float64), round16(m, bf16).astype(np.float64)
    return round16((q.astype(np.float64) * d16 + m16).astype(np.float32), bf16)


def run_gemm(prod, qt, bf16, M, N, K, epi, x, raw, bias, resid=None, naive=0, scale=0.125):
    """scale: the Q scale EPI_STORE16 applies to the first N/2 features (0.125 = 1/sqrt(64) unless a test asks otherwise)"""
    y = np.empty((M, N), np.float32)
    ms = C.c_float(0)
    fp = C.POINTER(C.c_float)
    buf = np.frombuffer(raw, np.uint8)
    rc = prod.lib.clip_b200_debug_gemm_scaled(QT[qt], int(bf16), M, N, K, epi, naive, scale, x.ctypes.data_as(fp), buf.ctypes.data,
                                              bias.ctypes.data_as(fp) if bias is not None else None,
                                              resid.ctypes.data_as(fp) if resid is not None else None, y.ctypes.data_as(fp),
                                              C.byref(ms))
    assert rc == 0, prod.last_error()
    return y, ms.value


def check_gelu(prod, qt, bf16, M, N, K, epi, x, raw, bias, y):
    """a GELU epilogue's 16-bit result y against the rule of tests/_epilogue_rule.py, at the fp32 value v that EPI_STORE32 gives for
    the same call (the same accumulator: tests/test_gpu_gemm_epilogue_exact.py)"""
    v, _ = run_gemm(prod, qt, bf16, M, N, K, EPI_STORE32, x, raw, bias)
    return rule.check(y, v, "gelu" if epi == EPI_GELU16 else "qgelu", bf16, (qt, M, N, K))


def expected(x, deq, bias, bf16, epi, resid, N):
    xr, wr = round16(x, bf16).astype(np.float64), unpacked(deq, bf16).astype(np.float64)
    acc = (xr @ wr.T).astype(np.float32)
    v = acc + (bias if bias is not None else 0)
    if epi == EPI_STORE32:
        return v
    if epi == EPI_REDADD32:
        return resid + v
    if epi == EPI_GELU16:
        v = 0.5 * v * (1 + np.tanh(0.7978845608 * v * (1 + 0.044715 * v * v)))
    elif epi == EPI_QGELU16:
        v = v / (1 + np.exp(-1.702 * v))
    else:
        v = v.copy()
        v[:, :N // 2] *= 0.125        # the hook scales the first N/2 features, like Q in the fused QKV GEMM
    return round16(v.astype(np.float32), bf16)


CASES = [(qt, bf) for qt in ("q4_0", "q4_1", "q5_0", "q5_1", "q8_0") for bf in (True, False)] + [("f16", False)]


@pytest.mark.parametrize("qt,bf16", CASES)
def test_gemm_all_types_store32(prod, qt, bf16):
    rng = np.random.default_rng(1)
    M, N, K = 300, 256, 192          # ragged token tile (300 = 256 + 44), 2 feature tiles, 3 k-blocks
    raw, deq = make_weight(qt, N, K, rng)
    x = rng.standard_normal((M, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    y, _ = run_gemm(prod, qt, bf16, M, N, K, EPI_STORE32, x, raw, bias)
    ref = expected(x, deq, bias, bf16, EPI_STORE32, None, N)
    err = np.abs(y - ref).max()
    assert err <= 2e-3 * max(1.0, np.abs(ref).max()), (qt, bf16, err)


@pytest.mark.parametrize("epi", [EPI_STORE16, EPI_GELU16, EPI_QGELU16, EPI_REDADD32, EPI_STORE32])
@pytest.mark.parametrize("bf16", [True, False])
def test_gemm_epilogues(prod, epi, bf16):
    rng = np.random.default_rng(2)
    M, N, K = 77, 128, 128
    raw, deq = make_weight("q4_0", N, K, rng)
    x = rng.standard_normal((M, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    resid = rng.standard_normal((M, N)).astype(np.float32)
    y, _ = run_gemm(prod, "q4_0", bf16, M, N, K, epi, x, raw, bias, resid)
    if epi in (EPI_GELU16, EPI_QGELU16):
        check_gelu(prod, "q4_0", bf16, M, N, K, epi, x, raw, bias, y)
    ref = expected(x, deq, bias, bf16, epi, resid, N)
    tol = 2e-2 if epi in (EPI_STORE16, EPI_GELU16, EPI_QGELU16) else 2e-3     # one 16-bit output ulp at |v|~2
    assert np.abs(y - ref).max() <= tol * max(1.0, np.abs(ref).max()), (epi, bf16, np.abs(y - ref).max())


@pytest.mark.parametrize("M", [1, 31, 256, 257, 1000])
def test_gemm_token_tails_and_multi_tile(prod, M):
    rng = np.random.default_rng(3)
    N, K = 384, 256
    raw, deq = make_weight("q8_0", N, K, rng)
    x = rng.standard_normal((M, K)).astype(np.float32)
    y, _ = run_gemm(prod, "q8_0", True, M, N, K, EPI_STORE32, x, raw, None)
    ref = expected(x, deq, None, True, EPI_STORE32, None, N)
    assert np.abs(y - ref).max() <= 2e-3 * max(1.0, np.abs(ref).max())


def test_gemm_matches_scalar_debug_kernel(prod):
    """wgmma path vs the scalar kernel that dequantises straight from ggml-format rows on the device."""
    rng = np.random.default_rng(4)
    M, N, K = 513, 256, 1024
    raw, _ = make_weight("q5_1", N, K, rng)
    x = rng.standard_normal((M, K)).astype(np.float32)
    # fp16 operands: d and m are exact in both kernels, so the two differ only by fp32 summation order
    a, _ = run_gemm(prod, "q5_1", False, M, N, K, EPI_STORE32, x, raw, None)
    b, _ = run_gemm(prod, "q5_1", False, M, N, K, EPI_STORE32, x, raw, None, naive=1)
    assert np.abs(a - b).max() <= 1e-3 * max(1.0, np.abs(b).max())


def test_gemm_large_persistent(prod):
    """More tiles than SMs (persistent loop, ring wrap-around, A-buffer reuse across tiles) at a ViT-L/14 layer shape."""
    rng = np.random.default_rng(5)
    M, N, K = 257 * 40, 1024, 1024
    raw, deq = make_weight("q4_0", N, K, rng)
    x = rng.standard_normal((M, K)).astype(np.float32)
    y, ms = run_gemm(prod, "q4_0", True, M, N, K, EPI_STORE32, x, raw, None)
    ref = expected(x, deq, None, True, EPI_STORE32, None, N)
    assert np.abs(y - ref).max() <= 2e-3 * max(1.0, np.abs(ref).max())
    print("gemm %dx%dx%d q4_0: %.3f ms  %.1f TFLOP/s" % (M, N, K, ms, 2.0 * M * N * K / ms / 1e9))


@pytest.mark.parametrize("qt,bf16", [(qt, bf) for qt in ("q4_0", "q4_1", "q5_0", "q5_1", "q8_0") for bf in (True, False)])
def test_gemm_wide_form_all_types(prod, qt, bf16):
    """Every weight type over more tiles than SMs (each CTA walks several tiles, rings wrap around), with a ragged last token tile."""
    rng = np.random.default_rng(21)
    M, N, K = 37 * 384 + 100, 512, 128           # 4 feature tiles x 74 token tiles = 296 tiles: > 2 per CTA on 132 SMs
    raw, deq = make_weight(qt, N, K, rng)
    x = rng.standard_normal((M, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    y, _ = run_gemm(prod, qt, bf16, M, N, K, EPI_STORE32, x, raw, bias)
    ref = expected(x, deq, bias, bf16, EPI_STORE32, None, N)
    assert np.abs(y - ref).max() <= 2e-3 * max(1.0, np.abs(ref).max()), (qt, bf16)


# ---- f16 weights: the form with both operands in shared memory (X box + W box per stage, a 5-deep ring) -------------------------
# It only takes fp16 activations.  f16 model files use it for every linear layer, and every model uses it for the patch embedding.

@pytest.mark.parametrize("epi", [EPI_STORE16, EPI_GELU16, EPI_QGELU16, EPI_REDADD32, EPI_STORE32])
def test_gemm_f16_weights_epilogues(prod, epi):
    """test_gemm_epilogues with f16 weights: STORE16 with the Q scale on the first N/2 features, both GELUs, the residual add"""
    rng = np.random.default_rng(12)
    M, N, K = 77, 128, 128
    raw, deq = make_weight("f16", N, K, rng)
    x = rng.standard_normal((M, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    resid = rng.standard_normal((M, N)).astype(np.float32)
    y, _ = run_gemm(prod, "f16", False, M, N, K, epi, x, raw, bias, resid)
    if epi in (EPI_GELU16, EPI_QGELU16):
        check_gelu(prod, "f16", False, M, N, K, epi, x, raw, bias, y)
    ref = expected(x, deq, bias, False, epi, resid, N)
    tol = 2e-2 if epi in (EPI_STORE16, EPI_GELU16, EPI_QGELU16) else 2e-3
    assert np.abs(y - ref).max() <= tol * max(1.0, np.abs(ref).max()), (epi, np.abs(y - ref).max())


def padded_f16_case(rng, M, N, K, K_real):
    """x and an f16 weight whose columns K_real..K are zero, as the patch embedding pads 3 P^2 up to kpad (make_linear)"""
    w = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
    x = rng.standard_normal((M, K)).astype(np.float32)
    w[:, K_real:] = 0
    x[:, K_real:] = 0
    return x, w.tobytes(), w.astype(np.float32)


@pytest.mark.parametrize("K,K_real", [(128, 128), (640, 588)], ids=["K128", "K640-patch14"])
def test_gemm_f16_weights_many_tiles(prod, K, K_real):
    """4 feature tiles x 75 token tiles (the last one ragged) = 300 tiles over 132 SMs: each CTA walks 2-3 tiles, so the ring's
    stage / phase bookkeeping carries across tiles.  K = 640 is the patch-embedding depth of a patch-14 model (588 + zero pad)."""
    rng = np.random.default_rng(K)
    M, N = 37 * 384 + 100, 512
    x, raw, w = padded_f16_case(rng, M, N, K, K_real)
    bias = rng.standard_normal(N).astype(np.float32)
    y, _ = run_gemm(prod, "f16", False, M, N, K, EPI_STORE32, x, raw, bias)
    ref = expected(x, w, bias, False, EPI_STORE32, None, N)
    assert np.abs(y - ref).max() <= 2e-3 * max(1.0, np.abs(ref).max()), K


# Bound at K = 5120 (the FC2 depth of a 1280-wide tower).  The reference is the fp64 product of the rounded operands, so only the
# kernel's fp32 accumulation differs: the tensor core sums each 16-deep k-step, and the accumulator adds K/16 = 320 of them in
# sequence, so |err| <= (320 + 4) u sum_k |x_k w_k|, u = 2^-24.  With |x| ~ N(0, 1) and |w| ~ 0.05 N(0, 1):
# sum_k |x_k w_k| ~ 0.8 * 0.04 K = 163 while max |ref| >= ~3.5 sqrt(K) 0.05 = 12.5, so err / max|ref| <= 2.6e-4 in the worst case --
# the 2e-3 bound used everywhere in this file still holds with room to spare.

def test_gemm_f16_weights_deep_k(prod):
    """K = 5120: 80 k-blocks, so the 5-stage ring wraps 16 times inside every tile"""
    rng = np.random.default_rng(5120)
    M, N, K = 1000, 512, 5120
    raw, deq = make_weight("f16", N, K, rng)
    x = rng.standard_normal((M, K)).astype(np.float32)
    y, _ = run_gemm(prod, "f16", False, M, N, K, EPI_STORE32, x, raw, None)
    ref = expected(x, deq, None, False, EPI_STORE32, None, N)
    assert np.abs(y - ref).max() <= 2e-3 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("epi", [EPI_STORE16, EPI_REDADD32])
def test_gemm_f16_weights_single_token(prod, epi):
    """M = 1: one token row in a 192-row tile, the rest zero-filled by the TMA"""
    rng = np.random.default_rng(1)
    M, N, K = 1, 256, 640
    raw, deq = make_weight("f16", N, K, rng)
    x = rng.standard_normal((M, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    resid = rng.standard_normal((M, N)).astype(np.float32)
    y, _ = run_gemm(prod, "f16", False, M, N, K, epi, x, raw, bias, resid)
    ref = expected(x, deq, bias, False, epi, resid, N)
    tol = 2e-2 if epi == EPI_STORE16 else 2e-3
    assert np.abs(y - ref).max() <= tol * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("K,M", [(64, 333), (5120, 1000)], ids=["K64", "K5120"])
@pytest.mark.parametrize("qt,bf16", [(qt, bf) for qt in ("q4_0", "q4_1", "q5_0", "q5_1", "q8_0") for bf in (True, False)])
def test_gemm_k_depth_edges(prod, qt, bf16, K, M):
    """K = 64 is a single k-block: only the tail kblock() after the paired loop runs.  K = 5120 is the FC2 depth of a 1280-wide
    tower: the packed-weight and X rings wrap many times inside each tile (bound: see the note above test_gemm_f16_weights_deep_k)."""
    rng = np.random.default_rng(K + M)
    N = 256
    raw, deq = make_weight(qt, N, K, rng)
    x = rng.standard_normal((M, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    y, _ = run_gemm(prod, qt, bf16, M, N, K, EPI_STORE32, x, raw, bias)
    ref = expected(x, deq, bias, bf16, EPI_STORE32, None, N)
    assert np.abs(y - ref).max() <= 2e-3 * max(1.0, np.abs(ref).max()), (qt, bf16, K)


@pytest.mark.parametrize("M", [74 * 384, 74 * 384 + 1, 75 * 384 - 191, 75 * 384 + 193, 111 * 384 + 7])
@pytest.mark.parametrize("epi", [EPI_STORE16, EPI_QGELU16, EPI_REDADD32])
def test_gemm_wide_form_tails_and_epilogues(prod, M, epi):
    """many token tiles: exact multiples of the tile, one extra row, ragged last tiles, partial last waves; 16-bit and residual epilogues"""
    rng = np.random.default_rng(M)
    N, K = 256, 192
    raw, deq = make_weight("q4_0", N, K, rng)
    x = rng.standard_normal((M, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    resid = rng.standard_normal((M, N)).astype(np.float32)
    y, _ = run_gemm(prod, "q4_0", True, M, N, K, epi, x, raw, bias, resid)
    if epi == EPI_QGELU16:
        check_gelu(prod, "q4_0", True, M, N, K, epi, x, raw, bias, y)
    ref = expected(x, deq, bias, True, epi, resid, N)
    assert np.abs(y - ref).max() <= 2e-2 * max(1.0, np.abs(ref).max())
