"""K1's 16-bit epilogues at every input they can see.  The weight is two stacked 128 x 128 identities (N = 256, K = 128), so feature n
reads input k = n % 128 with weight 1: every product but one is an exact zero and the accumulator is the 16-bit input itself.  The
first 128 features carry the hook's Q scale, the other 128 do not.

  * every finite 16-bit input (128 columns x ~500 rows), GELU16 and QGELU16 against the rule of tests/_epilogue_rule.py;
  * fp32 inputs between the 16-bit points and in the tails: per-feature biases make z = fl(x + b) dense in [-40, 40], put it where
    the GELU's cubic term overflows fp32 (|z| ~ 1e12 .. 1e14), and out to 1e30 in magnitude.  z is EPI_STORE32's result for the same
    call, and equals fl(x + b) bit for bit;
  * EPI_STORE16 bit for bit as RNE16(fl(fl(z) s)) on the scaled features for s = 0.125 and s = fl(1/sqrt(80)), RNE16(z) on the
    others, with inputs where the single-FMA form fma(x, s, fl(b s)) rounds to another 16-bit value, so the two orders differ.

Three weight / operand pairings (separate kernel instantiations: the f16-weight form, q8_0 with bf16 and with fp16 operands), each
on the wgmma kernel and on the scalar debug kernel (which runs common.cuh's GELUs directly)."""
import numpy as np
import pytest

import _epilogue_rule as rule
from _util import fmaf32
from test_gpu_gemm import EPI_GELU16, EPI_QGELU16, EPI_STORE16, EPI_STORE32, decode_blocks, run_gemm, unpacked

pytestmark = pytest.mark.gpu

N, K = 256, 128
FORMS = [("f16", False), ("q8_0", True), ("q8_0", False)]
KERNELS = [0, 1]                               # use_naive
S80 = float(np.float32(1.0 / np.sqrt(80.0)))
F32 = np.float32


def identity_weight(qt, bf16):
    """raw ggml rows of the stacked identities; q8_0 blocks are written with d = 1 and q = 1 on the diagonal, so that the
    unpacked operand-type weight is exactly 1 (a quantizer would store d = fp16(1/127), q = 127: 0.99994)"""
    w = np.zeros((N, K), np.float32)
    w[np.arange(N), np.arange(N) % K] = 1.0
    if qt == "f16":
        return w.astype(np.float16).tobytes()
    blk = np.zeros((N, K // 32, 34), np.uint8)
    blk[:, :, 0:2] = np.frombuffer(np.float16(1.0).tobytes(), np.uint8)
    blk[:, :, 2:] = w.reshape(N, K // 32, 32).astype(np.int8).view(np.uint8)
    raw = blk.tobytes()
    assert np.array_equal(unpacked(decode_blocks(qt, raw, N, K), bf16), w)
    return raw


def as16(a, bf16):
    return rule.round16(np.asarray(a, np.float32), bf16)


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a, np.float32).view(np.uint32), np.ascontiguousarray(b, np.float32).view(np.uint32))


def run_all(qt, bf16, naive, prod, x, bias):
    """z from EPI_STORE32 and the 16-bit outputs of the other epilogues, all for the same x and bias"""
    raw = identity_weight(qt, bf16)
    M = x.shape[0]
    xx = np.concatenate([x, np.zeros((M, K - x.shape[1]), F32)], 1) if x.shape[1] < K else x
    go = lambda epi, s=0.125: run_gemm(prod, qt, bf16, M, N, K, epi, xx, raw, bias, naive=naive, scale=s)[0]
    return go(EPI_STORE32), {"gelu": go(EPI_GELU16), "qgelu": go(EPI_QGELU16), 0.125: go(EPI_STORE16), S80: go(EPI_STORE16, S80)}


def check_store16(out, z, s, bf16, what):
    want = z.copy()
    want[:, :N // 2] = (z[:, :N // 2] * F32(s)).astype(F32)
    assert same_bits(out, as16(want, bf16)), (what, s)


# ---- every finite 16-bit input ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("naive", KERNELS, ids=["wgmma", "naive"])
@pytest.mark.parametrize("qt,bf16", FORMS)
def test_every_16bit_input(prod, qt, bf16, naive):
    v = rule.finite16(bf16)
    rows = -(-v.size // K)
    x = np.concatenate([v, np.zeros(rows * K - v.size, F32)]).reshape(rows, K)
    z, out = run_all(qt, bf16, naive, prod, x, None)
    xz = np.concatenate([x, x], 1)
    # the accumulator is the input: exactly, but for bf16 inputs below the smallest fp32 normal, which may arrive as 0
    sub = (xz != 0) & (np.abs(xz) < np.finfo(F32).tiny)
    assert np.all((z == xz) | (sub & (z == 0))), (qt, bf16, naive)
    what = (qt, "naive" if naive else "wgmma", "all 16-bit inputs")
    for fn in ("gelu", "qgelu"):
        rule.check(out[fn], z, fn, bf16, what)
    for s in (0.125, S80):
        check_store16(out[s], z, s, bf16, what)


# ---- fp32 inputs: dense, where the cubic overflows, far tails; and the Q-scale order ------------------------------------------
DENSE, CUBE, FAR = slice(0, 64), slice(64, 96), slice(96, 128)      # input columns k, and features k and k + 128


def order_differs(x, b, s, bf16):
    """inputs (x, b) where RNE16(fl(fl(x + b) s)) and RNE16(fma(x, s, fl(b s))) are different 16-bit values"""
    x, b = np.asarray(x, F32), np.asarray(b, F32)
    two_step = (((x + b).astype(F32)) * F32(s)).astype(F32)
    one_fma = fmaf32(x, F32(s), (b * F32(s)).astype(F32))
    return as16(two_step, bf16) != as16(one_fma, bf16)


def split_near_midpoint(rng, s, bf16):
    """(x, b) with x a 16-bit value and b = z - x exact, where z s lies within a few fp32 ulps of a 16-bit rounding midpoint and the
    two Q-scale orders round to different 16-bit values"""
    cand = rule.finite16(bf16)
    while True:
        v = float(as16(rng.uniform(0.3, 2.0), bf16)[()])
        m = v + rule.ulp16(v, bf16) / 2                             # a midpoint between two 16-bit values: exact in fp32
        z0 = F32(m / s)
        for j in range(-3, 4):
            z = F32(z0 + F32(j) * np.spacing(z0))
            x = cand[(cand >= z / 2) & (cand <= z)]                  # Sterbenz: z - x is exact
            b = (z - x).astype(F32)
            hit = np.flatnonzero(order_differs(x, b, s, bf16))
            if hit.size:
                sign = F32(1 if rng.integers(0, 2) else -1)
                return sign * x[hit[0]], sign * b[hit[0]]


def fp32_inputs(bf16, seed):
    """x [512, 128] of 16-bit values and bias [256] fp32.  Dense columns: x uniform in [-20, 20]; on the scaled features b comes
    from split_near_midpoint (|b| < 20, full fp32 mantissa), on the others b is uniform in [-20, 20].  The first rows of each
    dense column hold its split x and the other 16-bit inputs in [-40, 40] for which the two Q-scale orders at s = fl(1/sqrt(80))
    round to different 16-bit values.  Cube columns: b = +-10^[12, 14] (x (1 + 0.044715 x^2) overflows fp32 from about 7e12).
    Far columns: b = +-10^[0, 30]."""
    rng = np.random.default_rng(seed)
    M = 512
    x = as16(rng.uniform(-20, 20, (M, K)), bf16)
    x[:, CUBE.start:] = as16(rng.uniform(-2, 2, (M, FAR.stop - CUBE.start)), bf16)
    b = np.empty(N, F32)
    for half in (0, K):
        b[half + DENSE.start:half + DENSE.stop] = rng.uniform(-20, 20, DENSE.stop - DENSE.start)
        sign = np.where(rng.integers(0, 2, K) == 1, 1.0, -1.0)
        b[half + CUBE.start:half + CUBE.stop] = (sign[CUBE] * 10.0 ** rng.uniform(12, 14, CUBE.stop - CUBE.start))
        b[half + FAR.start:half + FAR.stop] = (sign[FAR] * 10.0 ** rng.uniform(0, 30, FAR.stop - FAR.start))
    cand = rule.finite16(bf16)
    cand = cand[np.abs(cand) <= 40]
    for k in range(DENSE.start, DENSE.stop):
        x0, b[k] = split_near_midpoint(rng, S80, bf16)
        hit = np.concatenate([[x0], cand[order_differs(cand, b[k], S80, bf16)]])[:M // 4]
        x[:hit.size, k] = hit
    return x, b


@pytest.mark.parametrize("naive", KERNELS, ids=["wgmma", "naive"])
@pytest.mark.parametrize("qt,bf16", FORMS)
def test_fp32_inputs_tails_and_q_scale(prod, qt, bf16, naive):
    x, b = fp32_inputs(bf16, 11 + bf16)
    z, out = run_all(qt, bf16, naive, prod, x, b)
    xz = np.concatenate([x, x], 1)
    assert same_bits(z, (xz + b).astype(F32)), (qt, bf16, naive)           # z = fl(x + b): one fp32 add of an exact accumulator
    assert np.abs(z).max() > 1e29 and np.count_nonzero((np.abs(z) > 7e12) & (np.abs(z) < 1e14)) > 1000
    what = (qt, "naive" if naive else "wgmma", "fp32 inputs")
    for fn in ("gelu", "qgelu"):
        rule.check(out[fn], z, fn, bf16, what)
    for s in (0.125, S80):
        check_store16(out[s], z, s, bf16, what)
    # the sweep tells the two orders apart at 1/sqrt(80) (for 0.125, a power of two, they agree)
    differs = order_differs(xz[:, :N // 2], b[:N // 2], S80, bf16)
    assert np.count_nonzero(differs) >= 32, (qt, bf16, np.count_nonzero(differs))
    assert not np.any(order_differs(xz[:, :N // 2], b[:N // 2], 0.125, bf16))
