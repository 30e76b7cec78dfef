"""K1's two activation epilogues (EPI_GELU16, EPI_QGELU16; csrc/common.cuh gelu_tanh / gelu_quick) and the rule a 16-bit result
must meet.  Shared by the GPU sweep (tests/test_gpu_gemm_epilogue_sweep.py), the GELU checks of tests/test_gpu_gemm.py and
tests/test_gpu_gemm_epilogue_staging.py, and the CPU test that shows what the rule accepts and rejects (tests/test_epilogue_rule.py).

References, in fp64, of the fp32 value z the epilogue sees:
    GELU(z)  = 0.5 z (1 + tanh(sqrt(2/pi) (z + 0.044715 z^3)))     evaluated as z / (1 + exp(-2u)), the same function: 1 + tanh
    QGELU(z) = z / (1 + exp(-1.702 z))                               cancels in fp64 too once tanh(u) rounds to -1 (z < -5.7)

Rule for a 16-bit result y against the reference r:
    RNE16(r) = +-inf                 y equals it;
    |r| >= smallest normal           |y - r| <= one ulp of the 16-bit type at r;
    |r| <  smallest normal           |y| <= smallest normal, and y is not of the opposite sign (0 of either sign is allowed).
A correctly rounded result is within half an ulp; the other half covers an fp32 evaluation with a relative error up to about
2^-13, where an ulp is at least 2^-11 |r| (fp16) or 2^-8 |r| (bf16)."""
import numpy as np

# (precision p in bits, exponent of the smallest normal, exponent of the largest binade)
FMT = {False: (11, -14, 15), True: (8, -126, 127)}
SQRT_2_OVER_PI = np.sqrt(2.0 / np.pi)


def gelu64(z):
    z = np.asarray(z, np.float64)
    u = SQRT_2_OVER_PI * (z + 0.044715 * z ** 3)
    with np.errstate(over="ignore"):
        return z / (1.0 + np.exp(-2.0 * u))


def qgelu64(z):
    z = np.asarray(z, np.float64)
    with np.errstate(over="ignore"):
        return z / (1.0 + np.exp(-1.702 * z))


REF = {"gelu": gelu64, "qgelu": qgelu64}


def tiny16(bf16):
    return 2.0 ** FMT[bf16][1]


def ulp16(r, bf16):
    """one ulp of the 16-bit type at |r| (fp64; the subnormal spacing below the smallest normal)"""
    p, emin, _ = FMT[bf16]
    _, e = np.frexp(np.abs(np.asarray(r, np.float64)))       # |r| = m 2^e, 0.5 <= m < 1
    return np.ldexp(1.0, np.maximum(e - 1, emin) - (p - 1))


def rne16(r, bf16):
    """fp64 values rounded once, to nearest even, to the 16-bit type (+-inf past its range), as fp64"""
    p, _, emax = FMT[bf16]
    r = np.asarray(r, np.float64)
    q = ulp16(r, bf16)
    y = np.rint(r / q) * q
    big = np.abs(y) > (2.0 - 2.0 ** (1 - p)) * 2.0 ** emax
    return np.where(big, np.copysign(np.inf, r), y)


def round16(a, bf16):
    """float32 values rounded once to the 16-bit type, as float32 (what the hook returns for a 16-bit output)"""
    return rne16(np.asarray(a, np.float32).astype(np.float64), bf16).astype(np.float32)


def accepts(y, r, bf16):
    """boolean mask: the 16-bit results y (float32 or fp64 values) meet the rule against the fp64 references r"""
    y = np.asarray(y, np.float64)
    r = np.asarray(r, np.float64)
    t = tiny16(bf16)
    inf = np.isinf(rne16(r, bf16))
    with np.errstate(invalid="ignore"):
        normal = np.abs(y - r) <= ulp16(r, bf16)
        small = (np.abs(y) <= t) & (y * r >= 0)
    return np.where(inf, y == rne16(r, bf16), np.where(np.abs(r) >= t, normal, small))


def ulp_error(y, r, bf16):
    """|y - r| in ulps of the 16-bit type at r, where |r| is at least the smallest normal and RNE16(r) is finite; 0 elsewhere"""
    y = np.asarray(y, np.float64)
    r = np.asarray(r, np.float64)
    m = (np.abs(r) >= tiny16(bf16)) & np.isfinite(rne16(r, bf16))
    with np.errstate(invalid="ignore"):
        return np.where(m, np.abs(y - r) / ulp16(r, bf16), 0.0)


def check(y, z, fn, bf16, what=""):
    """assert the rule for 16-bit results y of the epilogue fn ('gelu' or 'qgelu') at fp32 inputs z; returns the worst ulp error"""
    z = np.asarray(z, np.float32)
    r = REF[fn](z.astype(np.float64))
    ok = accepts(y, r, bf16)
    bad = np.flatnonzero(~ok.ravel())
    worst = float(ulp_error(y, r, bf16).max())
    print("epilogue rule %s %s %s: worst %.3g ulp, %d of %d outside the rule" % (what, fn, "bf16" if bf16 else "fp16", worst, bad.size,
                                                                                  ok.size))
    assert bad.size == 0, (what, fn, "bf16" if bf16 else "fp16", bad.size, z.ravel()[bad[:6]], np.asarray(y).ravel()[bad[:6]],
                           r.ravel()[bad[:6]])
    return worst


def finite16(bf16):
    """every finite 16-bit value (each bit pattern once, so -0 and +0 both), as float32"""
    b = np.arange(65536, dtype=np.uint32)
    if bf16:
        v = (b << 16).view(np.float32)
    else:
        v = b.astype(np.uint16).view(np.float16).astype(np.float32)
    return v[np.isfinite(v)]
