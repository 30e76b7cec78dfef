"""The epilogue rule of tests/_epilogue_rule.py, checked without a GPU.  It accepts the correctly rounded result and a float32
emulation of the kernel's form (csrc/common.cuh mul_sigmoid_exp2, with ex2.approx's and rcp.approx's errors in either direction), and it
rejects five wrong epilogues at the inputs that expose each one, for fp16 and bf16 results."""
import numpy as np
import pytest
from scipy.special import erf

from _epilogue_rule import REF, accepts, finite16, gelu64, qgelu64, rne16, tiny16
from _util import fmaf32

F32 = np.float32


def inputs(bf16):
    """every finite 16-bit value, dense fp32 values in [-20, 20] off the 16-bit grid, and both tails out to 1e30 in magnitude"""
    rng = np.random.default_rng(7 + bf16)
    dense = rng.uniform(-20, 20, 200000).astype(F32)
    tails = (10.0 ** rng.uniform(-40, 30, 20000)).astype(F32)
    return np.concatenate([finite16(bf16), dense, tails, -tails])


def rejected(y, z, fn, bf16):
    """number of inputs whose result breaks the rule"""
    return int(np.count_nonzero(~accepts(y, REF[fn](z.astype(np.float64)), bf16)))


# ---- the kernel's form, in float32 ------------------------------------------------------------------------------------------
def kernel_form(z, fn, ex2_rel=0.0, rcp_rel=0.0):
    """mul_sigmoid_exp2 of csrc/common.cuh step by step in float32; ex2.approx's result scaled by (1 + ex2_rel) and flushed to zero
    below the smallest fp32 normal (.ftz), rcp.approx's by (1 + rcp_rel)"""
    x = np.asarray(z, F32)
    with np.errstate(over="ignore", invalid="ignore"):
        a = x * fmaf32(F32(0.10294323958), x * x, F32(2.3022081981)) if fn == "gelu" else F32(2.4554669596) * x
        es = (np.exp2(64.0 - np.abs(a.astype(np.float64))) * (1.0 + ex2_rel)).astype(F32)
        es = np.where(es < np.finfo(F32).tiny, F32(0), es)
        d = fmaf32(es, F32(2.0 ** -64), F32(1))
        r = ((1.0 / d.astype(np.float64)) * (1.0 + rcp_rel)).astype(F32)
        n = np.where(a >= 0, x, (x * es) * F32(2.0 ** -64))
        return (n * r).astype(F32)


@pytest.mark.parametrize("fn", ["gelu", "qgelu"])
@pytest.mark.parametrize("bf16", [False, True])
def test_accepts_the_correctly_rounded_result(fn, bf16):
    z = inputs(bf16)
    assert rejected(rne16(REF[fn](z.astype(np.float64)), bf16), z, fn, bf16) == 0


@pytest.mark.parametrize("ex2_rel,rcp_rel", [(0.0, 0.0), (2.0 ** -22, 2.0 ** -22), (-2.0 ** -22, -2.0 ** -22)])
@pytest.mark.parametrize("fn", ["gelu", "qgelu"])
@pytest.mark.parametrize("bf16", [False, True])
def test_accepts_the_kernel_form(fn, bf16, ex2_rel, rcp_rel):
    z = inputs(bf16)
    y = kernel_form(z, fn, ex2_rel, rcp_rel)
    assert rejected(rne16(y.astype(np.float64), bf16), z, fn, bf16) == 0
    # the form's limits: x for large positive inputs, -0 for large negative ones (the exponential is then 0 or flushed)
    big = np.array([1e4, 1e13, 1e20, 1e30], F32)
    assert np.array_equal(rne16(kernel_form(big, fn, ex2_rel, rcp_rel), bf16), rne16(big, bf16))
    neg = kernel_form(-big, fn, ex2_rel, rcp_rel)
    assert np.all(neg == 0) and np.all(np.signbit(neg))


# ---- five wrong epilogues ---------------------------------------------------------------------------------------------------
def tanh_form(z, fn, rel):
    """the epilogues this rule replaced: 0.5 x (1 + t) with t = tanh.approx(u), here tanh scaled by (1 + rel)"""
    x = np.asarray(z, F32)
    with np.errstate(over="ignore", invalid="ignore"):
        if fn == "gelu":
            u = F32(0.7978845608) * x * (F32(1) + F32(0.044715) * x * x)
        else:
            u = F32(0.851) * x
        t = (np.tanh(u.astype(np.float64)) * (1.0 + rel)).astype(F32)
        return x * fmaf32(F32(0.5), t, F32(0.5))


def wrong(kind, z):
    z64 = np.asarray(z, np.float64)
    with np.errstate(over="ignore"):
        if kind == "erf":
            return 0.5 * z64 * (1.0 + erf(z64 / np.sqrt(2.0)))
        if kind == "qgelu_1.7":
            return z64 / (1.0 + np.exp(-1.7 * z64))
        if kind == "gelu_0.0447":
            return z64 / (1.0 + np.exp(-2.0 * np.sqrt(2.0 / np.pi) * (z64 + 0.0447 * z64 ** 3)))
    raise ValueError(kind)


# tanh.approx's documented relative error, 2^-11, in either direction.  Towards -1 (rel > 0) 1 + t reaches 0 or below and the
# result of a negative input is zero or of the wrong sign; towards 0 (rel < 0) it is |x| 2^-12 too large in magnitude.  Both GELUs
# break the rule at every negative input from about z = -0.6 down in fp16, from about z = -1.3 down in bf16.
@pytest.mark.parametrize("rel", [2.0 ** -11, -2.0 ** -11], ids=["towards_minus_1", "towards_0"])
@pytest.mark.parametrize("fn", ["gelu", "qgelu"])
@pytest.mark.parametrize("bf16", [False, True])
def test_rejects_tanh_with_its_documented_error(fn, bf16, rel):
    z = inputs(bf16)
    assert rejected(rne16(tanh_form(z, fn, rel).astype(np.float64), bf16), z, fn, bf16) > 0


# Where each wrong function breaks the rule: erf-GELU, z in [-4.2, -0.73] in fp16 and [-10.1, -2.0] in bf16 (tens of percent off
# in the tail); quick-GELU with 1.7, z in [-6.8, 1.1] in fp16 and [-53.6, -1.3] in bf16 (a factor exp(0.002 |z|) for negative z);
# 0.0447 in GELU, z in [-4.0, -2.5] in fp16 and [-10.1, -4.6] in bf16 (the exponent moves by 2 sqrt(2/pi) 1.5e-5 |z|^3).
@pytest.mark.parametrize("kind,fn", [("erf", "gelu"), ("qgelu_1.7", "qgelu"), ("gelu_0.0447", "gelu")])
@pytest.mark.parametrize("bf16", [False, True])
def test_rejects_the_wrong_function(kind, fn, bf16):
    z = inputs(bf16)
    assert rejected(rne16(wrong(kind, z), bf16), z, fn, bf16) > 0


# results in the lowest normal binade of the 16-bit type flushed to zero: the tiny positive inputs, and the negative inputs down to
# z = -4.0 (GELU) and -6.8 (quick-GELU) in fp16, -10.1 and -53.6 in bf16
@pytest.mark.parametrize("fn", ["gelu", "qgelu"])
@pytest.mark.parametrize("bf16", [False, True])
def test_rejects_normal_results_flushed_to_zero(fn, bf16):
    z = inputs(bf16)
    y = rne16(REF[fn](z.astype(np.float64)), bf16)
    y = np.where(np.abs(y) < 2 * tiny16(bf16), 0.0, y)
    assert rejected(y, z, fn, bf16) > 0


def test_reference_tails():
    """the fp64 references stay accurate where 1 + tanh cancels: their ratio to the asymptotic forms, and exact limits"""
    z = np.array([-8.0, -10.0, -12.0])
    u = np.sqrt(2.0 / np.pi) * (z + 0.044715 * z ** 3)
    np.testing.assert_allclose(gelu64(z), z * np.exp(2.0 * u), rtol=1e-12)
    np.testing.assert_allclose(qgelu64(np.array([-40.0, -60.0])), np.array([-40.0, -60.0]) * np.exp(1.702 * np.array([-40.0, -60.0])),
                               rtol=1e-12)
    assert gelu64(np.float64(-1e30)) == 0 and np.signbit(gelu64(np.float64(-1e30)))
    assert gelu64(np.float64(1e30)) == 1e30 and qgelu64(np.float64(1e30)) == 1e30
    assert np.isinf(rne16(65520.0, False)) and rne16(65519.0, False) == 65504.0
