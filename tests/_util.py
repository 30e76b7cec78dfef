"""Shared helpers for the test-suite: model files from seeds, golden fixtures, tolerances."""
import os

import numpy as np

import binding as bd
import synth_gguf as sg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
FTYPES = {"f32": 0, "f16": 1, "q4_0": 2, "q4_1": 3, "q5_0": 6, "q5_1": 7, "q8_0": 8}
SEED = 1234
TOK_LENS = [77, 5, 2, 33, 16, 77, 9, 64]

# tolerances from BASELINE.json north_star: 1 - cos <= 1e-3 for f16 (and f32), <= 1e-2 for q4_0 (applied to all q*)
TOL = {"f32": 1e-3, "f16": 1e-3, "q4_0": 1e-2, "q4_1": 1e-2, "q5_0": 1e-2, "q5_1": 1e-2, "q8_0": 1e-2}


def reference_runs():
    """what the reference returned for the inputs of the tests that compare against it (tests/golden/make_reference_runs.py)"""
    z = np.load(os.path.join(GOLDEN, "reference_runs.npz"))
    return {k: z[k] for k in z.files}


def golden(geom):
    p = os.path.join(GOLDEN, "%s-s%d.npz" % (geom, SEED))
    if not os.path.exists(p):
        return None
    z = np.load(p)
    return {k: z[k] for k in z.files}


def model_file(geom: str, ftype: str, prod: "bd.ClipLib") -> str:
    """(geom, SEED, ftype) -> path; f16/f32 written from the seed, q* made with the PRODUCT's clip_model_quantize
    (byte-identical to the reference's: tests/test_host_side.py)."""
    path = sg.model_path(geom, SEED, ftype)
    if not os.path.exists(path):
        if ftype in ("f32", "f16"):
            sg.write_model(path, sg.GEOMETRIES[geom], SEED, FTYPES[ftype])
        else:
            src = model_file(geom, "f16", prod)
            assert prod.quantize(src, path + ".tmp", FTYPES[ftype]), prod.last_error()
            os.replace(path + ".tmp", path)
    return path


_sha_cache = {}


def check_sha(path, expect):
    """The file must be the one the golden vectors were produced from."""
    key = (path, os.path.getmtime(path))
    if key not in _sha_cache:
        _sha_cache[key] = sg.sha256_file(path)
    assert _sha_cache[key] == str(expect), "model file %s drifted from the golden fixture (generator changed?)" % path


def token_seqs(n, tok_seed=99):
    return [sg.synth_tokens(1, TOK_LENS[i % len(TOK_LENS)], tok_seed + i)[0] for i in range(n)]


# ---- device scoring references (tests/test_gpu_scoring.py, tests/test_gpu_scoring_exact.py) -----------------------------------
def fmaf32(a, b, c):
    """fmaf(a, b, c) of float32 values (numpy arrays, broadcast), correctly rounded to nearest even, as float32.  The product of
    two float32 is exact in fp64 (24 + 24 <= 53 bits).  The fp64 sum p + c is then rounded to odd: TwoSum gives its rounding
    error, and a nonzero error on an even mantissa moves the sum one ulp towards it.  Rounding that once to float32 is the
    correctly rounded fma, because 53 >= 24 + 2 (a plain fp64 sum could land on a float32 tie the exact value is not on)."""
    p = np.asarray(a, np.float64) * np.asarray(b, np.float64)
    c = np.asarray(c, np.float64)
    s = p + c
    t = s - p
    err = (p - (s - t)) + (c - t)
    bits = s.view(np.int64)
    odd = (err != 0) & ((bits & 1) == 0) & np.isfinite(s)
    bits += odd * np.where((err > 0) == (s > 0), 1, -1)
    return s.astype(np.float32)


def fmaf_chain_dot(a, b):
    """S[i, j] = acc after acc = fmaf(a[i, k], b[j, k], acc) for k = 0 .. d-1 from acc = +0, as float32 [len(a), len(b)]: one
    sequential fused chain per entry, the order csrc/search.cu's sim_kernel accumulates in."""
    a = np.asarray(a, np.float64)
    bt = np.ascontiguousarray(np.asarray(b, np.float64).T)
    s = np.empty((len(a), bt.shape[1]), np.float32)
    rows = max(1, 32768 // bt.shape[1])                      # a few rows at a time keep the working set in cache
    for r0 in range(0, len(a), rows):
        acc = np.zeros((len(a[r0:r0 + rows]), bt.shape[1]), np.float32)
        for k in range(a.shape[1]):
            acc = fmaf32(a[r0:r0 + rows, k:k + 1], bt[k], acc)
        s[r0:r0 + rows] = acc
    return s


def softmax_sorted(s):
    """softmax_with_sorting's arithmetic (clip.cpp:1599-1607) per row -- e = float32(exp(float64(s)) + 1e-9), the sum of the
    rounded e in fp64, p = float32(e / sum) -- sorted by (p descending, index ascending): returns (p sorted, order)."""
    s = np.asarray(s, np.float32)
    e = (np.exp(s.astype(np.float64)) + 1e-9).astype(np.float32)
    p = (e.astype(np.float64) / e.astype(np.float64).sum(-1, keepdims=True)).astype(np.float32)
    order = np.argsort(-p, axis=-1, kind="stable")
    return np.take_along_axis(p, order, -1), order


def ulp_dist(a, b):
    """|a - b| in float32 ulps, for float32 arrays of one sign (the integer views are then ordered like the values)"""
    return np.abs(np.asarray(a, np.float32).view(np.int32).astype(np.int64) - np.asarray(b, np.float32).view(np.int32))


def one_minus_cos(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    num = (a * b).sum(-1)
    den = np.linalg.norm(a, axis=-1) * np.linalg.norm(b, axis=-1)
    return 1.0 - num / den


# ---- LayerNorm test rows and their fp64 reference (tests/test_gpu_rows.py, tests/test_oracle_pin.py) ----------------------------
# Row contents, each aimed at one way a LayerNorm goes subtly wrong:
#   normal       standard normal
#   offset       mean 1e3, std 1e-2: a one-pass E[x^2] - mean^2 variance cancels catastrophically
#   eps_scale    std 3e-3, so the variance (9e-6) is about eps: a missing or misplaced eps moves every output
#   const_half   constant 0.5, const_m3 constant -3: dyadic, so every partial sum is exact and the output is exactly beta
#   outlier      standard normal with one +-1e4 element
LN_KINDS = ("normal", "offset", "eps_scale", "const_half", "const_m3", "outlier")
LN_KIND_SCALE = {"normal": 1.0, "offset": 1e-2, "eps_scale": 3e-3, "const_half": 0.0, "const_m3": 0.0, "outlier": 1.0}


def ln_rows(rows, h, rng, first=0):
    """x [rows, h] float32 whose row r has content LN_KINDS[(first + r) % len(LN_KINDS)]; returns (x, kind names)."""
    kinds = [LN_KINDS[(first + r) % len(LN_KINDS)] for r in range(rows)]
    x = rng.standard_normal((rows, h))
    for r, k in enumerate(kinds):
        if k == "offset":
            x[r] = 1e3 + 1e-2 * x[r]
        elif k == "eps_scale":
            x[r] *= 3e-3
        elif k == "const_half":
            x[r] = 0.5
        elif k == "const_m3":
            x[r] = -3.0
        elif k == "outlier":
            x[r, rng.integers(h)] = 1e4 if r % 2 else -1e4
    return x.astype(np.float32), kinds


def ln_ref64(x, eps):
    """fp64 LayerNorm without the affine, of the fp32 values in x: returns (x_hat, rstd [rows, 1], mean |x| [rows, 1]).
    eps enters as the fp32 value the kernels add."""
    x = np.asarray(x, np.float64)
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    rstd = 1.0 / np.sqrt(var + float(np.float32(eps)))
    return (x - mu) * rstd, rstd, np.abs(x).mean(-1, keepdims=True)
