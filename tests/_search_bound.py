"""K10's scores (clip_b200_topk_search_16, csrc/search.cu): an fp64 reference on the 16-bit operands, the per-score bound the header
states, and a numpy emulation of the kernel's arithmetic.  Shared by the GPU test (tests/test_gpu_search_16.py) and by the CPU test
that checks the bound against the emulation and against two wrong results (tests/test_search_bound.py).

Notation: u = 2^-24.  q, x are the 16-bit operands (exact in fp64); every product q_i x_i is exact in fp32.  The kernel accumulates
the products in fp32 on the tensor cores in k16 steps (ceil(dim / 16) of them; zero-filled columns past dim add exact zeros).
As in tests/_attention_bound.py step 1, each step is allowed one rounding of up to 2u relative to the partial sum, |partial| <=
sum_i |q_i x_i|, plus 4u for the rest:
    |score - q.x| <= B = (2 ceil(dim / 16) + 4) u sum_i |q_i x_i|."""
import numpy as np

U = 2.0 ** -24


def bf16(x):
    """float32 -> bf16 (round to nearest even) as float32"""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(np.uint32).view(np.float32)


def round16(x, bf):
    """float32 values rounded once (to nearest even) to the 16-bit type, returned as float32"""
    x = np.asarray(x, np.float32)
    return bf16(x) if bf else x.astype(np.float16).astype(np.float32)


def bits16(x, bf):
    """the 16-bit encoding (uint16) of float32 values rounded to the 16-bit type"""
    if bf:
        return (bf16(x).view(np.uint32) >> 16).astype(np.uint16)
    with np.errstate(over="ignore"):                  # beyond the f16 range: +-inf, as RNE gives
        return np.asarray(x, np.float32).astype(np.float16).view(np.uint16)


def exact(q, x):
    """fp64 dot products of the 16-bit operands: [n_q, n_db]"""
    return np.asarray(q, np.float64) @ np.asarray(x, np.float64).T


def bound(q, x):
    """the per-score bound B [n_q, n_db] of the module docstring"""
    dim = np.shape(q)[1]
    return (2 * -(-dim // 16) + 4) * U * (np.abs(np.asarray(q, np.float64)) @ np.abs(np.asarray(x, np.float64)).T)


def _trunc32(v):
    """fp64 -> fp32 rounded toward zero (the worst case of one rounding)"""
    f = v.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(v)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f


def emulate(q, x, drop_last=False):
    """K10's arithmetic: fp32 accumulation of exact products in k16 steps, each step's sum truncated once.  drop_last skips
    the last k16 step (a wrong result the bound must reject)."""
    q, x = np.asarray(q, np.float64), np.asarray(x, np.float64)
    dim = q.shape[1]
    steps = -(-dim // 16)
    acc = np.zeros((len(q), len(x)), np.float32)
    for s in range(steps - (1 if drop_last else 0)):
        k = slice(16 * s, min(dim, 16 * s + 16))
        acc = _trunc32(acc.astype(np.float64) + q[:, k] @ x[:, k].T)
    return acc


def exceed(got, ref, b):
    """max |got - ref| / b (<= 1 where the bound holds)"""
    return float((np.abs(np.asarray(got, np.float64) - ref) / b).max())


def unit_rows(rng, n, dim, bf):
    """seeded unit-norm rows rounded to the 16-bit type (float32)"""
    v = rng.standard_normal((n, dim))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    return round16(v.astype(np.float32), bf)
