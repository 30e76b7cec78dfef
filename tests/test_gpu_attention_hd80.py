"""K3 (wgmma attention) at head_dim 80, the ViT-H/14 vision tower (1280 / 16), against an fp64 numpy restatement of
clip.cpp:1082-1108 / 1363-1388 through the C-ABI test hook clip_b200_debug_attention_hd.  Every Q, K and V tile of an 80-wide
head reaches shared memory as two pieces, columns 0-63 and 64-79; the cases below are built so that a fault in the 16-column tail
piece alone (S step, P.V product, store) or a read across a head boundary shows up."""
import ctypes as C

import numpy as np
import pytest

from _util import one_minus_cos

pytestmark = pytest.mark.gpu

DH = 80
SCALE = 1.0 / np.sqrt(DH)


def _bf16(x):
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(np.uint32).view(np.float32)


def _round(x, bf):
    return _bf16(x) if bf else x.astype(np.float16).astype(np.float32)


def ref_attention(qkv, nseq, T, H, causal, bf, dh=DH):
    """fp64 softmax(Q K^T [causal]) V of the operands rounded to the kernel's 16-bit type; Q already scaled"""
    x = _round(qkv, bf).reshape(nseq, T, 3, H, dh).astype(np.float64)
    q, k, v = x[:, :, 0], x[:, :, 1], x[:, :, 2]
    s = np.einsum("bthd,bshd->bhts", q, k)
    if causal:
        s = np.where(np.tril(np.ones((T, T), bool))[None, None], s, -np.inf)
    p = np.exp(s - s.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    return np.einsum("bhts,bshd->bthd", p, v).reshape(nseq * T, H * dh)


def run(prod, qkv, nseq, T, H, causal, bf=1, legacy=0, dh=DH):
    qkv = np.ascontiguousarray(qkv, np.float32)
    out = np.empty((nseq * T, H * dh), np.float32)
    fp = C.POINTER(C.c_float)
    rc = prod.lib.clip_b200_debug_attention_hd(bf, nseq, T, H, dh, causal, legacy, qkv.ctypes.data_as(fp), out.ctypes.data_as(fp), None)
    assert rc == 0, prod.last_error()
    return out


def check(got, want, tol=2e-2):
    assert np.isfinite(got).all()
    scale = np.abs(want).max() + 1e-6
    assert np.abs(got - want).max() / scale < tol, (np.abs(got - want).max(), scale)
    assert one_minus_cos(got.ravel(), want.ravel()) < 1e-4


def random_qkv(rng, nseq, T, H, qmag=3.0):
    qkv = rng.standard_normal((nseq * T, 3 * H * DH)).astype(np.float32)
    qkv[:, : H * DH] *= SCALE * qmag          # scaled queries, scores of a few units
    return qkv


@pytest.mark.parametrize("T", [1, 5, 50, 128, 129, 256, 257, 577])
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("bf", [1, 0])
def test_random(prod, T, causal, bf):
    rng = np.random.default_rng(T * 7 + causal * 3 + bf)
    nseq, H = 2, 3
    qkv = random_qkv(rng, nseq, T, H)
    got = run(prod, qkv, nseq, T, H, causal, bf)
    want = ref_attention(qkv, nseq, T, H, causal, bf)
    check(got, want)
    # the tail columns on their own: a fault confined to the 16-column piece must not hide behind 64 good columns
    g3, w3 = got.reshape(nseq * T, H, DH), want.reshape(nseq * T, H, DH)
    check(g3[:, :, 64:], w3[:, :, 64:])


@pytest.mark.parametrize("T,causal,nseq,H", [(257, 0, 40, 8), (17, 0, 90, 4), (77, 1, 64, 4), (129, 0, 20, 16)])
def test_many_items_per_cta(prod, T, causal, nseq, H):
    """More (sequence, head) items than the 132 SMs, several query tiles per item, both K/V ring stages."""
    rng = np.random.default_rng(T + nseq)
    qkv = random_qkv(rng, nseq, T, H, 2.0)
    check(run(prod, qkv, nseq, T, H, causal, 1), ref_attention(qkv, nseq, T, H, causal, 1))


@pytest.mark.parametrize("T", [257, 577])
@pytest.mark.parametrize("pattern", ["ramp_up", "late_spike", "early_spike"])
def test_running_max_from_tail_columns(prod, T, pattern):
    """Scores whose row maximum moves from key block to key block -- every block raises the running maximum and rescales O (ramp
    up), only the last does (late spike), none after the first (early spike) -- carried by column 70 alone: the head columns hold
    small noise, so the tail k16 step of S decides the scores."""
    rng = np.random.default_rng(3 + T)
    nseq, H = 2, 2
    qkv = (rng.standard_normal((nseq * T, 3 * H * DH)) * 0.05).astype(np.float32)
    x = qkv.reshape(nseq, T, 3, H, DH)
    u = np.zeros(DH, np.float32); u[70] = 1.0
    j = np.arange(T, dtype=np.float32)
    amp = {"ramp_up": 0.2 * j, "late_spike": np.where(j == T - 3, 60.0, 0.0), "early_spike": np.where(j == 2, 60.0, 0.0)}[pattern].astype(np.float32)
    x[:, :, 0, :, :] += u
    x[:, :, 1, :, :] += amp[None, :, None, None] * u
    got = run(prod, qkv, nseq, T, H, 0, 1)
    check(got, ref_attention(qkv, nseq, T, H, 0, 1), tol=3e-2)


@pytest.mark.parametrize("bf", [1, 0])
def test_tail_of_v_checked_on_its_own(prod, bf):
    """V whose columns 64-79 come from a different distribution (offset and sign pattern) than columns 0-63: the m64n16 P.V piece
    and the tail stores are compared separately from the m64n64 piece."""
    rng = np.random.default_rng(80 + bf)
    nseq, T, H = 3, 257, 2
    qkv = random_qkv(rng, nseq, T, H)
    v = qkv.reshape(nseq * T, 3, H, DH)[:, 2]
    v[:, :, 64:] = 4.0 * np.sign(np.arange(16) - 7.5)[None, None, :] + 0.5 * v[:, :, 64:]
    got = run(prod, qkv, nseq, T, H, 0, bf).reshape(nseq * T, H, DH)
    want = ref_attention(qkv, nseq, T, H, 0, bf).reshape(nseq * T, H, DH)
    check(got[:, :, :64], want[:, :, :64])
    check(got[:, :, 64:], want[:, :, 64:])


@pytest.mark.parametrize("T,causal", [(257, 0), (77, 1)])
@pytest.mark.parametrize("bf", [1, 0])
def test_heads_are_isolated(prod, T, causal, bf):
    """Neighbouring heads 10^3 apart in magnitude (V and K times m, Q divided by m, so every head's scores stay of order one),
    compared head by head: any column read across a head boundary, in S or in P.V, pulls in data of the wrong magnitude."""
    rng = np.random.default_rng(T + 17 * bf)
    nseq, H = 2, 4
    qkv = random_qkv(rng, nseq, T, H)
    x = qkv.reshape(nseq * T, 3, H, DH)
    m = np.array([1.0, 1e3, 1.0, 1e3], np.float32) if bf else np.array([1.0, 30.0, 1.0, 30.0], np.float32)
    if bf:
        x[:, 0] /= m[None, :, None]
        x[:, 1] *= m[None, :, None]
        x[:, 2] *= m[None, :, None]
    else:
        # fp16 holds 6.5e4 at most and loses Q below 6e-5: magnitudes 30 apart in Q and K, 10^3 apart in V
        x[:, 0] /= m[None, :, None]
        x[:, 1] *= m[None, :, None]
        x[:, 2] *= (m * m * 1e3 / 900.0)[None, :, None]
    got = run(prod, qkv, nseq, T, H, causal, bf).reshape(nseq * T, H, DH)
    want = ref_attention(qkv, nseq, T, H, causal, bf).reshape(nseq * T, H, DH)
    for h in range(H):
        check(got[:, h], want[:, h])


def test_head_dim_64_through_the_new_hook_is_unchanged(prod):
    """clip_b200_debug_attention is the head_dim 64 call of the same hook: identical bits"""
    rng = np.random.default_rng(64)
    nseq, T, H = 2, 257, 3
    qkv = rng.standard_normal((nseq * T, 3 * H * 64)).astype(np.float32)
    qkv[:, : H * 64] *= 0.3
    a = run(prod, qkv, nseq, T, H, 0, 1, dh=64)
    b = np.empty_like(a)
    fp = C.POINTER(C.c_float)
    assert prod.lib.clip_b200_debug_attention(1, nseq, T, H, 0, 0, qkv.ctypes.data_as(fp), b.ctypes.data_as(fp), None) == 0
    assert np.array_equal(a, b)


def test_legacy_kernel_and_other_head_dims_are_refused(prod):
    qkv = np.zeros((5, 3 * 2 * 88), np.float32)
    out = np.zeros((5, 2 * 88), np.float32)
    fp = C.POINTER(C.c_float)
    q, o = qkv.ctypes.data_as(fp), out.ctypes.data_as(fp)
    assert prod.lib.clip_b200_debug_attention_hd(1, 1, 5, 2, 80, 0, 1, q, o, None) != 0
    assert "head_dim 64 only" in prod.last_error()
    assert prod.lib.clip_b200_debug_attention_hd(1, 1, 5, 2, 88, 0, 0, q, o, None) != 0
    assert "64 or 80" in prod.last_error()
