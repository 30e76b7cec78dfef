"""K3 (wgmma attention) against a numpy restatement of clip.cpp:1082-1108 / 1363-1388 (scaled Q.K^T, optional causal mask,
soft_max ggml.c:12201-12270, .V), through the C-ABI test hook.  Includes score patterns whose row maximum moves from key block to key
block, which exercises the online-softmax rescale."""
import ctypes as C
import numpy as np
import pytest

from _util import one_minus_cos

pytestmark = pytest.mark.gpu


def _bf16(x):
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(np.uint32).view(np.float32)


def _round(x, bf):
    return _bf16(x) if bf else x.astype(np.float16).astype(np.float32)


def ref_attention(qkv, nseq, T, H, causal, bf):
    hid = H * 64
    x = _round(qkv, bf).reshape(nseq, T, 3, H, 64).astype(np.float64)
    q, k, v = x[:, :, 0], x[:, :, 1], x[:, :, 2]
    s = np.einsum("bthd,bshd->bhts", q, k)
    if causal:
        s = np.where(np.tril(np.ones((T, T), bool))[None, None], s, -np.inf)
    p = np.exp(s - s.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    return np.einsum("bhts,bshd->bthd", p, v).reshape(nseq * T, hid).astype(np.float32)


def run(prod, qkv, nseq, T, H, causal, bf=1, legacy=0):
    qkv = np.ascontiguousarray(qkv, np.float32)
    out = np.empty((nseq * T, H * 64), np.float32)
    fp = C.POINTER(C.c_float)
    rc = prod.lib.clip_b200_debug_attention(bf, nseq, T, H, causal, legacy, qkv.ctypes.data_as(fp), out.ctypes.data_as(fp), None)
    assert rc == 0, prod.last_error()
    return out


def check(prod, qkv, nseq, T, H, causal, bf=1, tol=2e-2):
    got = run(prod, qkv, nseq, T, H, causal, bf)
    want = ref_attention(qkv, nseq, T, H, causal, bf)
    assert np.isfinite(got).all()
    scale = np.abs(want).max() + 1e-6
    assert np.abs(got - want).max() / scale < tol, (np.abs(got - want).max(), scale)
    assert one_minus_cos(got.ravel(), want.ravel()) < 1e-4


@pytest.mark.parametrize("T,causal", [(257, 0), (256, 0), (129, 0), (128, 0), (50, 0), (197, 0), (77, 1), (33, 1), (1, 0), (5, 1)])
@pytest.mark.parametrize("bf", [1, 0])
def test_random(prod, T, causal, bf):
    rng = np.random.default_rng(T * 7 + causal + bf)
    nseq, H = 3, 2
    qkv = rng.standard_normal((nseq * T, 3 * H * 64)).astype(np.float32)
    qkv[:, : H * 64] *= 0.125 * 3.0          # scaled queries, scores of a few units
    check(prod, qkv, nseq, T, H, causal, bf)


@pytest.mark.parametrize("T", [257, 200, 77])
@pytest.mark.parametrize("pattern", ["ramp_up", "ramp_down", "late_spike", "early_spike", "second_half"])
def test_offset_rescale_paths(prod, T, pattern):
    """Scores that grow along the key axis by far more than 2^8 per 32-key chunk: every chunk after the first raises the
    exponent offset (slow path), and the two column halves of a row pair finish with different offsets."""
    rng = np.random.default_rng(11)
    nseq, H = 2, 2
    qkv = (rng.standard_normal((nseq * T, 3 * H * 64)) * 0.05).astype(np.float32)
    x = qkv.reshape(nseq, T, 3, H, 64)
    u = np.zeros(64, np.float32); u[0] = 1.0
    j = np.arange(T, dtype=np.float32)
    amp = {"ramp_up": 0.5 * j, "ramp_down": 0.5 * (T - 1 - j), "late_spike": np.where(j == T - 3, 60.0, 0.0),
           "early_spike": np.where(j == 2, 60.0, 0.0), "second_half": np.where(j >= 140, 40.0, 0.0)}[pattern].astype(np.float32)
    x[:, :, 0, :, :] += u            # q has a unit component along u
    x[:, :, 1, :, :] += amp[None, :, None, None] * u
    causal = 1 if T == 77 else 0
    check(prod, qkv, nseq, T, H, causal, 1, tol=3e-2)


def test_matches_legacy_kernel(prod):
    rng = np.random.default_rng(5)
    nseq, T, H = 4, 257, 3
    qkv = rng.standard_normal((nseq * T, 3 * H * 64)).astype(np.float32)
    qkv[:, : H * 64] *= 0.3
    a = run(prod, qkv, nseq, T, H, 0, 1, 0)
    b = run(prod, qkv, nseq, T, H, 0, 1, 1)
    assert np.abs(a - b).max() < 2e-2


@pytest.mark.parametrize("T,causal,nseq,H", [(17, 0, 90, 4), (5, 0, 200, 2), (50, 0, 60, 12), (257, 0, 40, 8), (77, 1, 64, 8), (20, 1, 100, 3)])
def test_many_items_per_cta(prod, T, causal, nseq, H):
    """More (sequence, head) items than SMs, several query tiles per item, both K/V ring stages."""
    rng = np.random.default_rng(T + nseq)
    qkv = rng.standard_normal((nseq * T, 3 * H * 64)).astype(np.float32)
    qkv[:, : H * 64] *= 0.3
    check(prod, qkv, nseq, T, H, causal, 1)


@pytest.mark.parametrize("T,causal", [(300, 0), (577, 0), (100, 1)])
def test_legacy_kernel_long_sequences(prod, T, causal):
    """the warp-level mma.sync flash kernel (the cross-check of the wgmma kernel) at T > 257 (e.g. ViT-L/14@336: 577 tokens)"""
    rng = np.random.default_rng(T)
    nseq, H = 2, 3
    qkv = rng.standard_normal((nseq * T, 3 * H * 64)).astype(np.float32)
    qkv[:, : H * 64] *= 0.3
    got = run(prod, qkv, nseq, T, H, causal, 1, legacy=1)
    want = ref_attention(qkv, nseq, T, H, causal, 1)
    assert np.abs(got - want).max() / (np.abs(want).max() + 1e-6) < 2e-2
    assert one_minus_cos(got.ravel(), want.ravel()) < 1e-4


@pytest.mark.parametrize("T,nseq,H", [(258, 3, 2), (300, 2, 3), (384, 2, 2), (385, 2, 2), (577, 2, 3), (577, 40, 16), (640, 1, 2)])
@pytest.mark.parametrize("bf", [1, 0])
def test_long_sequences_on_tcgen05(prod, T, nseq, H, bf):
    """257 < T <= 640 (ViT-L/14@336: 577 tokens): the wgmma kernel over several 128-key blocks, ragged last block, many (sequence, head)
    items in the (577, 40, 16) case -- against the numpy restatement and against the warp-level kernel."""
    rng = np.random.default_rng(T + nseq)
    qkv = rng.standard_normal((nseq * T, 3 * H * 64)).astype(np.float32)
    qkv[:, : H * 64] *= 0.3
    got = run(prod, qkv, nseq, T, H, 0, bf)
    assert np.isfinite(got).all()
    if nseq * H <= 64:
        want = ref_attention(qkv, nseq, T, H, 0, bf)
        assert np.abs(got - want).max() / (np.abs(want).max() + 1e-6) < 2e-2
        assert one_minus_cos(got.ravel(), want.ravel()) < 1e-4
    legacy = run(prod, qkv, nseq, T, H, 0, bf, legacy=1)
    assert np.abs(got - legacy).max() < 2e-2


@pytest.mark.parametrize("pattern", ["ramp_up", "late_spike", "early_spike"])
def test_long_sequences_running_max(prod, pattern):
    """scores whose maximum moves from key block to key block: every block raises the running maximum and rescales O (ramp up), only the
    last does (late spike), or none after the first (early spike)"""
    rng = np.random.default_rng(3)
    nseq, T, H = 2, 577, 2
    qkv = (rng.standard_normal((nseq * T, 3 * H * 64)) * 0.05).astype(np.float32)
    x = qkv.reshape(nseq, T, 3, H, 64)
    u = np.zeros(64, np.float32); u[0] = 1.0
    j = np.arange(T, dtype=np.float32)
    amp = {"ramp_up": 0.2 * j, "late_spike": np.where(j == T - 3, 60.0, 0.0), "early_spike": np.where(j == 2, 60.0, 0.0)}[pattern].astype(np.float32)
    x[:, :, 0, :, :] += u
    x[:, :, 1, :, :] += amp[None, :, None, None] * u
    check(prod, qkv, nseq, T, H, 0, 1, tol=3e-2)
