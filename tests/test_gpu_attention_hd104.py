"""K3 (wgmma attention) at head_dim 104, the ViT-bigG/14 vision tower (1664 / 16), against the fp64 restatement of clip.cpp:1082-1108 /
1363-1388 in tests/test_gpu_attention_hd80.py, through the C-ABI test hook clip_b200_debug_attention_hd.  The hook lays the unpadded
[rows, 3*H*104] input out as the loader lays out the QKV activations: each head padded to 112 columns, the last 8 zero.  Every Q, K
and V tile then reaches shared memory as three pieces, columns 0-63, 64-95 and 96-111, and keys come in 64-key blocks through a
three-stage ring; the cases below are built so that a fault in one piece alone (S step, P.V product, store), a wrong S width on a
ragged last block, or a read across a head boundary shows up."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_attention_hd80 import check, ref_attention, run

pytestmark = pytest.mark.gpu

DH = 104
SCALE = 1.0 / np.sqrt(DH)
PIECES = ((0, 64), (64, 96), (96, 104))


def random_qkv(rng, nseq, T, H, qmag=3.0):
    qkv = rng.standard_normal((nseq * T, 3 * H * DH)).astype(np.float32)
    qkv[:, : H * DH] *= SCALE * qmag          # scaled queries, scores of a few units
    return qkv


def check_pieces(got, want, nseq, T, H):
    """the whole output, then each column piece on its own: a fault confined to 32 or 8 columns must not hide behind the rest"""
    check(got, want)
    g3, w3 = got.reshape(nseq * T, H, DH), want.reshape(nseq * T, H, DH)
    for a, b in PIECES:
        check(g3[:, :, a:b], w3[:, :, a:b])


# T = 72, 88, 114: last 64-key blocks of 8, 24 and 50 keys (S 16, 32 and 64 wide); 64, 65, 128, 129 end a block or one past it
@pytest.mark.parametrize("T,causal", [(1, 0), (5, 0), (50, 0), (64, 0), (65, 0), (72, 0), (88, 0), (114, 0), (128, 0), (129, 0),
                                      (257, 0), (577, 0), (1025, 0), (77, 1), (88, 1), (129, 1), (257, 1)])
@pytest.mark.parametrize("bf", [1, 0])
def test_random(prod, T, causal, bf):
    rng = np.random.default_rng(T * 7 + causal * 3 + bf)
    nseq, H = (2, 3) if T < 1025 else (1, 4)
    qkv = random_qkv(rng, nseq, T, H)
    got = run(prod, qkv, nseq, T, H, causal, bf, dh=DH)
    check_pieces(got, ref_attention(qkv, nseq, T, H, causal, bf, dh=DH), nseq, T, H)


@pytest.mark.parametrize("bf", [1, 0])
def test_long_causal(prod, bf):
    """a long causal sequence: 65 key blocks on the last query group, every ring stage reused many times"""
    rng = np.random.default_rng(4161 + bf)
    nseq, T, H = 1, 4161, 2
    qkv = random_qkv(rng, nseq, T, H)
    got = run(prod, qkv, nseq, T, H, 1, bf, dh=DH)
    check_pieces(got, ref_attention(qkv, nseq, T, H, 1, bf, dh=DH), nseq, T, H)


@pytest.mark.parametrize("T,causal,nseq,H", [(257, 0, 40, 8), (17, 0, 90, 4), (77, 1, 64, 4), (129, 0, 20, 16)])
def test_many_items_per_cta(prod, T, causal, nseq, H):
    """More (sequence, head) items than the 132 SMs, several query groups per item, every K / V ring stage."""
    rng = np.random.default_rng(T + nseq)
    qkv = random_qkv(rng, nseq, T, H, 2.0)
    check(run(prod, qkv, nseq, T, H, causal, 1, dh=DH), ref_attention(qkv, nseq, T, H, causal, 1, dh=DH))


@pytest.mark.parametrize("col", [80, 100])
@pytest.mark.parametrize("T", [257, 577])
@pytest.mark.parametrize("pattern", ["ramp_up", "late_spike", "early_spike"])
def test_running_max_from_one_piece(prod, col, T, pattern):
    """Scores whose row maximum moves from key block to key block -- every block raises the running maximum and rescales O (ramp
    up), only the last does (late spike), none after the first (early spike) -- carried by one column of the 64-95 piece (80) or
    of the 96-103 piece (100) alone: the other columns hold small noise, so that piece's k16 steps of S decide the scores."""
    rng = np.random.default_rng(3 + T + col)
    nseq, H = 2, 2
    qkv = (rng.standard_normal((nseq * T, 3 * H * DH)) * 0.05).astype(np.float32)
    x = qkv.reshape(nseq, T, 3, H, DH)
    u = np.zeros(DH, np.float32); u[col] = 1.0
    j = np.arange(T, dtype=np.float32)
    amp = {"ramp_up": 0.2 * j, "late_spike": np.where(j == T - 3, 60.0, 0.0), "early_spike": np.where(j == 2, 60.0, 0.0)}[pattern].astype(np.float32)
    x[:, :, 0, :, :] += u
    x[:, :, 1, :, :] += amp[None, :, None, None] * u
    got = run(prod, qkv, nseq, T, H, 0, 1, dh=DH)
    check(got, ref_attention(qkv, nseq, T, H, 0, 1, dh=DH), tol=3e-2)


@pytest.mark.parametrize("bf", [1, 0])
def test_v_pieces_checked_on_their_own(prod, bf):
    """V whose columns 64-95 and 96-103 come from distributions of their own (offsets and sign patterns) unlike columns 0-63: the
    m64n32 and m64n16 P.V products and their stores are compared separately from the m64n64 piece."""
    rng = np.random.default_rng(104 + bf)
    nseq, T, H = 3, 257, 2
    qkv = random_qkv(rng, nseq, T, H)
    v = qkv.reshape(nseq * T, 3, H, DH)[:, 2]
    v[:, :, 64:96] = 4.0 * np.sign(np.arange(32) - 15.5)[None, None, :] + 0.5 * v[:, :, 64:96]
    v[:, :, 96:] = -6.0 + 0.25 * np.arange(8)[None, None, :] + 0.5 * v[:, :, 96:]
    got = run(prod, qkv, nseq, T, H, 0, bf, dh=DH).reshape(nseq * T, H, DH)
    want = ref_attention(qkv, nseq, T, H, 0, bf, dh=DH).reshape(nseq * T, H, DH)
    for a, b in PIECES:
        check(got[:, :, a:b], want[:, :, a:b])


@pytest.mark.parametrize("T,causal", [(257, 0), (77, 1)])
@pytest.mark.parametrize("bf", [1, 0])
def test_heads_are_isolated(prod, T, causal, bf):
    """Neighbouring heads far apart in magnitude, compared head by head (as at head_dim 80), and then a NaN in every Q, K and V
    column of head h + 1: head h must come out with the same bits, since no piece of head h reaches past its own 112 columns."""
    rng = np.random.default_rng(T + 17 * bf)
    nseq, H = 2, 4
    qkv = random_qkv(rng, nseq, T, H)
    x = qkv.reshape(nseq * T, 3, H, DH)
    m = np.array([1.0, 30.0, 1.0, 30.0], np.float32)
    x[:, 0] /= m[None, :, None]
    x[:, 1] *= m[None, :, None]
    x[:, 2] *= (m * m)[None, :, None]
    got = run(prod, qkv, nseq, T, H, causal, bf, dh=DH)
    want = ref_attention(qkv, nseq, T, H, causal, bf, dh=DH)
    g3, w3 = got.reshape(nseq * T, H, DH), want.reshape(nseq * T, H, DH)
    for h in range(H):
        check(g3[:, h], w3[:, h])
    for h in range(H - 1):
        poisoned = qkv.copy()
        poisoned.reshape(nseq * T, 3, H, DH)[:, :, h + 1] = np.nan
        gp = run(prod, poisoned, nseq, T, H, causal, bf, dh=DH).reshape(nseq * T, H, DH)
        assert np.array_equal(gp[:, h].view(np.uint32), g3[:, h].view(np.uint32)), h
        assert np.isnan(gp[:, h + 1]).all()


def test_head_dim_88_and_legacy_are_refused(prod):
    """104 is accepted next to 64 and 80; 88 (ViT-g/14) is still refused, and the legacy kernel stays head_dim 64 only"""
    qkv = np.zeros((5, 3 * 2 * DH), np.float32)
    out = np.zeros((5, 2 * DH), np.float32)
    fp = C.POINTER(C.c_float)
    q, o = qkv.ctypes.data_as(fp), out.ctypes.data_as(fp)
    assert prod.lib.clip_b200_debug_attention_hd(1, 1, 5, 2, DH, 0, 1, q, o, None) == 2
    assert "head_dim 64 only" in prod.last_error()
    assert prod.lib.clip_b200_debug_attention_hd(1, 1, 5, 2, 88, 0, 0, q, o, None) == 2
    assert "64 or 80" in prod.last_error() and "104" in prod.last_error()
