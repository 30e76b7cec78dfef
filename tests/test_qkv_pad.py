"""The loader's QKV padding at head_dim 104 (ViT-bigG/14) on the CPU, through clip_b200_debug_pad_qkv: every head's rows of Q, K and V
(and of the bias) are followed by 8 rows of zero bytes, so that each head takes 112 output columns of the QKV GEMM and the 8 extra ones
are exact zeros.  All-zero bytes are an exact zero in f32, f16 and every ggml block type.  Needs no GPU."""
import ctypes as C

import numpy as np
import pytest

BLOCK = {0: (1, 4), 1: (1, 2), 2: (32, 18), 3: (32, 20), 6: (32, 22), 7: (32, 24), 8: (32, 34)}     # qtype -> (elements, bytes)
H, DH, DHP = 16, 104, 112


def pad(prod, qtype, K, src, h=H, dh=DH, dhp=DHP):
    out = np.full(3 * h * dhp * (src.size // (3 * h * dh)), 0xA5, np.uint8)
    rc = prod.lib.clip_b200_debug_pad_qkv(qtype, h, dh, dhp, K, src.ctypes.data, out.ctypes.data)
    return rc, out


@pytest.mark.parametrize("qtype", sorted(BLOCK))
def test_rows_move_and_pad_rows_are_zero(prod, qtype):
    K = 128
    be, bb = BLOCK[qtype]
    rb = K // be * bb
    rng = np.random.default_rng(qtype)
    src = rng.integers(1, 256, size=(3 * H * DH, rb), dtype=np.uint8)      # no zero byte: a pad row can only come from padding
    rc, out = pad(prod, qtype, K, src)
    assert rc == 0, prod.last_error()
    got = out.reshape(3, H, DHP, rb)
    want = src.reshape(3, H, DH, rb)
    assert np.array_equal(got[:, :, :DH], want)
    assert (got[:, :, DH:] == 0).all()


def test_bias(prod):
    """qtype 0 with K = 1: the f32 bias, padded the same way; the pad entries are +0.0"""
    rng = np.random.default_rng(7)
    b = rng.standard_normal(3 * H * DH).astype(np.float32)
    rc, out = pad(prod, 0, 1, b.view(np.uint8))
    assert rc == 0, prod.last_error()
    got = out.view(np.float32).reshape(3, H, DHP)
    assert np.array_equal(got[:, :, :DH], b.reshape(3, H, DH))
    assert (got[:, :, DH:].view(np.uint32) == 0).all()


def test_bad_arguments(prod):
    src = np.zeros((3 * 2 * 8, 64), np.uint8)
    out = np.zeros(1 << 16, np.uint8)
    L = prod.lib
    assert L.clip_b200_debug_pad_qkv(2, 2, 8, 4, 64, src.ctypes.data, out.ctypes.data) == 1        # dhp < dh
    assert L.clip_b200_debug_pad_qkv(2, 2, 8, 16, 48, src.ctypes.data, out.ctypes.data) == 1       # K not whole blocks
    assert L.clip_b200_debug_pad_qkv(5, 2, 8, 16, 64, src.ctypes.data, out.ctypes.data) == 1       # unknown type
    assert L.clip_b200_debug_pad_qkv(2, 2, 8, 16, 64, None, out.ctypes.data) == 1
