"""Images of different sizes in one call (clip_b200_image_encode_device_mixed, clip_b200_image_tokens_device_mixed and the host forms
clip_b200_image_batch_encode_mixed / clip_b200_image_tokens_mixed): rows packed back to back into one forward pass, attention by K3's
variable-length instance.

  1. The variable-length kernel (clip_b200_debug_attention_mixed) equals K3 run on each sequence alone, bit for bit, and a sequence
     holding Inf / NaN leaves every other sequence's bits unchanged.
  2. Each image of a mixed call equals that image alone through the *_device_hw form, byte for byte: pooled, and tokens at several
     flags and every out_type, on head_dim 64, 80 and 104 models, at sizes that put T on both sides of multiples of 64 and 128.
  3. Order, pass boundaries and a NaN neighbour change nothing; one size equals the *_hw call, the native size the native call; host
     forms equal device forms; tiny against the CPU oracle.
  4. Refusals, in order, with their messages.  5. Devices mode equals one GPU."""
import ctypes as C

import numpy as np
import pytest

import binding as bd
import synth_gguf as sg
from _oracle_anyres import AnyresOracle
from _util import TOL, model_file
from test_gpu_anyres import cos_rows, encode_dev, images, tokens_dev
from test_gpu_tokens import Ctx, bits
from test_pos_resample import pos_resample_ref

pytestmark = pytest.mark.gpu

FP = C.POINTER(C.c_float)
IP = C.POINTER(C.c_int)


def image(H, W, seed):
    return images(1, H, W, seed)[0]


def sizes_arrays(imgs):
    h = np.array([im.shape[0] for im in imgs], np.int32)
    w = np.array([im.shape[1] for im in imgs], np.int32)
    return h, w


def upload_packed(prod, ctx, imgs):
    flat = np.concatenate([im.reshape(-1) for im in imgs]).astype(np.float32) if imgs else np.zeros(1, np.float32)
    d = prod.lib.clip_b200_device_malloc(ctx, flat.nbytes)
    assert prod.lib.clip_b200_memcpy_h2d(ctx, d, flat.ctypes.data, flat.nbytes)
    return d


def encode_mixed_dev(prod, ctx, imgs, normalize=True):
    n, dim = len(imgs), prod.vision_hparams(ctx).projection_dim
    h, w = sizes_arrays(imgs)
    out = np.empty((n, dim), np.float32)
    d_in = upload_packed(prod, ctx, imgs)
    d_out = prod.lib.clip_b200_device_malloc(ctx, max(out.nbytes, 1))
    try:
        assert prod.lib.clip_b200_image_encode_device_mixed(ctx, d_in, n, h.ctypes.data_as(IP), w.ctypes.data_as(IP), d_out, normalize), \
            prod.last_error()
        assert prod.lib.clip_b200_memcpy_d2h(ctx, out.ctypes.data, d_out, out.nbytes)
    finally:
        prod.lib.clip_b200_device_free(ctx, d_in)
        prod.lib.clip_b200_device_free(ctx, d_out)
    return out


def width_of(prod, ctx, flags):
    hp = prod.vision_hparams(ctx)
    return hp.projection_dim if flags & bd.TOKENS_PROJECT else hp.hidden_size


def tokens_mixed_dev(prod, ctx, imgs, layer, flags, ot=bd.OUT_F32):
    h, w = sizes_arrays(imgs)
    rows = prod.mixed_token_rows(ctx, [im.shape[:2] for im in imgs], flags)
    flat = np.empty((sum(rows), width_of(prod, ctx, flags)), bd.OUT_DTYPES[ot])
    d_in = upload_packed(prod, ctx, imgs)
    d_out = prod.lib.clip_b200_device_malloc(ctx, max(flat.nbytes, 1))
    try:
        assert prod.lib.clip_b200_image_tokens_device_mixed(ctx, d_in, len(imgs), h.ctypes.data_as(IP), w.ctypes.data_as(IP), layer, flags,
                                                            ot, d_out), prod.last_error()
        assert prod.lib.clip_b200_memcpy_d2h(ctx, flat.ctypes.data, d_out, flat.nbytes)
    finally:
        prod.lib.clip_b200_device_free(ctx, d_in)
        prod.lib.clip_b200_device_free(ctx, d_out)
    return np.split(flat, np.cumsum(rows)[:-1])


# ---- 1. the variable-length attention kernel ------------------------------------------------------------------------------------

LENS = [1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 257, 577, 1025]


def qkv_of(rng, rows, H, dh):
    return (rng.standard_normal((rows, 3 * H * dh)) * 0.5).astype(np.float32)


def hook_mixed(prod, bf16, lens, H, dh, qkv):
    out = np.empty((sum(lens), H * dh), np.float32)
    ln = np.array(lens, np.int32)
    rc = prod.lib.clip_b200_debug_attention_mixed(bf16, len(lens), ln.ctypes.data_as(IP), H, dh, qkv.ctypes.data_as(FP), out.ctypes.data_as(FP))
    assert rc == 0, (rc, prod.last_error())
    return out


def hook_alone(prod, bf16, T, H, dh, qkv):
    out = np.empty((T, H * dh), np.float32)
    rc = prod.lib.clip_b200_debug_attention_hd(bf16, 1, T, H, dh, 0, 0, np.ascontiguousarray(qkv).ctypes.data_as(FP), out.ctypes.data_as(FP), None)
    assert rc == 0, (rc, prod.last_error())
    return out


@pytest.mark.parametrize("bf16", [0, 1])
@pytest.mark.parametrize("dh", [64, 80, 104])
def test_varlen_kernel_equals_each_sequence_alone(prod, dh, bf16):
    rng = np.random.default_rng(dh * 10 + bf16)
    H = 2
    for order in range(2):
        lens = list(rng.permutation(LENS)) if order else LENS
        qkv = qkv_of(rng, sum(lens), H, dh)
        got = hook_mixed(prod, bf16, lens, H, dh, qkv)
        r0 = 0
        for T in lens:
            want = hook_alone(prod, bf16, T, H, dh, qkv[r0:r0 + T])
            assert np.array_equal(bits(got[r0:r0 + T]), bits(want)), (dh, bf16, lens, T)
            r0 += T


@pytest.mark.parametrize("dh", [64, 80, 104])
def test_varlen_kernel_isolates_non_finite_sequences(prod, dh):
    rng = np.random.default_rng(7 + dh)
    H = 2
    lens = [65, 129, 1, 63, 193, 2, 128]
    qkv = qkv_of(rng, sum(lens), H, dh)
    clean = hook_mixed(prod, 0, lens, H, dh, qkv)
    offs = np.concatenate([[0], np.cumsum(lens)])
    cols = H * dh
    for k in range(len(lens)):
        for part in range(3):                     # Q, K, V of sequence k
            for bad in (np.inf, -np.inf, np.nan):
                x = qkv.copy()
                x[offs[k]:offs[k + 1], part * cols:(part + 1) * cols:3] = bad
                got = hook_mixed(prod, 0, lens, H, dh, x)
                for j in range(len(lens)):
                    if j != k:
                        assert np.array_equal(bits(got[offs[j]:offs[j + 1]]), bits(clean[offs[j]:offs[j + 1]])), (dh, k, part, bad, j)


# ---- 2. each image against itself alone -----------------------------------------------------------------------------------------

# per geometry: the native size, a one-patch grid (T = 2), rectangles, and T at 63 / 64 / 65, 127 / 128 / 129 or near them
SIZES = {
    "tiny": [(64, 64), (16, 16), (32, 496), (112, 144), (128, 128), (144, 224), (16, 2032), (128, 256), (112, 48), (64, 128)],
    "small-p14": [(224, 224), (14, 14), (98, 126), (14, 882), (112, 112), (126, 252), (14, 1778), (112, 224), (224, 448)],
    "huge-w640": [(224, 224), (14, 14), (98, 126), (112, 112), (126, 252), (112, 224), (224, 126)],
    "bigg-w1664": [(224, 224), (14, 14), (98, 126), (112, 112), (112, 224), (224, 126)],
}
TOKEN_FLAGS = [0, bd.TOKENS_POST_LN, bd.TOKENS_PROJECT | bd.TOKENS_NORMALIZE, bd.TOKENS_NO_CLS]


@pytest.mark.parametrize("geom", list(SIZES))
def test_each_image_equals_itself_alone(prod, geom):
    path = model_file(geom, "f16", prod)
    imgs = [image(H, W, 100 + k) for k, (H, W) in enumerate(SIZES[geom])]
    with Ctx(prod, path) as ctx:
        for normalize in (True, False):
            got = encode_mixed_dev(prod, ctx, imgs, normalize)
            for k, im in enumerate(imgs):
                assert np.array_equal(bits(got[k]), bits(encode_dev(prod, ctx, im[None], normalize)[0])), (geom, k, normalize)
        for flags in TOKEN_FLAGS:
            for ot in (bd.OUT_F32, bd.OUT_F16, bd.OUT_BF16):
                got = tokens_mixed_dev(prod, ctx, imgs, -2, flags, ot)
                for k, im in enumerate(imgs):
                    want = tokens_dev(prod, ctx, im[None], -2, flags, ot)[0]
                    assert got[k].shape == want.shape, (geom, k, flags)
                    assert np.array_equal(bits(got[k]), bits(want)), (geom, k, flags, ot)


# ---- 3. order, passes, neighbours, the fixed-size forms, host forms, the oracle --------------------------------------------------

def tiny_batch(seed=5):
    return [image(H, W, seed + k) for k, (H, W) in enumerate(SIZES["tiny"])]


def test_permuted_batch_gives_permuted_outputs(prod):
    imgs = tiny_batch()
    perm = np.random.default_rng(3).permutation(len(imgs))
    with Ctx(prod, model_file("tiny", "q4_0", prod)) as ctx:
        e, ep = encode_mixed_dev(prod, ctx, imgs), encode_mixed_dev(prod, ctx, [imgs[p] for p in perm])
        t = tokens_mixed_dev(prod, ctx, imgs, -1, bd.TOKENS_NO_CLS | bd.TOKENS_POST_LN, bd.OUT_F16)
        tp = tokens_mixed_dev(prod, ctx, [imgs[p] for p in perm], -1, bd.TOKENS_NO_CLS | bd.TOKENS_POST_LN, bd.OUT_F16)
    for i, p in enumerate(perm):
        assert np.array_equal(bits(ep[i]), bits(e[p])), (i, p)
        assert np.array_equal(bits(tp[i]), bits(t[p])), (i, p)


def test_pass_boundaries_change_nothing(prod):
    """micro_batch 2 of tiny: 34 rows and 2 images a pass, so passes hold one or two images and end at every position"""
    sizes = [(64, 64), (16, 16), (64, 128), (32, 48), (16, 32), (48, 48), (16, 16), (64, 112), (16, 64)]
    imgs = [image(H, W, 40 + k) for k, (H, W) in enumerate(sizes)]
    path = model_file("tiny", "f16", prod)
    with Ctx(prod, path) as ctx:
        want_e = encode_mixed_dev(prod, ctx, imgs)
        want_t = tokens_mixed_dev(prod, ctx, imgs, -2, bd.TOKENS_PROJECT, bd.OUT_BF16)
    for shift in range(3):
        batch = imgs[shift:] + imgs[:shift]
        with Ctx(prod, path, (2, 0)) as ctx:
            got_e = encode_mixed_dev(prod, ctx, batch)
            got_t = tokens_mixed_dev(prod, ctx, batch, -2, bd.TOKENS_PROJECT, bd.OUT_BF16)
        for i in range(len(batch)):
            k = (i + shift) % len(imgs)
            assert np.array_equal(bits(got_e[i]), bits(want_e[k])), (shift, i)
            assert np.array_equal(bits(got_t[i]), bits(want_t[k])), (shift, i)


@pytest.mark.parametrize("bad", [np.nan, np.inf])
def test_non_finite_image_leaves_its_neighbours_alone(prod, bad):
    imgs = tiny_batch(9)
    with Ctx(prod, model_file("tiny", "f16", prod)) as ctx:
        clean_e = encode_mixed_dev(prod, ctx, imgs)
        clean_t = tokens_mixed_dev(prod, ctx, imgs, -1, 0)
        for k in (0, 3, len(imgs) - 1):
            x = [im.copy() for im in imgs]
            x[k][:] = bad
            got_e = encode_mixed_dev(prod, ctx, x)
            got_t = tokens_mixed_dev(prod, ctx, x, -1, 0)
            for j in range(len(imgs)):
                if j != k:
                    assert np.array_equal(bits(got_e[j]), bits(clean_e[j])), (k, j)
                    assert np.array_equal(bits(got_t[j]), bits(clean_t[j])), (k, j)


def test_one_size_equals_the_fixed_size_forms(prod):
    path = model_file("small-p14", "q4_0", prod)
    with Ctx(prod, path) as ctx:
        rect = images(5, 126, 252, 61)
        assert np.array_equal(bits(encode_mixed_dev(prod, ctx, list(rect))), bits(encode_dev(prod, ctx, rect)))
        got = tokens_mixed_dev(prod, ctx, list(rect), 3, bd.TOKENS_NO_CLS, bd.OUT_F16)
        assert np.array_equal(bits(np.stack(got)), bits(tokens_dev(prod, ctx, rect, 3, bd.TOKENS_NO_CLS, bd.OUT_F16)))
        native = sg.synth_images(6, 224, 62)
        assert np.array_equal(bits(prod.image_batch_encode_mixed(ctx, list(native))), bits(prod.image_batch_encode(ctx, native)))
        got = prod.image_tokens_mixed(ctx, list(native), -1, bd.TOKENS_POST_LN)
        assert np.array_equal(bits(np.stack(got)), bits(prod.image_tokens(ctx, native, -1, bd.TOKENS_POST_LN)))


def pinned_like(prod, shape, dtype):
    nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
    p = prod.lib.clip_b200_host_malloc(nbytes)
    assert p
    return p, np.frombuffer((C.c_uint8 * nbytes).from_address(p), dtype).reshape(shape)


def test_host_forms_equal_device_forms(prod):
    imgs = tiny_batch(21)
    flags = bd.TOKENS_NO_CLS | bd.TOKENS_PROJECT
    with Ctx(prod, model_file("tiny", "q4_0", prod)) as ctx:
        want_e = encode_mixed_dev(prod, ctx, imgs)
        want_t = tokens_mixed_dev(prod, ctx, imgs, -3, flags, bd.OUT_F16)
        assert np.array_equal(bits(prod.image_batch_encode_mixed(ctx, imgs)), bits(want_e))
        got = prod.image_tokens_mixed(ctx, imgs, -3, flags, bd.OUT_F16)          # pageable out
        for k in range(len(imgs)):
            assert np.array_equal(bits(got[k]), bits(want_t[k])), k
        rows = prod.mixed_token_rows(ctx, [im.shape[:2] for im in imgs], flags)
        batch, keep = prod.make_mixed_batch(imgs)
        p, out = pinned_like(prod, (sum(rows), width_of(prod, ctx, flags)), np.float16)
        try:
            assert prod.lib.clip_b200_image_tokens_mixed(ctx, C.byref(batch), -3, flags, bd.OUT_F16, p), prod.last_error()
            assert np.array_equal(bits(out), bits(np.concatenate(want_t)))
        finally:
            prod.lib.clip_b200_host_free(p)
        p, vec = pinned_like(prod, (len(imgs), prod.vision_hparams(ctx).projection_dim), np.float32)
        try:
            assert prod.lib.clip_b200_image_batch_encode_mixed(ctx, C.byref(batch), C.cast(p, FP), True), prod.last_error()
            assert np.array_equal(bits(vec), bits(want_e))
        finally:
            prod.lib.clip_b200_host_free(p)


def test_tiny_against_oracle(prod):
    path = model_file("tiny", "f16", prod)
    om = AnyresOracle(path)
    g = sg.GEOMETRIES["tiny"]
    P = g.patch_size
    sizes = [(64, 64), (16, 16), (64, 128), (112, 48), (128, 80)]
    imgs = [image(H, W, 70 + k) for k, (H, W) in enumerate(sizes)]
    pos = [om.position_table_hw(H // P, W // P, pos_resample_ref) for H, W in sizes]
    with Ctx(prod, path) as ctx:
        got = prod.image_batch_encode_mixed(ctx, imgs)
        toks = prod.image_tokens_mixed(ctx, imgs, 4, 0)
    for k, im in enumerate(imgs):
        assert float(cos_rows(got[k], om.encode_image_hw(im, pos[k], True))) <= TOL["f16"], k
        assert cos_rows(toks[k], om.image_tokens_hw(im, pos[k], 4)).max() <= TOL["f16"], k


# ---- 4. refusals ----------------------------------------------------------------------------------------------------------------

def test_refusals_in_order(prod):
    path = model_file("tiny", "f16", prod)
    good = [image(64, 64, 1), image(32, 48, 2)]
    h, w = sizes_arrays(good)
    with Ctx(prod, path, (2, 0)) as ctx:
        d_in = upload_packed(prod, ctx, good)
        d_out = prod.lib.clip_b200_device_malloc(ctx, 1 << 20)
        L = prod.lib

        def enc(n, hh, ww, di=d_in, do=d_out, c=ctx):
            return L.clip_b200_image_encode_device_mixed(c, di, n, hh.ctypes.data_as(IP) if hh is not None else None,
                                                         ww.ctypes.data_as(IP) if ww is not None else None, do, True)

        def tok(n, hh, ww, layer=-1, flags=0, ot=0, di=d_in, do=d_out):
            return L.clip_b200_image_tokens_device_mixed(ctx, di, n, hh.ctypes.data_as(IP) if hh is not None else None,
                                                         ww.ctypes.data_as(IP) if ww is not None else None, layer, flags, ot, do)

        def refused(ok, msg):
            assert not ok
            assert msg in prod.last_error(), (msg, prod.last_error())

        try:
            refused(enc(2, h, w, c=None), "clip_b200_image_encode_device_mixed: null context")
            bad_h = np.array([64, 40], np.int32)
            refused(enc(2, bad_h, w), "clip_b200_image_encode_device_mixed: image 1: height and width must be positive multiples of "
                                      "patch_size (16) and at most 4096, not 40 x 48")
            refused(enc(2, np.array([64, 4112], np.int32), np.array([64, 16], np.int32)), "image 1: height and width")
            refused(tok(2, bad_h, w, layer=99), "image 1: height and width")            # the size before the request
            assert enc(0, None, None, di=None, do=None)                                   # n == 0
            assert tok(0, None, None, layer=99, di=None, do=None)
            refused(enc(2, h, w, di=None), "clip_b200_image_encode_device_mixed: null device pointer")
            refused(tok(2, h, w, do=None, layer=99), "clip_b200_image_tokens_device_mixed: null device pointer")
            refused(enc(2, None, w), "clip_b200_image_encode_device_mixed: null heights or widths")
            refused(tok(2, h, w, layer=99), "clip_b200_image_tokens_device_mixed: layer 99 is outside")
            refused(tok(2, h, w, flags=bd.TOKENS_NORMALIZE), "NORMALIZE needs")
            refused(tok(2, h, w, ot=7), "unknown out_type 7")
            refused(tok(2, h, w, flags=bd.TOKENS_ATTENTION), "clip_b200_image_tokens_device_mixed: CLIP_B200_TOKENS_ATTENTION is not "
                                                             "supported at mixed sizes")
            big = [image(64, 64, 3), image(128, 128, 4)]                                 # T = 65 > 2 x 17 rows
            d_big = upload_packed(prod, ctx, big)
            bh, bw = sizes_arrays(big)
            refused(enc(2, bh, bw, di=d_big), "clip_b200_image_encode_device_mixed: image 1: one 128 x 128 image needs 65 rows, more than "
                                              "the workspace holds (34)")
            prod.lib.clip_b200_device_free(ctx, d_big)
            # host forms: n == 0, null pointers, then each image's pixels and size, then the request
            batch, keep = prod.make_mixed_batch([good[0], image(64, 40, 5)])
            vec = np.empty((2, prod.vision_hparams(ctx).projection_dim), np.float32)
            assert L.clip_b200_image_batch_encode_mixed(ctx, None, None, True)
            refused(L.clip_b200_image_batch_encode_mixed(ctx, C.byref(batch), None, True), "clip_b200_image_batch_encode_mixed: null output")
            refused(L.clip_b200_image_batch_encode_mixed(ctx, C.byref(batch), vec.ctypes.data_as(FP), True),
                    "clip_b200_image_batch_encode_mixed: image 1: height and width must be positive multiples of patch_size (16) and at "
                    "most 4096, not 64 x 40")
            refused(L.clip_b200_image_tokens_mixed(ctx, C.byref(batch), 99, 0, 0, vec.ctypes.data), "clip_b200_image_tokens_mixed: image 1")
            nopix = bd.clip_image_f32_batch((bd.clip_image_f32 * 1)(), 1)
            refused(L.clip_b200_image_batch_encode_mixed(ctx, C.byref(nopix), vec.ctypes.data_as(FP), True),
                    "clip_b200_image_batch_encode_mixed: image 0 has no pixels")
            batch, keep = prod.make_mixed_batch(good)
            refused(L.clip_b200_image_tokens_mixed(ctx, C.byref(batch), 0, bd.TOKENS_ATTENTION, 0, vec.ctypes.data),
                    "clip_b200_image_tokens_mixed: CLIP_B200_TOKENS_ATTENTION needs layer >= 1")
        finally:
            L.clip_b200_device_free(ctx, d_in)
            L.clip_b200_device_free(ctx, d_out)


# ---- 5. devices mode ------------------------------------------------------------------------------------------------------------

def test_devices_mode_equals_one_gpu(prod, monkeypatch):
    if prod.lib.clip_b200_cuda_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    imgs = [image(16 * (1 + k % 5), 16 * (1 + k % 7), 200 + k) for k in range(23)]
    path = model_file("tiny", "q4_0", prod)
    with Ctx(prod, path) as ctx:
        one_e = prod.image_batch_encode_mixed(ctx, imgs)
        one_t = prod.image_tokens_mixed(ctx, imgs, -2, bd.TOKENS_NO_CLS, bd.OUT_F16)
    monkeypatch.setenv("CLIP_B200_DEVICES", "all")
    with Ctx(prod, path) as ctx:
        assert prod.lib.clip_b200_device_count(ctx) >= 2
        assert np.array_equal(bits(prod.image_batch_encode_mixed(ctx, imgs)), bits(one_e))
        got = prod.image_tokens_mixed(ctx, imgs, -2, bd.TOKENS_NO_CLS, bd.OUT_F16)
        for k in range(len(imgs)):
            assert np.array_equal(bits(got[k]), bits(one_t[k])), k
