"""Attention probabilities through the public calls (CLIP_B200_TOKENS_ATTENTION / ATTENTION_CLS on every *_tokens call).

  * Every checked layer (1, middle, -2, -1) of both towers against the CPU oracle (tests/_oracle_attn.py), per query row at the
    hidden-state tests' bars, on tiny f16 / q4_0, tiny-gelu, small-p14-336 and huge-w640 (head_dim 80).
  * Slabs byte for byte: an attention slab of a _layers call equals the single-layer call; adding attention entries leaves every other
    slab unchanged; {-1 PROJECT, -1 ATTENTION} in either order gives the attention slab of ATTENTION alone (the stop order keeps qkv).
  * The same bytes on every path: host = device, pinned = pageable, several passes = one call per item, _hw at the native size =
    the native call, devices mode = one GPU; a rectangular _hw size against the oracle.
  * Text rows before the padding do not depend on the pad id; causal entries above the diagonal are +0.
  * One more launch per attention entry per micro-batch; the 16-byte slab padding; an attention slab past 2^32 bytes; every refusal."""
import ctypes as C

import numpy as np
import pytest

import binding as bd
import synth_gguf as sg
from _oracle_attn import AttnOracle
from _util import TOL, model_file, token_seqs
from test_gpu_anyres import images
from test_gpu_tokens import Ctx, bits, padded
from test_gpu_tokens_layers import check_slabs, pinned_like
from test_pos_resample import pos_resample_ref

pytestmark = pytest.mark.gpu

ATT, CLS = bd.TOKENS_ATTENTION, bd.TOKENS_ATTENTION | bd.TOKENS_ATTENTION_CLS
NO_CLS, PROJ = bd.TOKENS_NO_CLS, bd.TOKENS_PROJECT
GEOMS = [("tiny", "f16"), ("tiny", "q4_0"), ("tiny-gelu", "f16"), ("small-p14-336", "f16"), ("huge-w640", "f16")]


def row_cos_worst(got, want):
    """max over query rows of 1 - cos(got row, want row); got / want [..., R, K]"""
    g = np.asarray(got, np.float64)
    w = np.asarray(want, np.float64)
    c = (g * w).sum(-1) / (np.linalg.norm(g, axis=-1) * np.linalg.norm(w, axis=-1))
    return float((1 - c).max())


# ---- 1. against the oracle ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("geom,ft", GEOMS)
def test_layers_against_oracle(prod, geom, ft):
    g = sg.GEOMETRIES[geom]
    path = model_file(geom, ft, prod)
    om = AttnOracle(path)
    imgs = sg.synth_images(1 if g.n_pos > 257 else 2, g.image_size, 44)
    seqs = token_seqs(3)[1:] + [token_seqs(1)[0]]           # lengths 5, 2, 77
    ids = padded(seqs)
    tol = TOL[ft]
    worst = 0.0
    with Ctx(prod, path) as ctx:
        for vision, nl in ((True, g.v_layers), (False, g.t_layers)):
            for layer in (1, nl // 2, -2, -1):
                if vision:
                    got = prod.image_tokens(ctx, imgs, layer, ATT)
                    cls = prod.image_tokens(ctx, imgs, layer, CLS)
                    assert np.array_equal(bits(cls), bits(got[:, :, :1])), (geom, layer)
                    for k, img in enumerate(imgs):
                        d = row_cos_worst(got[k], om.image_attention(img, layer))
                        worst = max(worst, d)
                        assert d <= tol, ("image", geom, ft, layer, k, d)
                else:
                    got = prod.text_tokens(ctx, ids, layer, ATT)
                    T = ids.shape[1]
                    assert (bits(got)[:, :, np.triu(np.ones((T, T), bool), 1)] == 0).all()
                    for k, s in enumerate(seqs):
                        n = len(s)
                        d = row_cos_worst(got[k, :, :n, :n], om.text_attention(s, layer))
                        worst = max(worst, d)
                        assert d <= tol, ("text", geom, ft, layer, k, d)
    print("%s %s: worst per-row 1 - cos = %.3g (bar %g)" % (geom, ft, worst, tol))


def test_rectangle_against_oracle(prod):
    g = sg.GEOMETRIES["tiny"]
    S, P = g.image_size, g.patch_size
    path = model_file("tiny", "f16", prod)
    om = AttnOracle(path)
    H, W = S - 2 * P, S + 4 * P
    pos = om.position_table_hw(H // P, W // P, pos_resample_ref)
    imgs = images(2, H, W, 5)
    with Ctx(prod, path) as ctx:
        for layer in (1, -2):
            got = prod.image_tokens_hw(ctx, imgs, layer, ATT)
            assert got.shape == (2, g.v_heads, (H // P) * (W // P) + 1, (H // P) * (W // P) + 1)
            for k in range(2):
                d = row_cos_worst(got[k], om.image_attention(imgs[k], layer, pos))
                assert d <= TOL["f16"], (layer, k, d)


# ---- 2. slabs and paths ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("geom", ["tiny", "huge-w640"])
def test_slabs_equal_single_calls(prod, geom):
    g = sg.GEOMETRIES[geom]
    imgs = sg.synth_images(3, g.image_size, 12)
    ids = padded(token_seqs(3))
    with Ctx(prod, model_file(geom, "f16", prod)) as ctx:
        for vision, nl in ((True, g.v_layers), (False, g.t_layers)):
            nc = NO_CLS if vision else 0
            cls = CLS if vision else ATT
            with_attn = ([-2, -2, 1, -1, -1, nl // 2], [nc, cls, ATT, PROJ, ATT, 0])
            without = ([-2, -1, nl // 2], [nc, PROJ, 0])
            for ot in (bd.OUT_F32, bd.OUT_F16, bd.OUT_BF16):
                if vision:
                    single = lambda l, f: prod.image_tokens(ctx, imgs, l, f, ot)
                    multi = lambda ls, fs: prod.image_tokens_layers(ctx, imgs, ls, fs, ot)
                    multi_dev = lambda ls, fs: prod.image_tokens_layers_device(ctx, imgs, ls, fs, ot)
                else:
                    single = lambda l, f: prod.text_tokens(ctx, ids, l, f, ot)
                    multi = lambda ls, fs: prod.text_tokens_layers(ctx, ids, ls, fs, ot)
                    multi_dev = lambda ls, fs: prod.text_tokens_layers_device(ctx, ids, ls, fs, ot)
                want = [single(l, f) for l, f in zip(*with_attn)]
                check_slabs(multi(*with_attn), want, (geom, vision, ot, "host"))
                check_slabs(multi_dev(*with_attn), want, (geom, vision, ot, "device"))
                check_slabs(multi(*without), [want[0], want[3], want[5]], (geom, vision, ot, "without attention"))
                for ls, fs, j in (([-1, -1], [PROJ, ATT], 1), ([-1, -1], [ATT, PROJ], 0)):
                    check_slabs([multi(ls, fs)[j]], [want[4]], (geom, vision, ot, "project and attention", fs))


def test_several_passes_pinned_and_single_items(prod):
    """micro batches of 4 images and 3 sequences (passes 4, 4, 3 and 3, 3, 2) = one call per item; host = device; pinned = pageable"""
    path = model_file("tiny", "f16", prod)
    imgs = sg.synth_images(11, 64, 18)
    ids = padded(token_seqs(8))
    layers = [-2, -2, 3, -1]
    fi, ft = [NO_CLS, CLS, ATT, ATT], [0, ATT, ATT, PROJ]
    ot = bd.OUT_F16
    with Ctx(prod, path, (4, 3)) as ctx:
        host_i = prod.image_tokens_layers(ctx, imgs, layers, fi, ot)
        host_t = prod.text_tokens_layers(ctx, ids, layers, ft, ot)
        check_slabs(prod.image_tokens_layers_device(ctx, imgs, layers, fi, ot), host_i, "image device = host")
        check_slabs(prod.text_tokens_layers_device(ctx, ids, layers, ft, ot), host_t, "text device = host")
        for name, fn, want, fl in (("image", lambda o: prod.image_tokens_layers(ctx, imgs, layers, fi, ot, o), host_i, fi),
                                   ("text", lambda o: prod.text_tokens_layers(ctx, ids, layers, ft, ot, o), host_t, ft)):
            offs = bd.slab_offsets([w.nbytes for w in want], fl)
            buf, p = pinned_like(prod, (offs[-1] + want[-1].nbytes) // 2, np.float16)
            try:
                check_slabs([v.copy() for v in fn(buf)], want, name + " pinned = pageable")
            finally:
                prod.lib.clip_b200_host_free(p)
    with Ctx(prod, path) as ctx:
        for k in range(len(imgs)):
            for j, (l, f) in enumerate(zip(layers, fi)):
                assert np.array_equal(bits(prod.image_tokens(ctx, imgs[k:k + 1], l, f, ot)[0]), bits(host_i[j][k])), (k, j)
        for k in range(len(ids)):
            for j, (l, f) in enumerate(zip(layers, ft)):
                assert np.array_equal(bits(prod.text_tokens(ctx, ids[k:k + 1], l, f, ot)[0]), bits(host_t[j][k])), (k, j)


def test_hw_native_size_equals_native_call(prod):
    g = sg.GEOMETRIES["huge-w640"]
    imgs = sg.synth_images(2, g.image_size, 3)
    with Ctx(prod, model_file("huge-w640", "f16", prod)) as ctx:
        for l, f in ((-1, ATT), (-2, CLS), (1, ATT)):
            assert np.array_equal(bits(prod.image_tokens_hw(ctx, imgs, l, f, bd.OUT_BF16)), bits(prod.image_tokens(ctx, imgs, l, f, bd.OUT_BF16)))


def test_text_rows_before_padding_do_not_depend_on_pad_id(prod):
    seqs = token_seqs(4)
    with Ctx(prod, model_file("tiny", "f16", prod)) as ctx:
        a = prod.text_tokens(ctx, padded(seqs, pad=0), -2, ATT)
        b = prod.text_tokens(ctx, padded(seqs, pad=407), -2, ATT)
        for k, s in enumerate(seqs):
            n = len(s)
            assert np.array_equal(bits(a[k, :, :n]), bits(b[k, :, :n])), k


def test_launch_count(prod):
    """one more launch per attention entry per micro-batch (passes of 4 images: 11 images -> 3)"""
    imgs = sg.synth_images(11, 64, 8)
    ids = padded(token_seqs(5))
    with Ctx(prod, model_file("tiny", "q4_0", prod), (4, 3)) as ctx:
        n = prod.lib.clip_b200_kernel_launches

        def count(fn):
            fn()
            a = n(ctx)
            fn()
            return n(ctx) - a

        base_i = count(lambda: prod.image_tokens_layers(ctx, imgs, [-2, -1], [NO_CLS, PROJ]))
        att_i = count(lambda: prod.image_tokens_layers(ctx, imgs, [-2, 1, -2, -1], [NO_CLS, ATT, CLS, PROJ]))
        assert att_i == base_i + 2 * 3, (base_i, att_i)
        base_t = count(lambda: prod.text_tokens_layers(ctx, ids, [-1], [PROJ]))
        att_t = count(lambda: prod.text_tokens_layers(ctx, ids, [-1, -1], [ATT, PROJ]))
        assert att_t == base_t + 2, (base_t, att_t)


def test_slab_padding(prod):
    """tiny, T = 17, 2 heads, the CLS row in f16: 68 bytes per image, so the next slab of a one-image call starts at byte 80"""
    g = sg.GEOMETRIES["tiny"]
    imgs = sg.synth_images(1, g.image_size, 2)
    layers, flags = [-2, -2, -1], [CLS, NO_CLS, CLS]
    with Ctx(prod, model_file("tiny", "f16", prod)) as ctx:
        want = [prod.image_tokens(ctx, imgs, l, f, bd.OUT_F16) for l, f in zip(layers, flags)]
        assert want[0].nbytes == 68
        offs = bd.slab_offsets([w.nbytes for w in want], flags)
        assert offs == [0, 80, 80 + want[1].nbytes]
        raw = np.full((offs[2] + want[2].nbytes) // 2, 0x5555, np.uint16)
        views = prod.image_tokens_layers(ctx, imgs, layers, flags, bd.OUT_F16, raw.view(np.float16))
        check_slabs(views, want, "views")
        b = raw.view(np.uint8)
        for o, w in zip(offs, want):
            assert np.array_equal(b[o:o + w.nbytes], np.ascontiguousarray(w).view(np.uint8).reshape(-1)), o
        assert (b[68:80] == 0x55).all()                       # the padding is not written
        # no attention entries: today's layout, byte for byte
        plain = prod.image_tokens_layers(ctx, imgs, [-2, -1], [NO_CLS, 0], bd.OUT_F16)
        assert plain[1].__array_interface__["data"][0] - plain[0].__array_interface__["data"][0] == plain[0].nbytes


def test_attention_slab_past_4_gib(prod):
    """device form, tiny at 1024 x 1024 (T = 4097, 2 heads, f32: 134 MB per image), 33 images: the slab is 4.43 GB and its last
    item starts past 2^32 bytes; it equals a one-image call"""
    g = sg.GEOMETRIES["tiny"]
    S = 1024
    T = (S // g.patch_size) ** 2 + 1
    n = 33
    item = g.v_heads * T * T * 4
    assert (n - 1) * item > 2 ** 32
    imgs = images(n, S, S, 9)
    L = prod.lib
    with Ctx(prod, model_file("tiny", "f16", prod)) as ctx:
        layer = C.c_int * 1
        d_in = L.clip_b200_device_malloc(ctx, imgs.nbytes)
        d_out = L.clip_b200_device_malloc(ctx, n * item)
        assert d_in and d_out
        try:
            assert L.clip_b200_memcpy_h2d(ctx, d_in, imgs.ctypes.data, imgs.nbytes)
            assert L.clip_b200_image_tokens_layers_device(ctx, d_in, n, S, S, layer(-1), layer(ATT), 1, bd.OUT_F32, d_out), prod.last_error()
            last = np.empty(item // 4, np.float32)
            assert L.clip_b200_memcpy_d2h(ctx, last.ctypes.data, d_out + (n - 1) * item, item)
            one = np.empty(item // 4, np.float32)
            assert L.clip_b200_memcpy_h2d(ctx, d_in, imgs[n - 1:].ctypes.data, imgs[n - 1:].nbytes)
            assert L.clip_b200_image_tokens_device_hw(ctx, d_in, 1, S, S, -1, ATT, bd.OUT_F32, d_out), prod.last_error()
            assert L.clip_b200_memcpy_d2h(ctx, one.ctypes.data, d_out, item)
        finally:
            L.clip_b200_device_free(ctx, d_in)
            L.clip_b200_device_free(ctx, d_out)
        assert np.array_equal(bits(last), bits(one))
        assert np.isfinite(last).all() and abs(last.reshape(g.v_heads, T, T).sum(-1) - 1).max() < 1e-3


# ---- 3. refusals and devices mode -----------------------------------------------------------------------------------------------

def test_refusals(prod):
    g = sg.GEOMETRIES["tiny"]
    imgs = sg.synth_images(1, g.image_size, 1)
    ids = padded(token_seqs(1))
    batch, keep = prod.make_image_batch(imgs)
    out = np.empty(1 << 20, np.float32)
    L = prod.lib

    def ci(vals):
        return (C.c_int * len(vals))(*vals)

    def expect(ok, *msgs):
        assert not ok, msgs
        for m in msgs:
            assert m in prod.last_error(), (m, prod.last_error())

    with Ctx(prod, model_file("tiny", "f16", prod)) as ctx:
        img = lambda l, f: L.clip_b200_image_tokens(ctx, C.byref(batch), l, f, 0, out.ctypes.data)
        txt = lambda l, f: L.clip_b200_text_tokens(ctx, ids.ctypes.data_as(C.POINTER(C.c_int32)), 1, 77, l, f, 0, out.ctypes.data)
        for call in (img, txt):
            expect(call(0, ATT), "ATTENTION needs layer >= 1")
            expect(call(-13, ATT), "ATTENTION needs layer >= 1")
            for extra in (bd.TOKENS_POST_LN, PROJ, PROJ | bd.TOKENS_NORMALIZE, NO_CLS):
                expect(call(-1, ATT | extra), "cannot be combined")
            expect(call(-1, bd.TOKENS_ATTENTION_CLS), "ATTENTION_CLS needs CLIP_B200_TOKENS_ATTENTION")
            expect(call(-1, 16 | ATT), "unknown flag")
        expect(txt(-1, CLS), "vision tower only")
        assert img(-1, CLS) and img(1, ATT) and txt(12, ATT) and txt(-12, ATT)
        expect(L.clip_b200_image_tokens_layers(ctx, C.byref(batch), ci([-1, 0]), ci([0, ATT]), 2, 0, out.ctypes.data), "entry 1", "layer >= 1")
        expect(L.clip_b200_text_tokens_layers(ctx, ids.ctypes.data_as(C.POINTER(C.c_int32)), 1, 77, ci([-1, -1]), ci([ATT, CLS]), 2, 0,
                                              out.ctypes.data), "entry 1", "vision tower only")
        expect(L.clip_b200_image_tokens_device_hw(ctx, None, 1, 64, 64, -1, ATT | NO_CLS, 0, None), "cannot be combined")


def test_devices_mode_equals_one_gpu(prod, monkeypatch):
    if prod.lib.clip_b200_cuda_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    g = sg.GEOMETRIES["tiny"]
    imgs = sg.synth_images(37, g.image_size, 71)
    ids = padded(token_seqs(19))
    path = model_file("tiny", "q4_0", prod)
    layers = [-2, -2, -1]
    fi, ft = [NO_CLS, CLS, ATT], [0, ATT, PROJ]
    with Ctx(prod, path) as ctx:
        one_i = prod.image_tokens_layers(ctx, imgs, layers, fi, bd.OUT_F16)
        one_t = prod.text_tokens_layers(ctx, ids, layers, ft, bd.OUT_BF16)
    monkeypatch.setenv("CLIP_B200_DEVICES", "all")
    with Ctx(prod, path) as ctx:
        assert prod.lib.clip_b200_device_count(ctx) >= 2
        check_slabs(prod.image_tokens_layers(ctx, imgs, layers, fi, bd.OUT_F16), one_i, "image")
        check_slabs(prod.text_tokens_layers(ctx, ids, layers, ft, bd.OUT_BF16), one_t, "text")
