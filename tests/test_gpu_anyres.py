"""The vision tower at any patch-multiple image size (clip_b200_image_encode_device_hw, clip_b200_image_tokens_device_hw and the
host forms clip_b200_image_batch_encode_hw / clip_b200_image_tokens_hw), with the position table resampled as HF's
interpolate_pos_encoding does.

  1. K8 equals the fp64 restatement (tests/test_pos_resample.py, itself checked against torch) bit for bit; rectangular K0 equals a
     numpy patchify exactly.
  2. At the model's own size every *_hw entry point equals its existing counterpart bit for bit.
  3. A model whose file carries the resampled table and the new image_size, loaded natively, equals *_hw on the original model.
  4. Rectangular sizes against the CPU oracle (tests/_oracle_anyres.py) at the project's 1 - cos bars, embeddings and every layer.
  5. Planning: several passes equal one call per image; a large first call leaves the workspace of the native size; the cached
     table follows the size.
  6. Refusals, with their messages.  7. Devices mode equals one GPU."""
import ctypes as C

import numpy as np
import pytest

import binding as bd
import oracle as orc
import synth_gguf as sg
from _oracle_anyres import AnyresOracle
from _util import TOL, model_file
from test_gpu_tokens import PROJ_N, Ctx, bits, on_device
from test_pos_resample import pos_resample_ref

pytestmark = pytest.mark.gpu

FP = C.POINTER(C.c_float)


def images(n, H, W, seed):
    """[n, H, W, 3] f32 NHWC, U(-2, 2), as synth_gguf.synth_images"""
    rng = np.random.Generator(np.random.PCG64(seed))
    return rng.random(size=(n, H, W, 3), dtype=np.float32) * np.float32(4.0) - np.float32(2.0)


def n_rows(prod, ctx, H, W):
    P = prod.vision_hparams(ctx).patch_size
    return (H // P) * (W // P) + 1


def encode_dev(prod, ctx, imgs, normalize=True):
    n, H, W = imgs.shape[:3]
    d = prod.vision_hparams(ctx).projection_dim
    return on_device(prod, ctx, lambda di, do: prod.lib.clip_b200_image_encode_device_hw(ctx, di, n, H, W, do, normalize),
                     imgs, (n, d), np.float32)


def tokens_dev(prod, ctx, imgs, layer, flags, ot=bd.OUT_F32):
    n, H, W = imgs.shape[:3]
    shape = prod.token_shape(ctx, True, n, n_rows(prod, ctx, H, W), flags)
    return on_device(prod, ctx, lambda di, do: prod.lib.clip_b200_image_tokens_device_hw(ctx, di, n, H, W, layer, flags, ot, do),
                     imgs, shape, bd.OUT_DTYPES[ot])


def cos_rows(got, want):
    got = np.asarray(got, np.float64)
    want = np.asarray(want, np.float64)
    return 1 - np.sum(got * want, -1) / (np.linalg.norm(got, axis=-1) * np.linalg.norm(want, axis=-1))


# ---- 1. the kernels alone -------------------------------------------------------------------------------------------------------

RESAMPLE = [(7, 12, 12), (16, 7, 7), (16, 24, 8), (4, 3, 6), (7, 1, 1), (7, 7, 7), (16, 24, 24), (16, 32, 32)]


@pytest.mark.parametrize("h", [128, 1280])
@pytest.mark.parametrize("g,gh,gw", RESAMPLE)
def test_pos_resample_kernel_is_the_restatement(prod, g, gh, gw, h):
    rng = np.random.default_rng(g * 1000 + gh * 10 + gw + h)
    table = (rng.standard_normal((g * g, h)) * 0.05).astype(np.float32)
    table[rng.integers(g * g), rng.integers(h)] = 3.0           # one large entry: its taps must not leak beyond 4 x 4 outputs
    out = np.empty((gh * gw, h), np.float32)
    assert prod.lib.clip_b200_debug_pos_resample(table.ctypes.data_as(FP), g, h, gh, gw, out.ctypes.data_as(FP)) == 0, prod.last_error()
    want = pos_resample_ref(table, g, gh, gw)
    assert np.array_equal(bits(out), bits(want)), (g, gh, gw, h, int((bits(out) != bits(want)).sum()))


def patchify(px, P, kpad):
    B, H, W, _ = px.shape
    gh, gw = H // P, W // P
    p = px.reshape(B, gh, P, gw, P, 3).transpose(0, 1, 3, 5, 2, 4).reshape(B * gh * gw, 3 * P * P)
    out = np.zeros((B * gh * gw, kpad), np.float32)
    out[:, :3 * P * P] = p.astype(np.float16).astype(np.float32)
    return out


@pytest.mark.parametrize("B,H,W,P,kpad", [(2, 64, 128, 16, 768), (3, 112, 48, 16, 768), (2, 42, 28, 14, 640), (1, 224, 448, 14, 640),
                                          (2, 64, 64, 16, 768)])
def test_im2col_rectangles(prod, B, H, W, P, kpad):
    px = images(B, H, W, B * H + W)
    out = np.empty((B * (H // P) * (W // P), kpad), np.float32)
    assert prod.lib.clip_b200_debug_im2col_hw(px.ctypes.data_as(FP), B, H, W, P, kpad, out.ctypes.data_as(FP)) == 0, prod.last_error()
    assert np.array_equal(bits(out), bits(patchify(px, P, kpad)))
    if H == W:                                                   # the square hook is the same kernel, the same bytes
        sq = np.empty_like(out)
        assert prod.lib.clip_b200_debug_im2col(px.ctypes.data_as(FP), B, H, P, kpad, sq.ctypes.data_as(FP)) == 0
        assert np.array_equal(bits(sq), bits(out))


# ---- 2. the model's own size ----------------------------------------------------------------------------------------------------

TOKEN_FLAGS = [0, bd.TOKENS_POST_LN, bd.TOKENS_PROJECT, PROJ_N, bd.TOKENS_NO_CLS, bd.TOKENS_POST_LN | bd.TOKENS_NO_CLS]


@pytest.mark.parametrize("ft", ["f16", "q4_0"])
@pytest.mark.parametrize("geom", ["tiny", "vit-b32"])
def test_native_size_equals_existing_entry_points(prod, geom, ft):
    g = sg.GEOMETRIES[geom]
    S = g.image_size
    imgs = sg.synth_images(3, S, 12)
    with Ctx(prod, model_file(geom, ft, prod)) as ctx:
        d = g.proj_dim
        for normalize in (True, False):
            want = prod.image_batch_encode(ctx, imgs, normalize=normalize)
            assert np.array_equal(bits(prod.image_batch_encode_hw(ctx, imgs, normalize)), bits(want)), normalize
            dev = on_device(prod, ctx, lambda di, do: prod.lib.clip_b200_image_encode_device(ctx, di, 3, do, normalize), imgs, (3, d), np.float32)
            assert np.array_equal(bits(encode_dev(prod, ctx, imgs, normalize)), bits(dev)), normalize
        for layer in (0, -2, -1):
            for flags in TOKEN_FLAGS:
                want = prod.image_tokens(ctx, imgs, layer, flags)
                assert np.array_equal(bits(prod.image_tokens_hw(ctx, imgs, layer, flags)), bits(want)), (layer, flags)
                dev = on_device(prod, ctx, lambda di, do: prod.lib.clip_b200_image_tokens_device(ctx, di, 3, layer, flags, bd.OUT_F16, do),
                                imgs, want.shape, np.float16)
                assert np.array_equal(bits(tokens_dev(prod, ctx, imgs, layer, flags, bd.OUT_F16)), bits(dev)), (layer, flags)


# ---- 3. a derived model with the resampled table --------------------------------------------------------------------------------

def write_derived(src, dst, image_size, pos):
    """src's tensors and keys, copied one for one, except clip.vision.image_size = image_size and v.position_embd.weight = pos (f32)"""
    g = orc.GGUF(src)
    w = sg._Writer()
    for key in g.kv_order:
        typ, val = g.kv[key]
        if key == "clip.vision.image_size":
            val = image_size
        if typ == sg.T_ARR:
            (w.add_array_str if val and isinstance(val[0], str) else w.add_array_f32)(key, val)
        else:
            w.add(key, typ, val)
    for name in g.order:
        t = g.tensors[name]
        if name == "v.position_embd.weight":
            w.add_tensor(name, np.ascontiguousarray(pos, np.float32))
            continue
        assert t.type in (orc.F32, orc.F16), (name, t.type)
        w.add_tensor(name, np.frombuffer(t.data, np.float32 if t.type == orc.F32 else np.float16).reshape(t.shape))
    w.write(dst)


@pytest.mark.parametrize("geom,S2", [("tiny", 48), ("tiny", 96), ("small-p14", 336)])
def test_derived_model_equals_hw(prod, tmp_path, geom, S2):
    path = model_file(geom, "f16", prod)
    om = AnyresOracle(path)
    g2 = S2 // om.patch
    pos = om.position_table_hw(g2, g2, pos_resample_ref)
    derived = str(tmp_path / ("%s-%d.gguf" % (geom, S2)))
    write_derived(path, derived, S2, pos)
    imgs = images(3, S2, S2, S2)
    calls = [lambda ctx, f: f.image_batch_encode(ctx, imgs, True), lambda ctx, f: f.image_batch_encode(ctx, imgs, False)]
    calls += [lambda ctx, f, l=layer, fl=flags: f.image_tokens(ctx, imgs, l, fl)
              for layer, flags in ((-1, bd.TOKENS_POST_LN), (-2, bd.TOKENS_NO_CLS), (-1, PROJ_N), (0, 0))]

    class Hw:      # the *_hw host forms under the names of the native ones
        def image_batch_encode(self, ctx, x, normalize):
            return prod.image_batch_encode_hw(ctx, x, normalize)

        def image_tokens(self, ctx, x, layer, flags):
            return prod.image_tokens_hw(ctx, x, layer, flags)

    with Ctx(prod, path) as ctx:
        got = [f(ctx, Hw()) for f in calls]
        got.append(encode_dev(prod, ctx, imgs))
        got.append(tokens_dev(prod, ctx, imgs, -2, bd.TOKENS_POST_LN, bd.OUT_BF16))
    with Ctx(prod, derived) as ctx:
        assert prod.vision_hparams(ctx).image_size == S2
        want = [f(ctx, prod) for f in calls]
        want.append(prod.image_batch_encode(ctx, imgs))
        want.append(prod.image_tokens(ctx, imgs, -2, bd.TOKENS_POST_LN, bd.OUT_BF16))
    assert want[2].shape[1] == g2 * g2 + 1
    for i, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(bits(a), bits(b)), (geom, S2, i)


# ---- 4. rectangles against the oracle -------------------------------------------------------------------------------------------

RECT = [("tiny", "f16", 64, 128), ("tiny", "q4_0", 64, 128), ("tiny", "f16", 112, 48), ("tiny", "q4_0", 112, 48),
        ("small-p14", "f16", 224, 448), ("small-p14", "q4_0", 224, 448)]


@pytest.mark.parametrize("geom,ft,H,W", RECT)
def test_rectangles_against_oracle(prod, geom, ft, H, W):
    g = sg.GEOMETRIES[geom]
    path = model_file(geom, ft, prod)
    om = AnyresOracle(path)
    P = g.patch_size
    pos = om.position_table_hw(H // P, W // P, pos_resample_ref)
    imgs = images(1 if H * W > 64 * 128 else 2, H, W, H + W)
    tol = TOL[ft]
    worst = 0.0
    with Ctx(prod, path) as ctx:
        for normalize in (True, False):
            got = prod.image_batch_encode_hw(ctx, imgs, normalize)
            for k, img in enumerate(imgs):
                d = float(cos_rows(got[k], om.encode_image_hw(img, pos, normalize)))
                assert d <= tol, (geom, ft, H, W, "embedding", normalize, d)
        for layer in (0, 1, g.v_layers // 2, -2, -1):
            raw = [om.image_tokens_hw(img, pos, layer) for img in imgs]
            for post_ln in (False, True):
                got = prod.image_tokens_hw(ctx, imgs, layer, bd.TOKENS_POST_LN if post_ln else 0)
                assert got.shape == (len(imgs), (H // P) * (W // P) + 1, g.v_hidden)
                for k in range(len(imgs)):
                    want = om.ln(raw[k], "v.post_ln.weight", "v.post_ln.bias", om.v_eps) if post_ln else raw[k]
                    d = cos_rows(got[k], want)
                    assert d.max() <= tol, (geom, ft, H, W, layer, post_ln, float(d.max()))
                    worst = max(worst, float(d.max()))
    print("%s %s %dx%d  worst per-token 1-cos %.2e (bar %.0e)" % (geom, ft, H, W, worst, tol))


# ---- 5. planning ----------------------------------------------------------------------------------------------------------------

def test_several_passes_equal_one_call_per_image(prod):
    """micro_batch 8 of tiny (T = 17): 136 rows; at 128 x 128 (T = 65) two images fit a pass, so 5 images take 3 passes"""
    path = model_file("tiny", "f16", prod)
    imgs = images(5, 128, 128, 3)
    flags = bd.TOKENS_POST_LN | bd.TOKENS_NO_CLS
    with Ctx(prod, path, (8, 0)) as ctx:
        launches = prod.lib.clip_b200_kernel_launches
        one_e = [prod.image_batch_encode_hw(ctx, imgs[k:k + 1], True) for k in range(5)]           # the first resamples the table
        a = launches(ctx)
        one_t = [prod.image_tokens_hw(ctx, imgs[k:k + 1], -2, flags, bd.OUT_F16) for k in range(5)]
        per_pass = (launches(ctx) - a) // 5
        a = launches(ctx)
        big_t = prod.image_tokens_hw(ctx, imgs, -2, flags, bd.OUT_F16)
        assert launches(ctx) - a == 3 * per_pass, (launches(ctx) - a, per_pass)
        big_e = prod.image_batch_encode_hw(ctx, imgs, True)
        big_d = encode_dev(prod, ctx, imgs)
    for k in range(5):
        assert np.array_equal(bits(big_e[k]), bits(one_e[k][0])), k
        assert np.array_equal(bits(big_d[k]), bits(one_e[k][0])), k
        assert np.array_equal(bits(big_t[k]), bits(one_t[k][0])), k


def test_large_first_call_keeps_the_native_workspace(prod):
    path = model_file("tiny", "q4_0", prod)
    native = sg.synth_images(4, 64, 8)
    large = images(3, 128, 128, 9)
    with Ctx(prod, path) as ctx:
        want_e = prod.image_batch_encode(ctx, native)
        want_t = prod.image_tokens(ctx, native, -1, bd.TOKENS_POST_LN)
    with Ctx(prod, path) as ctx:
        prod.image_batch_encode_hw(ctx, large)
        got_e = prod.image_batch_encode(ctx, native)
        got_t = prod.image_tokens(ctx, native, -1, bd.TOKENS_POST_LN)
    assert np.array_equal(bits(got_e), bits(want_e))
    assert np.array_equal(bits(got_t), bits(want_t))


def test_table_cache_follows_the_size(prod):
    """sizes A, B, A in one context give what fresh contexts give"""
    path = model_file("tiny", "f16", prod)
    a = images(2, 96, 64, 10)
    b = images(2, 48, 112, 11)
    fresh = {}
    for name, x in (("a", a), ("b", b)):
        with Ctx(prod, path) as ctx:
            fresh[name] = (prod.image_batch_encode_hw(ctx, x), prod.image_tokens_hw(ctx, x, -1, 0))
    with Ctx(prod, path) as ctx:
        seq = [(prod.image_batch_encode_hw(ctx, x), prod.image_tokens_hw(ctx, x, -1, 0)) for x in (a, b, a)]
    for got, name in zip(seq, ("a", "b", "a")):
        assert np.array_equal(bits(got[0]), bits(fresh[name][0])), name
        assert np.array_equal(bits(got[1]), bits(fresh[name][1])), name


# ---- 6. refusals ----------------------------------------------------------------------------------------------------------------

def test_refusals(prod, tmp_path):
    L = prod.lib
    out = np.empty(1 << 22, np.float32)
    path = model_file("tiny", "f16", prod)

    def dev_enc(ctx, H, W, n=1):
        return L.clip_b200_image_encode_device_hw(ctx, out.ctypes.data, n, H, W, out.ctypes.data, True)

    def dev_tok(ctx, H, W, layer=-1, flags=0, ot=0, n=1):
        return L.clip_b200_image_tokens_device_hw(ctx, out.ctypes.data, n, H, W, layer, flags, ot, out.ctypes.data)

    def host(ctx, x, tokens=False, layer=-1):
        batch, keep = prod.make_image_batch(x)
        if tokens:
            return L.clip_b200_image_tokens_hw(ctx, C.byref(batch), layer, 0, 0, out.ctypes.data)
        return L.clip_b200_image_batch_encode_hw(ctx, C.byref(batch), out.ctypes.data_as(FP), True)

    def expect(ok, msg):
        assert not ok, msg
        assert msg in prod.last_error(), (msg, prod.last_error())

    with Ctx(prod, path) as ctx:
        for H, W in ((65, 64), (64, 0), (0, 64), (-16, 64), (64, 4112), (4112, 4112)):
            expect(dev_enc(ctx, H, W), "positive multiples of patch_size (16)")
            expect(dev_tok(ctx, H, W), "positive multiples of patch_size (16)")
        expect(host(ctx, images(2, 70, 64, 1)), "positive multiples of patch_size (16)")
        expect(host(ctx, images(1, 48, 40, 1), True), "positive multiples of patch_size (16)")
        expect(dev_tok(ctx, 64, 128, 13), "layer 13")
        expect(dev_tok(ctx, 64, 128, -1, bd.TOKENS_NORMALIZE), "needs")
        expect(dev_tok(ctx, 64, 128, -1, 0, 3), "out_type")
        expect(host(ctx, images(1, 64, 128, 1), True, 13), "layer 13")
        # mixed sizes in one host call
        x1, x2 = images(1, 64, 64, 1), images(1, 64, 128, 2)
        arr = (bd.clip_image_f32 * 2)()
        for i, x in enumerate((x1, x2)):
            arr[i] = bd.clip_image_f32(x.shape[2], x.shape[1], x.ctypes.data_as(FP), x.size)
        mixed = bd.clip_image_f32_batch(arr, 2)
        expect(L.clip_b200_image_batch_encode_hw(ctx, C.byref(mixed), out.ctypes.data_as(FP), True), "same size")
        expect(L.clip_b200_image_tokens_hw(ctx, C.byref(mixed), -1, 0, 0, out.ctypes.data), "same size")
        # n == 0
        empty = bd.clip_image_f32_batch(None, 0)
        assert L.clip_b200_image_batch_encode_hw(ctx, C.byref(empty), None, True)
        assert L.clip_b200_image_tokens_hw(ctx, C.byref(empty), -1, 0, 0, None)
        assert L.clip_b200_image_encode_device_hw(ctx, None, 0, 64, 128, None, True)
        assert L.clip_b200_image_tokens_device_hw(ctx, None, 0, 64, 128, -1, 0, 0, None)
        # the existing entry points still take the model's size only
        batch, keep = prod.make_image_batch(images(1, 128, 128, 1))
        expect(L.clip_image_batch_encode(ctx, 1, C.byref(batch), out.ctypes.data_as(FP), True), "image_size x image_size")
        expect(L.clip_b200_image_tokens(ctx, C.byref(batch), -1, 0, 0, out.ctypes.data), "image_size x image_size")
    # one image too large for the workspace: micro_batch 1 of tiny holds 17 rows, 128 x 128 needs 65
    with Ctx(prod, path, (1, 0)) as ctx:
        expect(host(ctx, images(1, 128, 128, 1)), "more than the workspace holds")
        expect(dev_tok(ctx, 128, 128), "more than the workspace holds")
        assert host(ctx, images(1, 32, 64, 1)), prod.last_error()      # 9 rows fit
        assert prod.image_batch_encode(ctx, sg.synth_images(1, 64, 1)).shape == (1, 128)
    text_only = sg.Geometry("text-only", image_size=64, patch_size=16, v_hidden=128, v_ff=256, v_heads=2, v_layers=1,
                            t_hidden=128, t_ff=256, t_heads=2, t_layers=2, proj_dim=128, has_vision=False)
    tpath = str(tmp_path / "text-only.gguf")
    sg.write_model(tpath, text_only, 1, 1)
    with Ctx(prod, tpath) as ctx:
        expect(dev_enc(ctx, 64, 64), "no vision encoder")
        expect(dev_tok(ctx, 64, 64), "no vision encoder")
        expect(host(ctx, images(1, 64, 64, 1)), "no vision encoder")
        expect(host(ctx, images(1, 64, 64, 1), True), "no vision encoder")


# ---- 7. devices mode ------------------------------------------------------------------------------------------------------------

def test_devices_mode_equals_one_gpu(prod, monkeypatch):
    if prod.lib.clip_b200_cuda_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    imgs = images(37, 64, 128, 77)
    path = model_file("tiny", "q4_0", prod)
    with Ctx(prod, path) as ctx:
        one_e = prod.image_batch_encode_hw(ctx, imgs)
        one_t = prod.image_tokens_hw(ctx, imgs, -2, bd.TOKENS_NO_CLS, bd.OUT_F16)
    monkeypatch.setenv("CLIP_B200_DEVICES", "all")
    with Ctx(prod, path) as ctx:
        assert prod.lib.clip_b200_device_count(ctx) >= 2
        assert np.array_equal(bits(prod.image_batch_encode_hw(ctx, imgs)), bits(one_e))
        assert np.array_equal(bits(prod.image_tokens_hw(ctx, imgs, -2, bd.TOKENS_NO_CLS, bd.OUT_F16)), bits(one_t))
