"""Several layers from one forward pass (clip_b200_image_tokens_layers / clip_b200_text_tokens_layers and their device forms).

  * Slab j of a multi-layer call equals the single-layer call with (layers[j], flags[j], out_type) bit for bit, for both towers, every
    out type, layer lists that are complete, sparse, unsorted with duplicates, mixed in flags or one entry long, at the native size
    and at two other image sizes (against the *_hw calls).
  * Several passes (a small micro_batch, a ragged last pass) equal one call per item; host = device; a pinned `out` = a pageable one.
  * The blocks run once, up to the deepest entry: the launch count is that of the deepest single call plus the other entries' tails.
  * Bad arguments are refused with a message that names the bad entry; devices mode equals one GPU."""
import ctypes as C

import numpy as np
import pytest

import binding as bd
import synth_gguf as sg
from _util import model_file, token_seqs
from test_gpu_tokens import Ctx, bits, on_device, padded

pytestmark = pytest.mark.gpu

PROJ_N = bd.TOKENS_PROJECT | bd.TOKENS_NORMALIZE
NO_CLS = bd.TOKENS_NO_CLS
OUT_TYPES = (bd.OUT_F32, bd.OUT_F16, bd.OUT_BF16)
MAX_LAYERS = 4096      # CLIP_B200_TOKENS_MAX_LAYERS (include/clip_b200.h)


def layer_lists(n, vision):
    """(name, layers, flags) of a tower of n blocks; flags None = NULL.  NO_CLS only where the tower is the vision one."""
    nc = NO_CLS if vision else 0
    llava = [l for l in (-2, -5, -8, -11) if l >= -(n + 1)]
    return [
        ("all", list(range(n + 1)), None),
        ("llava", llava, [nc] * len(llava)),
        ("sdxl", [-2, -1], [0, bd.TOKENS_PROJECT]),
        ("unsorted", [5, -1, 0, 5, 2, -1], [0, bd.TOKENS_POST_LN, 0, 0, bd.TOKENS_POST_LN, 0]),
        ("layer0", [0], None),
        ("mixed", [-1, 3, -2, 1, 3], [nc | bd.TOKENS_POST_LN, PROJ_N, bd.TOKENS_POST_LN, bd.TOKENS_PROJECT, nc]),
        ("one", [-2], [bd.TOKENS_POST_LN]),
    ]


def images(n, H, W, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    return rng.random(size=(n, H, W, 3), dtype=np.float32) * np.float32(4.0) - np.float32(2.0)


def check_slabs(got, want, what):
    assert len(got) == len(want), what
    for j, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape and a.dtype == b.dtype, (what, j, a.shape, b.shape)
        assert np.array_equal(bits(a), bits(b)), (what, j)


# ---- 1. slabs equal single calls ------------------------------------------------------------------------------------------------

GEOMS = [("tiny", "f16"), ("tiny", "q4_0"), ("tiny-gelu", "f16"), ("small-p14-336", "f16"), ("huge-w640", "f16")]


@pytest.mark.parametrize("geom,ft", GEOMS)
def test_slabs_equal_single_calls(prod, geom, ft):
    g = sg.GEOMETRIES[geom]
    imgs = sg.synth_images(2, g.image_size, 91)
    ids = padded(token_seqs(3))
    with Ctx(prod, model_file(geom, ft, prod)) as ctx:
        memo = {}

        def single(vision, layer, flags, ot):
            key = (vision, layer, flags, ot)
            if key not in memo:
                memo[key] = prod.image_tokens(ctx, imgs, layer, flags, ot) if vision else prod.text_tokens(ctx, ids, layer, flags, ot)
            return memo[key]

        for vision, n in ((True, g.v_layers), (False, g.t_layers)):
            for li, (name, layers, flags) in enumerate(layer_lists(n, vision)):
                ot = OUT_TYPES[li % 3]
                fl = flags or [0] * len(layers)
                want = [single(vision, l, f, ot) for l, f in zip(layers, fl)]
                if vision:
                    host = prod.image_tokens_layers(ctx, imgs, layers, flags, ot)
                    dev = prod.image_tokens_layers_device(ctx, imgs, layers, flags, ot)
                else:
                    host = prod.text_tokens_layers(ctx, ids, layers, flags, ot)
                    dev = prod.text_tokens_layers_device(ctx, ids, layers, flags, ot)
                check_slabs(host, want, (geom, ft, vision, name, ot, "host"))
                check_slabs(dev, want, (geom, ft, vision, name, ot, "device"))


def tokens_device_hw(prod, ctx, imgs, layer, flags, ot, shape):
    n, H, W = imgs.shape[:3]
    return on_device(prod, ctx, lambda di, do: prod.lib.clip_b200_image_tokens_device_hw(ctx, di, n, H, W, layer, flags, ot, do),
                     imgs, shape, bd.OUT_DTYPES[ot])


@pytest.mark.parametrize("geom", ["tiny", "huge-w640"])
def test_image_sizes_equal_hw_calls(prod, geom):
    """the native size, a larger square and a rectangle; host and device forms against clip_b200_image_tokens_hw / _device_hw"""
    g = sg.GEOMETRIES[geom]
    S, P = g.image_size, g.patch_size
    layers, flags = [-2, 0, 3, -1, 3], [NO_CLS, 0, bd.TOKENS_POST_LN, PROJ_N, bd.TOKENS_PROJECT]
    with Ctx(prod, model_file(geom, "f16", prod)) as ctx:
        for (H, W), ot, seed in (((S, S), bd.OUT_F32, 1), ((S + 2 * P, S + 2 * P), bd.OUT_F16, 2), ((S - 2 * P, S + 4 * P), bd.OUT_BF16, 3)):
            imgs = images(3, H, W, seed)
            want = [prod.image_tokens_hw(ctx, imgs, l, f, ot) for l, f in zip(layers, flags)]
            want_dev = [tokens_device_hw(prod, ctx, imgs, l, f, ot, w.shape) for l, f, w in zip(layers, flags, want)]
            check_slabs(want_dev, want, (geom, H, W, "device_hw = hw"))
            check_slabs(prod.image_tokens_layers(ctx, imgs, layers, flags, ot), want, (geom, H, W, "host"))
            check_slabs(prod.image_tokens_layers_device(ctx, imgs, layers, flags, ot), want, (geom, H, W, "device"))
            if (H, W) == (S, S):
                check_slabs([prod.image_tokens(ctx, imgs, l, f, ot) for l, f in zip(layers, flags)], want, (geom, "native"))


# ---- 2. several passes, host = device, pinned = pageable ------------------------------------------------------------------------

def pinned_like(prod, n_elems, dtype):
    """a pinned host buffer (clip_b200_host_malloc) seen as a numpy array; (array, pointer to free)"""
    nbytes = n_elems * np.dtype(dtype).itemsize
    p = prod.lib.clip_b200_host_malloc(nbytes)
    assert p
    return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p)).view(dtype), p


def test_several_passes_equal_one_call_per_item(prod):
    """micro batches of 4 images and 3 sequences: 11 images take passes of 4, 4, 3 and 8 sequences 3, 3, 2"""
    path = model_file("tiny", "f16", prod)
    imgs = sg.synth_images(11, 64, 17)
    ids = padded(token_seqs(8))
    layers = [-2, 0, -1, 4, -2]
    fi = [NO_CLS, bd.TOKENS_POST_LN, PROJ_N, 0, bd.TOKENS_PROJECT]
    ft = [0, bd.TOKENS_POST_LN, PROJ_N, 0, bd.TOKENS_PROJECT]
    ot = bd.OUT_F16
    with Ctx(prod, path, (4, 3)) as ctx:
        host_i = prod.image_tokens_layers(ctx, imgs, layers, fi, ot)
        host_t = prod.text_tokens_layers(ctx, ids, layers, ft, ot)
        check_slabs(prod.image_tokens_layers_device(ctx, imgs, layers, fi, ot), host_i, "image device = host")
        check_slabs(prod.text_tokens_layers_device(ctx, ids, layers, ft, ot), host_t, "text device = host")
        for name, fn, want in (("image", lambda o: prod.image_tokens_layers(ctx, imgs, layers, fi, ot, o), host_i),
                               ("text", lambda o: prod.text_tokens_layers(ctx, ids, layers, ft, ot, o), host_t)):
            buf, p = pinned_like(prod, sum(w.size for w in want), np.float16)
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


# ---- 3. the deepest layer bounds the work ---------------------------------------------------------------------------------------

EMBED_LAUNCHES = {True: 3, False: 1}      # vision: im2col, patch GEMM, class + position + pre_ln;  text: token + position embedding


def test_deepest_layer_bounds_the_work(prod):
    """launches(list) = launches(single call at the deepest entry) + the tails of the other entries, where an entry's tail is its
    single call's launches less the embedding and its 7 launches per block; {-2} alone launches as the single -2 call does"""
    g = sg.GEOMETRIES["tiny"]
    imgs = sg.synth_images(3, g.image_size, 66)
    ids = padded(token_seqs(3))
    layers = [-2, 0, 5, -1, 5, -1]
    with Ctx(prod, model_file("tiny", "q4_0", prod)) as ctx:
        n = prod.lib.clip_b200_kernel_launches

        def count(fn):
            a = n(ctx)
            fn()
            return n(ctx) - a

        for vision, nl in ((True, g.v_layers), (False, g.t_layers)):
            nc = NO_CLS if vision else 0
            flags = [nc, 0, bd.TOKENS_POST_LN, PROJ_N, bd.TOKENS_PROJECT, 0]
            if vision:
                multi = lambda: prod.image_tokens_layers(ctx, imgs, layers, flags)
                one = lambda l, f: prod.image_tokens(ctx, imgs, l, f)
                two = lambda: prod.image_tokens_layers(ctx, imgs, [-2], [nc])
            else:
                multi = lambda: prod.text_tokens_layers(ctx, ids, layers, flags)
                one = lambda l, f: prod.text_tokens(ctx, ids, l, f)
                two = lambda: prod.text_tokens_layers(ctx, ids, [-2], [nc])
            multi()                                                   # warm-up at the same size
            got = count(multi)
            singles = [count(lambda: one(l, f)) for l, f in zip(layers, flags)]
            blocks = [l if l >= 0 else nl + 1 + l for l in layers]
            deepest = int(np.argmax(blocks))
            tails = [s - EMBED_LAUNCHES[vision] - 7 * b for s, b in zip(singles, blocks)]
            assert got == singles[deepest] + sum(t for j, t in enumerate(tails) if j != deepest), (vision, got, singles)
            assert count(two) == count(lambda: one(-2, nc)), vision


# ---- 4. refusals ----------------------------------------------------------------------------------------------------------------

def test_refusals(prod, tmp_path):
    g = sg.GEOMETRIES["tiny"]
    imgs = sg.synth_images(1, g.image_size, 1)
    ids = padded(token_seqs(1))
    batch, keep = prod.make_image_batch(imgs)
    mixed_imgs = [images(1, 64, 64, 2), images(1, 32, 64, 3)]
    mixed_arr = (bd.clip_image_f32 * 2)()
    for i, x in enumerate(mixed_imgs):
        mixed_arr[i].ny, mixed_arr[i].nx, mixed_arr[i].size = x.shape[1], x.shape[2], x.size
        mixed_arr[i].data = x.ctypes.data_as(C.POINTER(C.c_float))
    mixed = bd.clip_image_f32_batch(mixed_arr, 2)
    out = np.empty(1 << 22, np.float32)
    L = prod.lib

    def ci(vals):
        return (C.c_int * max(len(vals), 1))(*vals)

    def img(layers, flags=None, ot=0, k=None, o=out, b=batch):
        return L.clip_b200_image_tokens_layers(ctx, C.byref(b), None if layers is None else ci(layers), None if flags is None else ci(flags),
                                               len(layers or []) if k is None else k, ot, None if o is None else o.ctypes.data)

    def txt(layers, flags=None, ot=0, k=None, seq_len=77):
        return L.clip_b200_text_tokens_layers(ctx, ids.ctypes.data_as(C.POINTER(C.c_int32)), 1, seq_len, ci(layers),
                                              None if flags is None else ci(flags), len(layers) if k is None else k, ot, out.ctypes.data)

    def expect(ok, *msgs):
        assert not ok, msgs
        for m in msgs:
            assert m in prod.last_error(), (m, prod.last_error())

    with Ctx(prod, model_file("tiny", "f16", prod)) as ctx:
        expect(img([-1], k=0), "n_layers")
        expect(img([-1], k=MAX_LAYERS + 1), "n_layers", str(MAX_LAYERS))
        expect(img(None, k=1), "null layers")
        expect(img([-1], o=None), "null output")
        expect(img([0, 13]), "entry 1", "layer 13")
        expect(img([0, -1, 2], [0, 0, 16]), "entry 2", "unknown flag")
        expect(img([3, 4], [bd.TOKENS_PROJECT, bd.TOKENS_NORMALIZE]), "entry 1", "needs")
        expect(img([-1], ot=3), "out_type")
        expect(img([-1], b=mixed), "same size")
        expect(txt([0, -14]), "entry 1", "outside")
        expect(txt([-1, 0], [0, NO_CLS]), "entry 1", "vision tower only")
        expect(txt([-1], ot=7), "out_type")
        expect(txt([-1], seq_len=78), "seq_len")
        expect(L.clip_b200_image_tokens_layers_device(ctx, None, 1, 65, 64, ci([-1]), None, 1, 0, None), "multiples of patch_size")
        expect(L.clip_b200_image_tokens_layers_device(ctx, None, 1, 64, 64, ci([-1]), None, 1, 0, None), "null device pointer")
        assert img([-13, 12, 0]) and txt([-13, 12])
        empty = bd.clip_image_f32_batch(None, 0)
        assert L.clip_b200_image_tokens_layers(ctx, C.byref(empty), ci([-1]), None, 1, 0, None)
        assert L.clip_b200_text_tokens_layers(ctx, None, 0, 77, ci([-1]), None, 1, 0, None)
        assert L.clip_b200_image_tokens_layers_device(ctx, None, 0, 64, 64, ci([-1]), None, 1, 0, None)
        assert L.clip_b200_text_tokens_layers_device(ctx, None, 0, 77, ci([-1]), None, 1, 0, None)
    text_only = sg.Geometry("text-only", image_size=64, patch_size=16, v_hidden=128, v_ff=256, v_heads=2, v_layers=1,
                            t_hidden=128, t_ff=256, t_heads=2, t_layers=2, proj_dim=128, has_vision=False)
    path = str(tmp_path / "text-only.gguf")
    sg.write_model(path, text_only, 1, 1)
    with Ctx(prod, path) as ctx:
        expect(img([-1]), "no vision encoder")
        expect(L.clip_b200_image_tokens_layers_device(ctx, None, 1, 64, 64, ci([-1]), None, 1, 0, None), "no vision encoder")
        assert txt([-1, 0], [bd.TOKENS_POST_LN, 0])


# ---- 5. devices mode ------------------------------------------------------------------------------------------------------------

def test_devices_mode_equals_one_gpu(prod, monkeypatch):
    if prod.lib.clip_b200_cuda_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    g = sg.GEOMETRIES["tiny"]
    imgs = sg.synth_images(37, g.image_size, 77)
    ids = padded(token_seqs(19))
    path = model_file("tiny", "q4_0", prod)
    layers = [-2, 0, -1]
    fi, ft = [NO_CLS, 0, PROJ_N], [0, bd.TOKENS_POST_LN, PROJ_N]
    with Ctx(prod, path) as ctx:
        one_i = prod.image_tokens_layers(ctx, imgs, layers, fi, bd.OUT_F16)
        one_t = prod.text_tokens_layers(ctx, ids, layers, ft, bd.OUT_BF16)
    monkeypatch.setenv("CLIP_B200_DEVICES", "all")
    with Ctx(prod, path) as ctx:
        assert prod.lib.clip_b200_device_count(ctx) >= 2
        check_slabs(prod.image_tokens_layers(ctx, imgs, layers, fi, bd.OUT_F16), one_i, "image")
        check_slabs(prod.text_tokens_layers(ctx, ids, layers, ft, bd.OUT_BF16), one_t, "text")
