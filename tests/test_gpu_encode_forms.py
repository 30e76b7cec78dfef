"""The pooled-embedding forms (clip_image_batch_encode, clip_text_batch_encode, the *_device, *_hw, *_all and u8 forms and
clip_b200_image_batch_preprocess_device) run through one table, so that they check their arguments alike and compute alike.

  * Every fault is refused by every form it applies to, with a message that starts with the form's name.
  * A call with two faults reports the one the documented order (include/clip_b200.h) puts first, on every form.
  * A model without the tower is refused first; the reference's forms print the reference's line instead and leave
    clip_b200_last_error as it was.
  * n == 0 returns true (outside ranks mode, where the *_all forms refuse it).
  * Every form that can run the same pass returns the same embedding bytes with the same number of kernel launches: native, *_hw
    at image_size, host, device and *_all outside ranks mode; the u8 form against clip_image_batch_preprocess + the f32 form."""
import ctypes as C

import numpy as np
import pytest

import binding as bd
import synth_gguf as sg
from _util import model_file, token_seqs
from test_gpu_tokens import padded

pytestmark = pytest.mark.gpu

G = sg.GEOMETRIES["tiny"]
S, P = G.image_size, G.patch_size
FP = C.POINTER(C.c_float)
NO_VISION = "This gguf file seems to have no vision encoder\n"
NO_TEXT = "This GGUF file seems to have no text encoder\n"


class Form:
    def __init__(self, name, vision, kind, hw=False, all_=False, ref=False):
        self.name, self.vision, self.kind, self.hw, self.all, self.ref = name, vision, kind, hw, all_, ref
        self.device = kind == "device"

    def __repr__(self):
        return self.name


FORMS = [
    Form("clip_image_batch_encode", True, "f32", ref=True),
    Form("clip_b200_image_batch_encode_hw", True, "f32", hw=True),
    Form("clip_b200_image_batch_encode_all", True, "f32", all_=True),
    Form("clip_b200_image_encode_device", True, "device"),
    Form("clip_b200_image_encode_device_hw", True, "device", hw=True),
    Form("clip_b200_image_encode_device_all", True, "device", all_=True),
    Form("clip_b200_image_batch_encode_u8", True, "u8"),
    Form("clip_b200_image_batch_preprocess_device", True, "u8"),
    Form("clip_text_batch_encode", False, "tokens", ref=True),
    Form("clip_b200_text_batch_encode_all", False, "tokens", all_=True),
    Form("clip_b200_text_encode_device", False, "device"),
    Form("clip_b200_text_encode_device_all", False, "device", all_=True),
]
IDS = [f.name for f in FORMS]


def f32_batch(arrays):
    """a clip_image_f32_batch of images of any sizes (None: an image without pixels); (batch, keep-alive)"""
    arr = (bd.clip_image_f32 * len(arrays))()
    for i, x in enumerate(arrays):
        if x is None:
            arr[i].ny = arr[i].nx = S
            continue
        arr[i].ny, arr[i].nx, arr[i].size = x.shape[0], x.shape[1], x.size
        arr[i].data = x.ctypes.data_as(FP)
    return bd.clip_image_f32_batch(arr, len(arrays)), (arr, arrays)


def tokens_array(seqs):
    arr = (bd.clip_tokens * len(seqs))()
    for i, s in enumerate(seqs):
        arr[i].data, arr[i].size = (s.ctypes.data_as(C.POINTER(C.c_int32)), s.size) if s is not None else (None, 0)
    return arr


def flush_stdout():
    C.CDLL(None).fflush(None)


class Env:
    """a model (the tiny f16 one by default) with two images (f32 and u8) and two sequences on the host and on the device, and
    output buffers on both"""

    def __init__(self, prod, path=None):
        self.prod, self.L = prod, prod.lib
        self.ctx = prod.load(path or model_file("tiny", "f16", prod), 0)
        self.imgs = sg.synth_images(2, S, 5)
        self.batch, self.keep = prod.make_image_batch(self.imgs)
        rng = np.random.default_rng(7)
        self.u8 = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in ((100, 150), (S, S))]
        self.u8_batch, self.u8_keep = prod._u8_batch(self.u8)
        self.seqs = token_seqs(2)                                   # 77 and 5 tokens: the host form pads to 77 as well
        self.ids = padded(self.seqs)
        self.lens = np.array([len(s) for s in self.seqs], np.int32)
        self.tokens = tokens_array(self.seqs)
        self.out = np.zeros(1 << 16, np.float32)
        self.dev = [self.L.clip_b200_device_malloc(self.ctx, a.nbytes) for a in (self.imgs, self.ids, self.lens, self.out)]
        assert all(self.dev)
        self.d_pix, self.d_ids, self.d_lens, self.d_out = self.dev
        for d, a in zip(self.dev[:3], (self.imgs, self.ids, self.lens)):
            assert self.L.clip_b200_memcpy_h2d(self.ctx, d, a.ctypes.data, a.nbytes)
        self.pixels = (bd.clip_image_f32 * 8)()
        self.pixels_batch = bd.clip_image_f32_batch(self.pixels, 8)

    def close(self):
        for p in self.dev:
            self.L.clip_b200_device_free(self.ctx, p)
        self.prod.free(self.ctx)

    def call(self, f, n=None, null_in=False, null_out=False, ctx=True, batch=None, hw=(S, S), seq_len=77, seqs=None):
        """one call of form f on every item (n=None), the first n items, or the given host batch / sequences"""
        L, c = self.L, (self.ctx if ctx else None)
        if f.kind == "device":
            nn = 2 if n is None else n
            o = None if null_out else self.d_out
            if f.vision:
                d = None if null_in else self.d_pix
                if f.hw:
                    return L.clip_b200_image_encode_device_hw(c, d, nn, hw[0], hw[1], o, True)
                return (L.clip_b200_image_encode_device_all if f.all else L.clip_b200_image_encode_device)(c, d, nn, o, True)
            d = None if null_in else self.d_ids
            return (L.clip_b200_text_encode_device_all if f.all else L.clip_b200_text_encode_device)(c, d, self.d_lens, nn, seq_len, o, True)
        if f.kind == "tokens":
            arr = self.tokens if seqs is None else tokens_array(seqs)
            nn = len(arr) if n is None else n
            o = None if null_out else self.out.ctypes.data_as(FP)
            return (L.clip_b200_text_batch_encode_all if f.all else L.clip_text_batch_encode)(c, 4, None if null_in else arr, nn, o, True)
        if f.kind == "u8":
            b = self.u8_batch if batch is None else batch
        else:
            b = self.batch if batch is None else batch
        b = type(b)(None if null_in or n == 0 else b.data, b.size if n is None else n)
        if f.name == "clip_b200_image_batch_preprocess_device":
            return L.clip_b200_image_batch_preprocess_device(c, C.byref(b), None if null_out else C.byref(self.pixels_batch))
        o = None if null_out else self.out.ctypes.data_as(FP)
        if f.kind == "u8":
            return L.clip_b200_image_batch_encode_u8(c, C.byref(b), o, True)
        if f.hw:
            return L.clip_b200_image_batch_encode_hw(c, C.byref(b), o, True)
        return (L.clip_b200_image_batch_encode_all if f.all else L.clip_image_batch_encode)(c, 4, C.byref(b), o, True)

    def refused(self, f, msg, **kw):
        """the call is refused with a message that starts with the form's name and contains msg"""
        assert not self.call(f, **kw), (f, msg, kw)
        err = self.prod.last_error()
        assert err.startswith(f.name + ": ") and msg in err, (f, msg, err)

    def result(self, f):
        """the embeddings of both items (device forms: downloaded) and the kernel launches of the call"""
        d = (self.prod.vision_hparams if f.vision else self.prod.text_hparams)(self.ctx).projection_dim
        self.out[:] = np.nan
        l0 = self.L.clip_b200_kernel_launches(self.ctx)
        assert self.call(f), (f, self.prod.last_error())
        launches = self.L.clip_b200_kernel_launches(self.ctx) - l0
        if f.device:
            assert self.L.clip_b200_memcpy_d2h(self.ctx, self.out.ctypes.data, self.d_out, 2 * d * 4)
        return self.out[:2 * d].reshape(2, d).copy(), launches


@pytest.fixture(scope="module")
def env(prod):
    e = Env(prod)
    yield e
    e.close()


def null_message(f, out):
    return "null device pointer" if f.device else "null output" if out else "null input"


# ---- 1. one refusal per fault, alike on every form ------------------------------------------------------------------------------

@pytest.mark.parametrize("f", FORMS, ids=IDS)
def test_refusals(env, f):
    env.refused(f, null_message(f, True), null_out=True)
    env.refused(f, null_message(f, False), null_in=True)
    if f.kind == "f32":
        big = sg.synth_images(2, S + P, 6)
        if f.hw:
            env.refused(f, "every image of one call must have the same size", batch=f32_batch([big[0], env.imgs[0]])[0])
            env.refused(f, "positive multiples of patch_size", batch=f32_batch([np.zeros((S + 1, S, 3), np.float32)])[0])
            env.refused(f, "image 1 has no pixels", batch=f32_batch([env.imgs[0], None])[0])
        else:
            env.refused(f, "every image must be image_size x image_size", batch=f32_batch(list(big))[0])
            env.refused(f, "every image must be image_size x image_size", batch=f32_batch([env.imgs[0], None])[0])
    if f.device and f.hw:
        env.refused(f, "positive multiples of patch_size", hw=(S + 1, S))
    if f.device and not f.vision:
        env.refused(f, "seq_len must be in [1, context_length]", seq_len=0)
        env.refused(f, "seq_len must be in [1, context_length]", seq_len=78)
    if f.kind == "tokens":
        env.refused(f, "empty token sequence", seqs=[env.seqs[0], None])
        env.refused(f, "token sequence longer than context_length (77)", seqs=[env.seqs[0], np.ones(78, np.int32)])
    if f.kind == "u8":
        empty = np.zeros((0, 5, 3), np.uint8)
        env.refused(f, "bad image", batch=env.prod._u8_batch([empty])[0])


# ---- 2. two faults: the first in the documented order wins ----------------------------------------------------------------------

@pytest.mark.parametrize("f", FORMS, ids=IDS)
def test_two_faults_report_the_first(env, f, capfd):
    if f.ref:                                                 # the reference's line, no message of our own
        env.refused(f, null_message(f, True), null_out=True)
        before = env.prod.last_error()
        capfd.readouterr()
        assert not env.call(f, ctx=False, null_out=True)
        flush_stdout()
        assert capfd.readouterr().out == (NO_VISION if f.vision else NO_TEXT)
        assert env.prod.last_error() == before
    else:
        assert not env.call(f, ctx=False, null_in=True, null_out=True)
        assert env.prod.last_error() == f.name + ": null context"
    if f.device and f.hw:                                     # the size argument before n == 0 and the pointers
        env.refused(f, "multiples of patch_size", hw=(S + 1, S), n=0)
        env.refused(f, "multiples of patch_size", hw=(S + 1, S), null_in=True, null_out=True)
    if f.device and not f.vision:                             # n == 0 before seq_len, seq_len before the pointers
        assert env.call(f, n=0, seq_len=78, null_in=True, null_out=True), env.prod.last_error()
        env.refused(f, "seq_len must be in [1, context_length]", seq_len=78, null_in=True, null_out=True)
    if f.kind == "f32":                                       # the pointers before the images
        bad = f32_batch(list(sg.synth_images(2, S + P, 6)) if not f.hw else [env.imgs[0], sg.synth_images(1, S + P, 6)[0]])[0]
        env.refused(f, "null output", batch=bad, null_out=True)
    if f.kind == "u8":
        env.refused(f, "null output", batch=env.prod._u8_batch([np.zeros((0, 5, 3), np.uint8)])[0], null_out=True)
    if f.kind == "tokens":
        env.refused(f, "null output", seqs=[env.seqs[0], None], null_out=True)
        env.refused(f, "empty token sequence", seqs=[None, np.ones(78, np.int32)])      # empty before too long, as in one pass


def missing_tower_model(tmp_path, vision):
    name = "text-only" if vision else "vision-only"
    geom = sg.Geometry(name, image_size=64, patch_size=16, v_hidden=128, v_ff=256, v_heads=2, v_layers=1, t_hidden=128, t_ff=256,
                       t_heads=2, t_layers=2, proj_dim=128, has_vision=not vision, has_text=vision)
    path = str(tmp_path / (name + ".gguf"))
    sg.write_model(path, geom, 1, 1)
    return path


@pytest.mark.parametrize("vision", [True, False], ids=["image", "text"])
def test_a_missing_tower_comes_first(prod, tmp_path, capfd, vision):
    e = Env(prod, missing_tower_model(tmp_path, vision))
    line = NO_VISION if vision else NO_TEXT
    try:
        forms = [f for f in FORMS if f.vision == vision]
        for f in sorted(forms, key=lambda f: f.ref):          # the reference's forms last, after a message of our own
            if not f.ref:
                msg = "this model has no %s encoder" % ("vision" if vision else "text")
                e.refused(f, msg, null_in=True, null_out=True, hw=(S + 1, S), seq_len=78)
                e.refused(f, msg, n=0)
                continue
            before = prod.last_error()
            capfd.readouterr()
            assert not e.call(f, null_in=True, null_out=True)
            flush_stdout()
            assert capfd.readouterr().out == line
            assert prod.last_error() == before
        # the single-item reference forms delegate to the batch forms
        if vision:
            img = bd.clip_image_f32(S, S, e.imgs[0].ctypes.data_as(FP), e.imgs[0].size)
            assert not prod.lib.clip_image_encode(e.ctx, 4, C.byref(img), e.out.ctypes.data_as(FP), True)
        else:
            tk = bd.clip_tokens(e.seqs[0].ctypes.data_as(C.POINTER(C.c_int32)), e.seqs[0].size)
            assert not prod.lib.clip_text_encode(e.ctx, 4, C.byref(tk), e.out.ctypes.data_as(FP), True)
        flush_stdout()
        assert capfd.readouterr().out == line
    finally:
        e.close()


# ---- 3. n == 0 ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("f", FORMS, ids=IDS)
def test_n0_returns_true(env, f):
    assert env.call(f, n=0, null_in=True, null_out=True), env.prod.last_error()
    if f.kind in ("f32", "u8"):                               # a NULL batch is an empty one
        L, o = env.L, env.out.ctypes.data_as(FP)
        calls = {"clip_image_batch_encode": lambda: L.clip_image_batch_encode(env.ctx, 4, None, o, True),
                 "clip_b200_image_batch_encode_hw": lambda: L.clip_b200_image_batch_encode_hw(env.ctx, None, o, True),
                 "clip_b200_image_batch_encode_all": lambda: L.clip_b200_image_batch_encode_all(env.ctx, 4, None, o, True),
                 "clip_b200_image_batch_encode_u8": lambda: L.clip_b200_image_batch_encode_u8(env.ctx, None, o, True),
                 "clip_b200_image_batch_preprocess_device":
                     lambda: L.clip_b200_image_batch_preprocess_device(env.ctx, None, C.byref(env.pixels_batch))}
        assert calls[f.name](), env.prod.last_error()
    if f.name == "clip_b200_image_batch_preprocess_device":   # the output batch reports its size, as the host preprocess does
        env.pixels_batch.size = 8
        assert env.call(f, n=0)
        assert env.pixels_batch.size == 0


# ---- 4. the same bytes and launches through every form --------------------------------------------------------------------------

@pytest.mark.parametrize("vision", [True, False], ids=["image", "text"])
def test_every_form_returns_the_same_bytes(env, vision):
    forms = [f for f in FORMS if f.vision == vision and f.kind != "u8"]
    want, launches = env.result(forms[0])
    assert np.isfinite(want).all() and launches > 0
    for f in forms[1:]:
        got, n = env.result(f)
        assert got.tobytes() == want.tobytes(), f
        assert n == launches, (f, n, launches)
    d = want.shape[1]
    for i in range(2):                                        # the single-item reference form
        one = np.zeros(d, np.float32)
        if vision:
            img = bd.clip_image_f32(S, S, env.imgs[i].ctypes.data_as(FP), env.imgs[i].size)
            assert env.L.clip_image_encode(env.ctx, 4, C.byref(img), one.ctypes.data_as(FP), True)
        else:
            tk = bd.clip_tokens(env.seqs[i].ctypes.data_as(C.POINTER(C.c_int32)), env.seqs[i].size)
            assert env.L.clip_text_encode(env.ctx, 4, C.byref(tk), one.ctypes.data_as(FP), True)
        if vision or i == 0:                                  # alone, the 5-token sequence pads to 8 tokens instead of 77
            assert one.tobytes() == want[i].tobytes(), i


def test_u8_equals_host_preprocess_then_f32(env):
    host_px = env.prod.batch_preprocess(env.ctx, env.u8)
    u8, pre = (next(f for f in FORMS if f.name == name) for name in ("clip_b200_image_batch_encode_u8", "clip_b200_image_batch_preprocess_device"))
    fused, n_u8 = env.result(u8)
    batch, keep = env.prod.make_image_batch(np.ascontiguousarray(host_px))
    env.batch, saved = batch, env.batch
    try:
        ref, n_f32 = env.result(FORMS[0])
    finally:
        env.batch = saved
    assert fused.tobytes() == ref.tobytes()
    assert n_u8 == n_f32, (n_u8, n_f32)
    # the preprocess-only form returns the same pixels
    assert env.call(pre), env.prod.last_error()
    assert env.pixels_batch.size == 2
    for i in range(2):
        px = env.pixels[i]
        got = np.ctypeslib.as_array(px.data, shape=(px.ny, px.nx, 3)).copy()
        env.L.clip_image_f32_clean(C.byref(px))
        assert got.tobytes() == host_px[i].tobytes(), i
