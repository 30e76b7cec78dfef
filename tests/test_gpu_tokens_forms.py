"""The ten per-token forms (clip_b200_image_tokens[_device], _hw, _device_hw, _layers, _layers_device and the four text forms) run
through one table, so that they check their arguments alike and compute alike.

  * Every bad request (layer, unknown flag, out_type, NO_CLS on text, ATTENTION misuse) and every null pointer is refused by every
    form it applies to, with the same message; the *_layers forms name the entry, the single-layer forms do not.
  * A call with two faults reports the one the documented order (include/clip_b200.h) puts first, on every form.
  * n == 0: a bad request is still refused, a good one returns true.
  * One (layer, flags) returns the same bytes through every form that can run it: native, *_hw at image_size, a one-entry *_layers
    list, host and device."""
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
NO_CLS, ATTN, POST_LN = bd.TOKENS_NO_CLS, bd.TOKENS_ATTENTION, bd.TOKENS_POST_LN
OUT_BYTES = 1 << 20      # every output below fits


class Form:
    def __init__(self, name, vision, host, hw=False, list_=False):
        self.name, self.vision, self.host, self.hw, self.list = name, vision, host, hw, list_

    def __repr__(self):
        return self.name


FORMS = [
    Form("clip_b200_image_tokens", True, True),
    Form("clip_b200_image_tokens_device", True, False),
    Form("clip_b200_image_tokens_hw", True, True, hw=True),
    Form("clip_b200_image_tokens_device_hw", True, False, hw=True),
    Form("clip_b200_image_tokens_layers", True, True, hw=True, list_=True),
    Form("clip_b200_image_tokens_layers_device", True, False, hw=True, list_=True),
    Form("clip_b200_text_tokens", False, True),
    Form("clip_b200_text_tokens_device", False, False),
    Form("clip_b200_text_tokens_layers", False, True, list_=True),
    Form("clip_b200_text_tokens_layers_device", False, False, list_=True),
]
IDS = [f.name for f in FORMS]


def ci(vals):
    return (C.c_int * max(len(vals), 1))(*vals)


def image_batch(arrays):
    """a clip_image_f32_batch of images of any sizes; (batch, keep-alive)"""
    arr = (bd.clip_image_f32 * len(arrays))()
    for i, x in enumerate(arrays):
        arr[i].ny, arr[i].nx, arr[i].size = x.shape[0], x.shape[1], x.size
        arr[i].data = x.ctypes.data_as(C.POINTER(C.c_float))
    return bd.clip_image_f32_batch(arr, len(arrays)), (arr, arrays)


class Env:
    """a model (the tiny f16 one by default) with two images and two sequences on the host and on the device, and output buffers on
    both"""

    def __init__(self, prod, path=None):
        self.prod, self.L = prod, prod.lib
        self.ctx = prod.load(path or model_file("tiny", "f16", prod), 0)
        self.imgs = sg.synth_images(2, S, 5)
        self.ids = padded(token_seqs(2))
        self.batch, self.keep = prod.make_image_batch(self.imgs)
        self.out = np.zeros(OUT_BYTES, np.uint8)
        self.dev = [self.L.clip_b200_device_malloc(self.ctx, n) for n in (self.imgs.nbytes, self.ids.nbytes, OUT_BYTES)]
        assert all(self.dev)
        self.d_pix, self.d_ids, self.d_out = self.dev
        assert self.L.clip_b200_memcpy_h2d(self.ctx, self.d_pix, self.imgs.ctypes.data, self.imgs.nbytes)
        assert self.L.clip_b200_memcpy_h2d(self.ctx, self.d_ids, self.ids.ctypes.data, self.ids.nbytes)

    def close(self):
        for p in self.dev:
            self.L.clip_b200_device_free(self.ctx, p)
        self.prod.free(self.ctx)

    def call(self, f, layer=-1, flags=0, ot=bd.OUT_F32, n=None, hw=(S, S), seq_len=77, null_in=False, null_out=False, batch=None,
             layers=True, n_layers=1, ctx=True):
        """one call of form f with a single (layer, flags) (a one-entry list for the *_layers forms); n=None: every item"""
        L, c = self.L, (self.ctx if ctx else None)
        entries, fl, k = (ci([layer]) if layers else None), ci([flags]), n_layers
        if f.vision and f.host:
            b = self.batch if batch is None else batch
            if n is not None:
                b = bd.clip_image_f32_batch(b.data if n else None, n)
            o = None if null_out else self.out.ctypes.data
            if f.list:
                return L.clip_b200_image_tokens_layers(c, C.byref(b), entries, fl, k, ot, o)
            return (L.clip_b200_image_tokens_hw if f.hw else L.clip_b200_image_tokens)(c, C.byref(b), layer, flags, ot, o)
        o = None if null_out else (self.d_out if not f.host else self.out.ctypes.data)
        if f.vision:
            nn, d = (len(self.imgs) if n is None else n), (None if null_in else self.d_pix)
            if f.list:
                return L.clip_b200_image_tokens_layers_device(c, d, nn, hw[0], hw[1], entries, fl, k, ot, o)
            if f.hw:
                return L.clip_b200_image_tokens_device_hw(c, d, nn, hw[0], hw[1], layer, flags, ot, o)
            return L.clip_b200_image_tokens_device(c, d, nn, layer, flags, ot, o)
        nn = len(self.ids) if n is None else n
        if f.host:
            d = None if null_in else self.ids.ctypes.data_as(C.POINTER(C.c_int32))
            if f.list:
                return L.clip_b200_text_tokens_layers(c, d, nn, seq_len, entries, fl, k, ot, o)
            return L.clip_b200_text_tokens(c, d, nn, seq_len, layer, flags, ot, o)
        d = None if null_in else self.d_ids
        if f.list:
            return L.clip_b200_text_tokens_layers_device(c, d, nn, seq_len, entries, fl, k, ot, o)
        return L.clip_b200_text_tokens_device(c, d, nn, seq_len, layer, flags, ot, o)

    def refused(self, f, msg, entry=False, **kw):
        """the call is refused with a message that starts with the form's name, contains msg, and names entry 0 only when the
        fault is in a request of a *_layers form"""
        assert not self.call(f, **kw), (f, msg, kw)
        err = self.prod.last_error()
        assert err.startswith(f.name + ": ") and msg in err, (f, msg, err)
        assert (": entry 0" in err) == (entry and f.list), (f, err)

    def result(self, f, layer, flags, ot):
        """the call's output bytes (device forms: downloaded)"""
        rows = (S // P) ** 2 + 1 if f.vision else self.ids.shape[1]
        nbytes = int(np.prod(self.prod.token_shape(self.ctx, f.vision, 2, rows, flags))) * np.dtype(bd.OUT_DTYPES[ot]).itemsize
        self.out[:] = 0xA5
        assert self.call(f, layer, flags, ot), (f, self.prod.last_error())
        if not f.host:
            assert self.L.clip_b200_memcpy_d2h(self.ctx, self.out.ctypes.data, self.d_out, nbytes)
        return self.out[:nbytes].copy()


@pytest.fixture(scope="module")
def env(prod):
    e = Env(prod)
    yield e
    e.close()


# ---- 1. one refusal per fault, alike on every form ------------------------------------------------------------------------------

def null_message(f):
    return "null device pointer" if not f.host else "null output" if f.vision else "null pointer"


@pytest.mark.parametrize("f", FORMS, ids=IDS)
def test_refusals(env, f):
    env.refused(f, "layer 13 is outside", entry=True, layer=13)
    env.refused(f, "layer -14 is outside", entry=True, layer=-14)
    env.refused(f, "unknown flag bits", entry=True, flags=16)
    env.refused(f, "unknown out_type 3", entry=True, ot=3)
    env.refused(f, "NORMALIZE needs CLIP_B200_TOKENS_PROJECT", entry=True, flags=bd.TOKENS_NORMALIZE)
    env.refused(f, "cannot be combined", entry=True, flags=ATTN | POST_LN)
    env.refused(f, "before the first block", entry=True, layer=0, flags=ATTN)
    env.refused(f, "ATTENTION_CLS needs", entry=True, flags=bd.TOKENS_ATTENTION_CLS)
    if not f.vision:
        env.refused(f, "NO_CLS is for the vision tower only", entry=True, flags=NO_CLS)
        env.refused(f, "ATTENTION_CLS is for the vision tower only", entry=True, flags=ATTN | bd.TOKENS_ATTENTION_CLS)
    env.refused(f, null_message(f), null_out=True)
    if not (f.vision and f.host):
        env.refused(f, null_message(f), null_in=True)
    if f.list:
        env.refused(f, "n_layers must be in [1, 4096], not 0", n_layers=0)
        env.refused(f, "null layers", layers=False)


# ---- 2. two faults: the first in the documented order wins ----------------------------------------------------------------------

@pytest.mark.parametrize("f", FORMS, ids=IDS)
def test_two_faults_report_the_first(env, f):
    assert not env.call(f, ctx=False, layer=13, null_out=True)
    assert env.prod.last_error() == f.name + ": null context"
    if f.vision and not f.host and f.hw:                      # the size argument comes before the request
        env.refused(f, "multiples of patch_size", hw=(S + 1, S), layer=13)
        env.refused(f, "multiples of patch_size", hw=(S + 1, S), n=0)
    if f.list:                                                # the list before its entries
        env.refused(f, "n_layers", n_layers=0, layer=13)
        env.refused(f, "null layers", layers=False, flags=16)
    env.refused(f, "layer 13", entry=True, layer=13, null_out=True)   # the request before the pointers (and the images below)
    if not f.vision:
        env.refused(f, "layer 13", entry=True, layer=13, seq_len=78)
        env.refused(f, "seq_len must be in [1, context_length]", seq_len=78, null_out=True)
        env.refused(f, "seq_len must be in [1, context_length]", seq_len=0, null_in=True)
    if f.vision and f.host:
        other = sg.synth_images(2, S + P, 6)
        if f.hw:
            bad, keep = image_batch([other[0], sg.synth_images(1, S, 7)[0]])
            msg = "every image of one call must have the same size"
        else:
            bad, keep = image_batch(list(other))
            msg = "every image must be image_size x image_size"
        env.refused(f, msg, batch=bad)
        env.refused(f, "layer 13", entry=True, layer=13, batch=bad)
        env.refused(f, "cannot be combined", entry=True, flags=ATTN | NO_CLS, batch=bad, null_out=True)
        env.refused(f, "null output", batch=bad, null_out=True)


def test_a_missing_tower_comes_first(prod, tmp_path):
    geom = sg.Geometry("text-only", image_size=64, patch_size=16, v_hidden=128, v_ff=256, v_heads=2, v_layers=1, t_hidden=128,
                       t_ff=256, t_heads=2, t_layers=2, proj_dim=128, has_vision=False)
    path = str(tmp_path / "text-only.gguf")
    sg.write_model(path, geom, 1, 1)
    e = Env(prod, path)
    try:
        for f in FORMS:
            if f.vision:
                e.refused(f, "this model has no vision encoder", layer=13, null_in=True, null_out=True, hw=(S + 1, S))
                e.refused(f, "this model has no vision encoder", n=0)
            else:
                e.refused(f, "layer 3 is outside", entry=True, layer=3, null_in=True, null_out=True)
    finally:
        e.close()


# ---- 3. n == 0 ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("f", FORMS, ids=IDS)
def test_n0_checks_the_request_only(env, f):
    env.refused(f, "layer 13", entry=True, layer=13, n=0, null_in=True, null_out=True)
    env.refused(f, "unknown out_type", entry=True, ot=5, n=0, null_in=True, null_out=True)
    env.refused(f, "cannot be combined", entry=True, flags=ATTN | POST_LN, n=0, null_in=True, null_out=True)
    if not f.vision:
        env.refused(f, "vision tower only", entry=True, flags=NO_CLS, n=0, null_in=True, null_out=True)
    assert env.call(f, layer=-1, n=0, null_in=True, null_out=True), env.prod.last_error()
    assert env.call(f, layer=1, flags=ATTN, n=0, null_in=True, null_out=True), env.prod.last_error()
    if not f.vision:
        assert env.call(f, layer=-1, n=0, seq_len=78, null_in=True, null_out=True), env.prod.last_error()


# ---- 4. the same bytes through every form ---------------------------------------------------------------------------------------

CASES = {
    True: [(-1, 0, bd.OUT_F32), (-2, NO_CLS, bd.OUT_F16), (1, ATTN, bd.OUT_BF16)],
    False: [(-1, 0, bd.OUT_F32), (-2, POST_LN, bd.OUT_F16), (1, ATTN, bd.OUT_BF16)],
}


@pytest.mark.parametrize("vision", [True, False], ids=["image", "text"])
def test_every_form_returns_the_same_bytes(env, vision):
    forms = [f for f in FORMS if f.vision == vision]
    for layer, flags, ot in CASES[vision]:
        want = env.result(forms[0], layer, flags, ot)
        assert not np.all(want == 0xA5)
        for f in forms[1:]:
            got = env.result(f, layer, flags, ot)
            assert np.array_equal(got, want), (f, layer, flags, ot)
