"""Per-token hidden states (clip_b200_image_tokens / clip_b200_text_tokens and their device forms) and the K7 token-row kernel.

  * The pooled rows are bit-exact: with PROJECT the CLS row of each image and the EOT row of each sequence equal the embeddings of
    clip_image_batch_encode / clip_text_batch_encode, with and without NORMALIZE.
  * Every layer against the CPU oracle (tests/_oracle_tokens.py) at the project's end-to-end bars, per token; layer 0 element-wise.
  * Layout and types are exact: NO_CLS drops row 0, f16 / bf16 are the round-to-nearest-even of the f32 rows, host = device, and an
    image's rows do not depend on the batch around it.
  * The row kernel alone against an fp64 LayerNorm at every MAXV width, and bit for bit against K2 in the operand type.
  * layer = -2 runs one block fewer; bad arguments are refused with a message; devices mode equals one GPU."""
import ctypes as C

import numpy as np
import pytest

import binding as bd
import synth_gguf as sg
from _oracle_tokens import TokenOracle
from _util import TOL, ln_ref64, ln_rows, model_file, token_seqs
from test_gpu_rows import affine, ln_bound, round16, spread_error

pytestmark = pytest.mark.gpu

FP = C.POINTER(C.c_float)
U = 2.0 ** -24
PROJ_N = bd.TOKENS_PROJECT | bd.TOKENS_NORMALIZE


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.itemsize == 4 else np.uint16)


def bf16_of(f32):
    """round-to-nearest-even bf16 bit patterns of float32 values"""
    return (round16(f32, True).view(np.uint32) >> 16).astype(np.uint16)


def padded(seqs, seq_len=77, pad=0):
    ids = np.full((len(seqs), seq_len), pad, np.int32)
    for i, s in enumerate(seqs):
        ids[i, :len(s)] = s
    return ids


class Ctx:
    def __init__(self, prod, path, micro_batch=(0, 0)):
        self.prod, self.ctx = prod, prod.load(path, 0)
        if micro_batch != (0, 0):
            prod.lib.clip_b200_set_micro_batch(self.ctx, *micro_batch)

    def __enter__(self):
        return self.ctx

    def __exit__(self, *a):
        self.prod.free(self.ctx)


def on_device(prod, ctx, fn, inp, out_shape, out_dtype):
    """upload inp, call fn(d_in, d_out), download [out_shape] of out_dtype"""
    out = np.empty(out_shape, out_dtype)
    d_in = prod.lib.clip_b200_device_malloc(ctx, inp.nbytes)
    d_out = prod.lib.clip_b200_device_malloc(ctx, max(out.nbytes, 1))
    try:
        assert prod.lib.clip_b200_memcpy_h2d(ctx, d_in, inp.ctypes.data, inp.nbytes)
        assert fn(d_in, d_out), prod.last_error()
        assert prod.lib.clip_b200_memcpy_d2h(ctx, out.ctypes.data, d_out, out.nbytes)
    finally:
        prod.lib.clip_b200_device_free(ctx, d_in)
        prod.lib.clip_b200_device_free(ctx, d_out)
    return out


# ---- 1. the pooled rows, bit-exact ----------------------------------------------------------------------------------------------

POOLED = [("tiny", "f16"), ("tiny", "q4_0"), ("tiny-gelu", "f16"), ("small-p14-336", "f16"), ("huge-w640", "f16")]


@pytest.mark.parametrize("geom,ft", POOLED)
def test_pooled_rows_are_bit_exact(prod, geom, ft):
    g = sg.GEOMETRIES[geom]
    imgs = sg.synth_images(3, g.image_size, 21)
    seqs = token_seqs(5)                                    # lengths 77, 5, 2, 33, 16
    ids = padded(seqs)
    with Ctx(prod, model_file(geom, ft, prod)) as ctx:
        for normalize in (True, False):
            flags = PROJ_N if normalize else bd.TOKENS_PROJECT
            pooled_i = prod.image_batch_encode(ctx, imgs, normalize=normalize)
            rows_i = prod.image_tokens(ctx, imgs, -1, flags)
            assert rows_i.shape == (3, g.n_pos, g.proj_dim)
            assert np.array_equal(bits(rows_i[:, 0]), bits(pooled_i)), (geom, ft, normalize)
            pooled_t = prod.text_batch_encode(ctx, seqs, normalize=normalize)
            rows_t = prod.text_tokens(ctx, ids, -1, flags)
            eot = rows_t[np.arange(len(seqs)), [len(s) - 1 for s in seqs]]
            assert np.array_equal(bits(eot), bits(pooled_t)), (geom, ft, normalize)


# ---- 2. every layer against the oracle ------------------------------------------------------------------------------------------

def preln_tol(om, img):
    """Element-wise bound between two fp32 evaluations of the pre_ln output (K4 after the patch GEMM; the oracle).  Both start
    from the same fp16 patches and fp16 weights, whose products are exact in fp32.  An fp32 sum of K products in any order, with
    the tensor cores' accumulation allowed 2u per addition, is within E_y = 2 K u sum|p w| of the fp64 sum; + pos adds u |x|.  An
    input error E moves LayerNorm's x_hat_i by at most r (E_i + mean E) + |x_hat_i| r^2 mean(|x - mu| E) to first order, and the
    LayerNorm's own roundings are ln_bound's.  Each side is within that of the fp64 value; the two are within twice it."""
    S, P, h = om.image_size, om.patch, om.v_hidden
    n = S // P
    planar = img.transpose(2, 0, 1)
    pt = planar.reshape(3, n, P, n, P).transpose(1, 3, 0, 2, 4).reshape(n * n, 3 * P * P)
    pt = pt.astype(np.float16).astype(np.float64)
    w = om.t("v.patch_embd.weight").f32().reshape(h, -1).astype(np.float64)
    y = pt @ w.T
    ey = 2 * w.shape[1] * U * (np.abs(pt) @ np.abs(w).T)
    x = np.concatenate([om.f32("v.class_embd")[None].astype(np.float64), y]) + om.f32("v.position_embd.weight")
    e = np.concatenate([np.zeros((1, h)), ey]) + U * np.abs(x)
    xh, r, mean_abs = ln_ref64(x, om.v_eps)
    mu = x.mean(-1, keepdims=True)
    dxh = r * (e + e.mean(-1, keepdims=True)) + np.abs(xh) * r * r * (np.abs(x - mu) * e).mean(-1, keepdims=True)
    g, b = om.f32("v.pre_ln.weight").astype(np.float64), om.f32("v.pre_ln.bias").astype(np.float64)
    return 2 * (np.abs(g) * dxh + ln_bound(xh, r, mean_abs, g, b, h, extra_roundings=2))


LAYER_CASES = [("tiny", "f16"), ("tiny", "q4_0"), ("tiny-gelu", "f16"), ("small-p14-336", "f16")]


@pytest.mark.parametrize("geom,ft", LAYER_CASES)
def test_layers_against_oracle(prod, geom, ft):
    g = sg.GEOMETRIES[geom]
    path = model_file(geom, ft, prod)
    om = TokenOracle(path)
    n_img = 1 if g.n_pos > 257 else 2
    imgs = sg.synth_images(n_img, g.image_size, 33)
    seqs = token_seqs(3)[1:]                                # lengths 5, 2 (+ 77 below)
    seqs.append(token_seqs(1)[0])
    ids = padded(seqs)
    tol = TOL[ft]
    worst = 0.0
    with Ctx(prod, path) as ctx:
        for layer in (0, 1, g.v_layers // 2, -2, -1):
            raw_i = [om.image_tokens(img, layer) for img in imgs]
            raw_t = [om.text_tokens(s, layer) for s in seqs]
            for post_ln in (False, True):
                flags = bd.TOKENS_POST_LN if post_ln else 0
                got_i = prod.image_tokens(ctx, imgs, layer, flags)
                for k, img in enumerate(imgs):
                    want = om.ln(raw_i[k], "v.post_ln.weight", "v.post_ln.bias", om.v_eps) if post_ln else raw_i[k]
                    d = 1 - np.sum(got_i[k].astype(np.float64) * want, -1) / (np.linalg.norm(got_i[k], axis=-1) * np.linalg.norm(want, axis=-1))
                    assert d.max() <= tol, (geom, ft, "image", layer, post_ln, float(d.max()))
                    worst = max(worst, float(d.max()))
                    if layer == 0 and not post_ln:
                        err = np.abs(got_i[k].astype(np.float64) - want)
                        bound = preln_tol(om, img)
                        assert (err <= bound).all(), (geom, ft, float((err / bound).max()))
                got_t = prod.text_tokens(ctx, ids, layer, flags)
                for k, s in enumerate(seqs):
                    want = om.ln(raw_t[k], "t.post_ln.weight", "t.post_ln.bias", om.t_eps) if post_ln else raw_t[k]
                    have = got_t[k, :len(s)]
                    if layer == 0 and not post_ln:
                        # token + position embeddings: one fp32 addition of the same dequantised values on both sides, so equal
                        # in value; a q4_0 zero may carry either sign (0 * d with d < 0), so bits are not compared
                        assert np.array_equal(have, want), (geom, ft, k, int((have != want).sum()))
                    d = 1 - np.sum(have.astype(np.float64) * want, -1) / (np.linalg.norm(have, axis=-1) * np.linalg.norm(want, axis=-1))
                    assert d.max() <= tol, (geom, ft, "text", layer, post_ln, float(d.max()))
                    worst = max(worst, float(d.max()))
    print("%s %s  worst per-token 1-cos %.2e (bar %.0e)" % (geom, ft, worst, tol))


# ---- 3. layout and types, exact -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("flags", [0, bd.TOKENS_POST_LN, bd.TOKENS_PROJECT, PROJ_N])
def test_layout_types_and_device_variants(prod, flags):
    g = sg.GEOMETRIES["tiny"]
    imgs = sg.synth_images(5, g.image_size, 44)
    ids = padded(token_seqs(4))
    with Ctx(prod, model_file("tiny", "f16", prod)) as ctx:
        for layer in (0, 5, -1):
            full = prod.image_tokens(ctx, imgs, layer, flags)
            no_cls = prod.image_tokens(ctx, imgs, layer, flags | bd.TOKENS_NO_CLS)
            assert np.array_equal(bits(no_cls), bits(full[:, 1:]))
            f16 = prod.image_tokens(ctx, imgs, layer, flags, bd.OUT_F16)
            b16 = prod.image_tokens(ctx, imgs, layer, flags, bd.OUT_BF16)
            assert np.array_equal(bits(f16), bits(full.astype(np.float16)))
            assert np.array_equal(b16, bf16_of(full))
            for ot, want in ((bd.OUT_F32, full), (bd.OUT_F16, f16), (bd.OUT_BF16, b16)):
                dev = on_device(prod, ctx, lambda di, do: prod.lib.clip_b200_image_tokens_device(ctx, di, len(imgs), layer, flags, ot, do),
                                imgs, want.shape, want.dtype)
                assert np.array_equal(bits(dev), bits(want)), (layer, flags, ot)
            t32 = prod.text_tokens(ctx, ids, layer, flags)
            t16 = prod.text_tokens(ctx, ids, layer, flags, bd.OUT_F16)
            tb16 = prod.text_tokens(ctx, ids, layer, flags, bd.OUT_BF16)
            assert np.array_equal(bits(t16), bits(t32.astype(np.float16)))
            assert np.array_equal(tb16, bf16_of(t32))
            for ot, want in ((bd.OUT_F32, t32), (bd.OUT_BF16, tb16)):
                dev = on_device(prod, ctx, lambda di, do: prod.lib.clip_b200_text_tokens_device(ctx, di, len(ids), 77, layer, flags, ot, do),
                                ids, want.shape, want.dtype)
                assert np.array_equal(bits(dev), bits(want)), (layer, flags, ot)


def test_rows_do_not_depend_on_the_batch(prod):
    """image 0 alone == image 0 .. 699 inside one call of 700 images in micro-batches of 64 (11 passes); the same for text rows
    in micro-batches of 3 sequences, and for the shorter seq_len of a second call"""
    g = sg.GEOMETRIES["tiny"]
    imgs = sg.synth_images(700, g.image_size, 55)
    ids = padded(token_seqs(8))
    path = model_file("tiny", "f16", prod)
    flags = bd.TOKENS_POST_LN | bd.TOKENS_NO_CLS
    with Ctx(prod, path, (64, 3)) as ctx:
        big = prod.image_tokens(ctx, imgs, -2, flags, bd.OUT_F16)
        big_t = prod.text_tokens(ctx, ids, -2, bd.TOKENS_POST_LN)
        short_t = prod.text_tokens(ctx, ids[:, :40], -2, bd.TOKENS_POST_LN)
    with Ctx(prod, path) as ctx:
        for k in (0, 63, 64, 699):
            one = prod.image_tokens(ctx, imgs[k:k + 1], -2, flags, bd.OUT_F16)
            assert np.array_equal(bits(one[0]), bits(big[k])), k
        for k in range(len(ids)):
            one = prod.text_tokens(ctx, ids[k:k + 1], -2, bd.TOKENS_POST_LN)
            assert np.array_equal(bits(one[0]), bits(big_t[k])), k
    assert np.array_equal(bits(short_t), bits(big_t[:, :40]))


# ---- 4. the row kernel alone ----------------------------------------------------------------------------------------------------

TR_WIDTHS = [128, 384, 512, 640, 1024, 1152, 1280, 1664, 2048]      # MAXV 4 | 8 | 16, full and partial lanes


def run_token_rows(prod, x, n, T, no_cls, gamma, beta, out_type, in_stride=None):
    h = x.shape[1]
    out = np.empty((n * (T - no_cls), h), bd.OUT_DTYPES[out_type])
    rc = prod.lib.clip_b200_debug_token_rows(n, T, h, in_stride or h, no_cls, 1e-5, x.ctypes.data_as(FP),
                                             None if gamma is None else gamma.ctypes.data_as(FP),
                                             None if beta is None else beta.ctypes.data_as(FP), out_type, out.ctypes.data)
    assert rc == 0, prod.last_error()
    return out


@pytest.mark.parametrize("strided", [False, True], ids=["dense", "stride3h"])
@pytest.mark.parametrize("h", TR_WIDTHS)
def test_token_rows_kernel(prod, h, strided):
    """n = 3 items of T = 13 rows (39 rows: several blocks of 8 warps, a partial last one).
      f32 + LN: within ln_bound of the fp64 LayerNorm (offset rows: the spread identity, as for K4's fp32 output).
      16-bit + LN: equal to clip_b200_debug_layernorm's output for the same rows in that operand type, and to the round-to-nearest
      -even of the f32 output.  No LN: an exact copy / rounding.  NO_CLS: rows 1 .. T-1 of each item."""
    rng = np.random.default_rng(h * 3 + int(strided))
    n, T = 3, 13
    x, kinds = ln_rows(n * T, h, rng, first=h)
    gamma, beta = affine(rng, h)
    stride = 3 * h if strided else h
    y32 = run_token_rows(prod, x, n, T, 0, gamma, beta, bd.OUT_F32, stride)
    xh, rstd, mean_abs = ln_ref64(x, 1e-5)
    g64, b64 = gamma.astype(np.float64), beta.astype(np.float64)
    ref = g64 * xh + b64
    s = ln_bound(xh, rstd, mean_abs, g64, b64, h)
    well = np.array([k != "offset" for k in kinds])
    err = np.abs(y32.astype(np.float64) - ref)
    assert (err[well] <= s[well]).all(), (h, float((err[well] / s[well]).max()))
    for r, k in enumerate(kinds):
        if k == "offset":
            assert spread_error(y32[r], x[r], g64, b64, 1e-5) <= 1e-5, (h, r)
    for ot, bf in ((bd.OUT_F16, False), (bd.OUT_BF16, True)):
        y16 = run_token_rows(prod, x, n, T, 0, gamma, beta, ot, stride)
        k2 = np.empty((n * T, h), np.float32)
        assert prod.lib.clip_b200_debug_layernorm(n * T, h, stride, 1e-5, x.ctypes.data_as(FP), gamma.ctypes.data_as(FP),
                                                  beta.ctypes.data_as(FP), None, int(bf), k2.ctypes.data_as(FP), None) == 0
        want16 = bf16_of(k2) if bf else k2.astype(np.float16)
        assert np.array_equal(bits(y16), bits(want16)), (h, ot)
        assert np.array_equal(bits(y16), bf16_of(y32) if bf else bits(y32.astype(np.float16))), (h, ot)
    drop = run_token_rows(prod, x, n, T, 1, gamma, beta, bd.OUT_F32, stride)
    assert np.array_equal(bits(drop), bits(y32.reshape(n, T, h)[:, 1:].reshape(-1, h)))
    raw = run_token_rows(prod, x, n, T, 1, None, None, bd.OUT_F32, stride)
    assert np.array_equal(bits(raw), bits(x.reshape(n, T, h)[:, 1:].reshape(-1, h)))
    raw16 = run_token_rows(prod, x, n, T, 0, None, None, bd.OUT_BF16, stride)
    assert np.array_equal(raw16, bf16_of(x))
    print("token_rows h=%d err/bound %.3f" % (h, float((err[well] / s[well]).max())))


# ---- 5. early exit, 6. refusals, 7. devices mode --------------------------------------------------------------------------------

def test_early_exit_skips_one_block(prod):
    """layer -2 launches exactly one block's kernels (LN, QKV, attention, out-proj, LN, FC1, FC2) fewer than layer -1"""
    g = sg.GEOMETRIES["tiny"]
    imgs = sg.synth_images(3, g.image_size, 66)
    ids = padded(token_seqs(3))
    with Ctx(prod, model_file("tiny", "q4_0", prod)) as ctx:
        n = prod.lib.clip_b200_kernel_launches
        counts = {}
        for layer in (-1, -2, 0):
            a = n(ctx)
            prod.image_tokens(ctx, imgs, layer, bd.TOKENS_NO_CLS)
            b = n(ctx)
            prod.text_tokens(ctx, ids, layer, bd.TOKENS_POST_LN)
            counts[layer] = (b - a, n(ctx) - b)
    assert counts[-1][0] - counts[-2][0] == 7 and counts[-1][1] - counts[-2][1] == 7, counts
    assert counts[-1][0] - counts[0][0] == 7 * g.v_layers and counts[-1][1] - counts[0][1] == 7 * g.t_layers, counts


def test_refusals(prod, tmp_path):
    g = sg.GEOMETRIES["tiny"]
    imgs = sg.synth_images(1, g.image_size, 1)
    ids = padded(token_seqs(1))
    batch, keep = prod.make_image_batch(imgs)
    out = np.empty(1 << 20, np.float32)
    L = prod.lib

    def img(layer, flags, ot=0):
        return L.clip_b200_image_tokens(ctx, C.byref(batch), layer, flags, ot, out.ctypes.data)

    def txt(layer, flags, ot=0):
        return L.clip_b200_text_tokens(ctx, ids.ctypes.data_as(C.POINTER(C.c_int32)), 1, 77, layer, flags, ot, out.ctypes.data)

    with Ctx(prod, model_file("tiny", "f16", prod)) as ctx:
        for call, msg in ((lambda: img(13, 0), "layer 13"), (lambda: img(-14, 0), "layer -14"), (lambda: txt(13, 0), "outside"),
                          (lambda: txt(0, bd.TOKENS_NO_CLS), "vision tower only"), (lambda: img(-1, bd.TOKENS_NORMALIZE), "needs"),
                          (lambda: img(-1, 16), "unknown flag"), (lambda: txt(-1, 0, 3), "out_type")):
            assert not call(), msg
            assert msg in prod.last_error(), (msg, prod.last_error())
        assert img(-13, 0) and img(12, 0) and txt(-13, 0)
        empty = bd.clip_image_f32_batch(None, 0)
        assert L.clip_b200_image_tokens(ctx, C.byref(empty), -1, 0, 0, None)
        assert L.clip_b200_text_tokens(ctx, None, 0, 77, -1, 0, 0, None)
        assert L.clip_b200_image_tokens_device(ctx, None, 0, -1, 0, 0, None)
    text_only = sg.Geometry("text-only", image_size=64, patch_size=16, v_hidden=128, v_ff=256, v_heads=2, v_layers=1,
                            t_hidden=128, t_ff=256, t_heads=2, t_layers=2, proj_dim=128, has_vision=False)
    path = str(tmp_path / "text-only.gguf")
    sg.write_model(path, text_only, 1, 1)
    with Ctx(prod, path) as ctx:
        assert not img(-1, 0)
        assert "no vision encoder" in prod.last_error()
        assert txt(-1, bd.TOKENS_POST_LN)


def test_devices_mode_equals_one_gpu(prod, monkeypatch):
    if prod.lib.clip_b200_cuda_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    g = sg.GEOMETRIES["tiny"]
    imgs = sg.synth_images(37, g.image_size, 77)
    ids = padded(token_seqs(19))
    path = model_file("tiny", "q4_0", prod)
    with Ctx(prod, path) as ctx:
        one_i = prod.image_tokens(ctx, imgs, -2, bd.TOKENS_NO_CLS, bd.OUT_F16)
        one_t = prod.text_tokens(ctx, ids, -1, PROJ_N)
    monkeypatch.setenv("CLIP_B200_DEVICES", "all")
    with Ctx(prod, path) as ctx:
        assert prod.lib.clip_b200_device_count(ctx) >= 2
        assert np.array_equal(bits(prod.image_tokens(ctx, imgs, -2, bd.TOKENS_NO_CLS, bd.OUT_F16)), bits(one_i))
        assert np.array_equal(bits(prod.text_tokens(ctx, ids, -1, PROJ_N)), bits(one_t))
