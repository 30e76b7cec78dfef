"""End-to-end parity of the CUDA path (through the reference-facing C ABI, host buffers) against golden vectors
produced by the reference itself (tests/golden/make_golden.py) and against the CPU oracle restatement.
Tolerances are BASELINE.json's: 1 - cos <= 1e-3 (f16/f32), <= 1e-2 (q*)."""
import numpy as np
import pytest

import synth_gguf as sg
from _util import FTYPES, TOL, check_sha, golden, model_file, one_minus_cos, token_seqs

pytestmark = pytest.mark.gpu


def _check(prod, geom, ft):
    g = golden(geom)
    assert g is not None and ("img_" + ft) in g, "golden fixture missing for %s/%s" % (geom, ft)
    path = model_file(geom, ft, prod)
    check_sha(path, g["sha_" + ft])
    geo = sg.GEOMETRIES[geom]
    imgs = sg.synth_images(int(g["n_img"]), geo.image_size, int(g["img_seed"]))
    seqs = token_seqs(int(g["n_txt"]), int(g["tok_seed"]))
    ctx = prod.load(path, 0)
    try:
        got_i = prod.image_batch_encode(ctx, imgs)
        got_t = prod.text_batch_encode(ctx, seqs)
        single = prod.image_encode(ctx, imgs[0])
        assert prod.lib.clip_b200_kernel_launches(ctx) > 0
    finally:
        prod.free(ctx)
    di, dt = one_minus_cos(got_i, g["img_" + ft]), one_minus_cos(got_t, g["txt_" + ft])
    print("%s %s  image 1-cos max %.2e  text 1-cos max %.2e" % (geom, ft, di.max(), dt.max()))
    assert np.isfinite(got_i).all() and np.isfinite(got_t).all()
    assert di.max() <= TOL[ft], (geom, ft, di)
    assert dt.max() <= TOL[ft], (geom, ft, dt)
    assert np.abs(np.linalg.norm(got_i, axis=1) - 1).max() < 1e-4
    # batch semantics == independent single-image encodes (SURVEY.md section 8c)
    assert one_minus_cos(single, got_i[0]) < 1e-6


@pytest.mark.parametrize("ft", list(FTYPES))
def test_tiny_all_file_types(prod, ft):
    _check(prod, "tiny", ft)


@pytest.mark.parametrize("ft", ["f16", "q4_0"])
def test_tiny_gelu_variant(prod, ft):
    _check(prod, "tiny-gelu", ft)


@pytest.mark.parametrize("ft", ["f16", "q4_0", "q8_0"])
def test_patch14_257_positions(prod, ft):
    _check(prod, "small-p14", ft)


@pytest.mark.parametrize("ft", ["f16", "q4_0"])
def test_patch14_336_577_positions(prod, ft):
    """ViT-L/14@336 token count (577 > 257: long-sequence attention path) end to end against the reference"""
    _check(prod, "small-p14-336", ft)


@pytest.mark.slow
@pytest.mark.parametrize("ft", ["f16", "q4_0", "q4_1", "q5_0", "q5_1", "q8_0"])
def test_vit_b32_true_geometry(prod, ft):
    _check(prod, "vit-b32", ft)


@pytest.mark.slow
@pytest.mark.parametrize("ft", ["f16", "q4_0", "q4_1", "q5_0", "q5_1", "q8_0"])
def test_vit_l14_true_geometry(prod, ft):
    _check(prod, "vit-l14", ft)


def test_against_cpu_oracle_unnormalized(prod):
    """normalize=false path + a model/seed with no golden fixture: compare with the oracle restatement directly."""
    import oracle as orc
    path = model_file("tiny", "q5_1", prod)
    imgs = sg.synth_images(2, 64, 4242)
    seqs = [sg.synth_tokens(1, n, 17 + n)[0] for n in (3, 40)]
    om = orc.OracleModel(path)
    ctx = prod.load(path, 0)
    try:
        gi = prod.image_batch_encode(ctx, imgs, normalize=False)
        gt = prod.text_batch_encode(ctx, seqs, normalize=False)
    finally:
        prod.free(ctx)
    for i in range(2):
        oi, ot = om.encode_image(imgs[i], normalize=False), om.encode_text(seqs[i], normalize=False)
        assert one_minus_cos(gi[i], oi) <= 1e-2 and one_minus_cos(gt[i], ot) <= 1e-2
        # un-normalised magnitudes must agree too, not only directions
        assert abs(np.linalg.norm(gi[i]) / np.linalg.norm(oi) - 1) < 0.05
        assert abs(np.linalg.norm(gt[i]) / np.linalg.norm(ot) - 1) < 0.05


@pytest.mark.parametrize("ft", ["f16", "q4_0"])
def test_wide_h1280_against_cpu_oracle(prod, ft):
    """1280-wide towers (wide-h1280): the only place the 16-float4-per-lane LayerNorm runs in the model schedule -- pre-LN, ln1 /
    ln2 and post-LN of both towers -- next to the f16 patch embedding at kpad 640 and FC2 at K = 5120.  No golden file: the
    oracle restatement is the reference."""
    import oracle as orc
    path = model_file("wide-h1280", ft, prod)
    imgs = sg.synth_images(3, 112, 1280)
    seqs = [sg.synth_tokens(1, n, 1280 + n)[0] for n in (2, 33, 77)]
    ctx = prod.load(path, 0)
    try:
        gi = prod.image_batch_encode(ctx, imgs, normalize=False)
        gt = prod.text_batch_encode(ctx, seqs, normalize=False)
        ni = prod.image_batch_encode(ctx, imgs)
        nt = prod.text_batch_encode(ctx, seqs)
    finally:
        prod.free(ctx)
    om = orc.OracleModel(path)
    for i in range(3):
        oi, ot = om.encode_image(imgs[i], normalize=False), om.encode_text(seqs[i], normalize=False)
        di, dt = one_minus_cos(ni[i], oi), one_minus_cos(nt[i], ot)
        print("wide-h1280 %s #%d  image 1-cos %.2e  text 1-cos %.2e" % (ft, i, di, dt))
        assert di <= TOL[ft] and dt <= TOL[ft], (ft, i, di, dt)
        assert abs(np.linalg.norm(gi[i]) / np.linalg.norm(oi) - 1) < 0.05
        assert abs(np.linalg.norm(gt[i]) / np.linalg.norm(ot) - 1) < 0.05
        assert one_minus_cos(gi[i], ni[i]) < 1e-6 and one_minus_cos(gt[i], nt[i]) < 1e-6


def test_edge_cases(prod):
    import ctypes as C
    import binding as bd
    path = model_file("tiny", "q4_0", prod)
    ctx = prod.load(path, 0)
    prod.lib.clip_b200_set_micro_batch(ctx, 64, 3)      # small micro-batches: the 300-image / 8-sequence cases below run in several passes
    try:
        # empty batch: succeeds, writes nothing
        empty = bd.clip_image_f32_batch(None, 0)
        assert prod.lib.clip_image_batch_encode(ctx, 1, C.byref(empty), None, True)
        assert prod.text_batch_encode(ctx, [], True).shape[0] == 0
        # wrong image size -> false, no crash (the reference GGML_ASSERTs, clip.cpp:1293)
        bad = np.zeros((1, 32, 32, 3), np.float32)
        with pytest.raises(RuntimeError):
            prod.image_batch_encode(ctx, bad)
        # sequence longer than context_length -> false
        with pytest.raises(RuntimeError):
            prod.text_batch_encode(ctx, [np.zeros(78, np.int32)])
        # shortest legal sequence (SOT, EOT) and the longest (77)
        out = prod.text_batch_encode(ctx, [np.array([49406, 49407], np.int32), sg.synth_tokens(1, 77, 1)[0]])
        assert np.isfinite(out).all()
        # ragged batch == one-at-a-time
        seqs = token_seqs(8)
        batch = prod.text_batch_encode(ctx, seqs)
        for i in (0, 2, 7):
            # same rows, same math; only the padded length differs (batch: 77, single: its own length rounded up to 8), which changes the
            # summation order inside the softmax.  The residual stream is fp32 end to end (no 16-bit branch rounding that would snap such
            # differences away), so they stay visible at the 1e-6 level
            dev = one_minus_cos(batch[i], prod.text_encode(ctx, seqs[i]))
            print("ragged vs single 1-cos", i, dev)
            assert dev < 1e-5
        # a batch larger than one micro-batch (several passes + balanced chunking), deterministic and order-preserving
        imgs = sg.synth_images(300, 64, 5)
        a = prod.image_batch_encode(ctx, imgs)
        b = prod.image_batch_encode(ctx, imgs)
        assert np.array_equal(a, b)
        perm = np.random.default_rng(0).permutation(300)
        c = prod.image_batch_encode(ctx, np.ascontiguousarray(imgs[perm]))
        assert one_minus_cos(c, a[perm]).max() < 1e-6
    finally:
        prod.free(ctx)
    assert prod.lib.clip_model_load(b"/nonexistent.gguf", 0) is None
    assert b"cannot open" in prod.lib.clip_b200_last_error()


def test_device_resident_entry_points(prod):
    import ctypes as C
    path = model_file("tiny", "q8_0", prod)
    ctx = prod.load(path, 0)
    try:
        imgs = sg.synth_images(5, 64, 11)
        host = prod.image_batch_encode(ctx, imgs)
        d_in = prod.lib.clip_b200_device_malloc(ctx, imgs.nbytes)
        d_out = prod.lib.clip_b200_device_malloc(ctx, host.nbytes)
        assert prod.lib.clip_b200_memcpy_h2d(ctx, d_in, imgs.ctypes.data, imgs.nbytes)
        assert prod.lib.clip_b200_image_encode_device(ctx, d_in, 5, d_out, True)
        got = np.empty_like(host)
        assert prod.lib.clip_b200_memcpy_d2h(ctx, got.ctypes.data, d_out, got.nbytes)
        assert np.array_equal(got, host)
        assert prod.lib.clip_b200_last_device_ms(ctx) > 0
        # zero-shot scoring on device vs the reference's softmax_with_sorting arithmetic on host
        seqs = token_seqs(6)
        txt = prod.text_batch_encode(ctx, seqs, normalize=False)
        img = prod.image_batch_encode(ctx, imgs, normalize=False)
        d_t = prod.lib.clip_b200_device_malloc(ctx, txt.nbytes)
        d_i = prod.lib.clip_b200_device_malloc(ctx, img.nbytes)
        prod.lib.clip_b200_memcpy_h2d(ctx, d_t, txt.ctypes.data, txt.nbytes)
        prod.lib.clip_b200_memcpy_h2d(ctx, d_i, img.ctypes.data, img.nbytes)
        scores = np.empty((5, 6), np.float32)
        idx = np.empty((5, 6), np.int32)
        assert prod.lib.clip_b200_zero_shot_batch(ctx, d_i, 5, d_t, 6, scores.ctypes.data_as(C.POINTER(C.c_float)),
                                                  idx.ctypes.data_as(C.POINTER(C.c_int)), 6)
        for i in range(5):
            s = (img[i] @ txt.T).astype(np.float32)
            e = np.exp(s.astype(np.float64)).astype(np.float32) + np.float32(1e-9)
            p = e / e.astype(np.float64).sum()
            order = np.argsort(-p, kind="stable")
            assert np.array_equal(idx[i], order)
            assert np.allclose(scores[i], p[order], rtol=1e-4, atol=1e-7)
        for d in (d_in, d_out, d_t, d_i):
            prod.lib.clip_b200_device_free(ctx, d)
    finally:
        prod.free(ctx)
