"""Both towers at the sequence lengths any-resolution images and long text contexts reach, against the CPU oracle at the
project's 1 - cos bars (TOL), per token.

  * Vision: tiny (f16, q4_0) at 512 x 512 (T = 1025) for the embedding and every checked layer, and at 1024 x 1024 (T = 4097) for
    layers 1 and 2; small-p14 at 448 x 448 (T = 1025) and 672 x 672 (T = 2305); huge-w640 (head_dim 80) at 448 x 448.  Several
    images in one call, in one pass and in several, equal each image alone bit for bit.
  * The largest pass: tiny at 4096 x 4096 (T = 65 537, one image in one pass of the default workspace) at layer 1, on sampled rows
    against the oracle's first block restated for those rows (its LayerNorm, mul_mat and GELU on every row, fp64 attention for
    the sampled query rows over all 65 537 keys).
  * Text: a tiny model with context_length 4096 (defined here, not one of synth_gguf's GEOMETRIES), text_tokens at 78, 248, 1000,
    2049 and 4096 tokens; a batch of mixed lengths equals each sequence alone bit for bit and the oracle's encode_text at TOL; a
    4097-token sequence is refused.
  * An oversized micro_batch is refused at the first encode with a message naming it and the limit, before any allocation, and
    the context then takes a valid one.
The oracle's attention is O(T^2) per head on the CPU, so the layers checked at each size are those it computes in seconds."""
import numpy as np
import pytest

import binding as bd
import synth_gguf as sg
from _oracle_anyres import AnyresOracle
from _util import TOL, model_file
from test_gpu_anyres import cos_rows, images
from test_gpu_tokens import Ctx, bits
from test_pos_resample import pos_resample_ref

pytestmark = pytest.mark.gpu


def check_layers(prod, ctx, om, imgs, layers, tol, tag):
    P = om.patch
    H, W = imgs.shape[1:3]
    pos = om.position_table_hw(H // P, W // P, pos_resample_ref)
    worst = 0.0
    for layer in layers:
        got = prod.image_tokens_hw(ctx, imgs, layer, 0)
        assert got.shape == (len(imgs), (H // P) * (W // P) + 1, om.v_hidden)
        for k, img in enumerate(imgs):
            d = cos_rows(got[k], om.image_tokens_hw(img, pos, layer))
            assert d.max() <= tol, (tag, layer, k, float(d.max()), int(d.argmax()))
            worst = max(worst, float(d.max()))
    print("%s layers %s  worst per-token 1-cos %.2e (bar %.0e)" % (tag, layers, worst, tol))
    return pos


VISION = [("tiny", "f16", 512, (0, 1, 6, -2, -1), True), ("tiny", "q4_0", 512, (0, 1, 6, -2, -1), True),
          ("tiny", "f16", 1024, (1, 2), False), ("tiny", "q4_0", 1024, (1, 2), False),
          ("small-p14", "f16", 448, (1, 2, -1), True), ("small-p14", "q4_0", 672, (1, 2), False),
          ("huge-w640", "f16", 448, (1, 2), False)]


@pytest.mark.parametrize("geom,ft,S,layers,embed", VISION)
def test_vision_tower_at_long_T(prod, geom, ft, S, layers, embed):
    path = model_file(geom, ft, prod)
    om = AnyresOracle(path)
    imgs = images(1, S, S, S + len(ft))
    with Ctx(prod, path) as ctx:
        pos = check_layers(prod, ctx, om, imgs, layers, TOL[ft], "%s %s %dx%d" % (geom, ft, S, S))
        if embed:
            for normalize in (True, False):
                got = prod.image_batch_encode_hw(ctx, imgs, normalize)
                d = float(cos_rows(got[0], om.encode_image_hw(imgs[0], pos, normalize)))
                assert d <= TOL[ft], (geom, ft, S, "embedding", normalize, d)


@pytest.mark.parametrize("micro_batch", [0, 130])
def test_images_in_one_call_equal_each_alone(prod, micro_batch):
    """3 images at 512 x 512 (T = 1025) in one call: one pass of the default workspace, or two with micro_batch 130 of T = 17
    (2210 rows: two images per pass)"""
    path = model_file("tiny", "f16", prod)
    imgs = images(3, 512, 512, 5)
    with Ctx(prod, path, (micro_batch, 0)) as ctx:
        all_t = prod.image_tokens_hw(ctx, imgs, -2, bd.TOKENS_POST_LN)
        all_e = prod.image_batch_encode_hw(ctx, imgs)
        for k in range(3):
            assert np.array_equal(bits(prod.image_tokens_hw(ctx, imgs[k:k + 1], -2, bd.TOKENS_POST_LN)[0]), bits(all_t[k])), k
            assert np.array_equal(bits(prod.image_batch_encode_hw(ctx, imgs[k:k + 1])[0]), bits(all_e[k])), k


def first_block_rows(om, x0, rows):
    """the oracle's block 0 (oracle.OracleModel._blocks, vision) for the residual rows `rows` of x0 [T, h]: ln1 and the QKV
    products on every row, softmax(Q K^T) V in fp64 for the given query rows over every key, the rest row by row"""
    b, eps, heads = "v.blk.0.", om.v_eps, om.v_heads
    hid = x0.shape[1]
    dh = hid // heads
    scale = np.float32(1.0) / np.float32(np.sqrt(np.float32(dh)))
    cur = om.ln(x0, b + "ln1.weight", b + "ln1.bias", eps)
    q = ((om.f32(b + "attn_q.bias") + om.mul_mat(b + "attn_q.weight", cur[rows])) * scale).astype(np.float64)
    k = (om.f32(b + "attn_k.bias") + om.mul_mat(b + "attn_k.weight", cur)).astype(np.float64)
    v = (om.f32(b + "attn_v.bias") + om.mul_mat(b + "attn_v.weight", cur)).astype(np.float64)
    att = np.empty((len(rows), hid), np.float32)
    for h in range(heads):
        sl = slice(h * dh, (h + 1) * dh)
        s = q[:, sl] @ k[:, sl].T
        p = np.exp(s - s.max(-1, keepdims=True))
        att[:, sl] = (p / p.sum(-1, keepdims=True)) @ v[:, sl]
    x = (om.f32(b + "attn_out.bias") + om.mul_mat(b + "attn_out.weight", att)) + x0[rows]
    cur = om.ln(x, b + "ln2.weight", b + "ln2.bias", eps)
    cur = om.gelu(om.f32(b + "ffn_down.bias") + om.mul_mat(b + "ffn_down.weight", cur))
    return x + (om.f32(b + "ffn_up.bias") + om.mul_mat(b + "ffn_up.weight", cur))


def test_largest_single_pass(prod):
    """tiny at 4096 x 4096: T = 65 537 rows in one pass (the default workspace holds 4472 x 17 = 76 024 rows), layer 1.  The call
    launches exactly what a one-pass call at 512 x 512 launches (both resample the table once)."""
    path = model_file("tiny", "f16", prod)
    om = AnyresOracle(path)
    img = images(1, 4096, 4096, 4096)
    small = images(1, 512, 512, 512)
    with Ctx(prod, path) as ctx:
        n = prod.lib.clip_b200_kernel_launches
        a = n(ctx)
        prod.image_tokens_hw(ctx, small, 1, 0)
        b = n(ctx)
        got = prod.image_tokens_hw(ctx, img, 1, 0)[0]
        assert n(ctx) - b == b - a, (n(ctx) - b, b - a)
    T = 256 * 256 + 1
    assert got.shape == (T, om.v_hidden)
    x0, _ = om._embed_hw(img[0], om.position_table_hw(256, 256, pos_resample_ref))
    rng = np.random.default_rng(7)
    rows = np.unique(np.concatenate([[0, 1, T - 1, T - 2], np.arange(128, T, 8192), np.arange(64, T, 8192) - 1,
                                     rng.integers(0, T, 192)]))
    want = first_block_rows(om, x0, rows)
    d = cos_rows(got[rows], want)
    print("tiny f16 4096x4096 layer 1: %d rows, worst 1-cos %.2e" % (len(rows), d.max()))
    assert d.max() <= TOL["f16"], (float(d.max()), int(rows[d.argmax()]))


# ---- text ----------------------------------------------------------------------------------------------------------------------
LONG_CTX = sg.Geometry("tiny-ctx4096", image_size=64, patch_size=16, v_hidden=128, v_ff=256, v_heads=2, v_layers=12, t_hidden=128,
                       t_ff=256, t_heads=2, t_layers=12, proj_dim=128, n_ctx=4096)
TEXT = [(78, (1, 2, -1)), (248, (1, 2, -1)), (1000, (1, 2, -1)), (2049, (1, 2, -1)), (4096, (1, 2))]


@pytest.fixture(scope="module")
def long_ctx_model(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("long_ctx") / "tiny-ctx4096.gguf")
    sg.write_model(path, LONG_CTX, 1234, 1)
    return path


@pytest.mark.parametrize("n,layers", TEXT)
def test_text_tokens_at_long_context(prod, long_ctx_model, n, layers):
    om = AnyresOracle(long_ctx_model)
    ids = sg.synth_tokens(1, n, 17 + n)
    worst = 0.0
    with Ctx(prod, long_ctx_model) as ctx:
        for layer in layers:
            got = prod.text_tokens(ctx, ids, layer, 0)[0]
            d = cos_rows(got, om.text_tokens(ids[0], layer))
            assert d.max() <= TOL["f16"], (n, layer, float(d.max()), int(d.argmax()))
            worst = max(worst, float(d.max()))
    print("text n=%d layers %s  worst per-token 1-cos %.2e" % (n, layers, worst))


def test_text_batch_at_long_context(prod, long_ctx_model):
    om = AnyresOracle(long_ctx_model)
    seqs = [sg.synth_tokens(1, n, 40 + n)[0] for n in (4096, 78, 1000, 2049, 5, 248)]
    with Ctx(prod, long_ctx_model) as ctx:
        batch = prod.text_batch_encode(ctx, seqs)
        for k, s in enumerate(seqs):
            assert np.array_equal(bits(prod.text_batch_encode(ctx, [s])[0]), bits(batch[k])), len(s)
        too_long = sg.synth_tokens(1, 4097, 3)
        with pytest.raises(RuntimeError, match="longer than context_length"):
            prod.text_batch_encode(ctx, [too_long[0]])
        with pytest.raises(RuntimeError, match=r"seq_len must be in \[1, context_length\]"):
            prod.text_tokens(ctx, too_long, -1, 0)
    for k, s in enumerate(seqs):
        d = float(cos_rows(batch[k], om.encode_text(s)))
        assert d <= TOL["f16"], (len(s), d)


# ---- micro_batch limit ---------------------------------------------------------------------------------------------------------
def test_oversized_micro_batch_is_refused_before_allocation(prod):
    """tiny: 17 rows per image x 768 (the padded patch width, its widest) and 77 rows per sequence x 384 (3 x hidden) must stay
    below 2^32, so at most 328 965 images and 145 257 sequences per pass.  One past each limit, and counts whose rows overflow an
    int, are refused at the first encode -- before allocating the ~40 GB the first would take -- and the same context then runs
    with a valid micro_batch as a fresh one does."""
    path = model_file("tiny", "f16", prod)
    imgs = sg.synth_images(3, 64, 9)
    seqs = [sg.synth_tokens(1, n, n)[0] for n in (77, 9)]
    with Ctx(prod, path, (8, 4)) as ctx:
        want_i, want_t = prod.image_batch_encode(ctx, imgs), prod.text_batch_encode(ctx, seqs)
    for images_mb, seqs_mb in ((328966, 145258), (200_000_000, 30_000_000)):
        with Ctx(prod, path, (images_mb, seqs_mb)) as ctx:
            with pytest.raises(RuntimeError, match="vision micro_batch %d is too large.*the limit is 328965" % images_mb):
                prod.image_batch_encode(ctx, imgs)
            with pytest.raises(RuntimeError, match="text micro_batch %d is too large.*the limit is 145257" % seqs_mb):
                prod.text_batch_encode(ctx, seqs)
            prod.lib.clip_b200_set_micro_batch(ctx, 8, 4)
            assert np.array_equal(bits(prod.image_batch_encode(ctx, imgs)), bits(want_i))
            assert np.array_equal(bits(prod.text_batch_encode(ctx, seqs)), bits(want_t))
