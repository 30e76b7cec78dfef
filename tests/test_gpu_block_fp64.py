"""Each encoder block on the GPU against fp64, fed the GPU's own residual rows (tests/_block_ref.py): for block l, one
*_tokens_layers call (flags 0, OUT_F32) returns x_l and x_{l+1} (HF numbering: the residual before and after block l), and every row
of every sequence must meet e_gpu <= C e_emu + floor.  The models have sharp attention (synth_gguf.write_model's qk_logit_std = 3),
so a wrong Q scale, mask or key moves the output; they are written into a temporary directory, and quantized by the product.

Two negative controls run on the GPU's numbers: emu built for fp16 operands where the GPU ran bf16, and x_{l-1} passed where x_l
belongs; both must miss the criterion."""
import numpy as np
import pytest

import _block_ref as br
import synth_gguf as sg
from _block_ref import C
from _oracle_tokens import TokenOracle
from _util import FTYPES
from test_gpu_tokens import Ctx, padded
from test_gpu_tokens_layers import images

pytestmark = pytest.mark.gpu

SHARP = 3.0
_files = {}


@pytest.fixture(scope="module")
def sharp(prod, tmp_path_factory):
    d = tmp_path_factory.mktemp("sharp")

    def path(geom, ft):
        key = (geom, ft)
        if key not in _files:
            if ft == "f16":
                p = str(d / ("%s-f16.gguf" % geom))
                sg.write_model(p, sg.GEOMETRIES[geom], 1234, 1, qk_logit_std=SHARP)
            else:
                p = str(d / ("%s-%s.gguf" % (geom, ft)))
                assert prod.quantize(path(geom, "f16"), p, FTYPES[ft]), prod.last_error()
            _files[key] = p
        return _files[key]
    return path


def text_ids(n):
    """n sequences padded to 77: one full length, the others shorter (their pad rows are causal rows like any other)"""
    return padded([sg.synth_tokens(1, L, 40 + i)[0] for i, L in enumerate([77, 33, 64][:n])])


def check(om, tower, l, x_in, x_out, lens, causal, bf16, what):
    blk = br.Block(om, tower, l)
    r = br.check_block(blk, x_in.reshape(-1, blk.hidden), x_out.reshape(-1, blk.hidden), lens, causal, bf16)
    print("%-48s block %2d: worst e_gpu/e_emu %.3f (C = %.2f)" % (what, l, r, C))
    return r


def run_layers(prod, om, path, geom, blocks, bf16, what, n_img=2, n_txt=3, towers=("v", "t")):
    """x before and after each block in `blocks` of each tower from one *_tokens_layers call, and the criterion on every row"""
    g = sg.GEOMETRIES[geom]
    worst = 0.0
    with Ctx(prod, path) as ctx:
        for tower in towers:
            vision = tower == "v"
            bl = blocks[tower] if isinstance(blocks, dict) else blocks
            bl = list(range(g.v_layers if vision else g.t_layers)) if bl == "all" else bl
            layers = sorted({l for b in bl for l in (b, b + 1)})
            if vision:
                imgs = sg.synth_images(n_img, g.image_size, 5)
                out = prod.image_tokens_layers(ctx, imgs, layers, None, 0)
                lens, causal = [g.n_pos] * n_img, False
            else:
                ids = text_ids(n_txt)
                out = prod.text_tokens_layers(ctx, ids, layers, None, 0)
                lens, causal = [77] * n_txt, True
            slab = dict(zip(layers, out))
            for b in bl:
                worst = max(worst, check(om, tower, b, slab[b], slab[b + 1], lens, causal, bf16, "%s %s %s" % (what, geom, tower)))
    return worst


TINY = [("f16", None)] + [(ft, op) for ft in ("q4_0", "q4_1", "q5_0", "q5_1", "q8_0") for op in ("bf16", "f16")]


@pytest.mark.parametrize("ft,operand", TINY)
def test_tiny_every_block(prod, sharp, monkeypatch, ft, operand):
    """dh 64, quick-GELU, both towers, all 12 blocks: f16 weights, and every quantized type at bf16 and at fp16 operands"""
    if operand:
        monkeypatch.setenv("CLIP_B200_OPERAND", operand)
    bf16 = operand == "bf16"
    path = sharp("tiny", ft)
    r = run_layers(prod, TokenOracle(path), path, "tiny", "all", bf16, "%s/%s" % (ft, "bf16" if bf16 else "fp16"))
    assert r <= C, r


GEOM_CASES = [
    ("tiny-gelu", "f16", "all"), ("tiny-gelu", "q4_0", "all"),
    ("small-p14", "f16", {"v": [0, 5, 11], "t": [0, 11]}), ("small-p14", "q8_0", {"v": [0, 5, 11], "t": [0, 11]}),
    ("small-p14-336", "f16", {"v": [0, 11], "t": [0]}),
    ("huge-w640", "f16", {"v": [0, 15, 31], "t": [0, 23]}), ("huge-w640", "q4_1", {"v": [0, 15, 31], "t": [0, 23]}),
    ("bigg-w1664", "f16", {"v": [0, 31], "t": [0]}), ("bigg-w1664", "q5_0", {"v": [0, 31], "t": [0]}),
    ("wide-h1280", "f16", {"v": [0, 1], "t": [0, 1]}), ("wide-h1280", "q4_0", {"v": [0, 1], "t": [0, 1]}),
]


@pytest.mark.parametrize("geom,ft,blocks", GEOM_CASES, ids=["%s-%s" % (g, f) for g, f, _ in GEOM_CASES])
def test_geometry_blocks(prod, sharp, geom, ft, blocks):
    """the tanh GELU; T = 257 (a ragged last key block); T = 577; head_dim 80; head_dim 104 padded to 112; width 1280 with FC2 K = 5120"""
    path = sharp(geom, ft)
    g = sg.GEOMETRIES[geom]
    r = run_layers(prod, TokenOracle(path), path, geom, blocks, ft != "f16", ft, n_img=1 if g.n_pos > 100 else 2,
                   n_txt=1 if g.t_hidden > 1024 else 3)
    assert r <= C, r


# ---- the single-layer packed, mixed and any-resolution forms, and the legacy attention kernel ------------------------------------

BLOCKS = (0, 6, 11)


def test_text_packed(prod, sharp):
    path = sharp("tiny", "f16")
    om = TokenOracle(path)
    seqs = [sg.synth_tokens(1, L, 70 + L)[0] for L in (1, 2, 63, 64, 65, 76, 77)]
    lens = [len(s) for s in seqs]
    worst = 0.0
    with Ctx(prod, path) as ctx:
        for b in BLOCKS:
            x0 = np.concatenate(prod.text_tokens_packed(ctx, seqs, b))
            x1 = np.concatenate(prod.text_tokens_packed(ctx, seqs, b + 1))
            worst = max(worst, check(om, "t", b, x0, x1, lens, True, False, "text_tokens_packed"))
    assert worst <= C, worst


def test_image_mixed_and_hw(prod, sharp):
    path = sharp("tiny", "f16")
    om = TokenOracle(path)
    P = om.patch
    mixed = [images(1, H, W, 80 + i)[0] for i, (H, W) in enumerate([(64, 64), (48, 80), (128, 128), (96, 64)])]
    lens = [(H // P) * (W // P) + 1 for H, W in [im.shape[:2] for im in mixed]]
    assert any(t % 64 for t in lens)
    hw = images(2, 160, 192, 90)
    worst = 0.0
    with Ctx(prod, path) as ctx:
        for b in BLOCKS:
            x0 = np.concatenate(prod.image_tokens_mixed(ctx, mixed, b))
            x1 = np.concatenate(prod.image_tokens_mixed(ctx, mixed, b + 1))
            worst = max(worst, check(om, "v", b, x0, x1, lens, False, False, "image_tokens_mixed"))
            x0, x1 = prod.image_tokens_hw(ctx, hw, b), prod.image_tokens_hw(ctx, hw, b + 1)
            worst = max(worst, check(om, "v", b, x0, x1, [x0.shape[1]] * 2, False, False, "image_tokens_hw 160x192"))
    assert worst <= C, worst


def test_legacy_attention(prod, sharp, monkeypatch):
    monkeypatch.setenv("CLIP_B200_ATTN", "legacy")
    path = sharp("tiny", "f16")
    r = run_layers(prod, TokenOracle(path), path, "tiny", list(BLOCKS), False, "CLIP_B200_ATTN=legacy")
    assert r <= C, r


# ---- negative controls on the GPU's numbers ------------------------------------------------------------------------------------

def test_negative_controls(prod, sharp):
    """a bf16 pass judged against emu built for fp16, and block l fed x_{l-1}: both must miss the criterion"""
    path = sharp("tiny", "q4_0")
    om = TokenOracle(path)
    imgs = sg.synth_images(2, om.image_size, 5)
    ids = text_ids(3)
    with Ctx(prod, path) as ctx:
        xi = prod.image_tokens_layers(ctx, imgs, [4, 5, 6], None, 0)
        xt = prod.text_tokens_layers(ctx, ids, [4, 5, 6], None, 0)
    for tower, x, lens, causal in (("v", xi, [(om.image_size // om.patch) ** 2 + 1] * 2, False), ("t", xt, [77] * 3, True)):
        ok = check(om, tower, 5, x[1], x[2], lens, causal, True, "control: right operand")
        wrong_op = check(om, tower, 5, x[1], x[2], lens, causal, False, "control: emu at fp16, GPU at bf16")
        stale = check(om, tower, 5, x[0], x[2], lens, causal, True, "control: x_{l-1} fed to block l")
        assert ok <= C and wrong_op > C and stale > C, (tower, ok, wrong_op, stale)
