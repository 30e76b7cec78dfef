"""ViT-H/14 models end to end through the C ABI: a vision tower with head_dim 80 (1280 / 16) next to a head_dim 64 text tower,
against golden vectors the reference produced (tests/golden/make_golden_huge.py).  huge-w640 has the huge tensor counts (32 vision and
24 text layers, 909 tensors) at width 640 with 8 heads; vit-h14 is the true LAION geometry.  Tolerances are BASELINE.json's."""
import numpy as np
import pytest

import synth_gguf as sg
from _util import TOL, check_sha, golden, model_file, one_minus_cos, token_seqs

pytestmark = pytest.mark.gpu


def check_golden_parity(prod, geom, ft):
    """Both towers of (geom, ft) through the C ABI against the golden vectors at the BASELINE tolerance TOL[ft]: batch image and
    text encodes, unit norms, and the first image encoded on its own equal to its row of the batch."""
    g = golden(geom)
    assert g is not None and ("img_" + ft) in g, "golden fixture missing for %s/%s" % (geom, ft)
    path = model_file(geom, ft, prod)
    check_sha(path, g["sha_" + ft])
    imgs = sg.synth_images(int(g["n_img"]), sg.GEOMETRIES[geom].image_size, int(g["img_seed"]))
    seqs = token_seqs(int(g["n_txt"]), int(g["tok_seed"]))
    ctx = prod.load(path, 0)
    try:
        got_i = prod.image_batch_encode(ctx, imgs)
        got_t = prod.text_batch_encode(ctx, seqs)
        single = prod.image_encode(ctx, imgs[0])
    finally:
        prod.free(ctx)
    di, dt = one_minus_cos(got_i, g["img_" + ft]), one_minus_cos(got_t, g["txt_" + ft])
    print("%s %s  image 1-cos max %.2e  text 1-cos max %.2e" % (geom, ft, di.max(), dt.max()))
    assert np.isfinite(got_i).all() and np.isfinite(got_t).all()
    assert di.max() <= TOL[ft], (geom, ft, di)
    assert dt.max() <= TOL[ft], (geom, ft, dt)
    assert np.abs(np.linalg.norm(got_i, axis=1) - 1).max() < 1e-4
    assert one_minus_cos(single, got_i[0]) < 1e-6


@pytest.mark.parametrize("ft", ["f16", "q4_0", "q5_1", "q8_0"])
def test_huge_w640(prod, ft):
    check_golden_parity(prod, "huge-w640", ft)


@pytest.mark.slow
@pytest.mark.parametrize("ft", ["f16", "q4_0", "q8_0"])
def test_vit_h14_true_geometry(prod, ft):
    check_golden_parity(prod, "vit-h14", ft)


def test_head_dim_88_is_refused(prod, tmp_path):
    """ViT-g/14 has head_dim 88 (1408 / 16); a small file with that head_dim is refused at load with a message naming 64 and 80"""
    geo = sg.Geometry("hd88", image_size=64, patch_size=16, v_hidden=704, v_ff=256, v_heads=8, v_layers=1,
                      t_hidden=128, t_ff=256, t_heads=2, t_layers=1, proj_dim=128)
    path = str(tmp_path / "hd88.gguf")
    sg.write_model(path, geo, 1, 1)
    assert prod.lib.clip_model_load(path.encode(), 0) is None
    err = prod.last_error()
    assert "vision tower" in err and "head_dim must be 64 or 80" in err, err


def test_legacy_attention_refuses_head_dim_80(prod, monkeypatch):
    """the mma.sync kernel (CLIP_B200_ATTN=legacy) is head_dim 64 only: with a head_dim 80 tower the load fails instead of
    computing a wrong result"""
    path = model_file("huge-w640", "q4_0", prod)
    monkeypatch.setenv("CLIP_B200_ATTN", "legacy")
    assert prod.lib.clip_model_load(path.encode(), 0) is None
    err = prod.last_error()
    assert "legacy" in err and "head_dim 64 only" in err, err
