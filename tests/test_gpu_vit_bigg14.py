"""ViT-bigG/14 models end to end through the C ABI: a vision tower with head_dim 104 (1664 / 16), whose QKV projection the loader pads
to 112 columns per head, next to a head_dim 64 text tower.  bigg-w1664 has the bigG vision layer (1664 wide, ff 8192, 257 positions,
GELU) at the huge tensor counts (909 tensors), so its golden vectors come from the reference itself (tests/golden/make_golden_bigg.py);
vit-bigg14 is the true LAION geometry (48 vision layers, a 1280-wide text tower of 20 heads over 32 layers, projection 1280), which the
reference refuses, so its golden vectors come from the CPU oracle (tests/golden/make_golden_bigg_oracle.py), pinned against the
reference on bigg-w1664 (tests/test_oracle_pin_bigg.py).  Tolerances are BASELINE.json's.  On its f16 file, the per-token paths against the CPU oracle: hidden rows of layer -2 without the
CLS row, the projected CLS rows bit for bit against the pooled call, an ATTENTION entry and its CLS row, and one _hw call at 336 x 336."""
import numpy as np
import pytest

import binding as bd
import synth_gguf as sg
from _oracle_attn import AttnOracle
from _util import TOL, golden, model_file, one_minus_cos
from test_gpu_anyres import images
from test_gpu_tokens import Ctx, bits
from test_gpu_tokens_attention import row_cos_worst
from test_gpu_vit_h14 import check_golden_parity
from test_pos_resample import pos_resample_ref

pytestmark = pytest.mark.gpu

ATT, CLS = bd.TOKENS_ATTENTION, bd.TOKENS_ATTENTION | bd.TOKENS_ATTENTION_CLS


@pytest.mark.parametrize("ft", ["f16", "q4_0", "q5_1", "q8_0"])
def test_bigg_w1664(prod, ft):
    check_golden_parity(prod, "bigg-w1664", ft)


@pytest.mark.slow
@pytest.mark.parametrize("ft", ["f16", "q4_0"])
def test_vit_bigg14_true_geometry(prod, ft):
    assert str(golden("vit-bigg14")["producer"]).startswith("oracle/oracle.py")
    check_golden_parity(prod, "vit-bigg14", ft)


def test_bigg_w1664_token_paths_against_oracle(prod):
    g = sg.GEOMETRIES["bigg-w1664"]
    path = model_file("bigg-w1664", "f16", prod)
    om = AttnOracle(path)
    imgs = sg.synth_images(2, g.image_size, 31)
    tol = TOL["f16"]
    with Ctx(prod, path) as ctx:
        rows = prod.image_tokens(ctx, imgs[:1], -2, bd.TOKENS_NO_CLS)
        assert rows.shape == (1, g.n_pos - 1, g.v_hidden)
        d = one_minus_cos(rows[0], om.image_tokens(imgs[0], -2)[1:])
        print("tokens layer -2 NO_CLS: worst per-row 1 - cos %.2e" % d.max())
        assert d.max() <= tol

        pooled = prod.image_batch_encode(ctx, imgs)
        proj = prod.image_tokens(ctx, imgs, -1, bd.TOKENS_PROJECT | bd.TOKENS_NORMALIZE)
        assert np.array_equal(bits(proj[:, 0]), bits(pooled))

        att = prod.image_tokens(ctx, imgs[:1], -1, ATT)
        assert att.shape == (1, g.v_heads, g.n_pos, g.n_pos)
        assert np.array_equal(bits(prod.image_tokens(ctx, imgs[:1], -1, CLS)), bits(att[:, :, :1]))
        d = row_cos_worst(att[0], om.image_attention(imgs[0], -1))
        print("attention layer -1: worst per-row 1 - cos %.2e" % d)
        assert d <= tol

        S = 336
        x = images(1, S, S, 5)
        pos = om.position_table_hw(S // g.patch_size, S // g.patch_size, pos_resample_ref)
        got = prod.image_batch_encode_hw(ctx, x)
        d = one_minus_cos(got[0], om.encode_image_hw(x[0], pos))
        print("_hw 336 x 336: 1 - cos %.2e" % d)
        assert d <= tol
