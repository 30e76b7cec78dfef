"""Pins the CPU oracle against the golden embeddings the reference produced for bigg-w1664 (tests/golden/make_golden_bigg.py): the bigG
vision layer, head_dim 104 with the 1/sqrt(104) query scale, ff 8192, GELU, at the huge tensor counts.  Same bounds as
tests/test_oracle_pin.py: 1e-5 for f16, 5e-4 for the quantized types.  Needs no GPU."""
import numpy as np
import pytest

import oracle as orc
import synth_gguf as sg
from _util import check_sha, golden, model_file, one_minus_cos, token_seqs
from test_oracle_pin_huge import PIN_TOL


@pytest.mark.parametrize("ft", sorted(PIN_TOL))
def test_oracle_matches_reference_golden_bigg_w1664(prod, ft):
    g = golden("bigg-w1664")
    path = model_file("bigg-w1664", ft, prod)
    check_sha(path, g["sha_" + ft])
    m = orc.OracleModel(path)
    imgs = sg.synth_images(int(g["n_img"]), sg.GEOMETRIES["bigg-w1664"].image_size, int(g["img_seed"]))
    seqs = token_seqs(int(g["n_txt"]), int(g["tok_seed"]))
    oi = np.stack([m.encode_image(im) for im in imgs])
    ot = np.stack([m.encode_text(s) for s in seqs])
    print("%s: image 1-cos %.2e, text 1-cos %.2e" % (ft, one_minus_cos(oi, g["img_" + ft]).max(), one_minus_cos(ot, g["txt_" + ft]).max()))
    assert one_minus_cos(oi, g["img_" + ft]).max() <= PIN_TOL[ft]
    assert one_minus_cos(ot, g["txt_" + ft]).max() <= PIN_TOL[ft]
