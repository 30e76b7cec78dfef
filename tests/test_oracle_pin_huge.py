"""Pins the CPU oracle against the golden embeddings the reference produced for huge-w640 (tests/golden/make_golden_huge.py): the huge
tensor counts, a head_dim 80 vision tower (640 / 8) with the 1/sqrt(80) query scale, and GELU.  Same bounds as
tests/test_oracle_pin.py: 1e-5 for f16, 5e-4 for the quantized types.  Needs no GPU."""
import numpy as np
import pytest

import oracle as orc
import synth_gguf as sg
from _util import check_sha, golden, model_file, one_minus_cos, token_seqs

PIN_TOL = {"f16": 1e-5, "q4_0": 5e-4}


@pytest.mark.parametrize("ft", ["f16", "q4_0"])
def test_oracle_matches_reference_golden_huge_w640(prod, ft):
    g = golden("huge-w640")
    path = model_file("huge-w640", ft, prod)
    check_sha(path, g["sha_" + ft])
    m = orc.OracleModel(path)
    imgs = sg.synth_images(int(g["n_img"]), sg.GEOMETRIES["huge-w640"].image_size, int(g["img_seed"]))
    seqs = token_seqs(int(g["n_txt"]), int(g["tok_seed"]))
    oi = np.stack([m.encode_image(im) for im in imgs])
    ot = np.stack([m.encode_text(s) for s in seqs])
    assert one_minus_cos(oi, g["img_" + ft]).max() <= PIN_TOL[ft]
    assert one_minus_cos(ot, g["txt_" + ft]).max() <= PIN_TOL[ft]
