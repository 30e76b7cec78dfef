"""The any-size oracle (tests/_oracle_anyres.py) at the model's own size, with the model's own table, is the pinned oracle: its rows
equal TokenOracle.image_tokens and its embedding equals encode_image, bit for bit.  CPU only."""
import numpy as np

import synth_gguf as sg
from _oracle_anyres import AnyresOracle
from test_pos_resample import pos_resample_ref


def test_native_size_is_the_pinned_oracle(tmp_path):
    path = str(tmp_path / "tiny.gguf")
    g = sg.GEOMETRIES["tiny"]
    sg.write_model(path, g, 1234, 1)
    om = AnyresOracle(path)
    img = sg.synth_images(1, g.image_size, 5)[0]
    n = g.image_size // g.patch_size
    pos = om.position_table_hw(n, n, pos_resample_ref)
    assert np.array_equal(pos, om.f32("v.position_embd.weight"))        # the identity resample is exact
    for layer in (0, 3, -1):
        assert np.array_equal(om.image_tokens_hw(img, pos, layer, True), om.image_tokens(img, layer, True)), layer
    assert np.array_equal(om.encode_image_hw(img, pos), om.encode_image(img))
    assert np.array_equal(om.encode_image_hw(img, pos, False), om.encode_image(img, False))
