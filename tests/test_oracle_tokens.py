"""CPU only: the oracle's per-token rows (tests/_oracle_tokens.py) are the rows its pooled encoders select.  The CLS row of
image_tokens(-1, post_ln) and the EOT row of text_tokens(-1, post_ln), projected (and normalised), equal encode_image / encode_text
bit for bit, so the GPU token tests compare against the same arithmetic the pinned encoders use."""
import os

import numpy as np
import pytest

import synth_gguf as sg
from _oracle_tokens import TokenOracle


@pytest.fixture(scope="module")
def tiny():
    path = sg.model_path("tiny", 1234, "f16")
    if not os.path.exists(path):
        sg.write_model(path, sg.GEOMETRIES["tiny"], 1234, 1)
    return TokenOracle(path)


@pytest.mark.parametrize("normalize", [True, False])
def test_oracle_cls_row_projected_is_encode_image(tiny, normalize):
    img = sg.synth_images(1, 64, 11)[0]
    rows = tiny.image_tokens(img, -1, post_ln=True)
    assert rows.shape == (17, 128)
    got = tiny.project_image(rows[:1], normalize)[0]
    assert np.array_equal(got.view(np.uint32), tiny.encode_image(img, normalize).view(np.uint32))


@pytest.mark.parametrize("n", [2, 9, 77])
def test_oracle_eot_row_projected_is_encode_text(tiny, n):
    ids = sg.synth_tokens(1, n, 40 + n)[0]
    rows = tiny.text_tokens(ids, -1, post_ln=True)
    got = tiny.project_text(rows[n - 1:n])[0]
    assert np.array_equal(got.view(np.uint32), tiny.encode_text(ids).view(np.uint32))


def test_oracle_layer_numbering(tiny):
    """-1 is layer n_layer, -(n_layer + 1) is layer 0 (the pre_ln output), and post_ln is a row-wise function of the raw rows"""
    img = sg.synth_images(1, 64, 12)[0]
    for a, b in ((-1, 12), (-2, 11), (-13, 0)):
        assert np.array_equal(tiny.image_tokens(img, a), tiny.image_tokens(img, b))
    raw = tiny.image_tokens(img, 3)
    assert np.array_equal(tiny.image_tokens(img, 3, post_ln=True), tiny.ln(raw, "v.post_ln.weight", "v.post_ln.bias", tiny.v_eps))
    with pytest.raises(AssertionError):
        tiny.image_tokens(img, 13)
