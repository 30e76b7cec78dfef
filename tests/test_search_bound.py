"""The score bound of tests/_search_bound.py, checked without a GPU: it holds for a numpy emulation of K10's arithmetic (fp32
accumulation in k16 steps, each step truncated) at every dim the GPU test uses and both 16-bit types; and it is tight enough to
reject two wrong results -- scores rounded to bf16, and a dot product missing its last k16 step."""
import numpy as np
import pytest

from _search_bound import bound, emulate, exact, exceed, round16, unit_rows

DIMS = [8, 40, 128, 768, 2048]


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("bf", [0, 1])
def test_bound_holds_for_the_emulation(dim, bf):
    rng = np.random.default_rng(dim + bf)
    q, x = unit_rows(rng, 6, dim, bf), unit_rows(rng, 300, dim, bf)
    x[:4] = q[:4]                                      # scores near 1 next to scores near 0
    assert exceed(emulate(q, x), exact(q, x), bound(q, x)) <= 1.0


@pytest.mark.parametrize("dim", [128, 768, 2048])
def test_bound_rejects_bf16_rounded_scores(dim):
    rng = np.random.default_rng(3)
    q, x = unit_rows(rng, 6, dim, 0), unit_rows(rng, 300, dim, 0)
    x[:4] = q[:4]
    ref = exact(q, x)
    assert exceed(round16(ref.astype(np.float32), 1), ref, bound(q, x)) > 1.0


@pytest.mark.parametrize("dim", DIMS)
def test_bound_rejects_a_dropped_last_step(dim):
    rng = np.random.default_rng(5)
    q, x = unit_rows(rng, 6, dim, 1), unit_rows(rng, 300, dim, 1)
    assert exceed(emulate(q, x, drop_last=True), exact(q, x), bound(q, x)) > 1.0
