"""The position-table resample of the *_hw entry points (K8) against HF's interpolate_pos_encoding, on the CPU.

pos_resample_ref is the fp64 restatement of K8's arithmetic, operation for operation (the GPU tests hold K8 to it bit for bit).
Here it is checked against tables that torch resampled (tests/golden/make_pos_resample_golden.py: F.interpolate(..., mode="bicubic",
align_corners=False), as HF does).  Torch evaluates the same formula in fp32, so the two agree within a bound derived from fp32
rounding of torch's coordinates, weights and sums, not bit for bit."""
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pos_resample_torch.npz")
A = -0.75
U = 2.0 ** -24          # unit roundoff of fp32


def cubic_taps(g, go):
    """per output index o of an axis g -> go: 4 clamped source indices [4, go] and 4 weights [4, go] (fp64), as K8 computes them"""
    o = np.arange(go, dtype=np.float64)
    src = (g / float(go)) * (o + 0.5) - 0.5             # not clamped (torch: area_pixel_compute_source_index, cubic)
    fi = np.floor(src)
    t = src - fi
    s = 1.0 - t

    def cc1(x):
        return ((A + 2) * x - (A + 3)) * x * x + 1

    def cc2(x):
        return ((A * x - 5 * A) * x + 8 * A) * x - 4 * A

    w = np.stack([cc2(t + 1.0), cc1(t), cc1(s), cc2(s + 1.0)])
    idx = np.stack([np.clip(fi.astype(np.int64) - 1 + k, 0, g - 1) for k in range(4)])
    return idx, w


def pos_resample_ref(table, g, gh, gw, keep64=False):
    """table [g*g, h] float32 -> [gh*gw, h]: each source row interpolated horizontally ((p0 w0 + p1 w1) + p2 w2) + p3 w3, then the
    four rows vertically in the same order, in fp64 (numpy never contracts a * b + c), rounded once to float32"""
    h = table.shape[1]
    t3 = np.asarray(table, np.float64).reshape(g, g, h)
    iy, wy = cubic_taps(g, gh)
    ix, wx = cubic_taps(g, gw)
    acc = None
    for j in range(4):
        rows = t3[iy[j]]                                # [gh, g, h]
        r = rows[:, ix[0]] * wx[0][None, :, None]
        for k in range(1, 4):
            r = r + rows[:, ix[k]] * wx[k][None, :, None]
        term = r * wy[j][:, None, None]
        acc = term if acc is None else acc + term
    acc = acc.reshape(gh * gw, h)
    return acc if keep64 else acc.astype(np.float32)


def torch_bound(table, g, gh, gw):
    """|torch - exact| + |ref - exact| per element.  Torch works in fp32:
      * source coordinate scale * (o + 0.5) - 0.5 with scale = fl(g / go): three roundings of values below g + 1, so
        |d src| <= 3 u (g + 1); t = src - floor(src) is then exact;
      * weights: the cubic polynomials have |w'| <= 1.5 on their intervals, and their fp32 evaluation makes at most 6 roundings of
        intermediates below 10, each carried through at most two products by |x| <= 2: |d w| <= 1.5 |d src| + 240 u;
      * the 16 products and 15 sums: at most 18 u sum |p| |wx| |wy|, with the perturbed weights;
    the restatement's own error is its final rounding, u |ref|."""
    h = table.shape[1]
    t3 = np.abs(np.asarray(table, np.float64)).reshape(g, g, h)
    iy, wy = cubic_taps(g, gh)
    ix, wx = cubic_taps(g, gw)
    dw_y = 1.5 * 3 * U * (g + 1) + 240 * U
    dw_x = dw_y
    s_exact = np.zeros((gh, gw, h))
    s_pert = np.zeros((gh, gw, h))
    for j in range(4):
        for k in range(4):
            p = t3[iy[j]][:, ix[k]]                         # [gh, gw, h]
            ay, ax = np.abs(wy[j])[:, None, None], np.abs(wx[k])[None, :, None]
            s_exact += p * ay * ax
            s_pert += p * ((ay + dw_y) * (ax + dw_x) - ay * ax)
    ref = np.abs(pos_resample_ref(table, g, gh, gw, keep64=True)).reshape(gh, gw, h)
    return (18 * U * (s_exact + s_pert) + s_pert + U * ref).reshape(gh * gw, h)


def golden_cases():
    z = np.load(GOLDEN)
    return sorted({k[:-3] for k in z.files if k.endswith("_in")})


@pytest.mark.parametrize("name", golden_cases())
def test_restatement_matches_torch(name):
    z = np.load(GOLDEN)
    g, gh, gw = (int(v) for v in z[name + "_shape"])
    table, want = z[name + "_in"], z[name + "_out"]
    got = pos_resample_ref(table, g, gh, gw)
    assert got.shape == want.shape == (gh * gw, table.shape[1])
    err = np.abs(got.astype(np.float64) - want)
    bound = torch_bound(table, g, gh, gw)
    assert (err <= bound).all(), (name, float((err / bound).max()))
    if (g, gh, gw) == (g, g, g):                        # identity: all weight on the centre tap, exactly
        assert np.array_equal(got, table)
    # in units of u times the table's largest output (per-element ulps mean little where a sum cancels towards zero)
    print("%s: max |ref - torch| / bound %.3f, = %.1f u max|out|" % (name, float((err / bound).max()), float(err.max() / (U * np.abs(want).max()))))


def test_bound_rejects_other_interpolations():
    """The bound is far tighter than the differences between interpolation choices: align_corners=True, the Keys A = -0.5 cubic
    (PIL's) and a bilinear table all leave it on the up-sampling case."""
    z = np.load(GOLDEN)
    g, gh, gw = (int(v) for v in z["up_7_12_shape"])
    table, want = z["up_7_12_in"], z["up_7_12_out"]
    bound = torch_bound(table, g, gh, gw)
    global A
    a0 = A
    try:
        A = -0.5
        other = pos_resample_ref(table, g, gh, gw)
    finally:
        A = a0
    assert (np.abs(other.astype(np.float64) - want) > bound).any()
    # bilinear, align_corners = False
    t3 = table.astype(np.float64).reshape(g, g, -1)

    def lin(go):
        src = np.clip((g / go) * (np.arange(go) + 0.5) - 0.5, 0, None)
        i0 = np.minimum(np.floor(src).astype(int), g - 1)
        return i0, np.minimum(i0 + 1, g - 1), src - i0

    y0, y1, ty = lin(gh)
    x0, x1, tx = lin(gw)
    rows = t3[y0] * (1 - ty)[:, None, None] + t3[y1] * ty[:, None, None]
    bil = (rows[:, x0] * (1 - tx)[None, :, None] + rows[:, x1] * tx[None, :, None]).reshape(gh * gw, -1)
    assert (np.abs(bil - want) > bound).any()


def test_weights_sum_to_one():
    for g, go in ((7, 12), (16, 7), (16, 24), (4, 3), (7, 1), (24, 32)):
        _, w = cubic_taps(g, go)
        assert np.allclose(w.sum(0), 1.0, rtol=0, atol=1e-15), (g, go)
