"""The row kernels of csrc/kernels.cu (LayerNorm, pre-LN assembly, im2col, text embedding, row gather, L2 norm, fill_last), each
run alone through its C-ABI test hook and compared with a plain fp64 (or exact) numpy restatement.

Every bound is derived from the rounding points the kernel declares.  u = 2^-24 is the fp32 unit roundoff; a sum of n fp32
terms evaluated as a tree of depth d is off by at most d * u * sum|terms|.  The LayerNorm kernels sum a row as: float4 pair sums
(depth 2), one running sum per lane over its ceil(h / 128) float4s, and a 5-level warp butterfly -- depth 7 + ceil(h / 128)."""
import ctypes as C

import numpy as np
import pytest

from _util import LN_KIND_SCALE, LN_KINDS, ln_ref64, ln_rows

pytestmark = pytest.mark.gpu

FP = C.POINTER(C.c_float)
I32P = C.POINTER(C.c_int32)
U = 2.0 ** -24


def _p(a, t=FP):
    return None if a is None else a.ctypes.data_as(t)


def round16(a, bf16):
    """fp32 -> fp16 / bf16 -> fp32, round to nearest even (like __float2half_rn / __float2bfloat16_rn)"""
    a = np.asarray(a, np.float32)
    if not bf16:
        return a.astype(np.float16).astype(np.float32)
    u = a.view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) >> 16 << 16
    return u.astype(np.uint32).view(np.float32)


def ulp16(m, bf16):
    """spacing of the 16-bit format at magnitude m (subnormal spacing below the smallest normal)"""
    emin, mant = (-126, 7) if bf16 else (-14, 10)
    e = np.floor(np.log2(np.maximum(np.abs(m), 2.0 ** emin)))
    return 2.0 ** (e - mant)


def ln_bound(xh, rstd, mean_abs, gamma, beta, h, extra_roundings=0):
    """s: how far the kernel's fp32 LayerNorm value may be from the fp64 one, element by element.
      mean: a depth-d sum and the division by h -> |dmu| <= (d + 1 + extra) u mean|x|; it shifts x_hat by rstd*dmu and adds
            dmu^2 to the variance (relative error (rstd*dmu)^2 / 2 in rstd).
      rstd: x - mean (1 rounding), the depth-d centred sum of squares (d + 2), / h and + eps (2), rsqrtf (2 ulp <= 4u), halved by
            the square root except rsqrtf's own error: <= (d/2 + 6) u relative.
      out:  (x - mean) * rstd * gamma + beta: three more roundings relative to |gamma x_hat| and one relative to |beta|.
    So s = u ((d/2 + 10) |gamma x_hat| + |beta|) + |gamma| rstd dmu + (rstd dmu)^2 / 2 |gamma x_hat|.  For a standard normal row at
    h = 2048 this is ~1.3e-6 relative: a few dozen fp32 ulps, far below half a 16-bit ulp.  On the offset rows (|mean| / std = 1e5)
    the mean term dominates -- an fp32 mean of values near 1e3 cannot be closer than ~1e-4 -- and those rows get a second check
    that does not depend on the mean."""
    d = 7 + -(-h // 128) + extra_roundings
    dmu = (d + 1) * U * mean_abs
    gx = np.abs(gamma * xh)
    return U * ((d / 2 + 10) * gx + np.abs(beta)) + np.abs(gamma) * rstd * dmu + 0.5 * (rstd * dmu) ** 2 * gx


def spread_error(y, x, gamma, beta, eps):
    """Relative error of the spread of z = (y - beta) / gamma on a row, checked without trusting the kernel's mean.  With the
    kernel's mean off by dmu, z = (x - mean - dmu) * r with r = 1 / sqrt(var + dmu^2 + eps) (the centred sum of squares picks up
    dmu^2).  So mean(z) = m = -dmu r and std(z) = sqrt(var) r, and eliminating dmu and r:  std(z)^2 = var (1 - m^2) / (var + eps).
    A wrong variance (one-pass cancellation, a lost eps) breaks this identity whatever dmu is."""
    z = (y.astype(np.float64) - beta) / gamma
    var = x.astype(np.float64).var()
    want = np.sqrt(var * (1 - z.mean() ** 2) / (var + float(np.float32(eps))))
    return abs(z.std() / want - 1)


def run_layernorm(prod, x, gamma, beta, eps, bf16, in_stride=None, delta=None):
    rows, h = x.shape
    y = np.empty((rows, h), np.float32)
    xo = np.empty((rows, h), np.float32)
    rc = prod.lib.clip_b200_debug_layernorm(rows, h, in_stride or h, eps, _p(x), _p(gamma), _p(beta), _p(delta), int(bf16),
                                            _p(y), _p(xo))
    assert rc == 0, prod.last_error()
    return y, xo


def affine(rng, h):
    """gamma and beta drawn per column, so that a column or lane mix-up shows"""
    return ((1.0 + 0.3 * rng.standard_normal(h)).astype(np.float32),
            (0.5 * rng.standard_normal(h)).astype(np.float32))


def check_layernorm(y, x, kinds, gamma, beta, eps, bf16, tag):
    xh, rstd, mean_abs = ln_ref64(x, eps)
    g, b = gamma.astype(np.float64), beta.astype(np.float64)
    ref = g * xh + b
    s = ln_bound(xh, rstd, mean_abs, g, b, x.shape[1])
    # the output is ONE round-to-nearest of an fp32 value within s of ref
    tol = 0.5 * ulp16(np.abs(ref) + s, bf16) + s
    err = np.abs(y.astype(np.float64) - ref)
    bad = ~(err <= tol)
    assert not bad.any(), (tag, sorted({kinds[r] for r in np.nonzero(bad)[0]}), float(np.nanmax(err / tol)), int(bad.sum()))
    # constant dyadic rows: every partial sum is exact, x - mean is 0, so the output is exactly beta rounded once
    for r, k in enumerate(kinds):
        if k.startswith("const"):
            assert np.array_equal(y[r], round16(beta, bf16)), (tag, k)
    # rows whose mean is well conditioned: nearly every element is the correctly rounded fp64 value
    well = np.array([k != "offset" for k in kinds])
    if well.any():
        exact = (y[well] == round16(ref[well].astype(np.float32), bf16)).mean()
        assert exact >= 0.99, (tag, exact)
    # offset rows: the spread identity, up to the 16-bit rounding of y -- independent errors of at most half an ulp, which
    # move the standard deviation of a unit-spread row by far less than one ulp at 1 (the bound used)
    for r, k in enumerate(kinds):
        if k == "offset":
            e = spread_error(y[r], x[r], g, b, eps)
            assert e <= ulp16(1.0, bf16), (tag, r, e)
    # how much of s the error uses beyond the 16-bit rounding itself
    return float(((err - 0.5 * ulp16(np.abs(ref) + s, bf16)) / s).max())


LN_WIDTHS = [128, 384, 512, 640, 1024, 1152, 1280, 1664, 2048]     # MAXV 4 | 8 | 16, full and partial lanes
LN_ROWS = [1, 7, 8, 9, 1031]                                        # 8 rows (warps) per block, walked last row first


@pytest.mark.parametrize("delta", [False, True], ids=["plain", "delta"])
@pytest.mark.parametrize("bf16", [False, True], ids=["f16", "bf16"])
@pytest.mark.parametrize("strided", [False, True], ids=["dense", "stride257"])
@pytest.mark.parametrize("rows", LN_ROWS)
@pytest.mark.parametrize("h", LN_WIDTHS)
def test_layernorm(prod, h, rows, strided, bf16, delta):
    """in_stride = h (ln1 / ln2), or T*h with T = 257 (the CLS-row post-LN reads row 0 of each sequence); the gaps between
    strided rows are poisoned, so a read outside the row turns into NaN.  The delta form first adds a 16-bit branch into x
    and writes x back: bit-exact against x + float(delta16) in fp32."""
    rng = np.random.default_rng(h * 7919 + rows)
    x, kinds = ln_rows(rows, h, rng, first=h + rows)
    gamma, beta = affine(rng, h)
    d = None
    if delta:
        # per row: noise at the row's own scale (constant rows get a dyadic constant and stay constant)
        d = np.stack([np.full(h, 0.25) if LN_KIND_SCALE[k] == 0 else LN_KIND_SCALE[k] * rng.standard_normal(h) for k in kinds])
        d = d.astype(np.float32)
    y, xo = run_layernorm(prod, x, gamma, beta, 1e-5, bf16, 257 * h if strided else h, d)
    x_new = x if d is None else (x + round16(d, bf16)).astype(np.float32)
    assert np.array_equal(xo.view(np.uint32), x_new.view(np.uint32))
    ratio = check_layernorm(y, x_new, kinds, gamma, beta, 1e-5, bf16, (h, rows, strided, bf16, delta))
    print("layernorm h=%d rows=%d (err - half ulp16)/s %.3f" % (h, rows, ratio))


@pytest.mark.parametrize("bf16", [False, True], ids=["f16", "bf16"])
@pytest.mark.parametrize("h", LN_WIDTHS)
def test_layernorm_eps_1e6(prod, h, bf16):
    """eps = 1e-6 (the eps_scale rows now have variance ~9 eps): eps must enter exactly once, under the square root"""
    rng = np.random.default_rng(h + 17)
    x, kinds = ln_rows(2 * len(LN_KINDS), h, rng)
    gamma, beta = affine(rng, h)
    y, _ = run_layernorm(prod, x, gamma, beta, 1e-6, bf16)
    ratio = check_layernorm(y, x, kinds, gamma, beta, 1e-6, bf16, (h, bf16))
    print("layernorm eps=1e-6 h=%d (err - half ulp16)/s %.3f" % (h, ratio))


# ---- pre-LN assembly -------------------------------------------------------------------------------------------------------

def run_preln(prod, patch, cls, pos, B, T, eps, gamma, beta):
    h = cls.size
    x = np.empty((B * T, h), np.float32)
    rc = prod.lib.clip_b200_debug_assemble_preln(_p(patch), _p(cls), _p(pos), B, T, h, eps, _p(gamma), _p(beta), _p(x))
    assert rc == 0, prod.last_error()
    return x


def preln_inputs(rng, B, T, h):
    patch, kinds = ln_rows(B * (T - 1), h, rng, first=T)
    cls = (0.3 + 0.5 * rng.standard_normal(h)).astype(np.float32)
    pos = (1e-3 * rng.standard_normal((T, h))).astype(np.float32)
    return patch, cls, pos, kinds


def preln_ref_input(patch, cls, pos, B, T):
    """the kernel's LN input: (class embedding | patch row) + position, one fp32 addition"""
    h = cls.size
    src = np.concatenate([cls[None, None, :].repeat(B, 0), patch.reshape(B, T - 1, h)], axis=1)
    return (src + pos[None]).astype(np.float32).reshape(B * T, h)


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("h", [128, 1024, 1280, 2048])
@pytest.mark.parametrize("T", [17, 50, 257, 577])
def test_assemble_preln(prod, T, h, B):
    """fp32 output: within s (ln_bound, with the two extra roundings of this kernel's mean = sum * fl(1/h)) of the fp64 LN of
    (cls | patch) + pos.  s is below 1e-5 (|gamma x_hat| + |beta|) except on the offset rows, which also get the spread check."""
    rng = np.random.default_rng(T * 31 + h + B)
    patch, cls, pos, kinds = preln_inputs(rng, B, T, h)
    gamma, beta = affine(rng, h)
    x = run_preln(prod, patch, cls, pos, B, T, 1e-5, gamma, beta)
    xin = preln_ref_input(patch, cls, pos, B, T)
    xh, rstd, mean_abs = ln_ref64(xin, 1e-5)
    g, b = gamma.astype(np.float64), beta.astype(np.float64)
    ref = g * xh + b
    s = ln_bound(xh, rstd, mean_abs, g, b, h, extra_roundings=2)
    err = np.abs(x - ref)
    assert (err <= s).all(), (T, h, B, float(np.nanmax(err / s)))
    print("assemble_preln T=%d h=%d B=%d err/bound %.3f" % (T, h, B, float((err / s).max())))
    rows_kind = [None if t == 0 else kinds[bb * (T - 1) + t - 1] for bb in range(B) for t in range(T)]
    # offset rows: fp32 output, so the spread identity holds to the variance's own rounding, (d/2 + 6) u ~ 1e-6
    for r, k in enumerate(rows_kind):
        if k == "offset":
            e = spread_error(x[r], xin[r], g, b, 1e-5)
            assert e <= 1e-5, (T, h, B, r, e)


def test_assemble_preln_class_row(prod):
    """row 0 of every image is LN(class_embd + pos[0]), not LN(patch[0] + pos[0]); rows t >= 1 take patch t - 1"""
    rng = np.random.default_rng(5)
    B, T, h = 2, 17, 1280
    patch, cls, pos, _ = preln_inputs(rng, B, T, h)
    gamma, beta = affine(rng, h)
    x = run_preln(prod, patch, cls, pos, B, T, 1e-5, gamma, beta).reshape(B, T, h)
    for bb in range(B):
        want_cls = gamma * ln_ref64(cls[None] + pos[:1], 1e-5)[0][0] + beta
        wrong = gamma * ln_ref64(patch[bb * (T - 1)][None] + pos[:1], 1e-5)[0][0] + beta
        assert np.abs(x[bb, 0] - want_cls).max() <= 1e-4
        assert np.abs(x[bb, 0] - wrong).max() > 0.1
        assert np.abs(x[bb, 1] - (gamma * ln_ref64(patch[bb * (T - 1)][None] + pos[1:2], 1e-5)[0][0] + beta)).max() <= 1e-4


# ---- im2col ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("S,P,B", [(224, 14, 8), (224, 32, 8), (64, 16, 96), (112, 14, 32)])
def test_im2col(prod, S, P, B):
    """bit-exact: NHWC pixels -> k = c P^2 + ky P + kx -> fp16 round-to-nearest-even, zeros in the padding columns up to kpad.
    Each B puts the total past the launcher's grid-stride cap (132 * 32 blocks of 256), so every thread walks more than one
    element.  The pixels are uniform fp32 draws with all mantissa bits live, so truncation would differ from RN."""
    K = 3 * P * P
    kpad = -(-K // 64) * 64
    n = S // P
    assert B * n * n * kpad > 132 * 32 * 256
    rng = np.random.default_rng(S + P)
    px = (rng.random((B, S, S, 3), dtype=np.float32) * np.float32(4.0) - np.float32(2.0))
    out = np.empty((B * n * n, kpad), np.float32)
    rc = prod.lib.clip_b200_debug_im2col(_p(px), B, S, P, kpad, _p(out))
    assert rc == 0, prod.last_error()
    cols = px.reshape(B, n, P, n, P, 3).transpose(0, 1, 3, 5, 2, 4).reshape(B * n * n, K)
    want = np.zeros((B * n * n, kpad), np.float32)
    want[:, :K] = cols.astype(np.float16).astype(np.float32)
    assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), (S, P, int((out != want).sum()))


# ---- text embedding, gather, fill_last, L2 norm --------------------------------------------------------------------------------

@pytest.mark.parametrize("h", [128, 768, 1280])
def test_text_embed(prod, h):
    """bit-exact pos + tok in fp32; ids -5 and n_vocab + 3 are clamped to 0 and n_vocab - 1"""
    rng = np.random.default_rng(h)
    nseq, T, n_vocab = 3, 77, 1000
    ids = rng.integers(0, n_vocab, (nseq, T)).astype(np.int32)
    ids[0, 3], ids[1, 0], ids[2, 76], ids[2, 5] = -5, n_vocab + 3, n_vocab - 1, 0
    tok = rng.standard_normal((n_vocab, h)).astype(np.float32)
    pos = rng.standard_normal((T, h)).astype(np.float32)
    x = np.empty((nseq * T, h), np.float32)
    rc = prod.lib.clip_b200_debug_text_embed(_p(ids, I32P), _p(tok), _p(pos), nseq, T, h, n_vocab, _p(x))
    assert rc == 0, prod.last_error()
    want = (tok[np.clip(ids, 0, n_vocab - 1)] + pos[None]).astype(np.float32).reshape(nseq * T, h)
    assert np.array_equal(x.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("bf16", [False, True], ids=["f16", "bf16"])
@pytest.mark.parametrize("with_delta", [False, True], ids=["plain", "delta"])
@pytest.mark.parametrize("with_offs", [False, True], ids=["stride", "offsets"])
def test_gather_rows(prod, with_offs, with_delta, bf16):
    """bit-exact: out[r] = src[r * stride_rows + offs[r]] (+ float(delta16) of that row, in fp32)"""
    rng = np.random.default_rng(int(with_offs) * 4 + int(with_delta) * 2 + int(bf16))
    nseq, T, h = 13, 77, 1280
    src = rng.standard_normal((nseq * T, h)).astype(np.float32)
    offs = rng.integers(0, T, nseq).astype(np.int32) if with_offs else None
    if with_offs:
        offs[0], offs[-1] = 0, T - 1
    delta = rng.standard_normal((nseq * T, h)).astype(np.float32) if with_delta else None
    out = np.empty((nseq, h), np.float32)
    rc = prod.lib.clip_b200_debug_gather_rows(_p(src), nseq * T, nseq, h, T, _p(offs, I32P), _p(delta), int(bf16), _p(out))
    assert rc == 0, prod.last_error()
    idx = np.arange(nseq) * T + (offs if with_offs else 0)
    want = src[idx] if delta is None else (src[idx] + round16(delta[idx], bf16)).astype(np.float32)
    assert np.array_equal(out.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("with_lens", [False, True])
def test_fill_last(prod, with_lens):
    """exact: clamp(lens ? lens[i] : seq_len, 1, seq_len) - 1, over more than one block of 256"""
    n, seq_len = 300, 77
    rng = np.random.default_rng(0)
    lens = None
    if with_lens:
        lens = rng.integers(-100, 200, n).astype(np.int32)
        lens[:7] = [0, 1, seq_len, seq_len + 5, -1, -(2 ** 31), 2 ** 31 - 1]
    last = np.empty(n, np.int32)
    assert prod.lib.clip_b200_debug_fill_last(_p(lens, I32P), n, seq_len, _p(last, I32P)) == 0, prod.last_error()
    want = np.clip(lens if with_lens else np.full(n, seq_len), 1, seq_len) - 1
    assert np.array_equal(last, want)


@pytest.mark.parametrize("d", [128, 512, 768, 1024, 1280])
def test_l2norm(prod, d):
    """normalize = 0 is a bit-exact copy.  normalize = 1: the sum of squares is a positive sum with ~(d/32 + 5) roundings, whose
    relative error is halved by the square root; 1/sqrt and the product add one rounding each.  Across the few rows here the
    observed error stays well inside 4 fp32 ulps of the fp64 result.  Rows span 1e-3 .. 1e3; there is no eps by design, so no
    all-zero row."""
    rng = np.random.default_rng(d)
    scales = np.array([1e-3, 1.0, 1e3, 3e-3, 7e2, 1.0, 0.5, 2e-3, 5e2, 1.0, 1e-3])
    v = (rng.standard_normal((scales.size, d)) * scales[:, None]).astype(np.float32)
    out = np.empty_like(v)
    assert prod.lib.clip_b200_debug_l2norm(_p(v), v.shape[0], d, 0, _p(out)) == 0, prod.last_error()
    assert np.array_equal(out.view(np.uint32), v.view(np.uint32))
    assert prod.lib.clip_b200_debug_l2norm(_p(v), v.shape[0], d, 1, _p(out)) == 0, prod.last_error()
    v64 = v.astype(np.float64)
    ref = v64 / np.sqrt((v64 * v64).sum(-1, keepdims=True))
    ulps = np.abs(out - ref) / np.spacing(np.abs(ref).astype(np.float32))
    assert ulps.max() <= 4, (d, float(ulps.max()))
    print("l2norm d=%d max ulps %.2f" % (d, float(ulps.max())))
