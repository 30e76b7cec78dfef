"""Token sequences of different lengths in one call, packed with no padding (clip_b200_text_encode_device_packed,
clip_b200_text_tokens_device_packed and the host forms clip_b200_text_batch_encode_packed / clip_b200_text_tokens_packed): rows packed
back to back into one forward pass, causal attention by K3's variable-length instance.

  1. The premise: a padded clip_text_batch_encode row equals its sequence alone at seq_len = len, byte for byte.
  2. The causal variable-length kernel (clip_b200_debug_attention_mixed_causal) equals K3's causal launch on each sequence alone,
     bit for bit, never writes its guard rows, and a sequence holding Inf / NaN leaves every other sequence's bits unchanged.
  3. Each sequence of a packed call equals that sequence alone through clip_b200_text_encode_device and clip_text_batch_encode's
     row, byte for byte, on text towers of width 128 (tiny, small-p14, huge-w640, bigg-w1664) and 1280 with 20 heads (wide-h1280).
  4. Token rows equal the first len rows of clip_b200_text_tokens_device at seq_len = len, at several layers, flags and every
     out_type; layer 0 equals numpy's tok[id] + pos[t] exactly.
  5. Order, pass boundaries, lengths 1 and context_length, a 4096-token context and the launch count of a pass.
  6. Host forms equal device forms.  7. tiny against the CPU oracle.  8. Refusals, in order.  9. Devices mode equals one GPU."""
import ctypes as C

import numpy as np
import pytest

import binding as bd
import synth_gguf as sg
from _oracle_anyres import AnyresOracle
from _util import TOL, model_file
from test_gpu_anyres import cos_rows
from test_gpu_long_sequences import LONG_CTX
from test_gpu_tokens import Ctx, bits, padded

pytestmark = pytest.mark.gpu

FP = C.POINTER(C.c_float)
IP = C.POINTER(C.c_int)
I32P = C.POINTER(C.c_int32)
OUT_TYPES = (bd.OUT_F32, bd.OUT_F16, bd.OUT_BF16)
FLAGS = [0, bd.TOKENS_POST_LN, bd.TOKENS_PROJECT, bd.TOKENS_PROJECT | bd.TOKENS_NORMALIZE]
# lengths on both sides of 8 (the padded forms' rounding) and of the 64-row query groups, 1 and context_length
LENS = [77, 1, 2, 9, 63, 64, 65, 33, 76, 16, 5, 8, 7]


def seqs_of(lens, seed):
    return [sg.synth_tokens(1, n, seed + 7 * k + n)[0] for k, n in enumerate(lens)]


class Dev:
    """device buffers of one test, freed together"""

    def __init__(self, prod, ctx):
        self.prod, self.ctx, self.ptrs = prod, ctx, []

    def up(self, a):
        a = np.ascontiguousarray(a)
        d = self.prod.lib.clip_b200_device_malloc(self.ctx, max(a.nbytes, 1))
        assert d
        self.ptrs.append(d)
        assert self.prod.lib.clip_b200_memcpy_h2d(self.ctx, d, a.ctypes.data, a.nbytes)
        return d

    def down(self, d, shape, dtype):
        out = np.empty(shape, dtype)
        assert self.prod.lib.clip_b200_memcpy_d2h(self.ctx, out.ctypes.data, d, out.nbytes)
        return out

    def __enter__(self):
        return self

    def __exit__(self, *a):
        for d in self.ptrs:
            self.prod.lib.clip_b200_device_free(self.ctx, d)


def text_width(prod, ctx, flags):
    hp = prod.text_hparams(ctx)
    return hp.projection_dim if flags & bd.TOKENS_PROJECT else hp.hidden_size


def encode_packed_dev(prod, ctx, seqs, normalize=True):
    lens = np.array([len(s) for s in seqs], np.int32)
    dim = prod.text_hparams(ctx).projection_dim
    with Dev(prod, ctx) as d:
        d_in, d_out = d.up(np.concatenate(seqs).astype(np.int32)), d.up(np.zeros((len(seqs), dim), np.float32))
        assert prod.lib.clip_b200_text_encode_device_packed(ctx, d_in, len(seqs), lens.ctypes.data_as(IP), d_out, normalize), prod.last_error()
        return d.down(d_out, (len(seqs), dim), np.float32)


def tokens_packed_dev(prod, ctx, seqs, layer, flags, ot=bd.OUT_F32):
    lens = np.array([len(s) for s in seqs], np.int32)
    shape = (int(lens.sum()), text_width(prod, ctx, flags))
    with Dev(prod, ctx) as d:
        d_in, d_out = d.up(np.concatenate(seqs).astype(np.int32)), d.up(np.zeros(shape, bd.OUT_DTYPES[ot]))
        assert prod.lib.clip_b200_text_tokens_device_packed(ctx, d_in, len(seqs), lens.ctypes.data_as(IP), layer, flags, ot, d_out), \
            prod.last_error()
        flat = d.down(d_out, shape, bd.OUT_DTYPES[ot])
    return np.split(flat, np.cumsum(lens)[:-1])


def encode_alone_dev(prod, ctx, s, normalize=True):
    dim = prod.text_hparams(ctx).projection_dim
    with Dev(prod, ctx) as d:
        d_in, d_out = d.up(np.asarray(s, np.int32)[None]), d.up(np.zeros(dim, np.float32))
        assert prod.lib.clip_b200_text_encode_device(ctx, d_in, None, 1, len(s), d_out, normalize), prod.last_error()
        return d.down(d_out, (dim,), np.float32)


def tokens_alone_dev(prod, ctx, s, layer, flags, ot=bd.OUT_F32):
    shape = (len(s), text_width(prod, ctx, flags))
    with Dev(prod, ctx) as d:
        d_in, d_out = d.up(np.asarray(s, np.int32)[None]), d.up(np.zeros(shape, bd.OUT_DTYPES[ot]))
        assert prod.lib.clip_b200_text_tokens_device(ctx, d_in, 1, len(s), layer, flags, ot, d_out), prod.last_error()
        return d.down(d_out, shape, bd.OUT_DTYPES[ot])


# ---- 1. the premise ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("ft", ["f16", "q4_0"])
def test_padded_batch_rows_equal_each_sequence_alone(prod, ft):
    seqs = seqs_of(LENS, 3)
    with Ctx(prod, model_file("tiny", ft, prod)) as ctx:
        batch = prod.text_batch_encode(ctx, seqs)
        for k, s in enumerate(seqs):
            assert np.array_equal(bits(batch[k]), bits(encode_alone_dev(prod, ctx, s))), (ft, len(s))


# ---- 2. the causal variable-length attention kernel ---------------------------------------------------------------------------

KLENS = [1, 2, 7, 8, 63, 64, 65, 76, 77, 127, 128, 129, 248, 1000]


def qkv_of(rng, rows, H, dh=64):
    return (rng.standard_normal((rows, 3 * H * dh)) * 0.5).astype(np.float32)


def hook_causal(prod, bf16, lens, H, qkv, dh=64):
    out = np.empty((sum(lens), H * dh), np.float32)
    ln = np.array(lens, np.int32)
    rc = prod.lib.clip_b200_debug_attention_mixed_causal(bf16, len(lens), ln.ctypes.data_as(IP), H, dh, qkv.ctypes.data_as(FP),
                                                         out.ctypes.data_as(FP))
    assert rc == 0, (rc, prod.last_error())         # rc 6: a guard row was written
    return out


def hook_alone(prod, bf16, T, H, qkv):
    out = np.empty((T, H * 64), np.float32)
    rc = prod.lib.clip_b200_debug_attention_hd(bf16, 1, T, H, 64, 1, 0, np.ascontiguousarray(qkv).ctypes.data_as(FP),
                                               out.ctypes.data_as(FP), None)
    assert rc == 0, (rc, prod.last_error())
    return out


@pytest.mark.parametrize("bf16", [0, 1])
def test_causal_varlen_kernel_equals_each_sequence_alone(prod, bf16):
    rng = np.random.default_rng(64 + bf16)
    H = 2
    mixes = [KLENS, list(rng.permutation(KLENS))] + [list(rng.integers(1, 300, size=int(rng.integers(2, 40)))) for _ in range(3)]
    for lens in mixes:
        lens = [int(t) for t in lens]
        qkv = qkv_of(rng, sum(lens), H)
        got = hook_causal(prod, bf16, lens, H, qkv)
        r0 = 0
        for T in lens:
            want = hook_alone(prod, bf16, T, H, qkv[r0:r0 + T])
            assert np.array_equal(bits(got[r0:r0 + T]), bits(want)), (bf16, lens, T)
            r0 += T


def test_causal_varlen_kernel_isolates_non_finite_sequences(prod):
    rng = np.random.default_rng(11)
    H = 2
    lens = [65, 129, 1, 63, 77, 2, 128, 8]
    qkv = qkv_of(rng, sum(lens), H)
    clean = hook_causal(prod, 0, lens, H, qkv)
    offs = np.concatenate([[0], np.cumsum(lens)])
    cols = H * 64
    for k in range(len(lens)):
        for part in range(3):                     # Q, K, V of sequence k
            for bad in (np.inf, -np.inf, np.nan):
                x = qkv.copy()
                x[offs[k]:offs[k + 1], part * cols:(part + 1) * cols:3] = bad
                got = hook_causal(prod, 0, lens, H, x)
                for j in range(len(lens)):
                    if j != k:
                        assert np.array_equal(bits(got[offs[j]:offs[j + 1]]), bits(clean[offs[j]:offs[j + 1]])), (k, part, bad, j)


def test_causal_varlen_hook_refuses_other_head_dims(prod):
    qkv = np.zeros((4, 3 * 80), np.float32)
    out = np.empty((4, 80), np.float32)
    ln = np.array([4], np.int32)
    assert prod.lib.clip_b200_debug_attention_mixed_causal(0, 1, ln.ctypes.data_as(IP), 1, 80, qkv.ctypes.data_as(FP),
                                                           out.ctypes.data_as(FP)) == 2
    assert "attention_mixed_causal: head_dim must be 64" in prod.last_error()


# ---- 3. and 4. each sequence against itself alone ------------------------------------------------------------------------------

GEOMS = [("tiny", "f16"), ("tiny", "q4_0"), ("small-p14", "f16"), ("huge-w640", "f16"), ("bigg-w1664", "f16"), ("wide-h1280", "f16")]


@pytest.mark.parametrize("geom,ft", GEOMS)
def test_each_sequence_equals_itself_alone(prod, geom, ft):
    seqs = seqs_of(LENS, 20)
    full = geom == "tiny"
    with Ctx(prod, model_file(geom, ft, prod)) as ctx:
        for normalize in (True, False):
            got = encode_packed_dev(prod, ctx, seqs, normalize)
            batch = prod.text_batch_encode(ctx, seqs, normalize)
            for k, s in enumerate(seqs):
                assert np.array_equal(bits(got[k]), bits(encode_alone_dev(prod, ctx, s, normalize))), (geom, ft, len(s), normalize)
                assert np.array_equal(bits(got[k]), bits(batch[k])), (geom, ft, len(s), normalize)
        for layer in ((0, 1, -2, -1) if full else (-2,)):
            for flags in FLAGS:
                for ot in OUT_TYPES:
                    got = tokens_packed_dev(prod, ctx, seqs, layer, flags, ot)
                    for k, s in enumerate(seqs):
                        want = tokens_alone_dev(prod, ctx, s, layer, flags, ot)
                        assert got[k].shape == want.shape, (geom, k, flags)
                        assert np.array_equal(bits(got[k]), bits(want)), (geom, ft, len(s), layer, flags, ot)


def test_layer_0_rows_are_token_plus_position(prod):
    path = model_file("tiny", "f16", prod)
    om = AnyresOracle(path)
    tok, pos = om.f32("t.token_embd.weight"), om.f32("t.position_embd.weight")
    seqs = seqs_of(LENS, 30)
    with Ctx(prod, path) as ctx:
        got = prod.text_tokens_packed(ctx, seqs, 0, 0)
    for k, s in enumerate(seqs):
        want = pos[:len(s)] + tok[s]
        assert np.array_equal(bits(got[k]), bits(want.astype(np.float32))), len(s)


# ---- 5. order, passes, lengths, long contexts, launches -------------------------------------------------------------------------

def test_permuted_batch_gives_permuted_outputs(prod):
    seqs = seqs_of(LENS, 40)
    perm = np.random.default_rng(5).permutation(len(seqs))
    with Ctx(prod, model_file("tiny", "q4_0", prod)) as ctx:
        e, ep = encode_packed_dev(prod, ctx, seqs), encode_packed_dev(prod, ctx, [seqs[p] for p in perm])
        t = tokens_packed_dev(prod, ctx, seqs, -1, bd.TOKENS_POST_LN, bd.OUT_F16)
        tp = tokens_packed_dev(prod, ctx, [seqs[p] for p in perm], -1, bd.TOKENS_POST_LN, bd.OUT_F16)
    for i, p in enumerate(perm):
        assert np.array_equal(bits(ep[i]), bits(e[p])), (i, p)
        assert np.array_equal(bits(tp[i]), bits(t[p])), (i, p)


@pytest.mark.parametrize("micro_batch", [1, 2])
def test_pass_boundaries_change_nothing(prod, micro_batch):
    """a text micro_batch of 1 or 2 makes passes of 77 or 154 rows; rotating the batch puts a pass boundary after every position"""
    lens = [77, 1, 40, 37, 30, 50, 2, 76, 1, 5, 64, 13]
    seqs = seqs_of(lens, 50)
    path = model_file("tiny", "f16", prod)
    with Ctx(prod, path) as ctx:
        want_e = encode_packed_dev(prod, ctx, seqs)
        want_t = tokens_packed_dev(prod, ctx, seqs, -2, bd.TOKENS_PROJECT, bd.OUT_BF16)
    with Ctx(prod, path, (0, micro_batch)) as ctx:
        for shift in range(len(seqs)):
            batch = seqs[shift:] + seqs[:shift]
            got_e = encode_packed_dev(prod, ctx, batch)
            got_t = tokens_packed_dev(prod, ctx, batch, -2, bd.TOKENS_PROJECT, bd.OUT_BF16)
            for i in range(len(batch)):
                k = (i + shift) % len(seqs)
                assert np.array_equal(bits(got_e[i]), bits(want_e[k])), (micro_batch, shift, i)
                assert np.array_equal(bits(got_t[i]), bits(want_t[k])), (micro_batch, shift, i)


def test_length_one_and_context_length(prod):
    with Ctx(prod, model_file("tiny", "f16", prod)) as ctx:
        for lens in ([1], [77], [1] * 9, [77] * 5, [1, 77, 1, 77]):
            seqs = seqs_of(lens, 60)
            got_e = encode_packed_dev(prod, ctx, seqs)
            got_t = tokens_packed_dev(prod, ctx, seqs, -1, 0)
            for k, s in enumerate(seqs):
                assert np.array_equal(bits(got_e[k]), bits(encode_alone_dev(prod, ctx, s))), (lens, k)
                assert np.array_equal(bits(got_t[k]), bits(tokens_alone_dev(prod, ctx, s, -1, 0))), (lens, k)


@pytest.fixture(scope="module")
def long_ctx_model(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("long_ctx_packed") / "tiny-ctx4096.gguf")
    sg.write_model(path, LONG_CTX, 1234, 1)
    return path


def test_long_context_sequences_next_to_short_ones(prod, long_ctx_model):
    seqs = seqs_of([2049, 5, 4096, 78, 1, 300], 70)
    with Ctx(prod, long_ctx_model) as ctx:
        got_e = encode_packed_dev(prod, ctx, seqs)
        got_t = tokens_packed_dev(prod, ctx, seqs, 1, bd.TOKENS_POST_LN)
        for k, s in enumerate(seqs):
            assert np.array_equal(bits(got_e[k]), bits(encode_alone_dev(prod, ctx, s))), len(s)
            assert np.array_equal(bits(got_t[k]), bits(tokens_alone_dev(prod, ctx, s, 1, bd.TOKENS_POST_LN))), len(s)


def test_one_pass_launches_the_same_whatever_n(prod):
    """one embedding, the blocks and the tail per pass: 3 sequences and 40 launch the same kernels"""
    with Ctx(prod, model_file("tiny", "f16", prod)) as ctx:
        n = prod.lib.clip_b200_kernel_launches
        counts = []
        for lens in ([9, 77, 1], [int(t) for t in np.random.default_rng(1).integers(1, 78, 40)]):
            seqs = seqs_of(lens, 80)
            a = n(ctx)
            encode_packed_dev(prod, ctx, seqs)
            b = n(ctx)
            tokens_packed_dev(prod, ctx, seqs, 0, 0)
            c = n(ctx)
            counts.append((b - a, c - b))
    assert counts[0] == counts[1], counts
    assert counts[0][1] == 2, counts              # layer 0: the packed embedding and the token rows


# ---- 6. host forms, 7. the oracle ----------------------------------------------------------------------------------------------

def pinned_like(prod, shape, dtype):
    nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
    p = prod.lib.clip_b200_host_malloc(nbytes)
    assert p
    return p, np.frombuffer((C.c_uint8 * nbytes).from_address(p), dtype).reshape(shape)


def test_host_forms_equal_device_forms(prod):
    seqs = seqs_of(LENS, 90)
    lens = np.array([len(s) for s in seqs], np.int32)
    ids = np.concatenate(seqs).astype(np.int32)
    flags = bd.TOKENS_PROJECT
    with Ctx(prod, model_file("tiny", "q4_0", prod)) as ctx:
        want_e = encode_packed_dev(prod, ctx, seqs)
        want_t = tokens_packed_dev(prod, ctx, seqs, -3, flags, bd.OUT_F16)
        assert np.array_equal(bits(prod.text_batch_encode_packed(ctx, seqs)), bits(want_e))          # pageable out
        got = prod.text_tokens_packed(ctx, seqs, -3, flags, bd.OUT_F16)
        for k in range(len(seqs)):
            assert np.array_equal(bits(got[k]), bits(want_t[k])), k
        p, out = pinned_like(prod, (int(lens.sum()), text_width(prod, ctx, flags)), np.float16)
        try:
            assert prod.lib.clip_b200_text_tokens_packed(ctx, ids.ctypes.data_as(I32P), len(seqs), lens.ctypes.data_as(IP), -3, flags,
                                                         bd.OUT_F16, p), prod.last_error()
            assert np.array_equal(bits(out), bits(np.concatenate(want_t)))
        finally:
            prod.lib.clip_b200_host_free(p)
        arr = (bd.clip_tokens * len(seqs))()
        for i, s in enumerate(seqs):
            arr[i].data = s.ctypes.data_as(I32P)
            arr[i].size = s.size
        p, vec = pinned_like(prod, (len(seqs), prod.text_hparams(ctx).projection_dim), np.float32)
        try:
            assert prod.lib.clip_b200_text_batch_encode_packed(ctx, arr, len(seqs), C.cast(p, FP), True), prod.last_error()
            assert np.array_equal(bits(vec), bits(want_e))
        finally:
            prod.lib.clip_b200_host_free(p)


def test_tiny_against_oracle(prod):
    path = model_file("tiny", "f16", prod)
    om = AnyresOracle(path)
    seqs = seqs_of([77, 1, 9, 64, 33], 100)
    with Ctx(prod, path) as ctx:
        got = prod.text_batch_encode_packed(ctx, seqs)
    for k, s in enumerate(seqs):
        assert float(cos_rows(got[k], om.encode_text(s))) <= TOL["f16"], len(s)


# ---- 8. refusals ----------------------------------------------------------------------------------------------------------------

def test_refusals_in_order(prod, tmp_path):
    L = prod.lib
    seqs = seqs_of([9, 5], 110)
    lens = np.array([9, 5], np.int32)
    ids = np.concatenate(seqs).astype(np.int32)
    out = np.empty(1 << 16, np.float32)

    def refused(ok, msg):
        assert not ok
        assert msg in prod.last_error(), (msg, prod.last_error())

    def enc(c, n, di, ln, do):
        return L.clip_b200_text_encode_device_packed(c, di, n, ln.ctypes.data_as(IP) if ln is not None else None, do, True)

    def tok(c, n, hi, ln, ho, layer=-1, flags=0, ot=0):
        return L.clip_b200_text_tokens_packed(c, hi.ctypes.data_as(I32P) if hi is not None else None, n,
                                              ln.ctypes.data_as(IP) if ln is not None else None, layer, flags, ot,
                                              ho.ctypes.data if ho is not None else None)

    refused(tok(None, 2, ids, lens, out), "clip_b200_text_tokens_packed: null context")
    no_text = sg.Geometry("vision-only", image_size=64, patch_size=16, v_hidden=128, v_ff=256, v_heads=2, v_layers=1, t_hidden=128,
                          t_ff=256, t_heads=2, t_layers=1, proj_dim=128, has_text=False)
    hd80 = sg.Geometry("text-hd80", image_size=64, patch_size=16, v_hidden=128, v_ff=256, v_heads=2, v_layers=1, t_hidden=640,
                       t_ff=1280, t_heads=8, t_layers=2, proj_dim=128)
    for g in (no_text, hd80):
        path = str(tmp_path / (g.name + ".gguf"))
        sg.write_model(path, g, 1, 1)
        with Ctx(prod, path) as ctx:
            msg = ("clip_b200_text_tokens_packed: this model has no text encoder" if g is no_text else
                   "clip_b200_text_tokens_packed: packed sequences need a text tower of head_dim 64, not 80 (hidden 640, heads 8)")
            refused(tok(ctx, 0, None, None, None), msg)           # before n == 0
            if g is hd80:
                assert prod.text_tokens(ctx, padded(seqs, 9), -1, 0).shape == (2, 9, 640)     # the unpacked forms still run
    with Ctx(prod, model_file("tiny", "f16", prod)) as ctx:
        with Dev(prod, ctx) as d:
            d_ids, d_out = d.up(ids), d.up(np.zeros(1 << 16, np.float32))
            assert enc(ctx, 0, None, None, None)                                           # n == 0
            assert tok(ctx, 0, None, None, None, layer=99)
            assert L.clip_b200_text_batch_encode_packed(ctx, None, 0, None, True)
            refused(enc(ctx, 2, None, None, None), "clip_b200_text_encode_device_packed: null input")
            refused(enc(ctx, 2, d_ids, None, None), "clip_b200_text_encode_device_packed: null lens")
            refused(enc(ctx, 2, d_ids, lens, None), "clip_b200_text_encode_device_packed: null output")
            refused(L.clip_b200_text_tokens_device_packed(ctx, d_ids, 2, lens.ctypes.data_as(IP), -1, 0, 0, None),
                    "clip_b200_text_tokens_device_packed: null output")
            for bad in ([9, 0], [9, 78], [9, -3]):
                bl = np.array(bad, np.int32)
                refused(enc(ctx, 2, d_ids, bl, d_out), "clip_b200_text_encode_device_packed: sequence 1 has length %d, outside "
                                                       "[1, context_length (77)]" % bad[1])
                refused(tok(ctx, 2, ids, bl, out, layer=99), "clip_b200_text_tokens_packed: sequence 1 has length")  # before the request
            arr = (bd.clip_tokens * 2)()
            arr[0].data, arr[0].size = seqs[0].ctypes.data_as(I32P), seqs[0].size
            vec = np.empty((2, 128), np.float32)
            refused(L.clip_b200_text_batch_encode_packed(ctx, arr, 2, None, True), "clip_b200_text_batch_encode_packed: null output")
            refused(L.clip_b200_text_batch_encode_packed(ctx, arr, 2, vec.ctypes.data_as(FP), True),
                    "clip_b200_text_batch_encode_packed: sequence 1 has no tokens")
            arr[1].data, arr[1].size = seqs[1].ctypes.data_as(I32P), 0
            refused(L.clip_b200_text_batch_encode_packed(ctx, arr, 2, vec.ctypes.data_as(FP), True),
                    "clip_b200_text_batch_encode_packed: sequence 1 has length 0")
            refused(tok(ctx, 2, ids, lens, out, layer=99), "clip_b200_text_tokens_packed: layer 99 is outside")
            refused(tok(ctx, 2, ids, lens, out, flags=bd.TOKENS_NO_CLS), "CLIP_B200_TOKENS_NO_CLS is for the vision tower only")
            refused(tok(ctx, 2, ids, lens, out, flags=bd.TOKENS_NORMALIZE), "NORMALIZE needs")
            refused(tok(ctx, 2, ids, lens, out, ot=7), "unknown out_type 7")
            refused(tok(ctx, 2, ids, lens, out, layer=0, flags=bd.TOKENS_ATTENTION), "CLIP_B200_TOKENS_ATTENTION needs layer >= 1")
            refused(tok(ctx, 2, ids, lens, out, flags=bd.TOKENS_ATTENTION),
                    "clip_b200_text_tokens_packed: CLIP_B200_TOKENS_ATTENTION is not supported at packed lengths")


# ---- 9. devices mode ------------------------------------------------------------------------------------------------------------

def test_devices_mode_equals_one_gpu(prod, monkeypatch):
    if prod.lib.clip_b200_cuda_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    lens = [int(t) for t in np.random.default_rng(4).integers(1, 78, 45)]
    seqs = seqs_of(lens, 120)
    path = model_file("tiny", "q4_0", prod)
    with Ctx(prod, path) as ctx:
        one_e = prod.text_batch_encode_packed(ctx, seqs)
        one_t = prod.text_tokens_packed(ctx, seqs, -2, bd.TOKENS_POST_LN, bd.OUT_F16)
    monkeypatch.setenv("CLIP_B200_DEVICES", "all")
    with Ctx(prod, path) as ctx:
        assert prod.lib.clip_b200_device_count(ctx) >= 2
        assert np.array_equal(bits(prod.text_batch_encode_packed(ctx, seqs)), bits(one_e))
        got = prod.text_tokens_packed(ctx, seqs, -2, bd.TOKENS_POST_LN, bd.OUT_F16)
        for k in range(len(seqs)):
            assert np.array_equal(bits(got[k]), bits(one_t[k])), k
