"""The per-block criterion of tests/_block_ref.py, checked without a GPU.

A second emulation of a block -- fp32 GEMM accumulation in 16-deep steps in a shuffled k order, fp32 LayerNorm, attention over
128-key blocks (64 at head_dim 104) with a running maximum as K3 keeps it, fp32 GELU -- must meet the criterion, and the same
emulation with one fault planted must miss it by at least 3 C: a Q scale from the padded or a 64 head_dim or none at all, the causal
mask one key off either way, one key dropped at a 64- or 128-key edge, the wrong GELU, LayerNorm eps x 10, the LN1 and LN2 weights
swapped, one GEMM's bias missing, the weights of the block before or after, a neighbouring sequence's keys visible to one row of a
packed pass, and bf16 operands where the GPU ran fp16.

The models are small synthetic files with sharp attention (synth_gguf.write_model's qk_logit_std = 3): head_dim 64 with quick-GELU, and head_dim 80
(vision) next to 104 (text) with the tanh GELU.  Each runs as f16 weights with fp16 operands and as q4_0 with bf16 operands.  The
inputs are random rows of different scales, down to a standard deviation of 0.02, where LayerNorm's eps starts to matter."""
import numpy as np
import pytest

import _block_ref as br
import _epilogue_rule as rule
import synth_gguf as sg
from _block_ref import C
from _oracle_tokens import TokenOracle
from _util import FTYPES

GEOMS = {
    "hd64": sg.Geometry("cpu-hd64", image_size=192, patch_size=16, v_hidden=128, v_ff=256, v_heads=2, v_layers=3, t_hidden=128,
                        t_ff=256, t_heads=2, t_layers=3, proj_dim=128, n_vocab=512),
    "hd80-104": sg.Geometry("cpu-hd80-104", image_size=192, patch_size=16, v_hidden=160, v_ff=320, v_heads=2, v_layers=3,
                            t_hidden=416, t_ff=832, t_heads=4, t_layers=3, proj_dim=128, n_vocab=512, use_gelu=True),
}
# (tower, lengths of the sequences of one pass, causal): two 145-row images (two 128-key blocks, the second ragged) and a packed
# text pass whose sequences straddle the 64-row edge
PASSES = {"v": ((145, 145), False), "t": ((1, 2, 63, 64, 65, 77), True)}
LAYER = 1
LOG2E = np.float32(1.4426950408889634)
F32 = np.float32


@pytest.fixture(scope="module")
def models(prod, tmp_path_factory):
    d = tmp_path_factory.mktemp("block_ref")
    out = {}
    for name, g in GEOMS.items():
        f16 = str(d / (name + "-f16.gguf"))
        sg.write_model(f16, g, 7, 1, qk_logit_std=3.0)
        q40 = str(d / (name + "-q4_0.gguf"))
        assert prod.quantize(f16, q40, FTYPES["q4_0"]), prod.last_error()
        out[name] = {"f16": TokenOracle(f16), "q4_0": TokenOracle(q40)}
    return out


# ---- the second emulation ------------------------------------------------------------------------------------------------------

def gemm32(a, w, rng):
    """a [M, K] . w [N, K]^T of 16-bit values: each 16-deep step exact and rounded to fp32, the steps added in fp32 in a shuffled
    order"""
    acc = np.zeros((a.shape[0], w.shape[0]), F32)
    for s in rng.permutation(a.shape[1] // 16):
        c = slice(16 * s, 16 * s + 16)
        acc = acc + (a[:, c] @ w[:, c].T).astype(F32)
    return acc


def ln32(x, gb, eps, bf):
    g, b = (v.astype(F32) for v in gb)
    mean = x.sum(-1, dtype=F32) / F32(x.shape[1])
    c = x - mean[:, None]
    rstd = F32(1) / np.sqrt((c * c).sum(-1, dtype=F32) / F32(x.shape[1]) + F32(eps))
    return rule.round16(c * rstd[:, None] * g + b, bf).astype(np.float64)


def gelu32(z, kind):
    if kind == "gelu":
        return F32(0.5) * z * (F32(1) + np.tanh(F32(0.7978845608) * (z + F32(0.044715) * z * z * z)))
    return z / (F32(1) + np.exp(F32(-1.702) * z))


def pass_mask(lens, causal, fault, kb):
    """which keys of the pass each row sees: its own sequence (up to itself when causal), with the mask faults planted"""
    M = sum(lens)
    vis = np.zeros((M, M), bool)
    for sl in br.seq_slices(lens):
        T = sl.stop - sl.start
        m = np.ones((T, T), bool)
        if causal:
            m = np.tri(T, T, {"causal+1": 1, "causal-1": -1}.get(fault, 0), bool)
            m[0, 0] = True
        edge = kb if T > kb else 64
        if fault == "drop_key" and T > edge:
            m[:, edge] = False
        vis[sl, sl] = m
    if fault == "neighbour":
        s0, s1 = br.seq_slices(lens)[-2:]
        vis[s1.start, s0] = True
    return vis


def attn32(q, k, v, vis, bf, kb):
    """K3 on one head of a pass: key blocks of kb in order, fp32 scores, running max, exp2, P rounded to 16 bits for P.V only"""
    s_all = (q @ k.T).astype(F32)
    M = len(q)
    m = np.full(M, -np.inf, F32)
    l = np.zeros(M, F32)
    o = np.zeros(v.shape, F32)
    with np.errstate(invalid="ignore"):
        for b0 in range(0, M, kb):
            c = slice(b0, b0 + kb)
            s = np.where(vis[:, c], s_all[:, c], F32(-np.inf))
            m_new = np.maximum(m, s.max(-1))
            mb = np.where(np.isfinite(m_new), m_new * LOG2E, F32(0)).astype(F32)
            alpha = np.where(np.isfinite(m), np.exp2((m * LOG2E).astype(F32) - mb), F32(0)).astype(F32)
            p = np.exp2((s * LOG2E).astype(F32) - mb[:, None]).astype(F32)
            l = l * alpha + p.sum(-1, dtype=F32)
            o = o * alpha[:, None] + (rule.round16(p, bf).astype(np.float64) @ v[c]).astype(F32)
            m = m_new
    return rule.round16(o * (F32(1) / l)[:, None], bf).astype(np.float64)


def second_emulation(om, tower, x, lens, causal, bf, fault=None, seed=0):
    """block LAYER of `tower` on fp32 rows x with fp32 arithmetic between the GPU's rounding points, with `fault` planted"""
    rng = np.random.default_rng(seed)
    blk = br.Block(om, tower, {"layer-1": LAYER - 1, "layer+1": LAYER + 1}.get(fault, LAYER))
    h, dh = blk.hidden, blk.dh
    kb = 64 if dh == 104 else 128
    ln1, ln2 = (blk.ln2, blk.ln1) if fault == "ln_swap" else (blk.ln1, blk.ln2)
    eps = F32(blk.eps) * F32(10) if fault == "eps_x10" else F32(blk.eps)
    gelu = {"gelu": "qgelu", "qgelu": "gelu"}[blk.gelu] if fault == "gelu" else blk.gelu
    bias = {n: (np.zeros_like(b) if fault == "no_bias_" + n else b).astype(F32) for n, b in blk.bias.items()}
    pad = {80: 128, 104: 112}.get(dh, dh)
    scale = {"scale_padded": 1 / np.sqrt(pad), "scale_64": 0.125, "scale_none": 1.0}.get(fault, 1 / np.sqrt(dh))
    W = {n: blk.w(n, bf) for n in ("qkv", "out", "fc1", "fc2")}

    x = np.asarray(x, F32)
    a = ln32(x, ln1, eps, bf)
    qkv = gemm32(a, W["qkv"], rng) + bias["qkv"]
    qkv[:, :h] *= F32(1) / np.sqrt(F32(dh)) if fault is None or not fault.startswith("scale") else F32(scale)
    qkv = rule.round16(qkv, bf).astype(np.float64)
    vis = pass_mask(lens, causal, fault, kb)
    o = np.empty((len(x), h))
    for hh in range(blk.heads):
        c = slice(hh * dh, (hh + 1) * dh)
        o[:, c] = attn32(qkv[:, c], qkv[:, h + c.start:h + c.stop], qkv[:, 2 * h + c.start:2 * h + c.stop], vis, bf, kb)
    x_mid = x + (gemm32(o, W["out"], rng) + bias["out"])
    a = ln32(x_mid, ln2, eps, bf)
    g = rule.round16(gelu32(gemm32(a, W["fc1"], rng) + bias["fc1"], gelu), bf).astype(np.float64)
    return (x_mid + (gemm32(g, W["fc2"], rng) + bias["fc2"])).astype(np.float64)


# ---- the cases -----------------------------------------------------------------------------------------------------------------

CONFIGS = [("f16", False), ("q4_0", True)]          # (weights, bf16 operands): what the GPU runs each file with by default
_memo = {}


def reference(models, name, ft, bf, tower):
    """(x, lens, causal, x_ref, x_emu, floor) of one case, computed once"""
    key = (name, ft, bf, tower)
    if key not in _memo:
        om = models[name][ft]
        lens, causal = PASSES[tower]
        blk = br.Block(om, tower, LAYER)
        rng = np.random.default_rng(11 if tower == "v" else 12)
        M = sum(lens)
        scale = np.exp(rng.uniform(np.log(0.02), np.log(2.0), (M, 1)))
        x = (rng.standard_normal((M, blk.hidden)) * scale + rng.standard_normal((M, 1)) * 0.1).astype(F32)
        x_emu, floor = br.emu(blk, x, lens, causal, bf)
        _memo[key] = (x, lens, causal, br.ref(blk, x, lens, causal), x_emu, floor)
    return _memo[key]


def worst_ratio(models, name, ft, bf, tower, fault=None, emu_bf=None, seed=0):
    x, lens, causal, x_ref, x_emu, floor = reference(models, name, ft, bf if emu_bf is None else emu_bf, tower)
    got = second_emulation(models[name][ft], tower, x, lens, causal, bf, fault, seed)
    return float(br.ratio(got, x_ref, x_emu, floor).max())


@pytest.mark.parametrize("ft,bf", CONFIGS)
@pytest.mark.parametrize("tower", ["v", "t"])
@pytest.mark.parametrize("name", list(GEOMS))
def test_second_emulation_meets_the_criterion(models, name, tower, ft, bf):
    for seed in range(3):
        r = worst_ratio(models, name, ft, bf, tower, seed=seed)
        print("accept %s %s %s %s seed %d: worst e_gpu/e_emu %.3f (C = %.2f)" % (name, tower, ft, "bf16" if bf else "fp16", seed, r, C))
        assert r <= C, r


FAULTS = ["scale_none", "scale_padded", "scale_64", "causal+1", "causal-1", "drop_key", "gelu", "eps_x10", "ln_swap", "no_bias_qkv",
          "no_bias_out", "no_bias_fc1", "no_bias_fc2", "layer-1", "layer+1", "neighbour"]


def applies(fault, name, tower):
    dh = {"hd64": 64, "hd80-104": 80 if tower == "v" else 104}[name]
    if fault in ("scale_padded", "scale_64") and dh == 64:
        return False                                   # head_dim 64 is neither padded nor other than 64
    return not (fault.startswith("causal") and tower == "v")


CASES = [(n, t, f) for n in GEOMS for t in ("v", "t") for f in FAULTS if applies(f, n, t)]
# Below 3 C at bf16 operands (see C in tests/_block_ref.py): the two GELUs differ by less than 1 % at the synthetic models' FC1
# pre-activations (standard deviation 0.3 - 0.6), and 1/sqrt(112) is 3.6 % off 1/sqrt(104); bf16 weights and activations carry
# 0.2 - 0.4 % per element.  strict: one that starts reaching 3 C must be moved back.
SHORT_AT_BF16 = {("gelu", n, t) for n in GEOMS for t in ("v", "t")} | {("scale_padded", "hd80-104", "t")}


@pytest.mark.parametrize("ft,bf", CONFIGS)
@pytest.mark.parametrize("name,tower,fault", CASES)
def test_planted_faults_break_the_criterion(models, name, tower, fault, ft, bf, request):
    if bf and (fault, name, tower) in SHORT_AT_BF16:
        request.applymarker(pytest.mark.xfail(reason="below 3 C at bf16 operands: see C in tests/_block_ref.py", strict=True))
    r = worst_ratio(models, name, ft, bf, tower, fault)
    print("fault %-12s %s %s %s %s: worst e_gpu/e_emu %.1f, %.1f C" % (fault, name, tower, ft, "bf16" if bf else "fp16", r, r / C))
    assert r >= 3 * C, r


@pytest.mark.parametrize("tower", ["v", "t"])
@pytest.mark.parametrize("name", list(GEOMS))
def test_bf16_operands_where_the_gpu_ran_fp16_break_the_criterion(models, name, tower):
    """q4_0 weights as the fp16-operand path unpacks them (CLIP_B200_OPERAND=f16), against a block that ran bf16 operands"""
    r = worst_ratio(models, name, "q4_0", True, tower, emu_bf=False)
    print("fault bf16-for-fp16 %s %s: worst e_gpu/e_emu %.1f, %.1f C" % (name, tower, r, r / C))
    assert r >= 3 * C, r
