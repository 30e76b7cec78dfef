"""Synthetic CLIP GGUF model files (numpy only, no `gguf` package needed).

There is no network and no real checkpoint on the build or GPU boxes, so every
parity test and benchmark runs on random-weight models of the *true geometries*
written in exactly the on-disk contract the reference's loader reads:

  * GGUF container layout:            /root/reference/ggml/src/ggml.c:19663-19697, 19751-20063
  * KV keys the loader looks up:      /root/reference/clip.cpp:41-58
  * tensor names:                     /root/reference/clip.cpp:64-79
  * dtype rules of the HF converter:  /root/reference/models/convert_hf_to_gguf.py:173-206
    (2-D `*.weight` -> f16/f32, `v.patch_embd.weight` always f16, everything else f32)
  * tensor counts the reference accepts (397 two-tower base, 589 two-tower large, 909 two-tower huge):
                                      /root/reference/clip.cpp:261-294

Weights are drawn from a seeded numpy PCG64 stream, so a (geometry, seed) pair
names one exact file; golden fixtures record the sha256 of the file they were
produced from and the tests refuse to compare against a drifted file.
"""
from __future__ import annotations

import hashlib
import os
import struct
from dataclasses import dataclass, field, asdict

import numpy as np

GGUF_MAGIC = 0x46554747
GGUF_VERSION = 3
GGUF_ALIGN = 32

# gguf value types (ggml.h:1844-1859)
T_U8, T_I8, T_U16, T_I16, T_U32, T_I32, T_F32, T_BOOL, T_STR, T_ARR, T_U64, T_I64, T_F64 = range(13)
# ggml tensor types used by clip.cpp
GGML_F32, GGML_F16 = 0, 1


@dataclass
class Geometry:
    """Hyper-parameters of a two-tower CLIP model (names follow clip.h:14-34)."""
    name: str
    image_size: int = 224
    patch_size: int = 32
    v_hidden: int = 768
    v_ff: int = 3072
    v_heads: int = 12
    v_layers: int = 12
    t_hidden: int = 512
    t_ff: int = 2048
    t_heads: int = 8
    t_layers: int = 12
    proj_dim: int = 512
    n_vocab: int = 49408
    n_ctx: int = 77
    eps: float = 1e-5
    use_gelu: bool = False          # OpenAI checkpoints: quick_gelu
    has_text: bool = True
    has_vision: bool = True

    @property
    def n_patches(self) -> int:
        return (self.image_size // self.patch_size) ** 2

    @property
    def n_pos(self) -> int:
        return self.n_patches + 1


GEOMETRIES = {
    # true geometries (SURVEY.md section 8)
    "vit-b32": Geometry("vit-b32"),
    "vit-l14": Geometry("vit-l14", patch_size=14, v_hidden=1024, v_ff=4096, v_heads=16, v_layers=24,
                        t_hidden=768, t_ff=3072, t_heads=12, t_layers=12, proj_dim=768),
    # ViT-L/14@336 (LLaVA-1.5's vision tower): 24 * 24 + 1 = 577 positions
    "vit-l14-336": Geometry("vit-l14-336", image_size=336, patch_size=14, v_hidden=1024, v_ff=4096, v_heads=16, v_layers=24,
                            t_hidden=768, t_ff=3072, t_heads=12, t_layers=12, proj_dim=768),
    # LAION ViT-H/14: vision head_dim 1280 / 16 = 80, text head_dim 1024 / 16 = 64, GELU
    "vit-h14": Geometry("vit-h14", patch_size=14, v_hidden=1280, v_ff=5120, v_heads=16, v_layers=32,
                        t_hidden=1024, t_ff=4096, t_heads=16, t_layers=24, proj_dim=1024, use_gelu=True),
    # small models for unit tests: same tensor counts as base (397) so the reference accepts them,
    # head_dim = 64 like every real CLIP model
    "tiny": Geometry("tiny", image_size=64, patch_size=16, v_hidden=128, v_ff=256, v_heads=2, v_layers=12,
                     t_hidden=128, t_ff=256, t_heads=2, t_layers=12, proj_dim=128),
    "tiny-gelu": Geometry("tiny-gelu", image_size=64, patch_size=16, v_hidden=128, v_ff=256, v_heads=2,
                          v_layers=12, t_hidden=128, t_ff=256, t_heads=2, t_layers=12, proj_dim=128,
                          use_gelu=True),
    # odd patch size (K = 3*14*14 = 588, not a multiple of 64) and 257 positions at small width
    "small-p14": Geometry("small-p14", image_size=224, patch_size=14, v_hidden=256, v_ff=512, v_heads=4,
                          v_layers=12, t_hidden=128, t_ff=256, t_heads=2, t_layers=12, proj_dim=128),
    # ViT-L/14@336 token count (24*24 + 1 = 577 > 257: the long-sequence attention path) at small width
    "small-p14-336": Geometry("small-p14-336", image_size=336, patch_size=14, v_hidden=128, v_ff=256, v_heads=2,
                              v_layers=12, t_hidden=128, t_ff=256, t_heads=2, t_layers=12, proj_dim=128),
    # ViT-H/14 width (1280 > 1024: the 16-float4-per-lane LayerNorm) in both towers, FC2 depth 5120, patch 14 (kpad 640), only
    # 2 layers; ~300 MB as f16
    "wide-h1280": Geometry("wide-h1280", image_size=112, patch_size=14, v_hidden=1280, v_ff=5120, v_heads=20, v_layers=2,
                           t_hidden=1280, t_ff=5120, t_heads=20, t_layers=2, proj_dim=1024),
    # the huge tensor counts (32 + 24 layers, 909 tensors) at low width, so the reference accepts it: vision head_dim 640 / 8 = 80
    # over 257 positions, GELU
    "huge-w640": Geometry("huge-w640", image_size=224, patch_size=14, v_hidden=640, v_ff=1280, v_heads=8, v_layers=32,
                          t_hidden=128, t_ff=256, t_heads=2, t_layers=24, proj_dim=128, use_gelu=True),
    # LAION ViT-bigG/14: vision head_dim 1664 / 16 = 104 (each head padded to 112 columns in the QKV projection at load), text
    # head_dim 1280 / 20 = 64, GELU; 1 293 tensors, more than the reference accepts
    "vit-bigg14": Geometry("vit-bigg14", patch_size=14, v_hidden=1664, v_ff=8192, v_heads=16, v_layers=48,
                           t_hidden=1280, t_ff=5120, t_heads=20, t_layers=32, proj_dim=1280, use_gelu=True),
    # the true bigG vision width and depth per layer with the huge tensor counts (32 + 24 layers, 909 tensors), so the reference
    # accepts it: head_dim 104 over 257 positions next to a tiny text tower; ~2.5 GB as f16
    "bigg-w1664": Geometry("bigg-w1664", image_size=224, patch_size=14, v_hidden=1664, v_ff=8192, v_heads=16, v_layers=32,
                           t_hidden=128, t_ff=256, t_heads=2, t_layers=24, proj_dim=128, use_gelu=True),
}


class _Writer:
    def __init__(self):
        self.kv = []        # (key, type, payload-bytes)
        self.tensors = []   # (name, np.ndarray)

    @staticmethod
    def _s(s: str) -> bytes:
        b = s.encode("utf-8")
        return struct.pack("<Q", len(b)) + b

    def add(self, key, typ, val):
        if typ == T_U32:
            p = struct.pack("<I", val)
        elif typ == T_F32:
            p = struct.pack("<f", val)
        elif typ == T_BOOL:
            p = struct.pack("<B", 1 if val else 0)
        elif typ == T_STR:
            p = self._s(val)
        else:
            raise ValueError(typ)
        self.kv.append((key, typ, p))

    def add_array_f32(self, key, vals):
        p = struct.pack("<IQ", T_F32, len(vals)) + struct.pack("<%df" % len(vals), *vals)
        self.kv.append((key, T_ARR, p))

    def add_array_str(self, key, strs):
        parts = [struct.pack("<IQ", T_STR, len(strs))]
        parts += [self._s(s) for s in strs]
        self.kv.append((key, T_ARR, b"".join(parts)))

    def add_tensor(self, name, arr: np.ndarray):
        assert arr.dtype in (np.float32, np.float16)
        self.tensors.append((name, np.ascontiguousarray(arr)))

    def write(self, path):
        head = [struct.pack("<IIQQ", GGUF_MAGIC, GGUF_VERSION, len(self.tensors), len(self.kv))]
        for key, typ, p in self.kv:
            head.append(self._s(key) + struct.pack("<I", typ) + p)
        off = 0
        offsets = []
        for name, arr in self.tensors:
            ne = list(arr.shape[::-1])          # ggml order: ne[0] is the fastest dimension
            head.append(self._s(name) + struct.pack("<I", len(ne)) +
                        struct.pack("<%dQ" % len(ne), *ne) +
                        struct.pack("<IQ", GGML_F32 if arr.dtype == np.float32 else GGML_F16, off))
            offsets.append(off)
            off += (arr.nbytes + GGUF_ALIGN - 1) // GGUF_ALIGN * GGUF_ALIGN
        meta = b"".join(head)
        pad = (-len(meta)) % GGUF_ALIGN
        with open(path, "wb") as f:
            f.write(meta + b"\0" * pad)
            for (name, arr), o in zip(self.tensors, offsets):
                b = arr.tobytes()
                f.write(b)
                f.write(b"\0" * ((-len(b)) % GGUF_ALIGN))


def _vocab(n):
    # Deterministic printable pseudo-vocabulary: bytes, "</w>" word forms and a few real words so the
    # tokenizer tests have something to match.  Ids 49406/49407 are SOT/EOT (clip.cpp:637,671).
    toks = []
    base = [chr(c) for c in range(33, 127)]
    toks += base
    toks += [c + "</w>" for c in base]
    words = ["a", "photo", "of", "the", "cat", "dog", "apple", "red", "white", "an", "image", "in", "on", "two"]
    toks += [w + "</w>" for w in words] + words
    i = 0
    while len(toks) < n:
        toks.append("tok%d</w>" % i)
        i += 1
    toks = toks[:n]
    if n > 49407:
        toks[49406] = "<|startoftext|>"
        toks[49407] = "<|endoftext|>"
    return toks


def write_model(path: str, geom: Geometry, seed: int = 1234, ftype: int = 1, qk_logit_std=None) -> str:
    """Write an f32 (ftype 0) or f16 (ftype 1) synthetic model; returns the sha256 of the file.

    qk_logit_std: draw each tower's attn_q / attn_k weights with std sqrt(qk_logit_std / hidden) instead of 0.03, so that the scaled
    attention logits q.k / sqrt(head_dim) have a standard deviation of about qk_logit_std at any head_dim (LayerNorm outputs have
    unit variance, so q and k entries have variance hidden std^2, and q.k / sqrt(head_dim) has standard deviation hidden std^2).
    At 3 the softmax is peaked, so a wrong Q scale, mask or key moves the output; the default std 0.03 gives hidden 9e-4 (0.1 at
    hidden 128), a nearly uniform softmax.  The
    draws are the same, only scaled, so None writes the same bytes as before the keyword existed."""
    assert ftype in (0, 1)
    g = geom
    rng = np.random.Generator(np.random.PCG64(seed))
    wdt = np.float32 if ftype == 0 else np.float16
    w = _Writer()
    w.add("general.architecture", T_STR, "clip")
    w.add("general.name", T_STR, "synthetic-" + g.name)
    w.add("general.description", T_STR, "synthetic random-weight CLIP (%s, seed %d)" % (g.name, seed))
    w.add("general.file_type", T_U32, ftype)
    w.add("clip.has_text_encoder", T_BOOL, g.has_text)
    w.add("clip.has_vision_encoder", T_BOOL, g.has_vision)
    w.add("clip.use_gelu", T_BOOL, g.use_gelu)

    def normal(shape, std, dtype=np.float32, mean=0.0):
        a = rng.standard_normal(size=shape, dtype=np.float32)
        a *= np.float32(std)
        if mean:
            a += np.float32(mean)
        return a.astype(dtype)

    def tower(p, hid, ff, heads, layers):
        for il in range(layers):
            pre = "%s.blk.%d." % (p, il)
            for nm in ("attn_q", "attn_k", "attn_v", "attn_out"):
                std = 0.02 if nm == "attn_out" else 0.03
                if qk_logit_std is not None and nm in ("attn_q", "attn_k"):
                    std = np.sqrt(qk_logit_std / hid)
                w.add_tensor(pre + nm + ".weight", normal((hid, hid), std, wdt))
                w.add_tensor(pre + nm + ".bias", normal((hid,), 0.02))
            w.add_tensor(pre + "ffn_down.weight", normal((ff, hid), 0.03, wdt))     # HF fc1 (h -> f)
            w.add_tensor(pre + "ffn_down.bias", normal((ff,), 0.02))
            w.add_tensor(pre + "ffn_up.weight", normal((hid, ff), 0.02, wdt))       # HF fc2 (f -> h)
            w.add_tensor(pre + "ffn_up.bias", normal((hid,), 0.02))
            for ln in ("ln1", "ln2"):
                w.add_tensor(pre + ln + ".weight", normal((hid,), 0.05, mean=1.0))
                w.add_tensor(pre + ln + ".bias", normal((hid,), 0.02))

    if g.has_text:
        w.add("clip.text.context_length", T_U32, g.n_ctx)
        w.add("clip.text.embedding_length", T_U32, g.t_hidden)
        w.add("clip.text.feed_forward_length", T_U32, g.t_ff)
        w.add("clip.text.block_count", T_U32, g.t_layers)
        w.add("clip.text.attention.head_count", T_U32, g.t_heads)
        w.add("clip.text.projection_dim", T_U32, g.proj_dim)
        w.add("clip.text.attention.layer_norm_epsilon", T_F32, g.eps)
        w.add_array_str("tokenizer.ggml.tokens", _vocab(g.n_vocab))
        w.add_tensor("t.token_embd.weight", normal((g.n_vocab, g.t_hidden), 0.05, wdt))
        w.add_tensor("t.position_embd.weight", normal((g.n_ctx, g.t_hidden), 0.02, wdt))
        tower("t", g.t_hidden, g.t_ff, g.t_heads, g.t_layers)
        w.add_tensor("t.post_ln.weight", normal((g.t_hidden,), 0.05, mean=1.0))
        w.add_tensor("t.post_ln.bias", normal((g.t_hidden,), 0.02))
        w.add_tensor("text_projection.weight", normal((g.proj_dim, g.t_hidden), 0.03, wdt))
    if g.has_vision:
        w.add("clip.vision.image_size", T_U32, g.image_size)
        w.add("clip.vision.patch_size", T_U32, g.patch_size)
        w.add("clip.vision.embedding_length", T_U32, g.v_hidden)
        w.add("clip.vision.feed_forward_length", T_U32, g.v_ff)
        w.add("clip.vision.block_count", T_U32, g.v_layers)
        w.add("clip.vision.attention.head_count", T_U32, g.v_heads)
        w.add("clip.vision.projection_dim", T_U32, g.proj_dim)
        w.add("clip.vision.attention.layer_norm_epsilon", T_F32, g.eps)
        w.add_array_f32("clip.vision.image_mean", [0.48145466, 0.4578275, 0.40821073])
        w.add_array_f32("clip.vision.image_std", [0.26862954, 0.26130258, 0.27577711])
        w.add_tensor("v.class_embd", normal((g.v_hidden,), 0.05))
        w.add_tensor("v.patch_embd.weight",
                     normal((g.v_hidden, 3, g.patch_size, g.patch_size), 0.03, np.float16))
        w.add_tensor("v.position_embd.weight", normal((g.n_pos, g.v_hidden), 0.05, wdt))
        w.add_tensor("v.pre_ln.weight", normal((g.v_hidden,), 0.05, mean=1.0))
        w.add_tensor("v.pre_ln.bias", normal((g.v_hidden,), 0.02))
        tower("v", g.v_hidden, g.v_ff, g.v_heads, g.v_layers)
        w.add_tensor("v.post_ln.weight", normal((g.v_hidden,), 0.05, mean=1.0))
        w.add_tensor("v.post_ln.bias", normal((g.v_hidden,), 0.02))
        w.add_tensor("visual_projection.weight", normal((g.proj_dim, g.v_hidden), 0.03, wdt))
    w.write(path)
    return sha256_file(path)


def sha256_file(path: str) -> str:
    h = hashlib.sha256()
    with open(path, "rb") as f:
        while True:
            b = f.read(1 << 24)
            if not b:
                break
            h.update(b)
    return h.hexdigest()


def synth_images(n: int, image_size: int, seed: int) -> np.ndarray:
    """[n, S, S, 3] f32 NHWC, U(-2, 2): the post-normalisation range (SURVEY.md section 8d)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    return (rng.random(size=(n, image_size, image_size, 3), dtype=np.float32) * np.float32(4.0)
            - np.float32(2.0))


def synth_tokens(n: int, length: int, seed: int, n_vocab: int = 49408) -> np.ndarray:
    """[n, length] int32: SOT, U{0..49405}, EOT (clip.cpp:637,671)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    t = rng.integers(0, min(n_vocab, 49406), size=(n, length), dtype=np.int32)
    t[:, 0] = 49406
    t[:, -1] = 49407
    return t


def cache_dir() -> str:
    d = os.environ.get("CLIP_B200_CACHE", "/tmp/clip_b200_cache")
    os.makedirs(d, exist_ok=True)
    return d


def model_path(geom_name: str, seed: int, ftype_name: str) -> str:
    return os.path.join(cache_dir(), "%s-s%d-%s.gguf" % (geom_name, seed, ftype_name))


if __name__ == "__main__":
    import sys
    gname = sys.argv[1] if len(sys.argv) > 1 else "tiny"
    out = sys.argv[2] if len(sys.argv) > 2 else model_path(gname, 1234, "f16")
    print(out, write_model(out, GEOMETRIES[gname]))
