#!/usr/bin/env python
"""Images of different sizes in one call (clip_b200_image_encode_device_mixed), ViT-L/14 q4_0, 512 device-resident images.

    python tools/bench_mixed.py [--steps 3] [--warmup 1] [--reps 3]

Workloads: "aspect" -- shorter side 336, longer side 336 .. 672 in steps of 14, either orientation (49 sizes), drawn from a seed, as
a photo collection resized to its own aspect ratio gives them; "uniform" -- every image 336 x 336.
  (a) aspect: one mixed call against one clip_b200_image_encode_device_hw call per distinct size.
  (b) aspect: one mixed call against one _hw call per image.
  (c) uniform: the mixed call against the single _hw call.
  (d) uniform: device time of the attention kernel (clip_b200_kernel_ms kind 1) in the mixed call (the variable-length instance)
      against the _hw call (the fixed-T instance), same rows, with CLIP_B200_PROFILE=1 in a context of its own.
Paired paths are alternated --reps times (host clock around calls that end in a device synchronise).  The card's name and power
limit are read in the same call.  One JSON line per case.  Model files are written from seeds into synth_gguf.cache_dir()."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "clip.cpp_b200"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)
import binding as bd  # noqa: E402
from bench_tokens import Dev, card, model, per_call  # noqa: E402

N, D, P = 512, 768, 14
IP = C.POINTER(C.c_int)


def sizes(workload, seed=11):
    if workload == "uniform":
        return [(336, 336)] * N
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(N):
        long = 336 + P * int(rng.integers(0, 25))
        out.append((336, long) if rng.integers(2) else (long, 336))
    return out


class Batch:
    """the images of one workload on the device, back to back (the mixed layout), and where each starts"""
    def __init__(self, lib, ctx, dev, hw, seed=1):
        rng = np.random.Generator(np.random.PCG64(seed))
        self.hw = hw
        self.h = np.array([a for a, _ in hw], np.int32)
        self.w = np.array([b for _, b in hw], np.int32)
        self.off = np.concatenate([[0], np.cumsum(self.h.astype(np.int64) * self.w * 3)])
        x = rng.random(int(self.off[-1]), dtype=np.float32) * np.float32(4.0) - np.float32(2.0)
        self.lib, self.ctx = lib, ctx
        self.d_pix, self.d_vec = dev.alloc(x.nbytes, x), dev.alloc(N * D * 4)
        # the images of each distinct size gathered together, for the one-call-per-size path
        order = sorted(range(N), key=lambda i: hw[i])
        xs = np.concatenate([x[self.off[i]:self.off[i + 1]] for i in order])
        self.d_sorted = dev.alloc(xs.nbytes, xs)
        self.groups, pos = [], 0
        for size in sorted(set(hw)):
            k = sum(1 for s in hw if s == size)
            self.groups.append((size, k, pos))
            pos += k * size[0] * size[1] * 3

    def mixed(self):
        return self.lib.lib.clip_b200_image_encode_device_mixed(self.ctx, self.d_pix, N, self.h.ctypes.data_as(IP), self.w.ctypes.data_as(IP),
                                                               self.d_vec, True)

    def per_size(self):
        ok = True
        for (H, W), k, pos in self.groups:
            ok &= self.lib.lib.clip_b200_image_encode_device_hw(self.ctx, self.d_sorted + pos * 4, k, H, W, self.d_vec, True)
        return ok

    def per_image(self):
        ok = True
        for i, (H, W) in enumerate(self.hw):
            ok &= self.lib.lib.clip_b200_image_encode_device_hw(self.ctx, self.d_pix + int(self.off[i]) * 4, 1, H, W, self.d_vec + i * D * 4, True)
        return ok

    def one_hw(self):
        H, W = self.hw[0]
        return self.lib.lib.clip_b200_image_encode_device_hw(self.ctx, self.d_pix, N, H, W, self.d_vec, True)


def alternate(calls, args):
    """{name: call} -> {name: images/s per rep, slowest first}, the calls alternated"""
    t = {k: [] for k in calls}
    for _ in range(args.reps):
        for k, f in calls.items():
            t[k].append(per_call(f, args.steps, args.warmup))
    return {k: [round(N / s, 1) for s in sorted(v, reverse=True)] for k, v in t.items()}


def ratio(r, a, b):
    """a over b in images/s, per rep (both lists slowest first)"""
    return [round(x / y, 3) for x, y in zip(r[a], r[b])]


def attention_ms(lib, path, args):
    """kind-1 device ms per call: the mixed call against the _hw call on the uniform workload"""
    os.environ["CLIP_B200_PROFILE"] = "1"
    ctx = lib.load(path, 0)
    dev = Dev(lib, ctx)
    out = {"mixed_attn_ms": [], "hw_attn_ms": []}
    try:
        b = Batch(lib, ctx, dev, sizes("uniform"))
        cnt = C.c_uint64(0)
        for _ in range(args.warmup):
            assert b.mixed() and b.one_hw()
        for _ in range(args.reps):
            for name, f in (("mixed_attn_ms", b.mixed), ("hw_attn_ms", b.one_hw)):
                lib.lib.clip_b200_kernel_ms(ctx, 1, C.byref(cnt))
                for _ in range(args.steps):
                    assert f()
                out[name].append(round(lib.lib.clip_b200_kernel_ms(ctx, 1, C.byref(cnt)) / args.steps, 3))
    finally:
        dev.free()
        lib.free(ctx)
        del os.environ["CLIP_B200_PROFILE"]
    out["mixed_over_hw"] = [round(x / y, 4) for x, y in zip(out["mixed_attn_ms"], out["hw_attn_ms"])]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    lib = bd.ClipLib(bd.PRODUCT_LIB)
    gpu = card()
    print("card, power limit:", gpu, flush=True)
    path = model(lib, "vit-l14", "q4_0")
    results = []
    ctx = lib.load(path, 0)
    dev = Dev(lib, ctx)
    try:
        b = Batch(lib, ctx, dev, sizes("aspect"))
        r = alternate({"mixed_img_s": b.mixed, "per_size_img_s": b.per_size, "per_image_img_s": b.per_image}, args)
        results.append(dict(case="(a, b) aspect: mixed vs one _hw call per size / per image, ViT-L/14 q4_0, n=512",
                            distinct_sizes=len(b.groups), rows=int(sum((h // P) * (w // P) + 1 for h, w in b.hw)),
                            mixed_over_per_size=ratio(r, "mixed_img_s", "per_size_img_s"),
                            mixed_over_per_image=ratio(r, "mixed_img_s", "per_image_img_s"), **r))
        b = Batch(lib, ctx, dev, sizes("uniform"), seed=2)
        r = alternate({"mixed_img_s": b.mixed, "hw_img_s": b.one_hw}, args)
        got, want = np.empty(N * D, np.float32), np.empty(N * D, np.float32)
        assert b.mixed()
        lib.lib.clip_b200_memcpy_d2h(ctx, got.ctypes.data, b.d_vec, got.nbytes)
        assert b.one_hw()
        lib.lib.clip_b200_memcpy_d2h(ctx, want.ctypes.data, b.d_vec, want.nbytes)
        results.append(dict(case="(c) uniform 336x336: mixed vs one _hw call, ViT-L/14 q4_0, n=512", mixed_over_hw=ratio(r, "mixed_img_s", "hw_img_s"),
                            bit_identical=bool(np.array_equal(got.view(np.uint32), want.view(np.uint32))), **r))
    finally:
        dev.free()
        lib.free(ctx)
    results.append(dict(case="(d) uniform 336x336: attention kernel ms per call (kind 1), varlen vs fixed-T instance", **attention_ms(lib, path, args)))
    for res in results:
        res["gpu"] = gpu
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
