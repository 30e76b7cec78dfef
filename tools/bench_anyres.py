#!/usr/bin/env python
"""The vision tower at non-native image sizes (clip_b200_image_encode_device_hw), ViT-L/14 q4_0, b = 256 device-resident images.

    python tools/bench_anyres.py [--steps 5] [--warmup 2] [--reps 3]

  (a) 224 x 224 through _hw on the 224 model against clip_b200_image_encode_device on the same context: the same work, so the
      _hw overhead should be nil.
  (b) 336 x 336 through _hw on the 224 model (T = 577) against the native ViT-L/14@336 geometry (same T, same work).
  (c) 448 x 448 (T = 1025) and 224 x 448 (T = 513) through _hw, as images/s.

Paired paths are alternated --reps times (host clock around calls that end in a device synchronise).  Per size, a second context
with CLIP_B200_PROFILE=1 gives the split of device time by kernel class (clip_b200_kernel_ms kinds 0-3) and the time of one K8
position-table resample (kind 5; the size alternates with another so that every call resamples), with K8's bytes and GB/s against
the H100 SXM data sheet's 3.35 TB/s.  The card's name and power limit are read in the same call.  One JSON line per case.  Model
files are written from seeds into synth_gguf.cache_dir(), never into the tree."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "clip.cpp_b200"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)
import binding as bd  # noqa: E402
import synth_gguf as sg  # noqa: E402
from bench_tokens import HBM_PEAK, Dev, card, model, per_call  # noqa: E402

KINDS = {0: "gemm", 1: "attention", 2: "layernorm", 3: "other"}
K_POS_RESAMPLE = 5
N = 256


def images(n, H, W, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    return rng.random(size=(n, H, W, 3), dtype=np.float32) * np.float32(4.0) - np.float32(2.0)


def hw_call(lib, ctx, dev, H, W, n=N, seed=1):
    x = images(n, H, W, seed)
    d_pix = dev.alloc(x.nbytes, x)
    d_vec = dev.alloc(n * 768 * 4)
    return lambda: lib.lib.clip_b200_image_encode_device_hw(ctx, d_pix, n, H, W, d_vec, True)


def profile(lib, path, H, W, args):
    """device ms per call by kernel class at H x W, and K8's ms per resample"""
    os.environ["CLIP_B200_PROFILE"] = "1"
    ctx = lib.load(path, 0)
    dev = Dev(lib, ctx)
    try:
        call = hw_call(lib, ctx, dev, H, W)
        for _ in range(args.warmup):
            assert call()
        cnt = C.c_uint64(0)
        for k in list(KINDS) + [K_POS_RESAMPLE]:
            lib.lib.clip_b200_kernel_ms(ctx, k, C.byref(cnt))
        for _ in range(args.steps):
            assert call()
        split = {KINDS[k]: round(lib.lib.clip_b200_kernel_ms(ctx, k, C.byref(cnt)) / args.steps, 3) for k in KINDS}
        # K8 alone: one image per call, the size alternating with a neighbour so that each call resamples
        g = 224 // 14
        one, other = hw_call(lib, ctx, dev, H, W, 1, 2), hw_call(lib, ctx, dev, H + 14, W, 1, 3)
        lib.lib.clip_b200_kernel_ms(ctx, K_POS_RESAMPLE, C.byref(cnt))
        for _ in range(args.steps):
            assert one() and other()
        ms = lib.lib.clip_b200_kernel_ms(ctx, K_POS_RESAMPLE, C.byref(cnt))
        k8 = ms / max(cnt.value, 1)
        out_rows = (H // 14) * (W // 14)
        k8_bytes = (out_rows + g * g) * 1024 * 4                 # output written once, table read once (its re-reads hit L1 / L2)
    finally:
        dev.free()
        lib.free(ctx)
        del os.environ["CLIP_B200_PROFILE"]
    total = sum(split.values())
    return {"device_ms_by_class": split, "share_by_class": {k: round(v / total, 3) for k, v in split.items()},
            "k8_ms_per_resample": round(k8, 4), "k8_resamples": cnt.value, "k8_bytes": k8_bytes,
            "k8_GBps": round(k8_bytes / (k8 * 1e-3) / 1e9, 1), "k8_hbm_share": round(k8_bytes / (k8 * 1e-3) / HBM_PEAK, 3)}


def alternate(calls, args):
    """{name: call} -> {name: images/s per rep, slowest first}, the calls alternated"""
    t = {k: [] for k in calls}
    for _ in range(args.reps):
        for k, f in calls.items():
            t[k].append(per_call(f, args.steps, args.warmup))
    return {k: [round(N / s) for s in sorted(v, reverse=True)] for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    lib = bd.ClipLib(bd.PRODUCT_LIB)
    gpu = card()
    print("card, power limit:", gpu, flush=True)
    l14, l14_336 = model(lib, "vit-l14", "q4_0"), model(lib, "vit-l14-336", "q4_0")
    results = []

    # (a) 224 through _hw against the native entry point, one context
    ctx = lib.load(l14, 0)
    dev = Dev(lib, ctx)
    try:
        x = sg.synth_images(N, 224, 1)
        d_pix, d_vec = dev.alloc(x.nbytes, x), dev.alloc(N * 768 * 4)
        d_vec2 = dev.alloc(N * 768 * 4)
        r = alternate({"hw_img_s": lambda: lib.lib.clip_b200_image_encode_device_hw(ctx, d_pix, N, 224, 224, d_vec, True),
                       "native_img_s": lambda: lib.lib.clip_b200_image_encode_device(ctx, d_pix, N, d_vec2, True)}, args)
        a, b = np.empty(N * 768, np.float32), np.empty(N * 768, np.float32)
        lib.lib.clip_b200_memcpy_d2h(ctx, a.ctypes.data, d_vec, a.nbytes)
        lib.lib.clip_b200_memcpy_d2h(ctx, b.ctypes.data, d_vec2, b.nbytes)
        r["bit_identical"] = bool(np.array_equal(a.view(np.uint32), b.view(np.uint32)))
    finally:
        dev.free()
        lib.free(ctx)
    results.append(dict(case="224x224: _hw vs native, ViT-L/14 q4_0, b=256", T=257, **r))

    # (b) 336 through _hw on the 224 model against the native 336 geometry (two contexts, alternated)
    ctx, ctx336 = lib.load(l14, 0), lib.load(l14_336, 0)
    dev, dev336 = Dev(lib, ctx), Dev(lib, ctx336)
    try:
        x = sg.synth_images(N, 336, 2)
        d_pix, d_vec = dev.alloc(x.nbytes, x), dev.alloc(N * 768 * 4)
        d_pix3, d_vec3 = dev336.alloc(x.nbytes, x), dev336.alloc(N * 768 * 4)
        r = alternate({"hw_on_224_model_img_s": lambda: lib.lib.clip_b200_image_encode_device_hw(ctx, d_pix, N, 336, 336, d_vec, True),
                       "native_336_model_img_s": lambda: lib.lib.clip_b200_image_encode_device(ctx336, d_pix3, N, d_vec3, True)}, args)
    finally:
        dev.free()
        dev336.free()
        lib.free(ctx)
        lib.free(ctx336)
    results.append(dict(case="336x336: _hw on ViT-L/14 vs native ViT-L/14@336, q4_0, b=256", T=577, **r))

    # (c) larger and rectangular sizes
    ctx = lib.load(l14, 0)
    dev = Dev(lib, ctx)
    try:
        r = alternate({"448x448_img_s": hw_call(lib, ctx, dev, 448, 448), "224x448_img_s": hw_call(lib, ctx, dev, 224, 448)}, args)
    finally:
        dev.free()
        lib.free(ctx)
    results.append(dict(case="448x448 (T=1025) and 224x448 (T=513) through _hw, ViT-L/14 q4_0, b=256", **r))

    for (H, W), res in zip(((224, 224), (336, 336), (448, 448), (224, 448)), (results[0], results[1], results[2], results[2])):
        res["profile_%dx%d" % (H, W)] = profile(lib, l14, H, W, args)
    for res in results:
        res["gpu"] = gpu
        print(json.dumps(res), flush=True)
    sys.exit(0 if results[0]["bit_identical"] else 1)


if __name__ == "__main__":
    main()
