#!/usr/bin/env python
"""Several layers' token rows from one forward pass (clip_b200_*_tokens_layers), against the single-layer calls they replace.

    python tools/bench_tokens_layers.py [--steps 3] [--warmup 1] [--reps 3] [--only all|llava|sdxl|host]

  all    ViT-L/14 q4_0, b = 256 device-resident images, all 25 hidden states, f16 rows: one _layers call, the 25 single-layer calls,
         and one pooled clip_b200_image_encode_device call.  The 25 slabs are checked byte for byte against the 25 single calls.
         Also the token-row kernel's CUDA-event time per call (kind 4 of clip_b200_kernel_ms, from a context with
         CLIP_B200_PROFILE=1), its bytes (fp32 rows read, f16 rows written) and rate against the H100 SXM data sheet's 3.35 TB/s.
  llava  ViT-L/14@336 q4_0, b = 256, layers -2 -5 -8 -11, NO_CLS, f16: one _layers call against the four single calls.
  sdxl   the ViT-L/14 text tower, 2048 x 77 ids, {-2: raw, -1: PROJECT}, f16: one _layers call against the two single calls.
  host   the first workload from host images into a pinned `out` (clip_b200_host_malloc) and a pageable one, against the device form
         and against a plain device-to-host copy of the same bytes into pinned memory.

Host clock around calls that end in a device synchronise; the compared forms alternate --reps times and every range is printed.
The card's name and power limit are read in the same call.  One JSON line per case.  Model files are written from seeds into
synth_gguf.cache_dir(), never into the tree."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from bench_tokens import HBM_PEAK, K_TOKEN_ROWS, Dev, bd, card, model, per_call, sg  # noqa: E402

F16 = bd.OUT_F16


def c_ints(v):
    return (C.c_int * len(v))(*v)


def ranges(n, times):
    return [round(n / t) for t in sorted(times, reverse=True)]


def timed(forms, n, args):
    """{name: fn}: the forms alternated --reps times -> {name: items/s of each rep, slowest first}"""
    t = {k: [] for k in forms}
    for _ in range(args.reps):
        for k, fn in forms.items():
            t[k].append(per_call(fn, args.steps, args.warmup))
    return {k + "_items_s": ranges(n, v) for k, v in t.items()}, {k: min(v) for k, v in t.items()}


def same_slabs(lib, ctx, d_multi, d_single, slab, k):
    """slab j of the _layers output == the single call's output, byte for byte, for every j"""
    a, b = np.empty(slab, np.uint8), np.empty(slab, np.uint8)
    for j in range(k):
        assert lib.lib.clip_b200_memcpy_d2h(ctx, a.ctypes.data, d_multi + j * slab, slab)
        assert lib.lib.clip_b200_memcpy_d2h(ctx, b.ctypes.data, d_single + j * slab, slab)
        if not np.array_equal(a, b):
            return False
    return True


def image_case(lib, name, geom, n, layers, flags, args, pooled=False):
    g = sg.GEOMETRIES[geom]
    rows = g.n_pos - (1 if flags & bd.TOKENS_NO_CLS else 0)
    slab = n * rows * g.v_hidden * 2
    k = len(layers)
    imgs = sg.synth_images(n, g.image_size, 7)
    path = model(lib, geom, "q4_0")
    res = {"case": name, "model": os.path.basename(path), "items": n, "layers": layers, "output_bytes": slab * k}
    ctx = lib.load(path, 0)
    dev = Dev(lib, ctx)
    try:
        d_pix = dev.alloc(imgs.nbytes, imgs)
        d_multi, d_single, d_vec = dev.alloc(slab * k), dev.alloc(slab * k), dev.alloc(n * g.proj_dim * 4)
        L, fl = c_ints(layers), c_ints([flags] * k)
        forms = {"layers_call": lambda: lib.lib.clip_b200_image_tokens_layers_device(ctx, d_pix, n, g.image_size, g.image_size, L, fl, k, F16, d_multi),
                 "single_calls": lambda: all(lib.lib.clip_b200_image_tokens_device(ctx, d_pix, n, l, flags, F16, d_single + j * slab)
                                             for j, l in enumerate(layers))}
        if pooled:
            forms["pooled_call"] = lambda: lib.lib.clip_b200_image_encode_device(ctx, d_pix, n, d_vec, True)
        r, best = timed(forms, n, args)
        res.update(r, speedup_vs_single=round(best["single_calls"] / best["layers_call"], 2),
                   slabs_equal_single_calls=same_slabs(lib, ctx, d_multi, d_single, slab, k))
    finally:
        dev.free()
        lib.free(ctx)
    return res


def k7(lib, geom, n, layers, args):
    """token-row kernel time per _layers call (all 25 layers of the first workload), from a profiling context"""
    g = sg.GEOMETRIES[geom]
    k, rows_bytes = len(layers), n * g.n_pos * g.v_hidden * (4 + 2) * len(layers)
    imgs = sg.synth_images(n, g.image_size, 7)
    os.environ["CLIP_B200_PROFILE"] = "1"
    ctx = lib.load(model(lib, geom, "q4_0"), 0)
    dev = Dev(lib, ctx)
    try:
        d_pix, d_out = dev.alloc(imgs.nbytes, imgs), dev.alloc(n * g.n_pos * g.v_hidden * 2 * k)
        L, fl = c_ints(layers), c_ints([0] * k)
        call = lambda: lib.lib.clip_b200_image_tokens_layers_device(ctx, d_pix, n, g.image_size, g.image_size, L, fl, k, F16, d_out)
        for _ in range(args.warmup):
            assert call()
        cnt = C.c_uint64(0)
        lib.lib.clip_b200_kernel_ms(ctx, K_TOKEN_ROWS, C.byref(cnt))
        for _ in range(args.steps):
            assert call()
        ms = lib.lib.clip_b200_kernel_ms(ctx, K_TOKEN_ROWS, C.byref(cnt)) / args.steps
    finally:
        dev.free()
        lib.free(ctx)
        del os.environ["CLIP_B200_PROFILE"]
    return {"row_kernel_ms_per_call": round(ms, 3), "row_kernel_launches_per_call": cnt.value // args.steps, "row_kernel_bytes": rows_bytes,
            "row_kernel_GBps": round(rows_bytes / (ms * 1e-3) / 1e9, 1), "row_kernel_hbm_share": round(rows_bytes / (ms * 1e-3) / HBM_PEAK, 3)}


def sdxl(lib, args):
    g = sg.GEOMETRIES["vit-l14"]
    n, T = 2048, 77
    ids = np.ascontiguousarray(sg.synth_tokens(n, T, 8))
    slab0, slab1 = n * T * g.t_hidden * 2, n * T * g.proj_dim * 2
    path = model(lib, "vit-l14", "q4_0")
    res = {"case": "sdxl conditioning: ViT-L/14 text q4_0, 2048 x 77, {-2: raw, -1: PROJECT}, f16", "model": os.path.basename(path), "items": n}
    ctx = lib.load(path, 0)
    dev = Dev(lib, ctx)
    try:
        d_ids = dev.alloc(ids.nbytes, ids)
        d_multi, d_single = dev.alloc(slab0 + slab1), dev.alloc(slab0 + slab1)
        L, fl = c_ints([-2, -1]), c_ints([0, bd.TOKENS_PROJECT])
        r, best = timed({"layers_call": lambda: lib.lib.clip_b200_text_tokens_layers_device(ctx, d_ids, n, T, L, fl, 2, F16, d_multi),
                         "single_calls": lambda: lib.lib.clip_b200_text_tokens_device(ctx, d_ids, n, T, -2, 0, F16, d_single) and
                         lib.lib.clip_b200_text_tokens_device(ctx, d_ids, n, T, -1, bd.TOKENS_PROJECT, F16, d_single + slab0)}, n, args)
        a, b = np.empty(slab0 + slab1, np.uint8), np.empty(slab0 + slab1, np.uint8)
        assert lib.lib.clip_b200_memcpy_d2h(ctx, a.ctypes.data, d_multi, a.nbytes)
        assert lib.lib.clip_b200_memcpy_d2h(ctx, b.ctypes.data, d_single, b.nbytes)
        res.update(r, speedup_vs_single=round(best["single_calls"] / best["layers_call"], 2), slabs_equal_single_calls=bool(np.array_equal(a, b)))
    finally:
        dev.free()
        lib.free(ctx)
    return res


def host(lib, args):
    g = sg.GEOMETRIES["vit-l14"]
    n, layers = 256, list(range(g.v_layers + 1))
    k, total = len(layers), n * g.n_pos * g.v_hidden * 2 * len(layers)
    imgs = sg.synth_images(n, g.image_size, 7)
    path = model(lib, "vit-l14", "q4_0")
    res = {"case": "host form: ViT-L/14 q4_0, b=256, all 25 hidden states, f16", "output_bytes": total}
    ctx = lib.load(path, 0)
    dev = Dev(lib, ctx)
    p = lib.lib.clip_b200_host_malloc(total)
    assert p
    try:
        pinned = np.ctypeslib.as_array((C.c_uint8 * total).from_address(p)).view(np.float16)
        pageable = np.empty(total // 2, np.float16)
        pageable.fill(0)                                           # touch every page before timing
        batch, keep = lib.make_image_batch(imgs)
        d_pix, d_out = dev.alloc(imgs.nbytes, imgs), dev.alloc(total)
        L = c_ints(layers)
        r, best = timed({"host_pinned": lambda: lib.lib.clip_b200_image_tokens_layers(ctx, C.byref(batch), L, None, k, F16, p),
                         "host_pageable": lambda: lib.lib.clip_b200_image_tokens_layers(ctx, C.byref(batch), L, None, k, F16, pageable.ctypes.data),
                         "device": lambda: lib.lib.clip_b200_image_tokens_layers_device(ctx, d_pix, n, g.image_size, g.image_size, L, None, k, F16, d_out),
                         "plain_d2h": lambda: lib.lib.clip_b200_memcpy_d2h(ctx, p, d_out, total)}, n, args)
        bound = max(best["device"], best["plain_d2h"])
        res.update(r, plain_d2h_GBps=round(total / best["plain_d2h"] / 1e9, 1), host_pinned_over_bound=round(best["host_pinned"] / bound, 3),
                   host_pageable_over_bound=round(best["host_pageable"] / bound, 3))
        assert lib.lib.clip_b200_image_tokens_layers(ctx, C.byref(batch), L, None, k, F16, p)
        assert lib.lib.clip_b200_image_tokens_layers(ctx, C.byref(batch), L, None, k, F16, pageable.ctypes.data)
        d = np.empty(total // 2, np.float16)
        assert lib.lib.clip_b200_image_tokens_layers_device(ctx, d_pix, n, g.image_size, g.image_size, L, None, k, F16, d_out)
        assert lib.lib.clip_b200_memcpy_d2h(ctx, d.ctypes.data, d_out, total)
        res["host_equals_device"] = bool(np.array_equal(pinned.view(np.uint16), d.view(np.uint16)) and np.array_equal(pageable.view(np.uint16), d.view(np.uint16)))
    finally:
        lib.lib.clip_b200_host_free(p)
        dev.free()
        lib.free(ctx)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", choices=["all", "llava", "sdxl", "host"])
    args = ap.parse_args()
    lib = bd.ClipLib(bd.PRODUCT_LIB)
    gpu = card()
    print("card, power limit:", gpu, flush=True)
    every = list(range(sg.GEOMETRIES["vit-l14"].v_layers + 1))
    cases = []
    if args.only in (None, "all"):
        cases.append(lambda: dict(image_case(lib, "all hidden states: ViT-L/14 q4_0, b=256, 25 layers, f16", "vit-l14", 256, every, 0, args, pooled=True),
                                  **k7(lib, "vit-l14", 256, every, args)))
    if args.only in (None, "llava"):
        cases.append(lambda: image_case(lib, "llava multi-layer: ViT-L/14@336 q4_0, b=256, layers -2 -5 -8 -11, NO_CLS, f16", "vit-l14-336", 256,
                                        [-2, -5, -8, -11], bd.TOKENS_NO_CLS, args))
    if args.only in (None, "sdxl"):
        cases.append(lambda: sdxl(lib, args))
    if args.only in (None, "host"):
        cases.append(lambda: host(lib, args))
    ok = True
    for case in cases:
        r = case()
        r["gpu"] = gpu
        ok = ok and r.get("slabs_equal_single_calls", True) and r.get("host_equals_device", True)
        print(json.dumps(r), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
