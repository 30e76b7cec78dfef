#!/usr/bin/env python
"""Attention probabilities (CLIP_B200_TOKENS_ATTENTION entries, kernel K9) on the workloads that read them.

    python tools/bench_attention_maps.py [--steps 3] [--warmup 1] [--reps 5] [--only prumerge|maps]

  prumerge  ViT-L/14@336 q4_0, b = 256 device-resident images, f16: one _layers call {-2 NO_CLS, -2 ATTENTION | ATTENTION_CLS} (the
            patch rows and the CLS row's attention a token-reduction front end ranks them by) against {-2 NO_CLS} alone, alternated.
  maps      ViT-L/14 q4_0, b = 256, all 24 full attention maps, f16, device form (24 x 541 MB): the call, and from a profiling
            context (CLIP_B200_PROFILE=1) K9's CUDA-event time per launch (kind 6 of clip_b200_kernel_ms), the bytes it writes
            and their rate as a share of the H100 SXM data sheet's 3.35 TB/s.  The floor is 541 MB / 3.35 TB/s = 0.16 ms per layer.

Host clock around calls that end in a device synchronise; the compared forms alternate --reps times and every rate is printed,
slowest first.  The card's name, power limit and SM clock are read in the same call.  One JSON line per case.  Model files are
written from seeds into synth_gguf.cache_dir(), never into the tree."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from bench_tokens import HBM_PEAK, Dev, bd, model, per_call, sg  # noqa: E402

F16 = bd.OUT_F16
K_ATTN_PROBS = 6
ATT_CLS = bd.TOKENS_ATTENTION | bd.TOKENS_ATTENTION_CLS


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    if q.returncode != 0:
        raise SystemExit("nvidia-smi failed: this benchmark needs the GPU it measures")
    return q.stdout.strip().splitlines()[0]


def c_ints(v):
    return (C.c_int * len(v))(*v)


def prumerge(lib, args):
    g = sg.GEOMETRIES["vit-l14-336"]
    n = 256
    rows = n * (g.n_pos - 1) * g.v_hidden * 2
    cls = n * g.v_heads * g.n_pos * 2
    imgs = sg.synth_images(n, g.image_size, 7)
    path = model(lib, "vit-l14-336", "q4_0")
    res = {"case": "prumerge: ViT-L/14@336 q4_0, b=256, {-2 NO_CLS, -2 ATTENTION|CLS} against {-2 NO_CLS}, f16",
           "model": os.path.basename(path), "items": n, "cls_row_bytes_per_image": cls // n}
    ctx = lib.load(path, 0)
    dev = Dev(lib, ctx)
    try:
        d_pix, d_out = dev.alloc(imgs.nbytes, imgs), dev.alloc(rows + 16 + cls)
        S = g.image_size
        with_att = lambda: lib.lib.clip_b200_image_tokens_layers_device(ctx, d_pix, n, S, S, c_ints([-2, -2]), c_ints([bd.TOKENS_NO_CLS, ATT_CLS]), 2, F16, d_out)
        rows_only = lambda: lib.lib.clip_b200_image_tokens_layers_device(ctx, d_pix, n, S, S, c_ints([-2]), c_ints([bd.TOKENS_NO_CLS]), 1, F16, d_out)
        t = {"with_attention": [], "rows_only": []}
        for _ in range(args.reps):
            t["with_attention"].append(per_call(with_att, args.steps, args.warmup))
            t["rows_only"].append(per_call(rows_only, args.steps, args.warmup))
        for k, v in t.items():
            res[k + "_items_s"] = [round(n / x) for x in sorted(v, reverse=True)]
        res["slowdown"] = round(min(t["with_attention"]) / min(t["rows_only"]) - 1, 4)
    finally:
        dev.free()
        lib.free(ctx)
    return res


def maps(lib, args):
    g = sg.GEOMETRIES["vit-l14"]
    n, layers = 256, list(range(1, g.v_layers + 1))
    k = len(layers)
    per_layer = n * g.v_heads * g.n_pos * g.n_pos * 2
    imgs = sg.synth_images(n, g.image_size, 7)
    path = model(lib, "vit-l14", "q4_0")
    res = {"case": "all attention maps: ViT-L/14 q4_0, b=256, 24 layers, f16, device form", "model": os.path.basename(path), "items": n,
           "bytes_per_layer": per_layer}
    os.environ["CLIP_B200_PROFILE"] = "1"
    ctx = lib.load(path, 0)
    dev = Dev(lib, ctx)
    try:
        d_pix, d_out = dev.alloc(imgs.nbytes, imgs), dev.alloc(per_layer * k)
        S = g.image_size
        L, fl = c_ints(layers), c_ints([bd.TOKENS_ATTENTION] * k)
        call = lambda: lib.lib.clip_b200_image_tokens_layers_device(ctx, d_pix, n, S, S, L, fl, k, F16, d_out)
        for _ in range(args.warmup):
            assert call()
        cnt = C.c_uint64(0)
        lib.lib.clip_b200_kernel_ms(ctx, K_ATTN_PROBS, C.byref(cnt))
        for _ in range(args.steps):
            assert call()
        ms = lib.lib.clip_b200_kernel_ms(ctx, K_ATTN_PROBS, C.byref(cnt))
        launches = cnt.value
        per = ms / launches
        call_s = per_call(call, args.steps, 0)
        res.update(k9_ms_per_launch=round(per, 4), k9_launches=launches, k9_GBps=round(per_layer * launches / (ms * 1e-3) / 1e9, 1),
                   k9_hbm_share=round(per_layer * launches / (ms * 1e-3) / HBM_PEAK, 3), floor_ms_per_layer=round(per_layer / HBM_PEAK * 1e3, 3),
                   call_ms_profiled=round(call_s * 1e3, 1))
    finally:
        dev.free()
        lib.free(ctx)
        del os.environ["CLIP_B200_PROFILE"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", choices=["prumerge", "maps"])
    args = ap.parse_args()
    lib = bd.ClipLib(bd.PRODUCT_LIB)
    gpu = card()
    print("card, power limit, SM clock, max SM clock:", gpu, flush=True)
    cases = []
    if args.only in (None, "prumerge"):
        cases.append(lambda: prumerge(lib, args))
    if args.only in (None, "maps"):
        cases.append(lambda: maps(lib, args))
    for case in cases:
        r = case()
        r["gpu"] = gpu
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
