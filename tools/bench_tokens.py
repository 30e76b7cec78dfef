#!/usr/bin/env python
"""Per-token hidden states at the two workloads they exist for, next to the pooled-embedding path on the same inputs.

    python tools/bench_tokens.py [--steps 10] [--warmup 3] [--reps 3] [--only llava|sd]

  (a) LLaVA-1.5's front end: ViT-L/14@336 (h 1024, 24 layers, T 577), q4_0 and f16 files, b = 256 device-resident images,
      layer -2, CLIP_B200_TOKENS_NO_CLS, f16 rows (256 x 576 x 1024).  Pooled: clip_b200_image_encode_device, normalised.
  (b) Stable Diffusion 1.x conditioning: the ViT-L/14 text tower (h 768, 12 layers), 2048 x 77 ids, layer -1,
      CLIP_B200_TOKENS_POST_LN, f16 rows.  Pooled: clip_b200_text_encode_device, normalised.

Per case it prints items/s of both paths (host clock around calls that end in a device synchronise, the two paths alternated
--reps times), the token-row kernel's CUDA-event time per call (kernel kind 4 of clip_b200_kernel_ms, from a second context with
CLIP_B200_PROFILE=1 so the timed context pays no event records), its bytes (fp32 rows read, output rows written) and GB/s against the
H100 SXM data sheet's 3.35 TB/s, and whether two runs gave the same output bytes.  The card's name and power limit are read in the
same call.  One JSON line per case.  Model files are written from seeds into synth_gguf.cache_dir(), never into the tree."""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "clip.cpp_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import binding as bd  # noqa: E402
import synth_gguf as sg  # noqa: E402

HBM_PEAK = 3.35e12
K_TOKEN_ROWS = 4


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        raise SystemExit("nvidia-smi failed: this benchmark needs the GPU it measures")
    return q.stdout.strip().splitlines()[0]


def model(lib, geom, ft):
    path = sg.model_path(geom, 1234, ft)
    if not os.path.exists(path):
        f16 = sg.model_path(geom, 1234, "f16")
        if not os.path.exists(f16):
            sg.write_model(f16, sg.GEOMETRIES[geom], 1234, 1)
        if ft != "f16":
            assert lib.quantize(f16, path + ".tmp", {"q4_0": 2, "q8_0": 8}[ft]), lib.last_error()
            os.replace(path + ".tmp", path)
    return path


class Dev:
    """device buffers of one context, freed together"""

    def __init__(self, lib, ctx):
        self.lib, self.ctx, self.ptrs = lib, ctx, []

    def alloc(self, nbytes, host=None):
        p = self.lib.lib.clip_b200_device_malloc(self.ctx, nbytes)
        assert p, self.lib.last_error()
        self.ptrs.append(p)
        if host is not None:
            assert self.lib.lib.clip_b200_memcpy_h2d(self.ctx, p, host.ctypes.data, host.nbytes)
        return p

    def free(self):
        for p in self.ptrs:
            self.lib.lib.clip_b200_device_free(self.ctx, p)


def per_call(fn, steps, warmup):
    for _ in range(warmup):
        assert fn()
    t0 = time.perf_counter()
    for _ in range(steps):
        assert fn()
    return (time.perf_counter() - t0) / steps


def run_case(lib, name, path, n, make_calls, out_bytes, row_bytes, args):
    """make_calls(ctx, dev) -> (tokens(), pooled(), fetch()): the two calls on device buffers and a copy of the token output"""
    res = {"case": name, "model": os.path.basename(path), "items": n}
    ctx = lib.load(path, 0)
    dev = Dev(lib, ctx)
    try:
        tokens, pooled, fetch = make_calls(ctx, dev)
        t_tok, t_pool = [], []
        for _ in range(args.reps):                       # alternate the two paths
            t_tok.append(per_call(tokens, args.steps, args.warmup))
            t_pool.append(per_call(pooled, args.steps, args.warmup))
        assert tokens()
        h1 = hashlib.sha256(fetch()).hexdigest()
        assert tokens()
        h2 = hashlib.sha256(fetch()).hexdigest()
        res.update(tokens_items_s=[round(n / t) for t in sorted(t_tok, reverse=True)],
                   pooled_items_s=[round(n / t) for t in sorted(t_pool, reverse=True)],
                   bit_identical_runs=h1 == h2, output_sha256=h1[:16], output_bytes=out_bytes)
    finally:
        dev.free()
        lib.free(ctx)
    os.environ["CLIP_B200_PROFILE"] = "1"
    ctx = lib.load(path, 0)
    dev = Dev(lib, ctx)
    try:
        tokens, _, _ = make_calls(ctx, dev)
        for _ in range(args.warmup):
            assert tokens()
        cnt = C.c_uint64(0)
        lib.lib.clip_b200_kernel_ms(ctx, K_TOKEN_ROWS, C.byref(cnt))
        for _ in range(args.steps):
            assert tokens()
        ms = lib.lib.clip_b200_kernel_ms(ctx, K_TOKEN_ROWS, C.byref(cnt)) / args.steps
        res.update(row_kernel_ms=round(ms, 4), row_kernel_launches_per_call=cnt.value // args.steps, row_kernel_bytes=row_bytes,
                   row_kernel_GBps=round(row_bytes / (ms * 1e-3) / 1e9, 1), row_kernel_hbm_share=round(row_bytes / (ms * 1e-3) / HBM_PEAK, 3))
    finally:
        dev.free()
        lib.free(ctx)
        del os.environ["CLIP_B200_PROFILE"]
    return res


def llava(lib, ft, args):
    g = sg.GEOMETRIES["vit-l14-336"]
    n, T, h = 256, g.n_pos, g.v_hidden
    imgs = sg.synth_images(n, g.image_size, 7)
    out_bytes = n * (T - 1) * h * 2

    def calls(ctx, dev):
        d_pix = dev.alloc(imgs.nbytes, imgs)
        d_tok = dev.alloc(out_bytes)
        d_vec = dev.alloc(n * g.proj_dim * 4)
        host = np.empty(out_bytes, np.uint8)

        def fetch():
            assert lib.lib.clip_b200_memcpy_d2h(ctx, host.ctypes.data, d_tok, out_bytes)
            return host.tobytes()
        return (lambda: lib.lib.clip_b200_image_tokens_device(ctx, d_pix, n, -2, bd.TOKENS_NO_CLS, bd.OUT_F16, d_tok),
                lambda: lib.lib.clip_b200_image_encode_device(ctx, d_pix, n, d_vec, True), fetch)
    return run_case(lib, "llava-1.5 front end: ViT-L/14@336 %s, b=256, layer -2, NO_CLS, f16" % ft, model(lib, "vit-l14-336", ft), n,
                    calls, out_bytes, n * (T - 1) * h * (4 + 2), args)


def sd(lib, ft, args):
    g = sg.GEOMETRIES["vit-l14"]
    n, T, h = 2048, 77, g.t_hidden
    ids = np.ascontiguousarray(sg.synth_tokens(n, T, 8))
    out_bytes = n * T * h * 2

    def calls(ctx, dev):
        d_ids = dev.alloc(ids.nbytes, ids)
        d_tok = dev.alloc(out_bytes)
        d_vec = dev.alloc(n * g.proj_dim * 4)
        host = np.empty(out_bytes, np.uint8)

        def fetch():
            assert lib.lib.clip_b200_memcpy_d2h(ctx, host.ctypes.data, d_tok, out_bytes)
            return host.tobytes()
        return (lambda: lib.lib.clip_b200_text_tokens_device(ctx, d_ids, n, T, -1, bd.TOKENS_POST_LN, bd.OUT_F16, d_tok),
                lambda: lib.lib.clip_b200_text_encode_device(ctx, d_ids, None, n, T, d_vec, True), fetch)
    return run_case(lib, "sd-1.x conditioning: ViT-L/14 text %s, 2048 x 77, layer -1, POST_LN, f16" % ft, model(lib, "vit-l14", ft), n,
                    calls, out_bytes, n * T * h * (4 + 2), args)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", choices=["llava", "sd"])
    args = ap.parse_args()
    lib = bd.ClipLib(bd.PRODUCT_LIB)
    gpu = card()
    print("card, power limit:", gpu, flush=True)
    cases = []
    if args.only in (None, "llava"):
        cases += [lambda: llava(lib, "q4_0", args), lambda: llava(lib, "f16", args)]
    if args.only in (None, "sd"):
        cases += [lambda: sd(lib, "f16", args), lambda: sd(lib, "q4_0", args)]
    ok = True
    for case in cases:
        r = case()
        r["gpu"] = gpu
        ok = ok and r["bit_identical_runs"]
        print(json.dumps(r), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
