#!/usr/bin/env python
"""K1 alone at the ViT-L/14 layer shapes, through the clip_b200_debug_gemm hook: one launch per call, CUDA-event time.

    python tools/bench_k1_shapes.py [--lib PATH] [--reps 5]

M = 25344 tokens = 99 token tiles of 256 (or 132 of 192): whole waves on 132 SMs for every shape below, q4_0 weights, bf16 operands.
Each shape runs `reps` times; the line reports the median of all but the first call.  REDADD32 and STORE32 at the same shape differ
only in the epilogue (read-add-write of the fp32 residual against a plain fp32 store), so their gap is what the residual add costs.

Next to TFLOP/s each line gives the bytes the launch's tiles read from L2 and their rate: every feature tile reads the activations
X once (M K 2 B), every token tile reads the packed weights once (N K / 32 blocks of 18 B), and the residual add reads x once (M N
4 B).  The tile comes from csrc/gemm.h; --tile FxT gives it for a library built with another one (e.g. --tile 128x192).
"""
import argparse
import ctypes as C
import json
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "clip.cpp_b200"))
import binding  # noqa: E402

EPI = {"STORE16": 0, "GELU16": 1, "QGELU16": 2, "REDADD32": 3, "STORE32": 4}
# (N, K, epilogue); the last four are the FC1 GEMMs of ViT-L/14 (4096 x 1024) and ViT-H/14 (5120 x 1280) under both GELUs
SHAPES = [(1024, 1024, "REDADD32"), (1024, 1024, "STORE32"), (1024, 4096, "REDADD32"), (1024, 4096, "STORE32"),
          (3072, 1024, "STORE16"), (4096, 1024, "QGELU16"), (4096, 1024, "GELU16"), (5120, 1280, "GELU16"), (5120, 1280, "QGELU16")]


def q4_0_rows(N, K, rng):
    """random ggml q4_0 rows: per 32 weights an fp16 scale and 16 bytes of nibbles"""
    blk = np.empty((N, K // 32, 18), np.uint8)
    blk[:, :, 0:2] = (rng.uniform(0.002, 0.02, (N, K // 32)).astype(np.float16)).view(np.uint8).reshape(N, K // 32, 2)
    blk[:, :, 2:] = rng.integers(0, 256, (N, K // 32, 16), dtype=np.uint8)
    return blk.tobytes()


def header_tile():
    """(features, tokens) per CTA tile: GEMM_BM and GEMM_BN of csrc/gemm.h"""
    src = open(os.path.join(ROOT, "clip.cpp_b200", "csrc", "gemm.h")).read()
    return tuple(int(re.search(r"constexpr int %s = (\d+);" % n, src).group(1)) for n in ("GEMM_BM", "GEMM_BN"))


def l2_read_bytes(M, N, K, epi, tile):
    bf, bt = tile
    x = -(-N // bf) * M * K * 2
    w = -(-M // bt) * N * (K // 32) * 18
    r = M * N * 4 if epi == "REDADD32" else 0
    return x + w + r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=binding.PRODUCT_LIB)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--M", type=int, default=25344)
    ap.add_argument("--tile", default="", help="FxT: the CTA tile (features x tokens) of the library under test (default: csrc/gemm.h)")
    ap.add_argument("--epi", default="", help="comma-separated epilogues to run (default: every shape)")
    args = ap.parse_args()
    lib = binding.ClipLib(args.lib)
    rng = np.random.default_rng(0)
    M = args.M
    fp = C.POINTER(C.c_float)
    tile = tuple(int(v) for v in args.tile.split("x")) if args.tile else header_tile()
    out = {"lib": os.path.basename(args.lib), "M": M, "tile": "%dx%d" % tile, "shapes": []}
    for N, K, epi in SHAPES:
        if args.epi and epi not in args.epi.split(","):
            continue
        x = rng.standard_normal((M, K)).astype(np.float32)
        raw = np.frombuffer(q4_0_rows(N, K, rng), np.uint8)
        bias = rng.standard_normal(N).astype(np.float32)
        resid = rng.standard_normal((M, N)).astype(np.float32) if epi == "REDADD32" else None
        y = np.empty((M, N), np.float32)
        ms = []
        for _ in range(args.reps):
            t = C.c_float(0)
            rc = lib.lib.clip_b200_debug_gemm(2, 1, M, N, K, EPI[epi], 0, x.ctypes.data_as(fp), raw.ctypes.data,
                                              bias.ctypes.data_as(fp), resid.ctypes.data_as(fp) if resid is not None else None,
                                              y.ctypes.data_as(fp), C.byref(t))
            assert rc == 0, lib.lib.clip_b200_last_error()
            ms.append(t.value)
        med = float(np.median(ms[1:]))
        rec = {"N": N, "K": K, "epi": epi, "ms": [round(v, 4) for v in ms], "median_ms": round(med, 4),
               "tflops": round(2.0 * M * N * K / med / 1e9, 1)}
        l2 = l2_read_bytes(M, N, K, epi, tile)
        rec.update(l2_read_gb=round(l2 / 1e9, 3), l2_tbps=round(l2 / med / 1e9, 2))
        out["shapes"].append(rec)
        print(json.dumps(rec), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
