#!/usr/bin/env python
"""K3 alone at the production attention shapes, through the clip_b200_debug_attention_hd hook: one launch per call, CUDA-event time.

    python tools/bench_k3_shapes.py [--lib PATH] [--reps 5]

Each shape runs `reps` calls (the hook times the last of three launches per call); the line reports the median of all but the first
call.  Useful FLOP: 4 T^2 dh per (sequence, head), halved for causal (dh the real head_dim: 104, not the 112 columns K3 multiplies).  HBM bytes: the fused QKV matrix read once and O written
once (3 + 1 rows of H dh 16-bit values per token), against the H100 SXM data sheet's 3.35 TB/s.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "clip.cpp_b200"))
import binding  # noqa: E402

HBM_PEAK = 3.35e12
# (name, nseq, T, heads, head_dim, causal): one micro-batch of each config (api.cu default_micro_batch)
SHAPES = [("vit-l14 (headline, cfg3)", 256, 257, 16, 64, 0),
          ("vit-b32 (cfg2)", 256, 50, 12, 64, 0),
          ("text (cfg4)", 683, 77, 12, 64, 1),
          ("vit-h14", 256, 257, 16, 80, 0),
          ("vit-bigg14", 256, 257, 16, 104, 0),
          ("vit-l14-336", 64, 577, 16, 64, 0)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=binding.PRODUCT_LIB)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    lib = binding.ClipLib(args.lib)
    rng = np.random.default_rng(0)
    fp = C.POINTER(C.c_float)
    out = {"lib": os.path.basename(args.lib), "shapes": []}
    for name, nseq, T, H, dh, causal in SHAPES:
        qkv = rng.standard_normal((nseq * T, 3 * H * dh)).astype(np.float32)
        qkv[:, : H * dh] *= 3.0 / np.sqrt(dh)
        o = np.empty((nseq * T, H * dh), np.float32)
        ms = []
        for _ in range(args.reps):
            t = C.c_float(0)
            rc = lib.lib.clip_b200_debug_attention_hd(1, nseq, T, H, dh, causal, 0, qkv.ctypes.data_as(fp), o.ctypes.data_as(fp),
                                                      C.byref(t))
            assert rc == 0, lib.last_error()
            ms.append(t.value)
        med = float(np.median(ms[1:]))
        flop = 4.0 * nseq * H * T * T * dh * (0.5 if causal else 1.0)
        hbm = 4.0 * nseq * T * H * dh * 2
        rec = {"shape": name, "nseq": nseq, "T": T, "H": H, "dh": dh, "causal": causal, "ms": [round(v, 4) for v in ms],
               "median_ms": round(med, 4), "tflops": round(flop / med / 1e9, 1), "hbm_gbs": round(hbm / med / 1e6, 1),
               "hbm_share": round(hbm / med * 1e3 / HBM_PEAK, 3)}
        out["shapes"].append(rec)
        print(json.dumps(rec), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
