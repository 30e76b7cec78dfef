#!/usr/bin/env python
"""ViT-H/14 q4_0 image-encode throughput, b = 512 per GPU: bench.py's image path and JSON line, on the ViT-H/14 geometry.

    python tools/bench_vit_h14.py --gpus 1 --steps 10 --warmup 3 [--no-cpu-baseline] [--dump-outputs DIR]

Every bench.py option applies.  The FLOPs entry is computed like bench.py's ViT-L/14 one: per layer 2·T·(4h² + 2h·ff) for the GEMMs
plus 4·T²·dh·H for attention, plus the patch embedding and the projection (T = 257, h = 1280, ff = 5120, H = 16, dh = 80, 32 layers).
The parity field compares 3 images with the reference's tests/golden/vit-h14-s1234.npz.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

bench.FLOPS[("vit-h14", "image")] = (334_590_279_680, 32 * 338_170_880)
bench.CONFIGS["vit-h14"] = dict(kind="image", geom="vit-h14", ftype="q4_0", batch=512,
                                workload="ViT-H/14 q4_0 image encode (h=1280, head_dim 80), b=512 per GPU, 224x224x3 synthetic")

if __name__ == "__main__":
    if "--config" not in sys.argv:
        sys.argv += ["--config", "vit-h14"]
    bench.main()
