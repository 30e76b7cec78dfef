#!/usr/bin/env python
"""ViT-bigG/14 image-encode throughput, b = 512 per GPU: bench.py's image path and JSON line, on the ViT-bigG/14 geometry.

    python tools/bench_vit_bigg14.py --gpus 1 --steps 10 --warmup 3 [--config vit-bigg14-f16] [--no-cpu-baseline] [--dump-outputs DIR]

Every bench.py option applies; --config vit-bigg14 (q4_0, the default) or vit-bigg14-f16.  The FLOPs entry is computed like
bench.py's ViT-L/14 one: per layer 2·T·(4h² + 2h·ff) for the GEMMs plus 4·T²·dh·H for attention, plus the patch embedding and the
projection (T = 257, h = 1664, ff = 8192, H = 16, dh = 104, 48 layers, projection 1280).  These are the model's FLOPs: the 8 zero
columns per head that the loader adds to the QKV projection (+7.7 % on that GEMM) are not counted.  The reference refuses the
1 293-tensor file; the parity field compares 2 images with tests/golden/vit-bigg14-s1234.npz, which the CPU oracle produced.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

T, H_, FF, HEADS, DH, LAYERS, P, PROJ = 257, 1664, 8192, 16, 104, 48, 14, 1280
ATTN = 4 * T * T * DH * HEADS
LAYER = 2 * T * (4 * H_ * H_ + 2 * H_ * FF) + ATTN
TOTAL = LAYERS * LAYER + 2 * (T - 1) * 3 * P * P * H_ + 2 * H_ * PROJ
assert TOTAL == 967_496_032_256

bench.FLOPS[("vit-bigg14", "image")] = (TOTAL, LAYERS * ATTN)
for name, ft in (("vit-bigg14", "q4_0"), ("vit-bigg14-f16", "f16")):
    bench.CONFIGS[name] = dict(kind="image", geom="vit-bigg14", ftype=ft, batch=512,
                               workload="ViT-bigG/14 %s image encode (h=1664, head_dim 104), b=512 per GPU, 224x224x3 synthetic" % ft)

_parity_check = bench.parity_check


def parity_check(b):
    """bench.py's parity field, labelled with where this geometry's fixture comes from"""
    r = _parity_check(b)
    if r is not None:
        r["against"] = "CPU oracle embeddings (tests/golden/vit-bigg14-s1234.npz, produced by oracle/oracle.py)"
    return r


bench.parity_check = parity_check

if __name__ == "__main__":
    if "--config" not in sys.argv:
        sys.argv += ["--config", "vit-bigg14"]
    bench.main()
