"""Writes tests/golden/pos_resample_torch.npz: position tables resampled by torch exactly as HF's interpolate_pos_encoding does it
(CLIPVisionEmbeddings: the patch rows as a [1, h, g, g] image, F.interpolate(size=(gh, gw), mode="bicubic", align_corners=False),
back to [gh * gw, h] rows), on the CPU in float32.  tests/test_pos_resample.py checks the fp64 restatement of K8 against it.

    python tests/golden/make_pos_resample_golden.py
"""
import os

import numpy as np
import torch

# name -> (g, gh, gw): up, down, rectangular both ways, to a single patch, identity
CASES = {"up_7_12": (7, 12, 12), "down_16_7": (16, 7, 7), "rect_16_24x8": (16, 24, 8), "rect_4_3x6": (4, 3, 6),
         "to_1x1": (7, 1, 1), "identity_7": (7, 7, 7)}
H = 64


def main():
    rng = np.random.default_rng(2024)
    out = {}
    for name, (g, gh, gw) in CASES.items():
        table = (rng.standard_normal((g * g, H)) * 0.05).astype(np.float32)
        x = torch.from_numpy(table).reshape(1, g, g, H).permute(0, 3, 1, 2)
        y = torch.nn.functional.interpolate(x, size=(gh, gw), mode="bicubic", align_corners=False)
        out[name + "_in"] = table
        out[name + "_out"] = y.permute(0, 2, 3, 1).reshape(gh * gw, H).numpy().astype(np.float32)
        out[name + "_shape"] = np.array([g, gh, gw], np.int32)
    out["torch_version"] = np.array(torch.__version__)
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "pos_resample_torch.npz"), **out)


if __name__ == "__main__":
    main()
