"""Generates the golden fixture of the true ViT-bigG/14 geometry (vit-bigg14: 48 vision layers of 1664 / 8192 with 16 heads of 104,
32 text layers of 1280 / 5120 with 20 heads, projection 1280) from the CPU ORACLE (oracle/oracle.py).  The reference refuses this
file (1 293 tensors), so it cannot produce the vectors itself; the oracle is pinned against the reference at the same vision layer in
tests/test_oracle_pin_bigg.py (bigg-w1664).  The fixture records this in its `producer` entry.  Same seeds, inputs and quantizer as
make_golden.py (the product's clip_model_quantize, byte-identical to the reference's: tests/test_host_side.py):

    python tests/golden/make_golden_bigg_oracle.py      # a 5 GB f16 and a 1.5 GB q4_0 file; a few minutes on 8 cores
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "clip.cpp_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import binding as bd          # noqa: E402
import make_golden as mg      # noqa: E402
import oracle as orc          # noqa: E402
import synth_gguf as sg       # noqa: E402

GEOM, FTYPES, N_IMG, N_TXT = "vit-bigg14", ["f16", "q4_0"], 2, 2


def main():
    prod = bd.ClipLib(bd.PRODUCT_LIB)
    g = sg.GEOMETRIES[GEOM]
    imgs = sg.synth_images(N_IMG, g.image_size, mg.IMG_SEED)
    seqs = mg.token_seqs(N_TXT)
    out = {"seed": mg.SEED, "img_seed": mg.IMG_SEED, "tok_seed": mg.TOK_SEED, "n_img": N_IMG, "n_txt": N_TXT,
           "tok_lens": np.array([len(s) for s in seqs]),
           "producer": "oracle/oracle.py (CPU oracle; the reference refuses this 1 293-tensor file)"}
    for ft in FTYPES:
        path = mg.ensure_model(GEOM, ft, prod.quantize)
        m = orc.OracleModel(path)
        out["sha_" + ft] = sg.sha256_file(path)
        out["img_" + ft] = np.stack([m.encode_image(im) for im in imgs]).astype(np.float32)
        out["txt_" + ft] = np.stack([m.encode_text(s) for s in seqs]).astype(np.float32)
        print("%s %-5s |img0|=%.4f" % (GEOM, ft, float(np.linalg.norm(out["img_" + ft][0]))), flush=True)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "%s-s%d.npz" % (GEOM, mg.SEED)), **out)


if __name__ == "__main__":
    main()
