"""Generates the ViT-bigG/14 golden fixture by running the REFERENCE ITSELF, with the machinery of make_golden.py (same seeds, inputs,
quantizer and one-process-per-model reference runs).  Needs the reference built into oracle/_ref:

    python tests/golden/make_golden_bigg.py        # bigg-w1664: the bigG vision layer (1664 wide, ff 8192, head_dim 104) at the
                                                   # huge tensor counts; a 2.5 GB f16 file, about a minute per file type
The true vit-bigg14 geometry has 1 293 tensors, which the reference refuses; its fixture comes from the oracle
(tests/golden/make_golden_bigg_oracle.py).
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg      # noqa: E402

BIGG = {"bigg-w1664": dict(ftypes=["f16", "q4_0", "q5_1", "q8_0"], n_img=2, n_txt=2)}

if __name__ == "__main__":
    mg.PLAN, mg.PLAN_FULL = {}, BIGG
    if "--only" not in sys.argv:
        sys.argv += ["--only", "bigg-w1664"]
    mg.main()
