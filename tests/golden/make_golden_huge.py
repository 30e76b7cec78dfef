"""Generates the ViT-H/14 golden fixtures by running the REFERENCE ITSELF, with the machinery of make_golden.py (same seeds, inputs,
quantizer and one-process-per-model reference runs).  Run in the build container (needs /root/reference built into oracle/_ref):

    python tests/golden/make_golden_huge.py                     # huge-w640 (huge tensor counts at width 640, head_dim 80)
    python tests/golden/make_golden_huge.py --only vit-h14      # the true LAION ViT-H/14 geometry (a 2 GB f16 file; minutes)
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg      # noqa: E402

HUGE = {
    "huge-w640": dict(ftypes=["f16", "q4_0", "q5_1", "q8_0"], n_img=2, n_txt=2),
    "vit-h14": dict(ftypes=["f16", "q4_0", "q8_0"], n_img=3, n_txt=3),
}

if __name__ == "__main__":
    mg.PLAN, mg.PLAN_FULL = {}, HUGE
    if "--only" not in sys.argv:
        sys.argv += ["--only", "huge-w640"]
    mg.main()
