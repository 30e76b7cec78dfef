"""Writes tests/golden/reference_runs.npz: what the unmodified reference (oracle/_ref, built by oracle/Makefile) returns for the inputs
of the tests that compare against it -- oracle embeddings (test_oracle_pin), tokenizer / preprocess / PNG and JPEG decode (test_host_side) and
the scoring entry points (test_gpu_scoring).  The tests read this file instead of running the reference, so they need nothing outside
the repository.  Re-run after changing any of those inputs:

    python tests/golden/make_reference_runs.py
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (os.path.join(ROOT, "clip.cpp_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import binding as bd  # noqa: E402
import ref_run  # noqa: E402
import synth_gguf as sg  # noqa: E402
import test_gpu_scoring as ts  # noqa: E402
import test_host_side as th  # noqa: E402
import test_oracle_pin as to  # noqa: E402
from _util import model_file  # noqa: E402


def main():
    assert ref_run.available(), "build oracle/_ref first (make -C oracle ref)"
    prod = bd.ClipLib(bd.PRODUCT_LIB)
    out = {}
    # test_oracle_pin.test_oracle_matches_live_reference
    imgs, seqs = to.live_inputs()
    for ft in to.LIVE_FTYPES:
        path = model_file("tiny", ft, prod)
        r = ref_run.run_reference(path, imgs, seqs, n_threads=2, normalize=False)
        out["oracle_%s_img" % ft], out["oracle_%s_txt" % ft] = r["img"], r["txt"]
        out["oracle_%s_sha" % ft] = np.array(sg.sha256_file(path))
    # test_host_side.test_tokenizer_and_preprocess_match_live_reference (the reference in its own process, as for every run here)
    ref = bd.ClipLib(ref_run.REF_LIB)
    path = model_file("tiny", "f16", prod)
    ctx = ref.load(path, 0)
    for i, t in enumerate(th.LIVE_TEXTS):
        out["tok_%d" % i] = np.array([int(v) for v in ref.tokenize(ctx, t)], np.int32)
    out["preprocess"] = np.asarray(ref.preprocess(ctx, th.live_u8()), np.float32)
    # test_host_side.test_png_decode_matches_live_reference
    with tempfile.TemporaryDirectory() as td:
        for name, im in th.live_pngs().items():
            p = os.path.join(td, name)
            im.save(p)
            out["png_" + name] = th._load_file(ref, p)
    # test_host_side.test_jpeg_decode_matches_live_reference
    import hashlib
    keys, fsha, rsha = [], [], []
    with tempfile.TemporaryDirectory() as td:
        for key, p in th.live_jpeg_cases(td):
            px = th._load_file(ref, p)
            keys.append(key)
            fsha.append(hashlib.sha256(open(p, "rb").read()).hexdigest())
            rsha.append(hashlib.sha256(px.tobytes()).hexdigest())
    out["jpeg_keys"], out["jpeg_file_sha"], out["jpeg_ref_sha"] = np.array(keys), np.array(fsha), np.array(rsha)
    # test_gpu_scoring.test_compare_and_zero_shot_label_match_live_reference
    for ft in ("f16", "q4_0"):
        path = model_file("tiny", ft, prod)
        r = ref_run.run_reference(path, u8_image=ts.live_u8(), texts=ts.TEXTS, n_threads=4)
        out["scoring_%s_cmp" % ft], out["scoring_%s_zsl_scores" % ft], out["scoring_%s_zsl_idx" % ft] = r["cmp"], r["zsl_scores"], r["zsl_idx"]
        out["scoring_%s_sha" % ft] = np.array(sg.sha256_file(path))
    np.savez_compressed(os.path.join(HERE, "reference_runs.npz"), **out)
    print("wrote", os.path.join(HERE, "reference_runs.npz"), sorted(out))


if __name__ == "__main__":
    main()
