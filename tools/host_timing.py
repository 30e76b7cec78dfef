"""Host-side members of the interface timed next to the reference's own implementation (no GPU involved): clip_image_load_from_file
(JPEG) and clip_image_preprocess's arithmetic.  Needs oracle/_ref/libclip_ref.so (make -C oracle ref) and PIL for the test images.

    python tools/host_timing.py            -> a markdown table on stdout
"""
import ctypes as C
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "clip.cpp_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import binding as bd          # noqa: E402
import ref_run                # noqa: E402
from _util import model_file  # noqa: E402


def load_ms(lib, path, reps):
    fn = lib.lib.clip_image_load_from_file
    fn.restype = C.c_bool
    fn.argtypes = [C.c_char_p, C.POINTER(bd.clip_image_u8)]
    lib.lib.clip_image_u8_clean.argtypes = [C.POINTER(bd.clip_image_u8)]
    best = 1e9
    for _ in range(reps):
        im = bd.clip_image_u8()
        t0 = time.perf_counter()
        assert fn(path.encode(), C.byref(im))
        best = min(best, (time.perf_counter() - t0) * 1e3)
        lib.lib.clip_image_u8_clean(C.byref(im))
    return best


def main():
    from PIL import Image
    prod, ref = bd.ClipLib(bd.PRODUCT_LIB), bd.ClipLib(ref_run.REF_LIB)
    rng = np.random.default_rng(0)
    big = np.clip(np.cumsum(rng.normal(0, 3, (3000, 4000, 3)), axis=1) + 128, 0, 255).astype(np.uint8)
    mid = big[:500, :600]
    files = []
    for name, arr, kw in [("600x500 baseline q90", mid, {}), ("600x500 progressive q90", mid, {"progressive": True}),
                          ("4000x3000 baseline q90", big, {}), ("4000x3000 progressive q90", big, {"progressive": True})]:
        p = "/tmp/host_timing_%d.jpg" % len(files)
        Image.fromarray(arr).save(p, quality=90, **kw)
        files.append((name, p))
    print("| JPEG decode (clip_image_load_from_file) | this library | reference (stb_image, SSE2) |\n|---|---|---|")
    for name, p in files:
        reps = 20 if "600" in name else 3
        print("| %s | %.1f ms | %.1f ms |" % (name, load_ms(prod, p, reps), load_ms(ref, p, reps)))

    S = 224
    mean = np.array([0.48145466, 0.4578275, 0.40821073], np.float32)
    std = np.array([0.26862954, 0.26130258, 0.27577711], np.float32)
    fp = C.POINTER(C.c_float)
    # the reference needs a model context whose image_size is 224: the synthetic ViT-B/32 geometry (f16)
    ctx = ref.load(model_file("vit-b32", "f16", prod))
    print("\n| bicubic preprocess to 224x224 | this library | reference (-mavx2 -mfma) | identical bits |\n|---|---|---|---|")
    for (h, w) in ((224, 224), (500, 600), (1080, 1920), (3000, 4000)):
        u8 = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        out = np.empty((S, S, 3), np.float32)
        tp = tr = 1e9
        for _ in range(3):
            t0 = time.perf_counter()
            rc = prod.lib.clip_b200_debug_preprocess(u8.ctypes.data_as(C.POINTER(C.c_uint8)), w, h, S, mean.ctypes.data_as(fp), std.ctypes.data_as(fp),
                                                     out.ctypes.data_as(fp))
            tp = min(tp, (time.perf_counter() - t0) * 1e3)
            assert rc == 0
            t0 = time.perf_counter()
            r = ref.preprocess(ctx, u8)
            tr = min(tr, (time.perf_counter() - t0) * 1e3)
        print("| %dx%d | %.1f ms | %.1f ms | %s |" % (w, h, tp, tr, np.array_equal(out.ravel(), np.asarray(r).ravel())))

    # file quantizer (clip_model_quantize, clip.cpp:1661-1844): single-threaded in both libraries, output files byte-identical
    import synth_gguf as sg
    print("\n| clip_model_quantize, ViT-L/14 f16 (857 MB) -> | this library | reference | identical file |\n|---|---|---|---|")
    src = sg.model_path("vit-l14", 1234, "f16")
    if not os.path.exists(src):
        sg.write_model(src, sg.GEOMETRIES["vit-l14"], 1234, 1)
    if True:
        for it, name in ((2, "q4_0"), (8, "q8_0")):
            t0 = time.perf_counter()
            assert prod.quantize(src, "/tmp/host_timing_p.gguf", it)
            tp = time.perf_counter() - t0
            t0 = time.perf_counter()
            assert ref.quantize(src, "/tmp/host_timing_r.gguf", it)
            tr = time.perf_counter() - t0
            same = open("/tmp/host_timing_p.gguf", "rb").read() == open("/tmp/host_timing_r.gguf", "rb").read()
            print("| %s | %.1f s | %.1f s | %s |" % (name, tp, tr, "yes" if same else "NO"))


if __name__ == "__main__":
    main()
