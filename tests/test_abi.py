"""The C-ABI library loads on a CPU-only box and exports every symbol include/clip_b200.h declares -- the 22 reference
symbols (clip.h:42-109) plus the additive ones.  No compute is called here."""
import ctypes
import os
import re

import binding as bd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions():
    src = open(os.path.join(ROOT, "include", "clip_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = re.findall(r"\b([a-z_][a-z0-9_]*)\s*\(", src)
    return sorted({n for n in names if n.startswith(("clip_", "softmax_with"))})


def test_header_and_binding_agree():
    decl = set(declared_functions())
    assert set(bd.REFERENCE_SYMBOLS) <= decl
    assert set(bd.EXTENSION_SYMBOLS) <= decl
    assert len(bd.REFERENCE_SYMBOLS) == 22


def test_library_exports_every_declared_symbol(prod):
    lib = ctypes.CDLL(bd.PRODUCT_LIB)
    missing = [n for n in declared_functions() if not hasattr(lib, n)]
    assert not missing, missing
    for n in ("ggml_time_init", "ggml_time_us", "ggml_time_ms"):      # include/ggml/ggml.h shim
        assert hasattr(lib, n)


def test_struct_layouts_match_reference_header():
    # clip.h:14-74 -- sizes on LP64
    assert ctypes.sizeof(bd.clip_text_hparams) == 32 and ctypes.sizeof(bd.clip_vision_hparams) == 32
    assert ctypes.sizeof(bd.clip_tokens) == 16
    assert ctypes.sizeof(bd.clip_image_u8) == 24 and ctypes.sizeof(bd.clip_image_f32) == 24
    assert ctypes.sizeof(bd.clip_image_u8_batch) == 16 and ctypes.sizeof(bd.clip_image_f32_batch) == 16


def test_no_cpu_fallback(prod):
    """Without a CUDA device clip_model_load must fail loudly (this test only runs its assertion on CPU-only hosts)."""
    import synth_gguf as sg
    path = sg.model_path("tiny", 1234, "f16")
    if not os.path.exists(path):
        sg.write_model(path, sg.GEOMETRIES["tiny"], 1234, 1)
    ctx = prod.lib.clip_model_load(path.encode(), 0)
    if ctx:                      # a GPU is present: nothing to assert here
        prod.free(ctx)
        return
    assert b"no CUDA device" in prod.lib.clip_b200_last_error() or b"sm_90" in prod.lib.clip_b200_last_error()


def test_product_does_not_reference_the_oracle():
    """The product sources never include / link / load anything under oracle/."""
    pkg = os.path.join(ROOT, "clip.cpp_b200")
    for dp, _, fns in os.walk(pkg):
        if "build" in dp:
            continue
        for fn in fns:
            if fn.endswith((".cu", ".cpp", ".h", ".hpp", ".cuh", ".py")) or fn == "Makefile":
                txt = open(os.path.join(dp, fn), errors="ignore").read()
                assert "liboracle" not in txt and "clip_oracle" not in txt and "import oracle" not in txt, fn
    out = os.popen("ldd %s" % bd.PRODUCT_LIB).read()
    assert "oracle" not in out
