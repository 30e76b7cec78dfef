"""Experiment driver: times one attention launch through the C-ABI test hook.  usage: attn_probe.py [nseq T H legacy]"""
import ctypes as C, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "clip.cpp_b200"))
import binding as bd
lib = bd.ClipLib()
nseq, T, H, legacy = [int(x) for x in (sys.argv[1:5] if len(sys.argv) > 4 else (82, 257, 16, 0))]
rng = np.random.default_rng(0)
qkv = rng.standard_normal((nseq * T, 3 * H * 64)).astype(np.float32); qkv[:, :H * 64] *= 0.3
out = np.empty((nseq * T, H * 64), np.float32)
fp = C.POINTER(C.c_float); ms = C.c_float(0)
best = 1e9
for i in range(3):
    rc = lib.lib.clip_b200_debug_attention(1, nseq, T, H, 0, legacy, qkv.ctypes.data_as(fp), out.ctypes.data_as(fp), C.byref(ms))
    assert rc == 0, lib.last_error()
    best = min(best, ms.value)
flops = 4.0 * nseq * H * T * T * 64
print("nseq=%d T=%d H=%d %s: %.1f us  %.0f TFLOP/s" % (nseq, T, H, "mma.sync kernel" if legacy else "wgmma kernel", best * 1e3, flops / best / 1e9))
