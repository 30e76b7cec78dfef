#!/usr/bin/env python
"""16-bit nearest-neighbour search (clip_b200_topk_search_16, kernel K10) on seeded unit-norm vectors, dim 768, f16.

    python tools/bench_search.py [--reps 3] [--only single|batched|knn|vs32]

  single   n_q = 1,     n_db = 1e7, k = 10: single-query latency, bound by HBM (15.4 GB / 3.35 TB/s = 4.6 ms)
  batched  n_q = 1024,  n_db = 1e7, k = 10: batched retrieval, bound by the tensor cores (15.7 TFLOP / 989 TFLOP/s = 16 ms)
  knn      n_q = n_db = 1e6, k = 16: a near-duplicate / kNN-graph pass (1.54 PFLOP)
  vs32     n_q = 1 and 1024 at n_db = 1e6, k = 10, against clip_b200_topk_search on the fp32 copies of the same vectors

The database is 65 536 distinct unit rows repeated (the scan's cost does not depend on the values).  Per case: the call's host
time (the call ends in a device synchronise) and K10's CUDA-event time (kind 7 of clip_b200_kernel_ms, CLIP_B200_PROFILE=1), the
achieved TFLOP/s (2 n_q n_db dim over K10's time) and the share of HBM bandwidth (database bytes over K10's time, against the H100
SXM data sheet's 3.35 TB/s).  Compared forms alternate --reps times; every value is printed, as [min, max].  The card's name, power
limit and SM clock are read in the same call.  One JSON line per case."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from bench_attention_maps import card  # noqa: E402
from bench_tokens import HBM_PEAK, Dev, bd, model  # noqa: E402

DIM, F16, K_KNN16, TC_PEAK = 768, 1, 7, 989e12
BLOCK = 65536


def unit_block(seed):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((BLOCK, DIM)).astype(np.float32)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    return v


class Data:
    """f32 block on the device; 16-bit (and optionally f32) databases of n rows made from it"""

    def __init__(self, lib, ctx, dev):
        self.lib, self.ctx, self.dev = lib, ctx, dev
        self.blk = unit_block(1)
        self.d_blk = dev.alloc(self.blk.nbytes, self.blk)

    def db16(self, n):
        p = self.dev.alloc(n * DIM * 2)
        for r0 in range(0, n, BLOCK):
            r = min(BLOCK, n - r0)
            assert self.lib.lib.clip_b200_rows_to_16bit(self.ctx, self.d_blk, r, DIM, F16, p + r0 * DIM * 2), self.lib.last_error()
        return p

    def db32(self, n):
        p = self.dev.alloc(n * DIM * 4)
        for r0 in range(0, n, BLOCK):
            r = min(BLOCK, n - r0)
            assert self.lib.lib.clip_b200_memcpy_h2d(self.ctx, p + r0 * DIM * 4, self.blk.ctypes.data, r * DIM * 4)
        return p


def timed(lib, ctx, fn):
    """(host seconds, K10 seconds or None) of one call"""
    n = C.c_uint64(0)
    lib.lib.clip_b200_kernel_ms(ctx, K_KNN16, C.byref(n))
    t0 = time.perf_counter()
    assert fn(), lib.last_error()
    t = time.perf_counter() - t0
    ms = lib.lib.clip_b200_kernel_ms(ctx, K_KNN16, C.byref(n))
    return t, (ms / 1e3 if n.value else None)


def rng_of(v):
    return [round(min(v), 6), round(max(v), 6)] if v else None


def search16(lib, ctx, d_q, nq, d_db, ndb, k):
    sc, ix = np.empty(nq * k, np.float32), np.empty(nq * k, np.int32)
    sp, ip = sc.ctypes.data_as(C.POINTER(C.c_float)), ix.ctypes.data_as(C.POINTER(C.c_int))
    return lambda: lib.lib.clip_b200_topk_search_16(ctx, d_q, nq, d_db, ndb, DIM, F16, k, sp, ip)


def search32(lib, ctx, d_q, nq, d_db, ndb, k):
    sc, ix = np.empty(nq * k, np.float32), np.empty(nq * k, np.int32)
    sp, ip = sc.ctypes.data_as(C.POINTER(C.c_float)), ix.ctypes.data_as(C.POINTER(C.c_int))
    return lambda: lib.lib.clip_b200_topk_search(ctx, d_q, nq, d_db, ndb, k, sp, ip)


def report(case, nq, ndb, k, host, kern, gpu, extra=None):
    flop, dbb = 2.0 * nq * ndb * DIM, ndb * DIM * 2.0
    r = {"case": case, "n_q": nq, "n_db": ndb, "dim": DIM, "k": k, "gpu": gpu, "host_s": rng_of(host), "k10_s": rng_of(kern)}
    if kern:
        r["tflops"] = rng_of([flop / t / 1e12 for t in kern])
        r["tc_peak_share"] = rng_of([flop / t / TC_PEAK for t in kern])
        r["hbm_share"] = rng_of([dbb / t / HBM_PEAK for t in kern])
    if extra:
        r.update(extra)
    print(json.dumps(r), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    os.environ["CLIP_B200_PROFILE"] = "1"
    lib = bd.ClipLib(bd.PRODUCT_LIB)
    ctx = lib.load(model(lib, "tiny", "f16"), 0)       # the search uses no tower; any context on the GPU will do
    dev = Dev(lib, ctx)
    gpu = card()
    try:
        data = Data(lib, ctx, dev)
        want = lambda c: not args.only or args.only == c
        if want("single") or want("batched"):
            db = data.db16(10_000_000)
            for case, nq in (("single", 1), ("batched", 1024)):
                if not want(case):
                    continue
                q = data.db16(nq)
                fn = search16(lib, ctx, q, nq, db, 10_000_000, 10)
                fn()
                runs = [timed(lib, ctx, fn) for _ in range(args.reps)]
                report(case, nq, 10_000_000, 10, [h for h, _ in runs], [t for _, t in runs if t], gpu)
            dev.free()
            dev.ptrs = []
            data = Data(lib, ctx, dev)
        if want("knn"):
            n = 1_000_000
            db = data.db16(n)
            fn = search16(lib, ctx, db, n, db, n, 16)
            fn()
            runs = [timed(lib, ctx, fn) for _ in range(args.reps)]
            report("knn", n, n, 16, [h for h, _ in runs], [t for _, t in runs if t], gpu)
        if want("vs32"):
            n = 1_000_000
            db16, db32 = data.db16(n), data.db32(n)
            for nq in (1, 1024):
                f16 = search16(lib, ctx, db16, nq, db16, n, 10)
                f32 = search32(lib, ctx, db32, nq, db32, n, 10)
                f16(), f32()
                h16, h32, k16 = [], [], []
                for _ in range(args.reps):              # alternated
                    a, b = timed(lib, ctx, f16)
                    h16.append(a)
                    if b:
                        k16.append(b)
                    h32.append(timed(lib, ctx, f32)[0])
                report("vs32", nq, n, 10, h16, k16, gpu, {"fp32_host_s": rng_of(h32),
                                                          "fp32_over_16bit": rng_of([x / y for x, y in zip(h32, h16)])})
    finally:
        dev.free()
        lib.free(ctx)


if __name__ == "__main__":
    main()
