#!/usr/bin/env python
"""16-bit and int8 nearest-neighbour search (clip_b200_topk_search_16 and clip_b200_topk_search_i8, kernel K10) on seeded unit-norm
vectors, dim 768, f16 or int8 with a scale per row (clip_b200_rows_to_int8).

    python tools/bench_search.py [--reps 3] [--only single|batched|knn|vs32|single_i8|batched_i8|knn_i8|vs16|recall_i8|
                                                 vs_i8_b1|ties_b1|rescore|recall_b1]

  single   n_q = 1,     n_db = 1e7, k = 10: single-query latency, bound by HBM (15.4 GB / 3.35 TB/s = 4.6 ms)
  batched  n_q = 1024,  n_db = 1e7, k = 10: batched retrieval, bound by the tensor cores (15.7 TFLOP / 989 TFLOP/s = 16 ms)
  knn      n_q = n_db = 1e6, k = 16: a near-duplicate / kNN-graph pass (1.54 PFLOP)
  vs32     n_q = 1 and 1024 at n_db = 1e6, k = 10, against clip_b200_topk_search on the fp32 copies of the same vectors
  single_i8, batched_i8, knn_i8   the same three cases in int8: n_db (dim + 4) bytes (7.72 GB / 3.35 TB/s = 2.3 ms at 1e7 rows)
           and 2 n_q n_db dim integer operations against the data sheet's 1 979 dense int8 TOP/s
  vs16     n_q = 1 and 1024 at n_db = 1e7, k = 10: the f16 and the int8 search on the same unit rows, alternated in one call
  recall_i8  recall@10 of the int8 search against clip_b200_topk_search, 1 000 queries over 1e6 distinct unit rows (information).
           clip_b200_topk_search scores the context's projection_dim features, so this case loads a small synthetic model with
           projection_dim 768, written to a temporary directory.
  vs_i8_b1 n_q = 1 and 1024 at n_db = 1e7, k = 10: the binary search (clip_b200_topk_search_b1, K11, kind 9; 96 bytes a row,
           0.96 GB / 3.35 TB/s = 0.29 ms at 1e7 rows) alternated with the int8 search on the same unit rows; 2 n_q n_db dim
           bit operations (AND + popcount) over K11's time as TOP/s, no share of peak (the BMMA rate is not published)
  ties_b1  n_q = 1024, n_db = 1e7: K11 on an all-identical database against random bits, alternated (every score a tie)
  rescore  n_q = 1024, n_cand = 100 random candidates, dim 768, f32 and f16 rows (clip_b200_topk_rescore, K12, kind 10): the
           bytes of the rows gathered over K12's time, against 3.35 TB/s
  recall_b1  recall@10 against clip_b200_topk_search over 1e6 random unit rows, 1 000 queries, for the binary search alone and
           for the binary search at k' = 100 followed by the f32 rescore (information; random rows are not CLIP embeddings)

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
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from bench_attention_maps import card  # noqa: E402
from bench_tokens import HBM_PEAK, Dev, bd, model, sg  # noqa: E402

DIM, F16, K_KNN16, TC_PEAK = 768, 1, 7, 989e12
K_KNN_I8, I8_PEAK = 8, 1979e12
K_KNN_B1, K_RESCORE = 9, 10
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

    def db8(self, n):
        """(codes, scales) of n rows in int8"""
        c, s = self.dev.alloc(n * DIM), self.dev.alloc(max(n * 4, 16))
        for r0 in range(0, n, BLOCK):
            r = min(BLOCK, n - r0)
            assert self.lib.lib.clip_b200_rows_to_int8(self.ctx, self.d_blk, r, DIM, c + r0 * DIM, s + r0 * 4), self.lib.last_error()
        return c, s

    def db32(self, n):
        p = self.dev.alloc(n * DIM * 4)
        for r0 in range(0, n, BLOCK):
            r = min(BLOCK, n - r0)
            assert self.lib.lib.clip_b200_memcpy_h2d(self.ctx, p + r0 * DIM * 4, self.blk.ctypes.data, r * DIM * 4)
        return p


def timed(lib, ctx, fn, kind=K_KNN16):
    """(host seconds, K10 seconds or None) of one call"""
    n = C.c_uint64(0)
    lib.lib.clip_b200_kernel_ms(ctx, kind, C.byref(n))
    t0 = time.perf_counter()
    assert fn(), lib.last_error()
    t = time.perf_counter() - t0
    ms = lib.lib.clip_b200_kernel_ms(ctx, kind, C.byref(n))
    return t, (ms / 1e3 if n.value else None)


def rng_of(v):
    return [round(min(v), 6), round(max(v), 6)] if v else None


def search16(lib, ctx, d_q, nq, d_db, ndb, k):
    sc, ix = np.empty(nq * k, np.float32), np.empty(nq * k, np.int32)
    sp, ip = sc.ctypes.data_as(C.POINTER(C.c_float)), ix.ctypes.data_as(C.POINTER(C.c_int))
    return lambda: lib.lib.clip_b200_topk_search_16(ctx, d_q, nq, d_db, ndb, DIM, F16, k, sp, ip)


def search_i8(lib, ctx, q, nq, db, ndb, k, out=None):
    sc, ix = np.empty(nq * k, np.float32), np.empty(nq * k, np.int32)
    if out is not None:
        out.extend([sc, ix])
    sp, ip = sc.ctypes.data_as(C.POINTER(C.c_float)), ix.ctypes.data_as(C.POINTER(C.c_int))
    return lambda: lib.lib.clip_b200_topk_search_i8(ctx, q[0], q[1], nq, db[0], db[1], ndb, DIM, k, sp, ip)


def search32(lib, ctx, d_q, nq, d_db, ndb, k):
    sc, ix = np.empty(nq * k, np.float32), np.empty(nq * k, np.int32)
    sp, ip = sc.ctypes.data_as(C.POINTER(C.c_float)), ix.ctypes.data_as(C.POINTER(C.c_int))
    return lambda: lib.lib.clip_b200_topk_search(ctx, d_q, nq, d_db, ndb, k, sp, ip)


def search_b1(lib, ctx, q, nq, db, ndb, k, out=None):
    sc, ix = np.empty(nq * k, np.float32), np.empty(nq * k, np.int32)
    if out is not None:
        out.extend([sc, ix])
    sp, ip = sc.ctypes.data_as(C.POINTER(C.c_float)), ix.ctypes.data_as(C.POINTER(C.c_int))
    return lambda: lib.lib.clip_b200_topk_search_b1(ctx, q, nq, db, ndb, DIM, k, sp, ip)


def db_b1(lib, ctx, dev, d_f32, n, nsrc=BLOCK):
    """bits of n rows, the nsrc f32 rows at d_f32 repeated"""
    p = dev.alloc(n * DIM // 8)
    for r0 in range(0, n, nsrc):
        r = min(nsrc, n - r0)
        assert lib.lib.clip_b200_rows_to_binary(ctx, d_f32, r, DIM, None, p + r0 * DIM // 8), lib.last_error()
    return p


def report(case, nq, ndb, k, host, kern, gpu, extra=None, i8=False):
    flop, dbb = 2.0 * nq * ndb * DIM, ndb * (DIM + 4.0 if i8 else DIM * 2.0)
    r = {"case": case, "n_q": nq, "n_db": ndb, "dim": DIM, "k": k, "gpu": gpu, "host_s": rng_of(host), "k10_s": rng_of(kern)}
    if kern:
        r["tops" if i8 else "tflops"] = rng_of([flop / t / 1e12 for t in kern])
        r["tc_peak_share"] = rng_of([flop / t / (I8_PEAK if i8 else TC_PEAK) for t in kern])
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
            dev.free()
            dev.ptrs = []
            data = Data(lib, ctx, dev)
        if want("single_i8") or want("batched_i8"):
            db = data.db8(10_000_000)
            for case, nq in (("single_i8", 1), ("batched_i8", 1024)):
                if not want(case):
                    continue
                fn = search_i8(lib, ctx, data.db8(nq), nq, db, 10_000_000, 10)
                fn()
                runs = [timed(lib, ctx, fn, K_KNN_I8) for _ in range(args.reps)]
                report(case, nq, 10_000_000, 10, [h for h, _ in runs], [t for _, t in runs if t], gpu, i8=True)
            dev.free()
            dev.ptrs = []
            data = Data(lib, ctx, dev)
        if want("knn_i8"):
            n = 1_000_000
            db = data.db8(n)
            fn = search_i8(lib, ctx, db, n, db, n, 16)
            fn()
            runs = [timed(lib, ctx, fn, K_KNN_I8) for _ in range(args.reps)]
            report("knn_i8", n, n, 16, [h for h, _ in runs], [t for _, t in runs if t], gpu, i8=True)
            dev.free()
            dev.ptrs = []
            data = Data(lib, ctx, dev)
        if want("vs16"):
            n = 10_000_000
            db16, db8 = data.db16(n), data.db8(n)
            for nq in (1, 1024):
                f16 = search16(lib, ctx, db16, nq, db16, n, 10)
                f8 = search_i8(lib, ctx, db8, nq, db8, n, 10)
                f16(), f8()
                h16, h8, k16, k8 = [], [], [], []
                for _ in range(args.reps):              # alternated
                    a, b = timed(lib, ctx, f16)
                    h16.append(a)
                    k16.append(b)
                    a, b = timed(lib, ctx, f8, K_KNN_I8)
                    h8.append(a)
                    k8.append(b)
                report("vs16", nq, n, 10, h8, [t for t in k8 if t], gpu, {
                    "f16_host_s": rng_of(h16), "f16_k10_s": rng_of([t for t in k16 if t]),
                    "f16_over_i8_host": rng_of([x / y for x, y in zip(h16, h8)]),
                    "f16_over_i8_k10": rng_of([x / y for x, y in zip(k16, k8) if x and y])}, i8=True)
            dev.free()
            dev.ptrs = []
            data = Data(lib, ctx, dev)
        if want("vs_i8_b1") or want("ties_b1"):
            n = 10_000_000
            db1 = db_b1(lib, ctx, dev, data.d_blk, n)
            if want("vs_i8_b1"):
                db8 = data.db8(n)
                for nq in (1, 1024):
                    q1 = db_b1(lib, ctx, dev, data.d_blk, nq)
                    f1, f8 = search_b1(lib, ctx, q1, nq, db1, n, 10), search_i8(lib, ctx, data.db8(nq), nq, db8, n, 10)
                    f1(), f8()
                    k1, k8 = [], []
                    for _ in range(args.reps):          # alternated
                        k1.append(timed(lib, ctx, f1, K_KNN_B1)[1])
                        k8.append(timed(lib, ctx, f8, K_KNN_I8)[1])
                    r = {"case": "vs_i8_b1", "n_q": nq, "n_db": n, "dim": DIM, "k": 10, "gpu": gpu, "k11_s": rng_of(k1), "k10_i8_s": rng_of(k8),
                         "i8_over_b1": rng_of([y / x for x, y in zip(k1, k8)]),
                         "bit_tops": rng_of([2.0 * nq * n * DIM / t / 1e12 for t in k1]),
                         "hbm_share": rng_of([n * DIM / 8 / t / HBM_PEAK for t in k1])}
                    print(json.dumps(r), flush=True)
            if want("ties_b1"):
                nq = 1024
                same = dev.alloc(n * DIM // 8)
                row = np.random.default_rng(3).integers(0, 256, DIM // 8, dtype=np.uint8)
                blk = np.tile(row, (BLOCK, 1))
                for r0 in range(0, n, BLOCK):
                    assert lib.lib.clip_b200_memcpy_h2d(ctx, same + r0 * DIM // 8, blk.ctypes.data, min(BLOCK, n - r0) * DIM // 8)
                q1 = db_b1(lib, ctx, dev, data.d_blk, nq)
                fr, fs = search_b1(lib, ctx, q1, nq, db1, n, 10), search_b1(lib, ctx, q1, nq, same, n, 10)
                fr(), fs()
                kr, ks = [], []
                for _ in range(args.reps):
                    kr.append(timed(lib, ctx, fr, K_KNN_B1)[1])
                    ks.append(timed(lib, ctx, fs, K_KNN_B1)[1])
                print(json.dumps({"case": "ties_b1", "n_q": nq, "n_db": n, "dim": DIM, "k": 10, "gpu": gpu, "random_k11_s": rng_of(kr),
                                  "identical_k11_s": rng_of(ks), "identical_over_random": rng_of([y / x for x, y in zip(kr, ks)])}), flush=True)
            dev.free()
            dev.ptrs = []
            data = Data(lib, ctx, dev)
        if want("rescore"):
            n, nq, nc = 10_000_000, 1024, 100
            cand = np.random.default_rng(4).integers(0, n, (nq, nc)).astype(np.int32)
            for name, t, eb in (("f32", 0, 4), ("f16", F16, 2)):
                db, q = (data.db32(n), data.db32(nq)) if t == 0 else (data.db16(n), data.db16(nq))
                sc, ix = np.empty(nq * 10, np.float32), np.empty(nq * 10, np.int32)
                fn = lambda: lib.lib.clip_b200_topk_rescore(ctx, q, nq, db, n, DIM, t, cand.ctypes.data_as(C.POINTER(C.c_int)), nc, 10,
                                                            sc.ctypes.data_as(C.POINTER(C.c_float)), ix.ctypes.data_as(C.POINTER(C.c_int)))
                fn()
                kt = [timed(lib, ctx, fn, K_RESCORE)[1] for _ in range(args.reps)]
                gathered = nq * nc * DIM * eb
                print(json.dumps({"case": "rescore", "type": name, "n_q": nq, "n_cand": nc, "n_db": n, "dim": DIM, "gpu": gpu,
                                  "k12_s": rng_of(kt), "gathered_bytes": gathered, "hbm_share": rng_of([gathered / x / HBM_PEAK for x in kt])}),
                      flush=True)
                dev.free()
                dev.ptrs = []
                data = Data(lib, ctx, dev)
        if want("recall_b1"):
            n, nq, k = 1_000_000, 1000, 10
            rng = np.random.default_rng(2)
            d32 = dev.alloc(n * DIM * 4)
            for r0 in range(0, n, BLOCK):
                v = rng.standard_normal((min(BLOCK, n - r0), DIM)).astype(np.float32)
                v /= np.linalg.norm(v, axis=1, keepdims=True)
                assert lib.lib.clip_b200_memcpy_h2d(ctx, d32 + r0 * DIM * 4, v.ctypes.data, v.nbytes)
            qv = rng.standard_normal((nq, DIM)).astype(np.float32)
            qv /= np.linalg.norm(qv, axis=1, keepdims=True)
            q32 = dev.alloc(qv.nbytes, qv)
            db1, q1 = db_b1(lib, ctx, dev, d32, n, n), db_b1(lib, ctx, dev, q32, nq, nq)
            o1, o100 = [], []
            assert search_b1(lib, ctx, q1, nq, db1, n, k, o1)() and search_b1(lib, ctx, q1, nq, db1, n, 100, o100)(), lib.last_error()
            rs, ri = np.empty(nq * k, np.float32), np.empty(nq * k, np.int32)
            assert lib.lib.clip_b200_topk_rescore(ctx, q32, nq, d32, n, DIM, 0, o100[1].ctypes.data_as(C.POINTER(C.c_int)), 100, k,
                                                  rs.ctypes.data_as(C.POINTER(C.c_float)), ri.ctypes.data_as(C.POINTER(C.c_int))), lib.last_error()
            sc, ix = np.empty(nq * k, np.float32), np.empty(nq * k, np.int32)
            with tempfile.TemporaryDirectory() as tmp:
                path = os.path.join(tmp, "p768.gguf")
                sg.write_model(path, sg.Geometry("p768", image_size=64, patch_size=16, v_hidden=128, v_ff=256, v_heads=2, v_layers=12,
                                                 t_hidden=128, t_ff=256, t_heads=2, t_layers=12, proj_dim=DIM), 1234, 1)
                ctx768 = lib.load(path, 0)
                assert ctx768, lib.last_error()
            try:
                assert lib.lib.clip_b200_topk_search(ctx768, q32, nq, d32, n, k, sc.ctypes.data_as(C.POINTER(C.c_float)),
                                                     ix.ctypes.data_as(C.POINTER(C.c_int))), lib.last_error()
            finally:
                lib.free(ctx768)
            want_i = ix.reshape(nq, k)
            rec = lambda got: round(float(np.mean([len(np.intersect1d(got[r], want_i[r])) / k for r in range(nq)])), 4)
            print(json.dumps({"case": "recall_b1", "n_q": nq, "n_db": n, "dim": DIM, "k": k, "gpu": gpu,
                              "recall_at_10_b1": rec(o1[1].reshape(nq, k)), "recall_at_10_b1_rescore_100": rec(ri.reshape(nq, k))}), flush=True)
            dev.free()
            dev.ptrs = []
            data = Data(lib, ctx, dev)
        if want("recall_i8"):
            n, nq, k = 1_000_000, 1000, 10
            rng = np.random.default_rng(2)
            d32 = dev.alloc(n * DIM * 4)
            for r0 in range(0, n, BLOCK):               # distinct rows: a repeated block would make every neighbour a tie
                v = rng.standard_normal((min(BLOCK, n - r0), DIM)).astype(np.float32)
                v /= np.linalg.norm(v, axis=1, keepdims=True)
                assert lib.lib.clip_b200_memcpy_h2d(ctx, d32 + r0 * DIM * 4, v.ctypes.data, v.nbytes)
            qv = rng.standard_normal((nq, DIM)).astype(np.float32)
            qv /= np.linalg.norm(qv, axis=1, keepdims=True)
            q32 = dev.alloc(qv.nbytes, qv)
            c8, s8 = dev.alloc(n * DIM), dev.alloc(n * 4)
            qc, qs = dev.alloc(nq * DIM), dev.alloc(nq * 4)
            assert lib.lib.clip_b200_rows_to_int8(ctx, d32, n, DIM, c8, s8) and lib.lib.clip_b200_rows_to_int8(ctx, q32, nq, DIM, qc, qs)
            o8, o32 = [], []
            assert search_i8(lib, ctx, (qc, qs), nq, (c8, s8), n, k, o8)(), lib.last_error()
            sc, ix = np.empty(nq * k, np.float32), np.empty(nq * k, np.int32)
            with tempfile.TemporaryDirectory() as tmp:
                path = os.path.join(tmp, "p768.gguf")
                sg.write_model(path, sg.Geometry("p768", image_size=64, patch_size=16, v_hidden=128, v_ff=256, v_heads=2, v_layers=12,
                                                 t_hidden=128, t_ff=256, t_heads=2, t_layers=12, proj_dim=DIM), 1234, 1)
                ctx768 = lib.load(path, 0)
                assert ctx768, lib.last_error()
            try:
                assert lib.lib.clip_b200_topk_search(ctx768, q32, nq, d32, n, k, sc.ctypes.data_as(C.POINTER(C.c_float)),
                                                     ix.ctypes.data_as(C.POINTER(C.c_int))), lib.last_error()
            finally:
                lib.free(ctx768)
            got, want_i = o8[1].reshape(nq, k), ix.reshape(nq, k)
            rec = np.mean([len(np.intersect1d(got[r], want_i[r])) / k for r in range(nq)])
            print(json.dumps({"case": "recall_i8", "n_q": nq, "n_db": n, "dim": DIM, "k": k, "gpu": gpu, "recall_at_10": round(float(rec), 4),
                              "top1_agree": round(float(np.mean(got[:, 0] == want_i[:, 0])), 4)}), flush=True)
    finally:
        dev.free()
        lib.free(ctx)


if __name__ == "__main__":
    main()
