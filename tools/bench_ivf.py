#!/usr/bin/env python
"""Inverted-file search over a 16-bit database (clip_b200_ivf_train_16 / _build_16 / _search_16) against the flat search
(clip_b200_topk_search_16) on the same rows: 10^7 x 768 f16 seeded clustered unit rows, n_lists = 4096, k = 10.

    python tools/bench_ivf.py [--reps 3] [--n 10000000] [--only single|batched|skew|train|build|recall]

  single   n_q = 1, nprobe = 32: the IVF call's host time against the flat search's, alternated --reps times
  batched  n_q = 1024, nprobe = 32: the same, plus the fine scan's kernel time (kind 11) and the bytes of the distinct probed
           lists' rows over it, as a share of the H100 SXM data sheet's 3.35 TB/s (the scan reads each probed list once per
           query tile, so this is a lower bound on the bytes it moves)
  skew     n_q = 1024, nprobe = 32 over an index with one list holding 50 % of the rows: time per probed row against the
           balanced index's
  train    20 iterations on the first 10^6 rows (information)
  build    the whole database (information)
  recall   recall@10 at nprobe 8, 32 and 128 against the flat search, 1 000 queries (information; the rows are synthetic
           clusters, not CLIP embeddings)

The rows: 4096 seeded cluster centres on the unit sphere, each row a centre plus Gaussian noise (sigma 0.6 / sqrt(768) a
feature), normalised; 65 536 such rows are made once and repeated (a scan's cost does not depend on the values).  Queries are
fresh rows of the same clusters.  Kernel times come from clip_b200_kernel_ms (CLIP_B200_PROFILE=1): kind 7 (the probes and the
assignments), 11 (the fine scan), 12 (the k-means update and the build's row gather).  The card's name, power limit and SM clock
are read in the same call.  One JSON line per case."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

os.environ.setdefault("CLIP_B200_PROFILE", "1")
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from bench_attention_maps import card  # noqa: E402
from bench_tokens import HBM_PEAK, Dev, bd, model  # noqa: E402

DIM, F16, L, K = 768, 1, 4096, 10
K_KNN16, K_IVF_SCAN, K_IVF_LAYOUT = 7, 11, 12
BLOCK = 65536
FP, IP = C.POINTER(C.c_float), C.POINTER(C.c_int)


def clustered(rng, centres, n, skew=False):
    c = np.zeros(n, np.int64) if skew else rng.integers(0, len(centres), n)
    v = centres[c] + rng.standard_normal((n, DIM)).astype(np.float32) * (0.6 / np.sqrt(DIM))
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


class Bench:
    def __init__(self, lib, ctx, args):
        self.lib, self.ctx, self.L_ = lib, ctx, lib.lib
        self.dev = Dev(lib, ctx)
        self.rng = np.random.default_rng(7)
        c = self.rng.standard_normal((L, DIM)).astype(np.float32)
        self.centres = c / np.linalg.norm(c, axis=1, keepdims=True)
        self.n = args.n

    def to16(self, x):
        d32 = self.dev.alloc(x.nbytes, x)
        d16 = self.dev.alloc(len(x) * DIM * 2)
        assert self.L_.clip_b200_rows_to_16bit(self.ctx, d32, len(x), DIM, F16, d16), self.lib.last_error()
        return d16

    def db(self, n, skew=False):
        """n rows: one block of BLOCK clustered rows repeated; skew: the first half from one cluster"""
        p = self.dev.alloc(n * DIM * 2)
        blocks = [self.to16(clustered(self.rng, self.centres, BLOCK))]
        if skew:
            blocks.append(self.to16(clustered(self.rng, self.centres, BLOCK, skew=True)))
        for r0 in range(0, n, BLOCK):
            r = min(BLOCK, n - r0)
            src = blocks[1] if skew and r0 < n // 2 else blocks[0]
            self.copy_d2d(p + r0 * DIM * 2, src, r * DIM * 2)
        return p

    def copy_d2d(self, dst, src, nbytes):
        """through the host: the C API has no device-to-device copy"""
        h = np.empty(nbytes, np.uint8)
        assert self.L_.clip_b200_memcpy_d2h(self.ctx, h.ctypes.data, src, nbytes)
        assert self.L_.clip_b200_memcpy_h2d(self.ctx, dst, h.ctypes.data, nbytes)

    def kernel_s(self, kind):
        n = C.c_uint64(0)
        return self.L_.clip_b200_kernel_ms(self.ctx, kind, C.byref(n)) / 1e3

    def index(self, d_db, n, d_cent):
        ix = dict(off=self.dev.alloc((L + 1) * 4), ids=self.dev.alloc(n * 4), rows=self.dev.alloc(n * DIM * 2), cent=d_cent)
        assert self.L_.clip_b200_ivf_build_16(self.ctx, d_db, n, DIM, F16, d_cent, L, ix["off"], ix["ids"], ix["rows"]), self.lib.last_error()
        off = np.empty(L + 1, np.int32)
        assert self.L_.clip_b200_memcpy_d2h(self.ctx, off.ctypes.data, ix["off"], off.nbytes)
        ix["sizes"] = np.diff(off)
        return ix

    def ivf(self, ix, d_q, nq, nprobe, n, k=K):
        s, i = np.empty(nq * k, np.float32), np.empty(nq * k, np.int32)
        f = lambda: self.L_.clip_b200_ivf_search_16(self.ctx, d_q, nq, DIM, F16, ix["cent"], L, ix["off"], ix["ids"], ix["rows"], n,
                                                    nprobe, k, s.ctypes.data_as(FP), i.ctypes.data_as(IP))
        return f, i

    def flat(self, d_q, nq, d_db, n, k=K):
        s, i = np.empty(nq * k, np.float32), np.empty(nq * k, np.int32)
        return (lambda: self.L_.clip_b200_topk_search_16(self.ctx, d_q, nq, d_db, n, DIM, F16, k, s.ctypes.data_as(FP),
                                                          i.ctypes.data_as(IP))), i

    def probed_rows(self, ix, d_q, nq, nprobe):
        """distinct rows of the probed lists, summed over queries, and over the distinct lists of the whole batch"""
        s, i = np.empty(nq * nprobe, np.float32), np.empty(nq * nprobe, np.int32)
        assert self.L_.clip_b200_topk_search_16(self.ctx, d_q, nq, ix["cent"], L, DIM, F16, nprobe, s.ctypes.data_as(FP),
                                                 i.ctypes.data_as(IP)), self.lib.last_error()
        i = i.reshape(nq, nprobe)
        return int(ix["sizes"][i].sum()), int(ix["sizes"][np.unique(i)].sum())


def timed(fn, b, kinds=()):
    for k in kinds:
        b.kernel_s(k)
    t0 = time.perf_counter()
    assert fn(), b.lib.last_error()
    t = time.perf_counter() - t0
    return t, [b.kernel_s(k) for k in kinds]


def rng_of(v):
    return [round(min(v), 6), round(max(v), 6)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    lib = bd.ClipLib(bd.PRODUCT_LIB)
    ctx = lib.load(model(lib, "tiny", "f16"), 0)
    assert ctx, lib.last_error()
    b = Bench(lib, ctx, args)
    gpu = card()
    want = lambda c: not args.only or c in args.only.split(",")
    out = lambda d: print(json.dumps(dict(d, card=gpu)), flush=True)
    n = b.n

    d_train = b.db(1_000_000)
    d_cent = b.dev.alloc(L * DIM * 2)
    t, (ks, ku) = timed(lambda: b.L_.clip_b200_ivf_train_16(ctx, d_train, 1_000_000, DIM, F16, L, 20, d_cent), b, (K_KNN16, K_IVF_LAYOUT))
    if want("train"):
        out(dict(case="train", n_train=1_000_000, n_lists=L, n_iter=20, call_s=round(t, 4), assign_kernel_s=round(ks, 4),
                 update_kernel_s=round(ku, 4)))
    d_db = b.db(n)
    t0 = time.perf_counter()
    ix = b.index(d_db, n, d_cent)
    t = time.perf_counter() - t0
    if want("build"):
        out(dict(case="build", n_db=n, n_lists=L, call_s=round(t, 4), largest_list=int(ix["sizes"].max()),
                 empty_lists=int((ix["sizes"] == 0).sum())))
    qs = clustered(np.random.default_rng(11), b.centres, 1024)
    d_q = b.to16(qs)                                   # 1024 queries; recall uses the first 1000
    for case, nq in (("single", 1), ("batched", 1024)):
        if not want(case):
            continue
        fi, _ = b.ivf(ix, d_q, nq, 32, n)
        ff, _ = b.flat(d_q, nq, d_db, n)
        fi(), ff()
        ti, tf, scan = [], [], []
        for _ in range(args.reps):
            t, (s,) = timed(fi, b, (K_IVF_SCAN,))
            ti.append(t), scan.append(s)
            tf.append(timed(ff, b)[0])
        per_q, distinct = b.probed_rows(ix, d_q, nq, 32)
        r = dict(case=case, n_q=nq, nprobe=32, ivf_call_s=rng_of(ti), flat_call_s=rng_of(tf),
                 speedup=[round(min(tf) / max(ti), 2), round(max(tf) / min(ti), 2)], scan_kernel_s=rng_of(scan),
                 probed_rows_per_query=round(per_q / nq), distinct_probed_rows=distinct)
        if case == "batched":
            r["scan_hbm_share_distinct_bytes"] = rng_of([distinct * DIM * 2 / s / HBM_PEAK for s in scan])
        out(r)
    if want("skew"):
        d_sk = b.db(n, skew=True)
        ix_s = b.index(d_sk, n, d_cent)
        res = {}
        for name, x, d in (("balanced", ix, d_db), ("skewed", ix_s, d_sk)):
            f, _ = b.ivf(x, d_q, 1024, 32, n)
            f()
            ts = [timed(f, b)[0] for _ in range(args.reps)]
            per_q, _ = b.probed_rows(x, d_q, 1024, 32)
            res[name] = dict(call_s=rng_of(ts), probed_rows=per_q, s_per_mrow=round(min(ts) / per_q * 1e6, 6))
        out(dict(case="skew", n_q=1024, nprobe=32, largest_list_share=round(float(ix_s["sizes"].max()) / n, 3), **res,
                 ratio_per_probed_row=round(res["skewed"]["s_per_mrow"] / res["balanced"]["s_per_mrow"], 3)))
    if want("recall"):
        fl, fi_ = b.flat(d_q, 1000, d_db, n)
        assert fl(), lib.last_error()
        rec = {}
        for npr in (8, 32, 128):
            f, got = b.ivf(ix, d_q, 1000, npr, n)
            assert f(), lib.last_error()
            g, w = got.reshape(1000, K), fi_.reshape(1000, K)
            rec[str(npr)] = round(float(np.mean([len(np.intersect1d(a, c)) / K for a, c in zip(g, w)])), 4)
        out(dict(case="recall", n_q=1000, k=K, recall_at_10=rec))
    b.dev.free()
    lib.free(ctx)


if __name__ == "__main__":
    main()
