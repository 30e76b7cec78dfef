#!/usr/bin/env python
"""Inverted-file search with product-quantised residuals (clip_b200_ivfpq_*) against the 16-bit IVF search
(clip_b200_ivf_search_16) on the same centroids and lists: tools/bench_ivf.py's data, 10^7 x 768 f16 seeded clustered rows,
n_lists = 4096, k = 10, m = 96.

    python tools/bench_ivfpq.py [--reps 3] [--n 10000000] [--only train,encode,batched,single,scale,recall]

  train    codebook k-means, 20 iterations on 10^6 rows (information)
  encode   the 10^7 rows in chunks of 10^6, then the build (information)
  batched  n_q = 1024, nprobe = 32: the PQ call against clip_b200_ivf_search_16, alternated --reps times; the ADC scan's kernel
           time (kind 13) and its shared-memory lookup bound, pairs x probed rows x m lookups over 132 SMs x 32 words a clock x the
           SM clock read right after each PQ call (the lowest of them; the card's maximum is reported beside it) (aims: the call no
           slower than the 16-bit IVF's; the scan within 3x of the bound)
  single   n_q = 1, nprobe = 32: the PQ call's time (information)
  scale    10^8 rows encoded in chunks of 10^6 from the repeated block, built and searched at n_q = 1024: the index's device bytes
           against the 16-bit IVF's (information)
  recall   recall@10 on 10^6 non-repeated rows at nprobe 8 / 32 / 128, PQ alone and PQ with an exact rescore of its top 100
           (information; synthetic clusters, not CLIP embeddings)

The card's name, power limit and SM clock are read in the same call.  One JSON line per case."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

os.environ.setdefault("CLIP_B200_PROFILE", "1")
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from bench_attention_maps import card  # noqa: E402
from bench_ivf import DIM, F16, FP, IP, K, L, Bench, clustered, rng_of, timed  # noqa: E402
from bench_tokens import bd, model  # noqa: E402

M = 96
K_ADC, K_PQ = 13, 14
CHUNK = 1_000_000


def sm_clocks_hz():
    """(current SM clock, maximum SM clock) in Hz"""
    out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"], capture_output=True,
                         text=True)
    cur, mx = out.stdout.splitlines()[0].split(",")
    return float(cur) * 1e6, float(mx) * 1e6


class Pq:
    def __init__(self, b, d_cent, d_books):
        self.b, self.L_, self.ctx, self.cent, self.books = b, b.L_, b.ctx, d_cent, d_books

    def encode(self, d_rows, n, d_lists, d_codes):
        assert self.L_.clip_b200_ivfpq_encode_16(self.ctx, d_rows, n, DIM, F16, self.cent, L, self.books, M, d_lists, d_codes), self.b.lib.last_error()

    def build(self, d_lists, d_codes, n):
        ix = dict(off=self.b.dev.alloc((L + 1) * 4), ids=self.b.dev.alloc(n * 4), codes=self.b.dev.alloc(n * M), n=n)
        assert self.L_.clip_b200_ivfpq_build(self.ctx, d_lists, d_codes, n, L, M, ix["off"], ix["ids"], ix["codes"]), self.b.lib.last_error()
        return ix

    def search(self, ix, d_q, nq, nprobe, k=K):
        s, i = np.empty(nq * k, np.float32), np.empty(nq * k, np.int32)
        return (lambda: self.L_.clip_b200_ivfpq_search_16(self.ctx, d_q, nq, DIM, F16, self.cent, L, self.books, M, ix["off"], ix["ids"],
                                                          ix["codes"], ix["n"], nprobe, k, s.ctypes.data_as(FP), i.ctypes.data_as(IP))), i

    def encoded(self, d_rows, n, chunk=CHUNK, src_rows=None):
        """lists and codes of n rows, encoded chunk by chunk (src_rows: a block of `chunk` rows repeated)"""
        d_l, d_k = self.b.dev.alloc(n * 4), self.b.dev.alloc(n * M)
        for r0 in range(0, n, chunk):
            c = min(chunk, n - r0)
            src = src_rows if src_rows is not None else d_rows + r0 * DIM * 2
            self.encode(src, c, d_l + r0 * 4, d_k + r0 * M)
        return d_l, d_k


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
    assert b.L_.clip_b200_ivf_train_16(ctx, d_train, 1_000_000, DIM, F16, L, 20, d_cent), lib.last_error()
    d_books = b.dev.alloc(M * 256 * (DIM // M) * 4)
    t, (ka, kp) = timed(lambda: b.L_.clip_b200_ivfpq_train_16(ctx, d_train, 1_000_000, DIM, F16, d_cent, L, M, 20, d_books), b, (7, K_PQ))
    if want("train"):
        out(dict(case="train", n_train=1_000_000, m=M, n_iter=20, call_s=round(t, 4), assign_kernel_s=round(ka, 4), pq_kernel_s=round(kp, 4)))
    pq = Pq(b, d_cent, d_books)
    d_db = b.db(n)
    t0 = time.perf_counter()
    d_l, d_k = pq.encoded(d_db, n)
    t_enc = time.perf_counter() - t0
    t0 = time.perf_counter()
    ix = pq.build(d_l, d_k, n)
    t_build = time.perf_counter() - t0
    if want("encode"):
        out(dict(case="encode", n_db=n, chunk=CHUNK, m=M, encode_s=round(t_enc, 4), build_s=round(t_build, 4)))
    qs = clustered(np.random.default_rng(11), b.centres, 1024)
    d_q = b.to16(qs)
    ix16 = b.index(d_db, n, d_cent)
    for case, nq in (("batched", 1024), ("single", 1)):
        if not want(case):
            continue
        fp, _ = pq.search(ix, d_q, nq, 32)
        fi, _ = b.ivf(ix16, d_q, nq, 32, n)
        fp(), fi()
        tp, ti, scan, tab, clocks = [], [], [], [], []
        for _ in range(args.reps):
            t, (s, tb) = timed(fp, b, (K_ADC, K_PQ))
            clocks.append(sm_clocks_hz())                  # read right after the PQ call, while the card is still loaded
            tp.append(t), scan.append(s), tab.append(tb)
            ti.append(timed(fi, b)[0])
        r = dict(case=case, n_q=nq, nprobe=32, m=M, pq_call_s=rng_of(tp), ivf16_call_s=rng_of(ti),
                 speedup_vs_ivf16=[round(min(ti) / max(tp), 2), round(max(ti) / min(tp), 2)], adc_kernel_s=rng_of(scan),
                 table_kernel_s=rng_of(tab))
        if case == "batched":
            per_q, _ = b.probed_rows(ix16, d_q, nq, 32)
            lookups = per_q * M
            clock = min(c for c, _ in clocks)               # the lowest SM clock read after a PQ call: the bound at that clock
            bound = lookups / (132 * 32 * clock)
            r.update(lookups=lookups, sm_clock_mhz_after_calls=[c / 1e6 for c, _ in clocks], sm_clock_max_mhz=clocks[0][1] / 1e6,
                     lookup_bound_s=round(bound, 6),
                     adc_over_bound=[round(min(scan) / bound, 2), round(max(scan) / bound, 2)])
        out(r)
    if want("recall"):
        b.dev.free()
        b.dev = type(b.dev)(lib, ctx)
        n_r = 1_000_000
        rng = np.random.default_rng(13)
        d_x = b.dev.alloc(n_r * DIM * 2)
        for r0 in range(0, n_r, 100_000):
            d16 = b.to16(clustered(rng, b.centres, 100_000))
            b.copy_d2d(d_x + r0 * DIM * 2, d16, 100_000 * DIM * 2)
        d_cent = b.dev.alloc(L * DIM * 2)
        assert b.L_.clip_b200_ivf_train_16(ctx, d_x, n_r, DIM, F16, L, 10, d_cent), lib.last_error()
        d_books = b.dev.alloc(M * 256 * (DIM // M) * 4)
        assert b.L_.clip_b200_ivfpq_train_16(ctx, d_x, n_r, DIM, F16, d_cent, L, M, 10, d_books), lib.last_error()
        pq = Pq(b, d_cent, d_books)
        d_l, d_k = pq.encoded(d_x, n_r)
        ixr = pq.build(d_l, d_k, n_r)
        d_q = b.to16(clustered(np.random.default_rng(17), b.centres, 1000))
        ff, truth = b.flat(d_q, 1000, d_x, n_r)
        assert ff(), lib.last_error()
        truth = truth.reshape(1000, K)
        rec = lambda got: round(float(np.mean([len(np.intersect1d(a, c)) / K for a, c in zip(got, truth)])), 4)
        res = {}
        for npr in (8, 32, 128):
            f, i100 = pq.search(ixr, d_q, 1000, npr, 100)
            assert f(), lib.last_error()
            i100 = i100.reshape(1000, 100)
            s, i = np.empty(1000 * K, np.float32), np.empty(1000 * K, np.int32)
            cand = np.ascontiguousarray(i100)
            assert b.L_.clip_b200_topk_rescore(ctx, d_q, 1000, d_x, n_r, DIM, F16, cand.ctypes.data_as(IP), 100, K, s.ctypes.data_as(FP),
                                               i.ctypes.data_as(IP)), lib.last_error()
            res[str(npr)] = dict(pq=rec(i100[:, :K]), pq_rescore_100=rec(i.reshape(1000, K)))
        out(dict(case="recall", n_db=n_r, n_q=1000, k=K, m=M, data="synthetic clusters", recall_at_10=res))
    if want("scale"):
        b.dev.free()
        b.dev = type(b.dev)(lib, ctx)
        n8 = 100_000_000
        blk = b.db(CHUNK)
        d_cent = b.dev.alloc(L * DIM * 2)
        assert b.L_.clip_b200_ivf_train_16(ctx, blk, CHUNK, DIM, F16, L, 10, d_cent), lib.last_error()
        d_books = b.dev.alloc(M * 256 * (DIM // M) * 4)
        assert b.L_.clip_b200_ivfpq_train_16(ctx, blk, CHUNK, DIM, F16, d_cent, L, M, 10, d_books), lib.last_error()
        pq = Pq(b, d_cent, d_books)
        t0 = time.perf_counter()
        d_l, d_k = pq.encoded(None, n8, src_rows=blk)
        t_enc = time.perf_counter() - t0
        t0 = time.perf_counter()
        ix8 = pq.build(d_l, d_k, n8)
        t_build = time.perf_counter() - t0
        d_q = b.to16(qs)
        f, _ = pq.search(ix8, d_q, 1024, 32)
        f()
        ts = [timed(f, b)[0] for _ in range(args.reps)]
        index_bytes = n8 * M + n8 * 4 + (L + 1) * 4 + L * DIM * 2 + M * 256 * (DIM // M) * 4
        out(dict(case="scale", n_db=n8, m=M, encode_s=round(t_enc, 3), build_s=round(t_build, 3), search_call_s=rng_of(ts), n_q=1024,
                 nprobe=32, index_device_gb=round(index_bytes / 1e9, 2), ivf16_rows_gb=round(n8 * DIM * 2 / 1e9, 1)))
    b.dev.free()
    lib.free(ctx)


if __name__ == "__main__":
    main()
