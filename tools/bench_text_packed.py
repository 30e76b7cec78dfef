#!/usr/bin/env python
"""Token sequences of different lengths in one packed call (clip_b200_text_*_packed), ViT-L/14 text tower q4_0, 16 384 sequences.

    python tools/bench_text_packed.py [--steps 3] [--warmup 1] [--reps 3]

Workloads: "captions" -- an ASSUMED stand-in for web captions, since no real caption set ships with the project: 90 % of the lengths
are 2 + lognormal(median 14, sigma 0.5) rounded and clipped to [3, 76], 10 % are exactly 77, drawn from a seed; "full" -- every
sequence 77 tokens.  Ids are drawn from a seed (SOT first, EOT last).
  (a) captions: clip_b200_text_encode_device_packed against clip_b200_text_encode_device at seq_len 77 with d_lens.
  (b) captions: clip_b200_text_batch_encode_packed against clip_text_batch_encode, the same clip_tokens.
  (c) captions: the packed device call against sort-by-length, one clip_b200_text_encode_device call per length bucket of 8.
  (d) full: the packed device call against clip_b200_text_encode_device at seq_len 77; the embeddings compared bit for bit.
  (e) full: device time of the attention kernel (clip_b200_kernel_ms kind 1) in (d)'s two calls -- the causal variable-length
      instance against the fixed-T causal one -- with CLIP_B200_PROFILE=1 in a context of its own.
Paired paths are alternated --reps times (host clock around calls that end in a device synchronise).  The card's name and power
limit are read in the same call.  One JSON line per case.  Model files are written from seeds into synth_gguf.cache_dir()."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "clip.cpp_b200"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)
import binding as bd  # noqa: E402
from bench_tokens import Dev, card, model, per_call  # noqa: E402

N, D, CTX = 16384, 768, 77
IP = C.POINTER(C.c_int)
I32P = C.POINTER(C.c_int32)


def lengths(workload, seed=7):
    if workload == "full":
        return np.full(N, CTX, np.int32)
    rng = np.random.default_rng(seed)
    short = np.clip(np.rint(2 + rng.lognormal(np.log(14.0), 0.5, N)), 3, 76).astype(np.int32)
    return np.where(rng.random(N) < 0.1, CTX, short).astype(np.int32)


class Batch:
    """one workload's sequences: packed and padded on the device, length buckets of 8, and host clip_tokens"""
    def __init__(self, lib, ctx, dev, lens, seed=1):
        rng = np.random.default_rng(seed)
        self.lib, self.ctx, self.lens = lib, ctx, lens
        self.seqs = []
        for n in lens:
            s = rng.integers(0, 49406, int(n), dtype=np.int32)
            s[0], s[-1] = 49406, 49407
            self.seqs.append(s)
        packed = np.concatenate(self.seqs)
        padded = np.zeros((N, CTX), np.int32)
        for i, s in enumerate(self.seqs):
            padded[i, :len(s)] = s
        self.d_packed, self.d_padded = dev.alloc(packed.nbytes, packed), dev.alloc(padded.nbytes, padded)
        self.d_lens = dev.alloc(lens.nbytes, lens)
        self.d_vec = dev.alloc(N * D * 4)
        # sort-by-length: bucket b holds the sequences of length 8b - 7 .. 8b, padded to min(8b, 77), one device call each
        self.buckets = []
        order = np.argsort(lens, kind="stable")
        keys = np.minimum((lens[order] + 7) // 8 * 8, CTX)
        for T in np.unique(keys):
            idx = order[keys == T]
            ids = np.zeros((len(idx), T), np.int32)
            for j, i in enumerate(idx):
                ids[j, :lens[i]] = self.seqs[i]
            bl = lens[idx].astype(np.int32)
            self.buckets.append((int(T), len(idx), dev.alloc(ids.nbytes, ids), dev.alloc(bl.nbytes, bl)))
        self.arr = (bd.clip_tokens * N)()
        for i, s in enumerate(self.seqs):
            self.arr[i].data = s.ctypes.data_as(I32P)
            self.arr[i].size = s.size
        self.vec = np.empty((N, D), np.float32)

    def packed_dev(self):
        return self.lib.lib.clip_b200_text_encode_device_packed(self.ctx, self.d_packed, N, self.lens.ctypes.data_as(IP), self.d_vec, True)

    def padded_dev(self):
        return self.lib.lib.clip_b200_text_encode_device(self.ctx, self.d_padded, self.d_lens, N, CTX, self.d_vec, True)

    def packed_host(self):
        return self.lib.lib.clip_b200_text_batch_encode_packed(self.ctx, self.arr, N, self.vec.ctypes.data_as(C.POINTER(C.c_float)), True)

    def padded_host(self):
        return self.lib.lib.clip_text_batch_encode(self.ctx, 4, self.arr, N, self.vec.ctypes.data_as(C.POINTER(C.c_float)), True)

    def bucketed_dev(self):
        ok = True
        for T, k, d_ids, d_lens in self.buckets:
            ok &= self.lib.lib.clip_b200_text_encode_device(self.ctx, d_ids, d_lens, k, T, self.d_vec, True)
        return ok

    def fetch(self):
        out = np.empty((N, D), np.float32)
        assert self.lib.lib.clip_b200_memcpy_d2h(self.ctx, out.ctypes.data, self.d_vec, out.nbytes)
        return out


def alternate(calls, args):
    """{name: call} -> {name: sequences/s per rep, slowest first}, the calls alternated"""
    t = {k: [] for k in calls}
    for _ in range(args.reps):
        for k, f in calls.items():
            t[k].append(per_call(f, args.steps, args.warmup))
    return {k: [round(N / s) for s in sorted(v, reverse=True)] for k, v in t.items()}


def ratio(r, a, b):
    return [round(x / y, 3) for x, y in zip(r[a], r[b])]


def attention_ms(lib, path, args):
    """kind-1 device ms per call on the full workload: the packed call against the padded one"""
    os.environ["CLIP_B200_PROFILE"] = "1"
    ctx = lib.load(path, 0)
    dev = Dev(lib, ctx)
    out = {"packed_attn_ms": [], "padded_attn_ms": []}
    try:
        b = Batch(lib, ctx, dev, lengths("full"))
        cnt = C.c_uint64(0)
        for _ in range(args.warmup):
            assert b.packed_dev() and b.padded_dev()
        for _ in range(args.reps):
            for name, f in (("packed_attn_ms", b.packed_dev), ("padded_attn_ms", b.padded_dev)):
                lib.lib.clip_b200_kernel_ms(ctx, 1, C.byref(cnt))
                for _ in range(args.steps):
                    assert f()
                out[name].append(round(lib.lib.clip_b200_kernel_ms(ctx, 1, C.byref(cnt)) / args.steps, 3))
    finally:
        dev.free()
        lib.free(ctx)
        del os.environ["CLIP_B200_PROFILE"]
    out["packed_over_padded"] = [round(x / y, 4) for x, y in zip(out["packed_attn_ms"], out["padded_attn_ms"])]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    lib = bd.ClipLib(bd.PRODUCT_LIB)
    gpu = card()
    print("card, power limit:", gpu, flush=True)
    path = model(lib, "vit-l14", "q4_0")
    results = []
    ctx = lib.load(path, 0)
    dev = Dev(lib, ctx)
    try:
        lens = lengths("captions")
        b = Batch(lib, ctx, dev, lens)
        shape = dict(n=N, mean_len=round(float(lens.mean()), 2), share_77=round(float((lens == CTX).mean()), 3), buckets=len(b.buckets))
        r = alternate({"packed_dev_seq_s": b.packed_dev, "padded_dev_seq_s": b.padded_dev, "bucketed_dev_seq_s": b.bucketed_dev}, args)
        results.append(dict(case="(a, c) captions, device: packed vs padded to 77 (d_lens) / one call per length bucket of 8, ViT-L/14 q4_0",
                            packed_over_padded=ratio(r, "packed_dev_seq_s", "padded_dev_seq_s"),
                            packed_over_bucketed=ratio(r, "packed_dev_seq_s", "bucketed_dev_seq_s"), **shape, **r))
        r = alternate({"packed_host_seq_s": b.packed_host, "padded_host_seq_s": b.padded_host}, args)
        results.append(dict(case="(b) captions, host: clip_b200_text_batch_encode_packed vs clip_text_batch_encode, ViT-L/14 q4_0",
                            packed_over_padded=ratio(r, "packed_host_seq_s", "padded_host_seq_s"), **shape, **r))
        b = Batch(lib, ctx, dev, lengths("full"), seed=2)
        r = alternate({"packed_dev_seq_s": b.packed_dev, "padded_dev_seq_s": b.padded_dev}, args)
        assert b.packed_dev()
        got = b.fetch()
        assert b.padded_dev()
        want = b.fetch()
        results.append(dict(case="(d) every sequence 77 tokens, device: packed vs padded, ViT-L/14 q4_0, n=%d" % N,
                            packed_over_padded=ratio(r, "packed_dev_seq_s", "padded_dev_seq_s"),
                            bit_identical=bool(np.array_equal(got.view(np.uint32), want.view(np.uint32))), **r))
    finally:
        dev.free()
        lib.free(ctx)
    results.append(dict(case="(e) every sequence 77 tokens: attention kernel ms per call (kind 1), causal varlen vs fixed-T causal",
                        **attention_ms(lib, path, args)))
    for res in results:
        res["gpu"] = gpu
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
