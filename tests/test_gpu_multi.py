"""Multi-GPU inside the library (SURVEY.md section 8e), needs >= 2 H100s (`python -m pytest tests -m gpu -k multi`; skips on one GPU):
  * devices mode -- CLIP_B200_DEVICES at clip_model_load, one context drives every GPU, results identical to one GPU;
  * ranks mode   -- one process per GPU, NCCL communicator built by the library from the launcher's environment (no torch),
                    clip_b200_*_all return every rank's embeddings in rank order."""
import os
import socket
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import synth_gguf as sg
from _util import model_file, token_seqs

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _n_gpus(prod):
    return prod.lib.clip_b200_cuda_device_count()


def test_devices_mode_matches_single_gpu(prod):
    if _n_gpus(prod) < 2:
        pytest.skip("needs >= 2 GPUs")
    path = model_file("tiny", "q4_0", prod)
    imgs = sg.synth_images(37, 64, 3)
    seqs = token_seqs(40, 11)
    labels = token_seqs(13, 500)
    one = prod.load(path, 0)
    try:
        want_i, want_t = prod.image_batch_encode(one, imgs), prod.text_batch_encode(one, seqs)
        want_s, want_x = prod.zero_shot_images(one, imgs, labels, 5, normalize=True)
    finally:
        prod.free(one)
    os.environ["CLIP_B200_DEVICES"] = "all" if _n_gpus(prod) <= 8 else "0,1"
    try:
        ctx = prod.load(path, 0)
    finally:
        del os.environ["CLIP_B200_DEVICES"]
    try:
        assert prod.lib.clip_b200_device_count(ctx) == min(_n_gpus(prod), 8)
        got_i, got_t = prod.image_batch_encode(ctx, imgs), prod.text_batch_encode(ctx, seqs)
        assert np.array_equal(got_i, want_i)                   # same kernels, same per-item math: bit-identical
        assert np.array_equal(got_t, want_t)
        got_s, got_x = prod.zero_shot_images(ctx, imgs, labels, 5, normalize=True)
        # labels are encoded in per-GPU shards whose padded length differs from the single-GPU batch's: identical math up to the
        # summation order inside the softmax (the ragged-batch test pins that at 1e-6), so scores agree to ~1e-6 and the ranking
        # may only differ where two probabilities agree to that precision
        assert np.allclose(got_s, want_s, rtol=1e-4)
        diff = got_x != want_x
        assert diff.mean() < 0.1 and np.allclose(got_s[diff], want_s[diff], rtol=1e-4)
        # raw u8 images: per-GPU preprocess + encode, sharded like the f32 path
        rng = np.random.default_rng(5)
        u8 = [rng.integers(0, 256, (int(rng.integers(40, 200)), int(rng.integers(40, 200)), 3), dtype=np.uint8) for _ in range(19)]
        got_u8 = prod.image_batch_encode_u8(ctx, u8)
        host_px = np.stack([prod.preprocess(ctx, im) for im in u8])
        assert np.array_equal(got_u8, prod.image_batch_encode(ctx, host_px))
        # fewer items than GPUs, and a single item
        assert np.array_equal(prod.image_batch_encode(ctx, imgs[:1]), want_i[:1])
        assert np.array_equal(prod.text_batch_encode(ctx, seqs[:3]), want_t[:3])
    finally:
        prod.free(ctx)


def test_devices_mode_rejects_bad_lists(prod):
    path = model_file("tiny", "q4_0", prod)
    for bad in ("0,0", "99", "a,b", ","):
        os.environ["CLIP_B200_DEVICES"] = bad
        try:
            assert prod.lib.clip_model_load(path.encode(), 0) is None
        finally:
            del os.environ["CLIP_B200_DEVICES"]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_ranks_mode_all_gather_without_torch(prod):
    world = min(_n_gpus(prod), 4)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    path = model_file("tiny", "q4_0", prod)
    n_img, n_lab = 9, 7
    with tempfile.TemporaryDirectory() as td:
        out = os.path.join(td, "res")
        env = dict(os.environ, WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(_free_port()))
        ps = [subprocess.Popen([sys.executable, os.path.join(HERE, "dist_worker.py"), path, out, str(n_img), str(n_lab)],
                               env=dict(env, RANK=str(r), LOCAL_RANK=str(r)), stdout=subprocess.PIPE, stderr=subprocess.STDOUT) for r in range(world)]
        logs = [p.communicate(timeout=600)[0].decode()[-3000:] for p in ps]
        assert all(p.returncode == 0 for p in ps), "\n".join(logs)
        res = [dict(np.load(out + ".rank%d.npz" % r)) for r in range(world)]
    want_img = np.concatenate([r["local_img"] for r in res])
    want_txt = np.concatenate([r["local_txt"] for r in res])
    for r, z in enumerate(res):
        assert np.array_equal(z["img_all"], want_img) and np.array_equal(z["dev_all"], want_img)     # every rank holds everything, in rank order
        assert np.array_equal(z["txt_all"], want_txt)
        assert list(z["maxes"]) == [world - 1.0, 0.0]
        assert int(z["nccl"]) > 20000
        # zero-shot of this rank's images against ALL labels
        s = (z["local_img"] @ want_txt.T).astype(np.float32)
        e = (np.exp(s.astype(np.float64)) + 1e-9).astype(np.float32)
        p = (e.astype(np.float64) / e.astype(np.float64).sum(1, keepdims=True)).astype(np.float32)
        order = np.argsort(-p, axis=1, kind="stable")[:, :5]
        assert np.array_equal(z["zs_idx"], order)
        assert np.allclose(z["zs_scores"], np.take_along_axis(p, order, 1), rtol=1e-4)
