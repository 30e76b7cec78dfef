"""K3 is persistent: each CTA strides over pairs of 64-row query groups numbered in (sequence, head, group) order, and a pair may
straddle two heads.  Where an item lands in that schedule -- which CTA, which iteration, which warpgroup, paired with which other
group, which ring stage (two stages of 128-key blocks at head_dim 64 and 80, three of 64-key blocks at 104) -- must not change a
single bit of its output.  Each case runs a batch, the same sequences in permuted
order, and a few of them alone, compares the bytes, and checks the sequences run alone against the fp64 restatement at the bound of
tests/test_gpu_attention.py."""
import numpy as np
import pytest

from test_gpu_attention_hd80 import check, ref_attention, run

pytestmark = pytest.mark.gpu

H = 3          # odd: with an odd number of groups per head, every other warpgroup pair straddles two heads
SMS = 132
# T (64-row groups per head: 1 1 1 1 1 1 2 2 2 3 3 4 5 5 10 17 4 16 33), causal
CASES = [(1, 0), (16, 0), (17, 0), (50, 0), (63, 0), (64, 0), (65, 0), (77, 1), (128, 0), (129, 0), (192, 0), (256, 0), (257, 0),
         (320, 0), (577, 0), (1025, 0), (248, 1), (1000, 1), (2049, 1)]
# groups in the launch against 2 x 132 (one pair per SM): below, about at, several times above
GROUPS = {"below": 40, "at": 2 * SMS, "above": 8 * SMS}


@pytest.mark.parametrize("load", list(GROUPS))
@pytest.mark.parametrize("T,causal", CASES)
@pytest.mark.parametrize("dh", [64, 80, 104])
@pytest.mark.parametrize("bf", [1, 0])
def test_output_independent_of_schedule(prod, T, causal, dh, bf, load):
    ngrp = -(-T // 64)
    nseq = max(2, -(-GROUPS[load] // (H * ngrp))) | 1      # odd: an odd group count when ngrp is odd leaves the last warpgroup idle
    rng = np.random.default_rng(T * 131 + dh + 7 * bf + GROUPS[load])
    qkv = rng.standard_normal((nseq, T, 3 * H * dh)).astype(np.float32)
    qkv[:, :, : H * dh] *= 3.0 / np.sqrt(dh)
    batch = run(prod, qkv.reshape(nseq * T, -1), nseq, T, H, causal, bf, dh=dh).reshape(nseq, T, H * dh)

    perm = rng.permutation(nseq)
    permuted = run(prod, qkv[perm].reshape(nseq * T, -1), nseq, T, H, causal, bf, dh=dh).reshape(nseq, T, H * dh)
    assert np.array_equal(permuted.view(np.uint32), batch[perm].view(np.uint32))

    for s in sorted({0, nseq // 2, nseq - 1}):
        alone = run(prod, qkv[s], 1, T, H, causal, bf, dh=dh)
        assert np.array_equal(alone.view(np.uint32), batch[s].view(np.uint32)), s
        check(alone, ref_attention(qkv[s], 1, T, H, causal, bf, dh=dh))
