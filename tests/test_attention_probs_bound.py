"""The bound of tests/_attention_probs_bound.py, checked without a GPU: it holds for a numpy emulation of K9's arithmetic at every
block structure the kernel meets (one ragged block, exact multiples of 64 and 128, one key past them, several blocks, ViT-L/14@336's
577 tokens) and at any-resolution lengths (2049 causal, 4097), both operand types and head_dim 64, 80 and 104 (the operands padded
to the 112 columns the kernel multiplies), causal or not; and it is tight enough to reject two wrong results -- a softmax of
exponentials rounded to fp16 (what K3 multiplies V with) and a probability row shifted by one key."""
import numpy as np
import pytest

from _attention_bound import pattern_head
from _attention_probs_bound import emulate, exceed, reference_probs, round16, to_out

TS = [1, 17, 64, 65, 128, 129, 257, 577]


def operands(T, dh, bf, causal, seed, pattern="random"):
    """Q and K of one (sequence, head), rounded to the operand type; head_dim 104 padded with zeros to 112 columns"""
    rng = np.random.default_rng(seed)
    q, k, _ = pattern_head(pattern, T, dh, causal, rng)
    q, k = round16(q, bf), round16(k, bf)
    if dh == 104:
        q, k = (np.concatenate([x, np.zeros((T, 8), np.float32)], 1) for x in (q, k))
    return q, k


@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("dh", [64, 80, 104])
@pytest.mark.parametrize("bf", [0, 1])
def test_bound_holds_for_the_emulation(T, dh, bf):
    causal = int(T in (65, 129))
    q, k = operands(T, dh, bf, causal, 7 * T + dh + bf)
    p32 = emulate(q, k, causal)
    for out_type in (0, 1, 2):
        pi, bound = reference_probs(q, k, causal, bf, out_type)
        assert exceed(to_out(p32, out_type), pi, bound) <= 1.0, (T, dh, bf, out_type)


@pytest.mark.parametrize("T,causal", [(2049, 1), (4097, 0)])
@pytest.mark.parametrize("dh", [64, 104])
@pytest.mark.parametrize("bf", [0, 1])
def test_bound_holds_at_long_sequences(T, causal, dh, bf):
    """17 and 33 blocks of 128 keys: l summed over many rescaled blocks, every row, every output type"""
    q, k = operands(T, dh, bf, causal, 7 * T + dh + bf)
    p32 = emulate(q, k, causal)
    worst = 0.0
    for r0 in range(0, T, 1024):                # row slices keep the fp64 [rows, T] intermediates small
        rows = np.arange(r0, min(T, r0 + 1024))
        for out_type in (0, 1, 2):
            pi, bound = reference_probs(q, k, causal, bf, out_type, rows=rows)
            worst = max(worst, exceed(to_out(p32[rows], out_type), pi, bound))
    print("T=%d causal=%d dh=%d bf=%d: worst err/bound %.3f" % (T, causal, dh, bf, worst))
    assert worst <= 1.0, worst


@pytest.mark.parametrize("pattern", ["needle", "ramp", "late_spike", "early_spike"])
@pytest.mark.parametrize("causal", [0, 1])
def test_bound_holds_where_the_running_max_moves(pattern, causal):
    q, k = operands(577, 64, 1, causal, 11, pattern)
    pi, bound = reference_probs(q, k, causal, 1)
    assert exceed(emulate(q, k, causal), pi, bound) <= 1.0


@pytest.mark.parametrize("bf", [0, 1])
def test_bound_rejects_fp16_rounded_exponentials(bf):
    """softmax with each e^(s - m) rounded to fp16 before the division, as K3's P is before P.V"""
    q, k = operands(257, 64, bf, 0, 5)
    pi, bound = reference_probs(q, k, 0, bf)
    s = np.asarray(q, np.float64) @ np.asarray(k, np.float64).T
    w = np.exp(s - s.max(-1, keepdims=True)).astype(np.float16).astype(np.float64)
    assert exceed(w / w.sum(-1, keepdims=True), pi, bound) > 1.0


@pytest.mark.parametrize("causal", [0, 1])
def test_bound_rejects_a_row_shifted_by_one_key(causal):
    q, k = operands(129, 80, 1, causal, 9)
    p32 = emulate(q, k, causal)
    pi, bound = reference_probs(q, k, causal, 1)
    assert exceed(np.roll(p32, 1, axis=1), pi, bound) > 1.0
