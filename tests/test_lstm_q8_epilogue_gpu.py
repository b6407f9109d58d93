"""GPU: k_lstm_layer_q8 cut into launches of fewer steps.

The decoder layer hands each gate tile's pre-activations to an epilogue warpgroup, and h_t to the next step's h-part, through
barriers whose phases count from the launch's first step.  A layer run as launches of 1, 2, 5 or 32 steps starts those
barriers at t0 > 0 and hands h and c over through HBM at every launch boundary; the results must be bit-identical to one
launch of all 33 steps, and padding rows must stay unwritten (the test hook reports a written padding row of y_f32 as an
error under poison)."""
import numpy as np
import pytest

from tests.test_lstm_int8_gpu import run_q8

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M", [1, 130, 1000, 8448])
def test_lstm_q8_launch_split(M):
    y, q, c = run_q8(M, persist=1, poison=1)
    assert np.isfinite(y).all() and np.isfinite(c).all()
    mt = -(-M // 128)
    pad = (np.arange(mt * 128) >= M).reshape(mt, 128)
    by_row = q.reshape(2, mt, -1, 128, 16).transpose(0, 1, 3, 2, 4)            # [2][mt][128 rows][k-chunks][16]
    assert (by_row[:, pad] == -1).all()
    for steps in (0, 2, 5, 32):                                                 # persist 0: one launch per step
        ys, qs, cs = run_q8(M, persist=steps, poison=1)
        assert np.array_equal(ys, y), (steps, np.abs(ys - y).max())
        assert np.array_equal(qs, q), steps
        assert np.array_equal(cs, c), steps                                     # c read back through c_index
        del ys, qs, cs
