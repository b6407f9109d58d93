"""GPU: the int8 slices the encoder LSTM layer hands the mode-2 decoder (k_lstm_layer_enc with the slice output).

The layer's fp16 output and fp32 copy are checked against the per-step path in test_tc_layers_gpu.py; its slice output is
not.  Each slice pair must be the 16-bit fixed-point split of the per-step path's fp32 h, bit for bit:
q = rint(h * 32512) (fp32 multiply, ties to even), q1 = floor((q + 128) / 256), q0 = q - 256 q1; and with the slice buffer
poisoned (0xff) before the launch, the padding rows of the last row tile keep the poison."""
import ctypes as C
import functools

import numpy as np
import pytest

from tests.test_tc_layers_gpu import VT, run_lstm, variant_inputs, variant_net

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _net():
    net = variant_net()
    net.L.pb_test_variant_enc_q8.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    return net


def slices_of(h):
    """fp32 h [..] -> (q1, q0) int8, the encoder epilogue's qbias split"""
    q = np.rint(h.astype(np.float32) * np.float32(32512.0)).astype(np.int64)
    q1 = (q + 128) >> 8
    return q1.astype(np.int8), (q - 256 * q1).astype(np.int8)


@pytest.mark.parametrize("M", [1, 130, 1000, 8448])
def test_encoder_q8_slices(M):
    from pepper_b200 import _lib
    net = _net()
    mt = -(-M // 128)
    x = np.ascontiguousarray(variant_inputs()[0][:M])
    raw = np.empty(2 * mt * VT * 8 * 128 * 64, np.int8)
    _lib.check(net.L.pb_test_variant_enc_q8(net.h, M, x.ctypes.data, 1, raw.ctypes.data), "pb_test_variant_enc_q8")
    # [slice][mt][t][k-tile][16-k chunk][row][16] -> [slice][row][t][feature d * 256 + unit]
    q = raw.reshape(2, mt, VT, 8, 4, 128, 16).transpose(0, 1, 5, 2, 3, 4, 6).reshape(2, mt * 128, VT, 512)
    assert (q[:, M:] == -1).all(), "a padding row of the slice tiles was written"
    y, _, _, _ = run_lstm(0, M, 1, 0, persist=0, poison=0, tiles=False)
    q1, q0 = slices_of(y)
    assert np.array_equal(q[0, :M], q1), np.argwhere(q[0, :M] != q1)[:5]
    assert np.array_equal(q[1, :M], q0), np.argwhere(q[1, :M] != q0)[:5]
