"""GPU: the int8-slice decoder LSTM layer (mode 2, k_lstm_layer_q8) against an integer model of its arithmetic, and the
mode-2 network against the fp32 oracle.

The model (no library code):
  - an input or hidden value v is q = rint(fp32(clamp(v, -1, 1) * 32512)) split into q1 = floor((q + 128) / 256) and
    q0 = q - 256 q1;
  - the decoder weight row n (K = [W_ih | W_hh]) is w = rint(W sw_n) with sw_n = 32512 / max_k |W[n][k]|, split the same way;
  - acc_hh = a1 . w1 and acc_mix = a1 . w0 + a0 . w1 in int64 (exact, like the int32 wgmma accumulators);
  - gate = (65536 acc_hh + 256 acc_mix) / (32512 sw_n) + bias in float64, then the torch LSTM cell.
The model is teacher forced: step t multiplies the h slices the kernel wrote at step t - 1.  With exact accumulation the
only differences are the fp32 epilogue's (one rounding of 256 acc_hh + acc_mix, the column scale, ex2.approx-based
sigmoid / tanh), so the tolerance is the fp16 path's epilogue noise floor, not an accumulation bound."""
import ctypes as C
import functools

import numpy as np
import pytest

from tests.test_tc_layers_gpu import VH, VT, lstm_params, rows_below, sigmoid, variant_inputs, variant_state

pytestmark = pytest.mark.gpu

QS = np.float32(32512.0)
TOL = 5e-6
QBYTES_PER_MT = VT * 8 * 8192
TOL_NET = 1e-3
MARGIN = 1e-4


def qsplit(q):
    q = q.astype(np.int64)
    q1 = np.floor_divide(q + 128, 256)
    return q1, q - 256 * q1


def quantize(v):
    """fp32 activations -> the 16-bit fixed-point integer the kernels split"""
    return np.rint(np.clip(v.astype(np.float32), -1, 1) * QS).astype(np.int64)


def slices_of(Wih, Whh, bias):
    W = np.concatenate([Wih, Whh], axis=1)                         # torch row order; each row has its own scale
    m = np.abs(W).max(axis=1)
    sw = 32512.0 / np.where(m > 0, m, 32512.0)                     # an all-zero row keeps sw = 1
    w1, w0 = qsplit(np.rint(W * sw[:, None]))
    return w1, w0, 1.0 / (32512.0 * sw), bias


@functools.lru_cache(maxsize=None)
def weight_slices(d):
    return slices_of(*lstm_params(1, d))


def untile_q(q, M, rows):
    """[2][Mt][33][8][4][128][16] slice bytes -> q1, q0 [rows][33][512] int64"""
    mt = -(-M // 128)
    t = q.reshape(2, mt, VT, 8, 4, 128, 16).transpose(0, 1, 5, 2, 3, 4, 6)       # [2][mt][128][33][8][4][16]
    r = np.asarray(rows)
    s = t[:, r // 128, r % 128].reshape(2, r.size, VT, 512).astype(np.int64)
    return s[0], s[1]


@functools.lru_cache(maxsize=None)
def variant_net_q8():
    from pepper_b200.variant import VariantNet
    net = VariantNet(variant_state())
    net.L.pb_test_variant_lstm_q8.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                              C.c_void_p]
    return net


def run_q8(M, persist, poison, net=None):
    from pepper_b200 import _lib
    net = net or variant_net_q8()
    x = np.ascontiguousarray(variant_inputs()[1][:M])
    mt = -(-M // 128)
    y = np.empty((M, VT, 512), np.float32)
    q = np.empty(2 * mt * QBYTES_PER_MT, np.int8)
    c = np.empty((2, VH, M), np.float32)
    _lib.check(net.L.pb_test_variant_lstm_q8(net.h, M, x.ctypes.data, persist, poison, y.ctypes.data, q.ctypes.data,
                                             c.ctypes.data), "pb_test_variant_lstm_q8")
    return y, q, c


def model_dir(x, d, fed1, fed0, slices=None):
    """x [R][33][512] fp32 input; fed1 / fed0 [R][33][256]: the kernel's h slices of direction d; slices: slices_of() of
    the direction's weights (default: variant_state()'s)"""
    w1, w0, inv, bias = slices or weight_slices(d)
    a1, a0 = qsplit(quantize(x))
    R = x.shape[0]
    c = np.zeros((R, VH))
    out = np.zeros((R, VT, VH))
    steps = range(VT - 1, -1, -1) if d else range(VT)
    prev = None
    for t in steps:
        b1, b0 = a1[:, t], a0[:, t]
        if prev is None:
            hh = b1 @ w1[:, :512].T
            mix = b1 @ w0[:, :512].T + b0 @ w1[:, :512].T
        else:
            b1 = np.concatenate([b1, fed1[:, prev]], axis=1)
            b0 = np.concatenate([b0, fed0[:, prev]], axis=1)
            hh = b1 @ w1.T
            mix = b1 @ w0.T + b0 @ w1.T
        g = (65536.0 * hh + 256.0 * mix) * inv + bias
        i, f, gg, o = sigmoid(g[:, :VH]), sigmoid(g[:, VH:2 * VH]), np.tanh(g[:, 2 * VH:3 * VH]), sigmoid(g[:, 3 * VH:])
        c = f * c + i * gg
        out[:, t] = o * np.tanh(c)
        prev = t
    return out, c


@pytest.mark.parametrize("M", [1, 130, 1000, 8448])
def test_lstm_q8_layer(M):
    rows = rows_below(M)
    y, q, c = run_q8(M, persist=1, poison=1)
    assert np.isfinite(y).all() and np.isfinite(c).all()
    # the per-step launches (h handed over through HBM at kernel boundaries) agree bit for bit
    y0, q0_, c0 = run_q8(M, persist=0, poison=0)
    assert np.array_equal(y, y0) and np.array_equal(c, c0), np.abs(y - y0).max()
    # padding rows of the slice output are never written (the poison's 0xff bytes stay); valid rows match the other path
    mt = -(-M // 128)
    by_row = q.reshape(2, mt, -1, 128, 16).transpose(0, 1, 3, 2, 4)            # [2][mt][128 rows][k-chunks][16]
    by_row0 = q0_.reshape(2, mt, -1, 128, 16).transpose(0, 1, 3, 2, 4)
    pad = (np.arange(mt * 128) >= M).reshape(mt, 128)
    assert (by_row[:, pad] == -1).all()
    assert np.array_equal(by_row[:, ~pad], by_row0[:, ~pad])
    del y0, q0_, c0, by_row, by_row0
    # the slices are the quantization of the layer's own fp32 output (layout of the slice tiles)
    s1, s0 = untile_q(q, M, rows)
    w1, w0 = qsplit(quantize(y[rows]))
    assert np.array_equal(s1, w1) and np.array_equal(s0, w0)
    # kernel vs the integer model, teacher forced on the kernel's h slices
    x = variant_inputs()[1][rows]
    err_y, err_c = 0.0, 0.0
    for d in range(2):
        out, cd = model_dir(x, d, s1[:, :, d * VH:(d + 1) * VH], s0[:, :, d * VH:(d + 1) * VH])
        err_y = max(err_y, np.abs(out - y[rows][:, :, d * VH:(d + 1) * VH]).max())
        err_c = max(err_c, np.abs(cd - c[d][:, rows].T).max())
    assert err_y < TOL and err_c < 2 * TOL, (err_y, err_c)


def _check_parity(probs, hid, want, whid):
    assert np.abs(hid - whid).max() < TOL_NET, np.abs(hid - whid).max()
    assert np.abs(probs - want).max() < TOL_NET, np.abs(probs - want).max()
    srt = np.sort(want, axis=1)
    clear = (srt[:, -1] - srt[:, -2]) > MARGIN
    assert np.array_equal(probs.argmax(1)[clear], want.argmax(1)[clear])


def test_mode2_golden():
    """the reference model's own outputs (tests/golden/make_golden_nets.py) on its seed-0 weights"""
    import os
    from oracle import nets
    from pepper_b200.variant import VariantNet
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "variant_net_seed0.npz"))
    net = VariantNet(nets.make_variant_weights(0))
    net.set_mode(2)
    probs, hid = net.predict(g["images"], return_hidden=True)
    _check_parity(probs, hid[:4], g["probs"], g["hidden"])


@pytest.mark.parametrize("n,seed", [(1, 1), (130, 2), (700, 3)])
def test_mode2_vs_oracle(n, seed):
    from oracle import nets
    from pepper_b200.variant import VariantNet
    from tests.test_nets_gpu import _variant_images
    state = nets.make_variant_weights(seed)
    x = _variant_images(n, seed)
    want, whid = nets.variant_predict(state, x, threads=8, return_hidden=True)
    net = VariantNet(state)
    p_default, h_default = net.predict(x, return_hidden=True)         # mode 2 is the default
    net.set_mode(2)
    got, hid = net.predict(x, return_hidden=True)
    assert np.array_equal(got, p_default) and np.array_equal(hid, h_default)
    _check_parity(got, hid, want, whid)
    net.set_lo_mask(0x1a)                                             # back to mode 1: the fp16 split's bits apply again
    p1 = net.predict(x)
    net.set_mode(1)
    assert np.array_equal(net.predict(x), p1)


def test_mode2_random_state_batch_invariance():
    """seeded random weights (pepper_b200.weights): a candidate's probabilities do not depend on the batch or on where
    the 8,448-candidate chunk boundary falls"""
    from pepper_b200 import weights
    from pepper_b200.variant import VariantNet
    from tests.test_nets_gpu import _variant_images
    net = VariantNet(weights.random_variant_state(7))
    net.set_mode(2)
    x = _variant_images(8448 + 300, 12)
    full = net.predict(x)
    assert np.isfinite(full).all() and np.allclose(full.sum(1), 1.0, atol=1e-5)
    for lo, hi in ((0, 130), (8400, 8500), (8448, 8748)):
        assert np.array_equal(net.predict(x[lo:hi]), full[lo:hi])
