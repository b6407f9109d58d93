"""linear_1 on int8 slices (mode 2, k_gemm_q8): the kernel against a float64 model of its integer arithmetic, the host packing
of linear_1's weights (CPU), and the guard that keeps linear_1 off weights its slices cannot hold.

The model (no library code): the decoder's h is q = rint(fp32(clamp(h, -1, 1) * 32512)) split into q1 = floor((q + 128) / 256)
and q0 = q - 256 q1; output row n of linear_1 is w = rint(W sw_n), sw_n = 32512 / max_k |W[n][k]|, split the same way;
acc_hh = a1 . w1 and acc_mix = a1 . w0 + a0 . w1 are exact (float64 holds every partial sum below 2^53);
y = SELU((256 acc_hh + acc_mix) 256 / (32512 sw_n) + bias).  The kernel rounds 256 acc_hh + acc_mix and the column scale to
fp32 once each and takes SELU's exp from __expf, so the tolerance is a few fp32 ulps of the output, not an accumulation bound.
Run with -s for the MEASURE lines of the guard."""
import ctypes as C
import functools
import re

import numpy as np
import pytest

from tests.test_lstm_int8_gpu import qsplit, quantize
from tests.test_tc_layers_gpu import VT, rows_below, variant_inputs, variant_state

K = VT * 512
N = 512
QS = 32512.0
RTOL = ATOL = 2e-6
SELU_A, SELU_S = 1.6732632423543772848170429916717, 1.0507009873554804934193349852946


def selu(x):
    return SELU_S * np.where(x > 0, x, SELU_A * np.expm1(np.minimum(x, 0)))


def lin1_slices(W):
    """float64 w1, w0 [N][K] and sw [N] of the documented packing"""
    W = np.asarray(W, np.float64)
    m = np.abs(W).max(axis=1)
    sw = QS / np.where(m > 0, m, QS)
    w1, w0 = qsplit(np.rint(W * sw[:, None]))
    return w1.astype(np.float64), w0.astype(np.float64), sw


def untile_w(t, rows, cols):
    """[rows / 128][cols / 64][4][128][16] slice bytes -> [rows][cols]"""
    return t.reshape(rows // 128, cols // 64, 4, 128, 16).transpose(0, 3, 1, 2, 4).reshape(rows, cols)


def slices(x):
    """fp32 h [M][K] -> int8 slices a1, a0 [M][K] (quantize / qsplit of test_lstm_int8_gpu, row blocks to bound memory)"""
    a1, a0 = np.empty(x.shape, np.int8), np.empty(x.shape, np.int8)
    for r in range(0, x.shape[0], 512):
        s1, s0 = qsplit(quantize(x[r:r + 512]))
        a1[r:r + 512], a0[r:r + 512] = s1, s0
    return a1, a0


def model(a1, a0, W, bias):
    """float64 forward of the int32 accumulators: a1, a0 [R][K] integer slices"""
    w1, w0, sw = lin1_slices(W)
    a1, a0 = a1.astype(np.float64), a0.astype(np.float64)
    hh = a1 @ w1.T
    mix = a1 @ w0.T + a0 @ w1.T
    return selu((256.0 * hh + mix) * (256.0 / (QS * sw)) + np.asarray(bias, np.float64))


# ------------------------------------------------------------------------------------------------ CPU
def test_head_threshold_matches_header():
    import os
    from pepper_b200 import abi
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "pepper_b200.h")).read()
    m = re.search(r"#define\s+PB_VARIANT_Q8_HEAD_MAX_ERR\s+(\S+)", src)
    assert m and float(m.group(1)) == abi.PB_VARIANT_Q8_HEAD_MAX_ERR


def q8_pack(W, a_quant):
    from pepper_b200 import _lib
    L = _lib.lib()
    L.pb_test_q8_pack.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    W = np.ascontiguousarray(W, np.float32)
    n, k = W.shape
    w1, w0 = np.empty(n * k, np.int8), np.empty(n * k, np.int8)
    cs, err = np.empty(n, np.float32), np.empty(n, np.float64)
    _lib.check(L.pb_test_q8_pack(n, k, W.ctypes.data, a_quant, w1.ctypes.data, w0.ctypes.data, cs.ctypes.data, err.ctypes.data),
               "pb_test_q8_pack")
    return untile_w(w1, n, k).astype(np.int64), untile_w(w0, n, k).astype(np.int64), cs, err


def test_pack_round_trip():
    """linear_1's packing: w = 256 w1 + w0 within half a step of W sw_n per row, the slices in range, the column scale, the
    zero row's sw = 1, and the guard's per-row estimate restated in float64"""
    from oracle import nets
    W = nets.make_variant_weights(0)["linear_1.weight"].numpy().copy()
    W[5] = 0
    W[7] *= 1e-6
    W[9, 100] = 30 * W.std()
    w1, w0, cs, err = q8_pack(W, 1)
    W64 = W.astype(np.float64)
    m = np.abs(W64).max(axis=1)
    sw = QS / np.where(m > 0, m, QS)
    assert w1.min() >= -127 and w1.max() <= 127 and w0.min() >= -128 and w0.max() <= 127
    q = 256 * w1 + w0
    assert np.abs(q).max() <= 32512
    assert (np.abs(q / sw[:, None] - W64) <= 0.5 / sw[:, None] * (1 + 1e-9)).all()
    assert np.array_equal(cs, (256.0 / (QS * sw)).astype(np.float32))
    assert not q[5].any() and cs[5] == np.float32(256.0 / QS)
    r = q / sw[:, None] - W64
    d = w0 / sw[:, None]
    want = np.sqrt((r * r).sum(1) + 128.0 ** 2 / 3 / QS ** 2 * (d * d).sum(1) + (W64 * W64).sum(1) / (12 * QS ** 2))
    assert np.allclose(err, want, rtol=1e-9, atol=0)
    assert np.allclose(q8_pack(W, 0)[3], np.sqrt((r * r).sum(1) + 128.0 ** 2 / 3 / QS ** 2 * (d * d).sum(1)), rtol=1e-9, atol=0)
    # the outlier row's estimate is the largest: its scale coarsens every other weight of the row
    assert err.argmax() == 9


# ------------------------------------------------------------------------------------------------ GPU
@functools.lru_cache(maxsize=None)
def head_net(state_key="default"):
    from pepper_b200.variant import VariantNet
    return VariantNet(variant_state() if state_key == "default" else extreme_state())


def run_head(net, a1, a0, poison=1):
    """a1, a0 [M][K] int slices -> (out [M][512] fp32, act hi / lo tiles uint16)"""
    from pepper_b200 import _lib
    L = net.L
    L.pb_test_variant_head_q8.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    M = a1.shape[0]
    mt = -(-M // 128)
    q = np.ascontiguousarray(np.stack([a1, a0]).astype(np.int8))
    out = np.empty((M, N), np.float32)
    hi = np.empty((mt, 16, 4, 128, 8), np.uint16)
    lo = np.empty_like(hi)
    _lib.check(L.pb_test_variant_head_q8(net.h, M, q.ctypes.data, poison, out.ctypes.data, hi.ctypes.data, lo.ctypes.data),
               "pb_test_variant_head_q8")
    return out, hi, lo


def untile_act(t, M):
    """[mt][16][4][128][8] -> [mt * 128][512]"""
    mt = t.shape[0]
    return t.transpose(0, 3, 1, 2, 4).reshape(mt * 128, N)


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 130, 1000, 8448])
def test_head_q8_kernel(M):
    st = variant_state()
    net = head_net()
    x = variant_inputs()[1][:M].reshape(M, K)
    a1, a0 = slices(x)
    out, hi, lo = run_head(net, a1, a0)
    assert np.isfinite(out).all()
    rows = np.arange(M) if M <= 1000 else rows_below(M)
    want = model(a1[rows], a0[rows], st["linear_1.weight"].numpy(), st["linear_1.bias"].numpy())
    err = np.abs(out[rows] - want)
    assert (err <= ATOL + RTOL * np.abs(want)).all(), err.max()
    # the fp16 operand tiles linear_2 reads: hi = fp16(y), lo = fp16(y - hi) on valid rows; padding rows keep the poison
    h16, l16 = untile_act(hi, M), untile_act(lo, M)
    assert (h16[M:] == 0xffff).all() and (l16[M:] == 0xffff).all()
    y = out.astype(np.float32)
    want_hi = y.astype(np.float16)
    want_lo = (y - want_hi.astype(np.float32)).astype(np.float16)
    assert np.array_equal(h16[:M], want_hi.view(np.uint16)) and np.array_equal(l16[:M], want_lo.view(np.uint16))


def extreme_state():
    """variant_state() with every linear_1 weight at q = 32384 (w1 = 127, w0 = -128) and one per row at the row maximum"""
    import torch
    st = dict(variant_state())
    W = np.full((N, K), 32384.0 / 32512.0, np.float32)
    W[np.arange(N), np.arange(N) * 17] = 1.0
    W[1::2] *= -1
    st["linear_1.weight"] = torch.from_numpy(W)
    return st


@pytest.mark.gpu
def test_head_q8_extreme_slices():
    """every slice and weight at its extreme over K = 16,896: |acc_hh| = 2.7e8 and |acc_mix| = 5.5e8 accumulate exactly
    in int32 (an overflow would be off by 2^32 / 2^24 of the result)"""
    st = extreme_state()
    net = head_net("extreme")
    M = 128
    a1 = np.empty((M, K), np.int64)
    a0 = np.empty((M, K), np.int64)
    pat = [(127, -128), (-127, -128), (127, 127), (-127, 127)]
    for r in range(M):
        a1[r], a0[r] = pat[r % 4]
    a1[4::8] = np.where(np.arange(K) % 2, 127, -127)                     # alternating signs: sums that cancel exactly
    w1, w0, _ = lin1_slices(st["linear_1.weight"].numpy())
    assert np.abs(w1).max() == 127 and (w0 == -128).sum() == N * (K - 1)
    out, _, _ = run_head(net, a1, a0)
    want = model(a1, a0, st["linear_1.weight"].numpy(), st["linear_1.bias"].numpy())
    hh = a1[0].astype(np.float64) @ w1[0]
    assert abs(hh) > 2.7e8
    err = np.abs(out - want)
    assert (err <= ATOL + RTOL * np.abs(want)).all(), err.max()


# ------------------------------------------------------------------------------------------------ the guard
@pytest.mark.gpu
def test_head_guard_keeps_default_states_in_mode2():
    from oracle import nets
    from pepper_b200 import weights
    from pepper_b200.abi import PB_VARIANT_Q8_HEAD_MAX_ERR
    from pepper_b200.variant import VariantNet
    states = [("make_variant_weights(%d)" % s, nets.make_variant_weights(s)) for s in range(4)]
    states += [("random_variant_state(%d)" % s, weights.random_variant_state(s)) for s in (0, 3, 7)]
    # default weights already use a third of the 1e-3 gate (DESIGN.md "linear_1 on int8 slices"), so the threshold cannot sit
    # far above their estimate; 1.5x is the margin asked of them
    for name, st in states:
        net = VariantNet(st)
        print("MEASURE head guard %s: head_err %.3g (threshold %.3g), mode %d" % (name, net.head_q8_err,
                                                                                 PB_VARIANT_Q8_HEAD_MAX_ERR, net.mode))
        assert net.mode == 2 and net.head_q8_err < PB_VARIANT_Q8_HEAD_MAX_ERR / 1.5, name
        net.close()


# linear_1 replacements (test_weight_distributions_gpu._linear): one weight per output row at +-6 / +-9 std puts the guard's
# estimate (5.4e-5 / 8.1e-5) just above the threshold, +-30 / +-100 std and Student-t far above it; edge weights (zero and
# 1e-6 rows) stay below
LIN1_DISTS = ["t3", "outlier6", "outlier9", "outlier30", "outlier100", "edge"]


@functools.lru_cache(maxsize=None)
def lin1_state(dist):
    """the seeded state of test_weight_distributions_gpu with only linear_1 replaced"""
    import torch
    from oracle import nets
    from tests.test_weight_distributions_gpu import BASE_SEED, _linear
    st = dict(nets.make_variant_weights(BASE_SEED))
    W = st["linear_1.weight"].numpy().astype(np.float64)
    rng = np.random.default_rng([BASE_SEED, LIN1_DISTS.index(dist), 3])
    st["linear_1.weight"] = torch.from_numpy(_linear(rng, dist, W).astype(np.float32))
    return st


@functools.lru_cache(maxsize=None)
def lin1_f64(dist, n):
    import torch
    from oracle import nets
    from tests.test_nets_gpu import _variant_images
    from tests.test_weight_distributions_gpu import IMAGES
    m = nets.VariantNet()
    m.load_state_dict(lin1_state(dist))
    m = m.double().eval()
    with torch.no_grad():
        p, h = m(torch.from_numpy(_variant_images(n, IMAGES[n]).astype(np.float64)), return_hidden=True)
    return p.numpy(), h.numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("dist", LIN1_DISTS)
def test_head_guard_heavy_tails(dist):
    """heavy tails in linear_1 only: the estimate is reported; forced mode 2 either passes the 1e-3 gate against the float64
    module or the guard has put the network in mode 1, and the default mode passes"""
    from pepper_b200.abi import PB_VARIANT_Q8_HEAD_MAX_ERR
    from pepper_b200.variant import VariantNet
    from tests.test_nets_gpu import _variant_images
    from tests.test_weight_distributions_gpu import GATE, IMAGES, parity, passes
    net = VariantNet(lin1_state(dist))
    default = net.mode
    res = {}
    for mode in ("default", 2):
        if mode != "default":
            net.set_mode(mode)
        r = [parity(*net.predict(_variant_images(n, IMAGES[n]), return_hidden=True), *lin1_f64(dist, n)) for n in IMAGES]
        res[mode] = (max(x[0] for x in r), max(x[1] for x in r), sum(x[2] for x in r))
        print("MEASURE head %-10s mode %-7s: max|dh| %.3g  max|dp| %.3g (margin %.3g)  argmax mismatches %d  "
              "[head_err %.3g (threshold %.3g), gate_err %.3g, default mode %d]"
              % (dist, mode, res[mode][0], res[mode][1], GATE - res[mode][1], res[mode][2], net.head_q8_err,
                 PB_VARIANT_Q8_HEAD_MAX_ERR, net.q8_gate_err, default))
    net.close()
    assert passes(res["default"]), res["default"]
    if not passes(res[2]):
        assert default == 1, ("int8 linear_1 misses the gate but the guard kept mode 2", res[2])
