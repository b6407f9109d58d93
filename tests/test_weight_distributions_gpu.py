"""GPU: the variant network and its LSTM layers on heavy-tailed and degenerate weights against float64, and the int8 guard
that keeps the decoder off weights its slices cannot hold.

Every other test runs on default-init (uniform) weights, where a gate row's largest |w| is about 1.7x its std.  Trained LSTM
weights are heavy-tailed, and mode 2 holds each decoder gate row as 16-bit integers at a scale set by the row's largest
|w|, so one large weight coarsens every other weight of its row.  The states here start from oracle.nets.make_variant_weights
and replace the chosen matrices:
  uniform     unchanged;
  t3          Student-t with 3 degrees of freedom, rescaled to the matrix's std;
  outlier30   one weight per gate row (linear_1: per output row) set to +-30 x the matrix's std in a random column, in the
  outlier100  W_ih columns on even rows and the W_hh columns on odd rows; +-100 x std;
  edge        a few all-zero gate rows (the quantizer's sw = 1 fallback), a few rows scaled by 1e-6 (very small column
              scales), and a forget-gate bias of +3 on every fourth unit.
Each is applied to the encoder only, the decoder only, or both LSTM layers plus linear_1 ("all").  A matrix gets the same
replacement in every scope it belongs to.

Checks:
  * layer, decoder in mode 2 (pb_test_variant_lstm_q8): the teacher-forced integer model of test_lstm_int8_gpu within its
    5e-6 on every distribution; free running against a float64 LSTM of the unquantized weights, within the parity gate
    wherever the guard keeps the network in mode 2;
  * layer, mode 1 (pb_test_variant_lstm_layer, every product on): against exact float64 within FP32_FACTOR x the error of a
    float32 torch layer (assertion 3 of test_tc_layers_gpu);
  * network: VariantNet in modes 0, 1 and its default mode against a float64 forward of the oracle's nn.Module, at the parity
    gate (hidden states and probabilities within 1e-3, argmax equal where the top-2 margin exceeds 1e-4); mode 2 forced is
    measured, and wherever it misses the gate the guard must have chosen mode 1.
Run with -s for the MEASURE lines (max |dh|, |dp| per distribution, scope and mode, and the margin to 1e-3)."""
import ctypes as C
import functools

import numpy as np
import pytest

from tests.test_lstm_int8_gpu import TOL, model_dir, run_q8, slices_of, untile_q
from tests.test_tc_layers_gpu import CHECK_ROWS, FP32_FACTOR, VH, lstm_dir, rows_below, run_lstm, variant_inputs
from tests.test_nets_gpu import _variant_images

pytestmark = pytest.mark.gpu

GATE = 1e-3
MARGIN = 1e-4
DISTS = ["uniform", "t3", "outlier30", "outlier100", "edge"]
HEAVY = DISTS[1:]
SCOPES = ["encoder", "decoder", "all"]
NET_CASES = [("uniform", "all")] + [(d, s) for d in HEAVY for s in SCOPES]
IMAGES = {1: 1, 130: 2, 700: 3}           # n -> image seed
BASE_SEED = 4


# ------------------------------------------------------------------------------------------------ weight states
def _t3(rng, W):
    X = rng.standard_t(3, size=W.shape)
    return X * (W.std() / X.std())


def _outliers(rng, W, k, rows):
    sd = W.std()
    W = W.copy()
    cols = rng.integers(0, W.shape[1], size=len(rows))
    W[rows, cols] = k * sd * rng.choice([-1.0, 1.0], size=len(rows))
    return W


def _lstm_direction(rng, dist, Wih, Whh, bias_ih):
    if dist == "t3":
        return _t3(rng, Wih), _t3(rng, Whh), bias_ih
    if dist.startswith("outlier"):
        k = float(dist[len("outlier"):])
        n = np.arange(Wih.shape[0])
        return _outliers(rng, Wih, k, n[0::2]), _outliers(rng, Whh, k, n[1::2]), bias_ih
    assert dist == "edge"
    Wih, Whh, bias_ih = Wih.copy(), Whh.copy(), bias_ih.copy()
    zero, tiny = [3, 260, 515, 1000], [9, 270, 777, 1023]      # rows of i, f, g and o gates
    Wih[zero] = 0
    Whh[zero] = 0
    Wih[tiny] *= 1e-6
    Whh[tiny] *= 1e-6
    bias_ih[VH:2 * VH:4] += 3.0                                 # forget gates of every fourth unit
    return Wih, Whh, bias_ih


def _linear(rng, dist, W):
    if dist == "t3":
        return _t3(rng, W)
    if dist.startswith("outlier"):
        return _outliers(rng, W, float(dist[len("outlier"):]), np.arange(W.shape[0]))
    W = W.copy()
    W[[5, 300]] = 0
    W[[7, 411]] *= 1e-6
    return W


@functools.lru_cache(maxsize=None)
def weight_state(dist, scope):
    """the seeded state_dict (torch fp32 tensors) of `dist` applied to `scope`"""
    import torch
    from oracle import nets
    st = {k: v.numpy().astype(np.float64) for k, v in nets.make_variant_weights(BASE_SEED).items()}
    if dist != "uniform":
        layers = {"encoder": ["encoder"], "decoder": ["decoder"], "all": ["encoder", "decoder"]}[scope]
        for li, layer in enumerate(["encoder", "decoder"]):
            if layer not in layers:
                continue
            for d, suf in enumerate(["", "_reverse"]):
                p = f"{layer}.%s_l0{suf}"
                rng = np.random.default_rng([BASE_SEED, DISTS.index(dist), li, d])
                st[p % "weight_ih"], st[p % "weight_hh"], st[p % "bias_ih"] = _lstm_direction(
                    rng, dist, st[p % "weight_ih"], st[p % "weight_hh"], st[p % "bias_ih"])
        if scope == "all":
            st["linear_1.weight"] = _linear(np.random.default_rng([BASE_SEED, DISTS.index(dist), 2]), dist,
                                            st["linear_1.weight"])
    return {k: torch.from_numpy(v.astype(np.float32)) for k, v in st.items()}


def lstm_weights(state, layer, d):
    """float64 W_ih, W_hh and the fp32 sum of the two biases (the packed bias) of one direction"""
    p = ("encoder" if layer == 0 else "decoder") + ".%s_l0" + ("_reverse" if d else "")
    f64 = lambda t: t.numpy().astype(np.float64)
    return f64(state[p % "weight_ih"]), f64(state[p % "weight_hh"]), f64(state[p % "bias_ih"] + state[p % "bias_hh"])


@functools.lru_cache(maxsize=None)
def variant_net(dist, scope):
    from pepper_b200.variant import VariantNet
    net = VariantNet(weight_state(dist, scope))
    L = net.L
    L.pb_test_variant_lstm_q8.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.pb_test_variant_lstm_layer.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return net


def layer_scope(layer):
    return "encoder" if layer == 0 else "decoder"


# ------------------------------------------------------------------------------------------------ layer references
@functools.lru_cache(maxsize=None)
def lstm_exact(dist, layer):
    """float64 layer output [CHECK_ROWS][33][512] on the unquantized weights"""
    st = weight_state(dist, layer_scope(layer))
    x = variant_inputs()[layer][CHECK_ROWS].astype(np.float64)
    return np.concatenate([lstm_dir(x, *lstm_weights(st, layer, d), 1, 1, d == 1, True)[0] for d in range(2)], axis=2)


@functools.lru_cache(maxsize=None)
def lstm_torch_fp32(dist, layer):
    import torch
    name = layer_scope(layer)
    st = weight_state(dist, name)
    m = torch.nn.LSTM(26 if layer == 0 else 512, VH, batch_first=True, bidirectional=True)
    m.load_state_dict({k[len(name) + 1:]: v for k, v in st.items() if k.startswith(name + ".")})
    with torch.no_grad():
        y, _ = m(torch.from_numpy(variant_inputs()[layer][CHECK_ROWS].astype(np.float32)))
    return y.numpy().astype(np.float64)


@pytest.mark.parametrize("M", [1, 130, 8448])
@pytest.mark.parametrize("dist", DISTS)
def test_q8_layer(dist, M):
    """mode 2's decoder layer: exact to the integer model, and within the gate of float64 where the guard keeps mode 2"""
    st = weight_state(dist, "decoder")
    net = variant_net(dist, "decoder")
    rows = rows_below(M)
    y, q, c = run_q8(M, persist=1, poison=1, net=net)
    assert np.isfinite(y).all() and np.isfinite(c).all()
    s1, s0 = untile_q(q, M, rows)
    x = variant_inputs()[1][rows]
    err_y, err_c = 0.0, 0.0
    for d in range(2):
        out, cd = model_dir(x, d, s1[:, :, d * VH:(d + 1) * VH], s0[:, :, d * VH:(d + 1) * VH],
                            slices=slices_of(*lstm_weights(st, 1, d)))
        err_y = max(err_y, np.abs(out - y[rows][:, :, d * VH:(d + 1) * VH]).max())
        err_c = max(err_c, np.abs(cd - c[d][:, rows].T).max())
    free = np.abs(y[rows] - lstm_exact(dist, 1)[np.searchsorted(CHECK_ROWS, rows)]).max()
    print("MEASURE q8 layer %-10s M %4d: |y - int model| %.3g  |c - int model| %.3g  free running vs float64 %.3g  "
          "(gate_err %.3g, mode %d)" % (dist, M, err_y, err_c, free, net.q8_gate_err, net.mode))
    assert err_y < TOL and err_c < 2 * TOL, (err_y, err_c)
    if net.mode == 2:
        assert free < GATE, free


@pytest.mark.parametrize("M", [1, 130, 8448])
@pytest.mark.parametrize("layer", [0, 1])
@pytest.mark.parametrize("dist", DISTS)
def test_mode1_layer(dist, layer, M):
    """the fp16-split layer (every product on, power-of-two per-matrix scale) stays within FP32_FACTOR of a float32 layer"""
    net = variant_net(dist, layer_scope(layer))
    rows = rows_below(M)
    y, c, _, _ = run_lstm(layer, M, 1, 1, persist=1, poison=0, tiles=False, net=net)
    assert np.isfinite(y).all() and np.isfinite(c).all()
    sel = np.searchsorted(CHECK_ROWS, rows)
    exact = lstm_exact(dist, layer)[sel]
    e_kernel = np.abs(y[rows] - exact).max()
    e_torch = np.abs(lstm_torch_fp32(dist, layer)[sel] - exact).max()
    print("MEASURE mode-1 layer %d %-10s M %4d: kernel vs float64 %.3g, torch fp32 vs float64 %.3g" % (layer, dist, M, e_kernel, e_torch))
    assert e_kernel <= FP32_FACTOR * e_torch, (e_kernel, e_torch)


# ------------------------------------------------------------------------------------------------ network
@functools.lru_cache(maxsize=None)
def net_f64(dist, scope, n):
    """float64 forward of the oracle's nn.Module: probabilities [n][3], hidden states [n][33][512]"""
    import torch
    from oracle import nets
    m = nets.VariantNet()
    m.load_state_dict(weight_state(dist, scope))
    m = m.double().eval()
    with torch.no_grad():
        p, h = m(torch.from_numpy(_variant_images(n, IMAGES[n]).astype(np.float64)), return_hidden=True)
    return p.numpy(), h.numpy()


def parity(probs, hid, want, whid):
    """(max |dh|, max |dp|, argmax mismatches where the float64 top-2 margin exceeds 1e-4)"""
    srt = np.sort(want, axis=1)
    clear = (srt[:, -1] - srt[:, -2]) > MARGIN
    return (float(np.abs(hid - whid).max()), float(np.abs(probs - want).max()),
            int((probs.argmax(1)[clear] != want.argmax(1)[clear]).sum()))


def passes(r):
    return r[0] < GATE and r[1] < GATE and r[2] == 0


@pytest.mark.parametrize("dist,scope", NET_CASES)
def test_network(dist, scope):
    net = variant_net(dist, scope)
    default = net.mode
    res = {}
    try:
        for mode in ("default", 0, 1, 2):
            if mode != "default":
                net.set_mode(mode)
                assert net.mode == mode                      # an explicit mode is honoured, the guard's choice included
            r = [parity(*net.predict(_variant_images(n, IMAGES[n]), return_hidden=True), *net_f64(dist, scope, n))
                 for n in IMAGES]
            res[mode] = (max(x[0] for x in r), max(x[1] for x in r), sum(x[2] for x in r))
            print("MEASURE network %-10s %-7s mode %-7s: max|dh| %.3g (margin %.3g)  max|dp| %.3g (margin %.3g)  "
                  "argmax mismatches %d  [gate_err %.3g, default mode %d]"
                  % (dist, scope, mode, res[mode][0], GATE - res[mode][0], res[mode][1], GATE - res[mode][1],
                     res[mode][2], net.q8_gate_err, default))
    finally:
        net.set_mode(default)
    for mode in ("default", 0, 1):
        assert passes(res[mode]), (mode, res[mode])
    if not passes(res[2]):
        assert default == 1, ("mode 2 misses the gate but the guard kept it", res[2], net.q8_gate_err)


# ------------------------------------------------------------------------------------------------ the guard
def test_guard_keeps_uniform_init_in_mode2():
    """default-init weights (the oracle's seeds, the product's seeded states, the benchmark's weights) keep mode 2"""
    from oracle import nets
    from pepper_b200 import weights
    from pepper_b200.abi import PB_VARIANT_Q8_MAX_GATE_ERR
    from pepper_b200.variant import VariantNet
    states = [("make_variant_weights(%d)" % s, nets.make_variant_weights(s)) for s in range(4)]
    states += [("random_variant_state(%d)" % s, weights.random_variant_state(s)) for s in (0, 3, 7)]
    for name, st in states:
        net = VariantNet(st)
        print("MEASURE guard %s: gate_err %.3g (threshold %.3g), mode %d" % (name, net.q8_gate_err, PB_VARIANT_Q8_MAX_GATE_ERR,
                                                                            net.mode))
        assert net.mode == 2 and net.q8_gate_err < PB_VARIANT_Q8_MAX_GATE_ERR / 2, name
        net.close()


@pytest.mark.parametrize("dist", ["outlier30", "outlier100"])
def test_guard_fallback_is_mode1(dist):
    """a network the guard put in mode 1 computes what set_mode(1) computes, bit for bit, and set_mode(2) still reaches the
    int8 decoder; the callers built on VariantNet take the same default"""
    from pepper_b200.dist import DistributedVariantCaller
    from pepper_b200.pipeline import VariantCaller
    from pepper_b200.variant import VariantNet
    st = weight_state(dist, "decoder")
    net = VariantNet(st)
    assert net.mode == 1
    x = _variant_images(300, 5)
    p, h = net.predict(x, return_hidden=True)
    net.set_mode(1)
    p1, h1 = net.predict(x, return_hidden=True)
    assert np.array_equal(p, p1) and np.array_equal(h, h1)
    net.set_mode(2)
    assert net.mode == 2
    p2, h2 = net.predict(x, return_hidden=True)
    assert not np.array_equal(h2, h1)
    net.close()
    vc = VariantCaller(st)
    assert vc.net.mode == 1
    vc.close()
    dvc = DistributedVariantCaller(st, 0, 1024, distributed=False)
    assert dvc.caller.net.mode == 1
    dvc.close()
