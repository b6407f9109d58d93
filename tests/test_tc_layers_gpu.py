"""GPU: the wgmma GEMM, LSTM-layer and GRU-layer kernels, one layer at a time, against a float64 model of the arithmetic
they are documented to perform.

The model (no library code: it splits, scales and accumulates by itself):
  - every fp32 operand value v is split into fp16 hi = rn(clamp(v, +-65504)) and lo = rn(v - hi);
  - each packed weight matrix W (an RNN direction: x-part and h-part together) is multiplied by s = 2^(15 - ceil(log2 max|W|))
    before the split, and the accumulator is multiplied by 1/s before the bias is added;
  - products: a_hi w_hi + a_hi w_lo, plus a_lo w_hi where that operand's lo flag is set, summed in float64;
  - cells with torch semantics (LSTM gates i, f, g, o; GRU r, z, n with n = tanh(W_in x + b_in + r (W_hn h + b_hn));
    SELU), h fed back to the next step as its fp16 hi + lo.

Each case asserts:
  1. kernel vs the model with the same flags: max |diff| <= tol (the accumulation / fast-math noise floor, derived below).
     The recurrent models are teacher forced: step t multiplies the h operands (hi, lo) the kernel wrote at step t - 1;
  2. the model with one flag flipped differs from the model by >= 5 tol on the same data and operands, so (1) can tell a
     dropped or misrouted product from noise;
  3. with every product on, kernel vs exact float64 within FP32_FACTOR x what a float32 torch layer gets on the same
     inputs.  Measured on H100 the ratio is 5.3 (LSTM encoder), 4.3 (decoder), 2.3 / 2.6 (GRU encoder / decoder, against
     the larger of torch and the 22-bit model), 2.5-3.8 for GEMMs up to K = 512, so the path is not "fp32-equivalent"
     against a float32 CPU layer, and at K = 16,896 a GEMM is 190x a blocked float32 CPU GEMM (see test_tc_gemm_layer);
  4. the persistent and the per-step LSTM paths are bit-identical;
  5. the output tiles reconstruct the fp32 output to 2^-22 relative; under poison (every operand buffer NaN before the
     launch) valid rows stay finite and the padding rows of the output tiles are never written.

The kernels run every row of M; the float64 model runs a fixed set of rows (tile edges, the last CTA's rows, random
rows), which is enough because rows never interact.

Tolerances.  A pre-activation sums K exact fp16 x fp16 products (K = x-part + h-part columns, x 2-3 products) in fp32
wgmma accumulators.  The accumulation order and rounding inside wgmma are not documented; measured on H100 the error
grows about linearly with K, from ~3 x 2^-24 sum_k |a_k w_k| at K = 32 to ~62 x 2^-24 at K = 16,896 (tol_gemm allows
(16 + K / 128) x 2^-24).  A gate of the variant encoder sums 26 products of |x| <= 128 and |w| <= 1/16 plus the h-part:
|p| sums of ~50 give ~3e-6 in z.  The epilogue adds the error of __expf / __fdividef (ex2.approx: 2 ulp, after a
multiply that carries |x| 2^-24 relative), ~2^-21 absolute on each sigmoid / tanh, and the cell state carries both over
the steps; the GRU output is read back as hi + lo (2^-23 relative).  Measured maxima on H100 (80GB HBM3, 700 W, SM clock
1560-1740 MHz under the power cap), teacher forced, over every M and flag set: LSTM encoder 4.0e-6, decoder 2.0e-6;
GRU encoder 2.7e-6, decoder 2.3e-6.  Smallest flag gaps on the same data: LSTM encoder h 1.5e-4; decoder h 2.1e-5,
x 1.2e-4; GRU encoder h 3.1e-4; decoder h 1.8e-4, x 4.9e-4."""
import ctypes as C
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FP16_MAX = 65504.0
MAX_M = 8448                 # the production k_lstm_layer grid: 66 row tiles x 2 directions = 132 CTAs
MS = [1, 127, 128, 129, 1000, 8448]
VT, VH, PT, PH = 33, 256, 100, 128

# noise floors (max |h_kernel - h_model| over every checked row, step and unit); see the module docstring
TOL_LSTM = {0: 8e-6, 1: 3e-6}      # measured 4.0e-6, 2.0e-6
TOL_GRU = {0: 1.5e-5, 1: 1e-5}     # measured 2.7e-6, 2.3e-6
FP32_FACTOR = 8                    # assertion 3: kernel vs exact within this many times the float32 torch layer's error


def tol_gemm(K):
    """per element, x sum_k |a_k w_k| (+ 2^-20 absolute for the SELU epilogue)"""
    return 2.0 ** -24 * (16 + K / 128)


# ------------------------------------------------------------------------------------------------ float64 model
def split16(v):
    """fp32 value -> (hi, lo) as float64, the hi / lo split of the operand packing and of the kernels' epilogues."""
    v32 = np.asarray(v, np.float64).astype(np.float32)
    hi = np.clip(v32, -FP16_MAX, FP16_MAX).astype(np.float16)
    lo = np.clip(v32 - hi.astype(np.float32), -FP16_MAX, FP16_MAX).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)


def pow2_scale(*mats):
    m = max(float(np.abs(w).max()) for w in mats)
    return 2.0 ** (15 - np.ceil(np.log2(m)))


class SplitLinear:
    """a -> a W^T on the tensor cores: W scaled by s and split once; `lo` adds the a_lo w_hi product.  exact=True: plain
    float64 a W^T (the reference the fp32-equivalence claim is measured against)."""

    def __init__(self, W, s, exact=False):
        self.exact = exact
        self.W = np.asarray(W, np.float64)
        if not exact:
            self.s = s
            wh, wl = split16(self.W * s)
            self.wsum, self.wh = (wh + wl).T.copy(), wh.T.copy()

    def __call__(self, a, lo, parts=None):
        if self.exact:
            return a @ self.W.T
        ah, al = split16(a) if parts is None else parts
        acc = ah @ self.wsum
        if lo:
            acc += al @ self.wh
        return acc / self.s


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def feed(h, exact):
    """what the next step multiplies: the fp16 hi + lo of the fp32 h (exact model: h itself)"""
    if exact:
        return h
    hi, lo = split16(h)
    return hi + lo


def lstm_dir(x, Wih, Whh, bias, lo_x, lo_h, reverse, exact, forced=None):
    """forced = (hi, lo) [R][T][256]: the operands the kernel fed back, used as the h-part of the next step (teacher
    forcing), so that a step is compared on exactly the operands the kernel multiplied"""
    s = pow2_scale(Wih, Whh)
    fx, fh = SplitLinear(Wih, s, exact), SplitLinear(Whh, s, exact)
    R, T, _ = x.shape
    zx = fx(x.reshape(R * T, -1), lo_x).reshape(R, T, -1)
    h = np.zeros((R, VH))
    c = np.zeros((R, VH))
    out = np.zeros((R, T, VH))
    prev = None
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        parts = None if forced is None or prev is None else (forced[0][:, prev], forced[1][:, prev])
        g = zx[:, t] + fh(feed(h, exact), lo_h, parts) + bias
        prev = t
        i, f, gg, o = sigmoid(g[:, :VH]), sigmoid(g[:, VH:2 * VH]), np.tanh(g[:, 2 * VH:3 * VH]), sigmoid(g[:, 3 * VH:])
        c = f * c + i * gg
        h = o * np.tanh(c)
        out[:, t] = h
    return out, c


def gru_dir(x, h0, Wih, Whh, bih, bhh, lo_x, lo_h, reverse, exact, forced=None):
    s = pow2_scale(Wih, Whh)
    fx, fh = SplitLinear(Wih, s, exact), SplitLinear(Whh, s, exact)
    R, T, _ = x.shape
    zx = fx(x.reshape(R * T, -1), lo_x).reshape(R, T, -1)
    brz = (bih[:2 * PH] + bhh[:2 * PH]).astype(np.float32).astype(np.float64)      # packed as one fp32 bias
    h = np.asarray(h0, np.float64)
    out = np.zeros((R, T, PH))
    prev = None
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        if forced is None or prev is None:
            hf = feed(h, exact)
            zh = fh(hf, lo_h)
        else:
            hf = forced[0][:, prev] + forced[1][:, prev]
            zh = fh(None, lo_h, (forced[0][:, prev], forced[1][:, prev]))
        prev = t
        r = sigmoid(zx[:, t, :PH] + zh[:, :PH] + brz[:PH])
        z = sigmoid(zx[:, t, PH:2 * PH] + zh[:, PH:2 * PH] + brz[PH:])
        n = np.tanh(zx[:, t, 2 * PH:] + bih[2 * PH:] + r * (zh[:, 2 * PH:] + bhh[2 * PH:]))
        h = (1.0 - z) * n + z * hf
        out[:, t] = h
    return out


def selu(x):
    a, s = 1.6732632423543772848170429916717, 1.0507009873554804934193349852946
    return np.where(x > 0, s * x, s * a * (np.exp(np.minimum(x, 0)) - 1.0))


# ------------------------------------------------------------------------------------------------ tiles
def tile_offsets(rows, cols, kt):
    r = np.asarray(rows, np.int64)[:, None]
    k = np.asarray(cols, np.int64)[None, :]
    return ((r // 128) * kt + k // 32) * 4096 + ((k % 32) // 8) * 1024 + (r % 128) * 8 + k % 8


def untile_parts(hi, lo, rows, ncols):
    o = tile_offsets(rows, np.arange(ncols), ncols // 32)
    return hi[o].view(np.float16).astype(np.float64), lo[o].view(np.float16).astype(np.float64)


def untile(hi, lo, rows, ncols):
    h, l = untile_parts(hi, lo, rows, ncols)
    return h + l


def check_padding_unwritten(hi, lo, M, ncols):
    pad = np.arange(M, -(-M // 128) * 128)
    if pad.size:
        o = tile_offsets(pad, np.arange(ncols), ncols // 32)
        assert np.all(hi[o] == 0xFFFF) and np.all(lo[o] == 0xFFFF), "a padding row of the output tiles was written"


def check_reconstruct(y, rec):
    """hi + lo of the fp32 output: 22 significant bits (2^-25 absolute where lo is an fp16 subnormal)"""
    err = np.abs(rec - y) - (2.0 ** -22 * np.abs(y) + 2.0 ** -25)
    assert err.max() <= 0, err.max()


# ------------------------------------------------------------------------------------------------ data
CHECK_ROWS = np.unique(np.concatenate([
    [0, 1, 2, 63, 64, 126, 127, 128, 129, 255, 256, 511, 640, 998, 999, 1000, 1023, 4095, 4096, 8191, 8192, 8320, 8383,
     8384, 8445, 8446, 8447],
    np.random.default_rng(99).choice(MAX_M, 48, replace=False)]))


def rows_below(M):
    return CHECK_ROWS[CHECK_ROWS < M]


@functools.lru_cache(maxsize=None)
def variant_inputs():
    from tests.test_nets_gpu import _variant_images
    x0 = _variant_images(MAX_M, 21)
    x0[::7, :, 5] = -128                                       # the int8 range ends
    x0[::11, :, 9] = 127
    rng = np.random.default_rng(22)
    x1 = rng.uniform(-1, 1, size=(MAX_M, VT, 512)).astype(np.float32)
    return x0, x1


@functools.lru_cache(maxsize=None)
def polish_inputs():
    rng = np.random.default_rng(23)
    cov = rng.integers(0, 255, size=(MAX_M, 1, 1))
    x0 = ((rng.random((MAX_M, PT, 10)) < 0.25) * cov).astype(np.uint8)
    x0[::5, :, 3] = 254
    x1 = rng.uniform(-1, 1, size=(MAX_M, PT, 256)).astype(np.float32)
    h0 = rng.uniform(-1, 1, size=(2, MAX_M, PH)).astype(np.float32)
    return x0, x1, h0


@functools.lru_cache(maxsize=None)
def variant_state():
    from oracle import nets
    return nets.make_variant_weights(3)


@functools.lru_cache(maxsize=None)
def polish_state():
    from oracle import nets
    return nets.make_polish_weights(6)


@functools.lru_cache(maxsize=None)
def variant_net():
    from pepper_b200.variant import VariantNet
    net = VariantNet(variant_state())
    net.L.pb_test_variant_lstm_layer.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                 C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return net


@functools.lru_cache(maxsize=None)
def polish_net():
    from pepper_b200.polish import PolishNet
    net = PolishNet(polish_state())
    net.L.pb_test_polish_gru_layer.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                               C.c_int, C.c_void_p, C.c_void_p]
    return net


def _f64(t):
    return t.detach().cpu().numpy().astype(np.float64)


# ------------------------------------------------------------------------------------------------ LSTM
def lstm_params(layer, d):
    st = variant_state()
    p = ("encoder" if layer == 0 else "decoder") + ".%s_l0" + ("_reverse" if d else "")
    Wih, Whh = _f64(st[p % "weight_ih"]), _f64(st[p % "weight_hh"])
    bias = (st[p % "bias_ih"] + st[p % "bias_hh"]).numpy().astype(np.float64)       # packed as one fp32 bias
    return Wih, Whh, bias


@functools.lru_cache(maxsize=None)
def lstm_model(layer, lo_x, lo_h, exact=False):
    """[rows][33][512] hidden sequence and [2][rows][256] final cell state of CHECK_ROWS"""
    x = variant_inputs()[layer][CHECK_ROWS].astype(np.float64)
    ys, cs = [], []
    for d in range(2):
        y, c = lstm_dir(x, *lstm_params(layer, d), lo_x, lo_h, d == 1, exact)
        ys.append(y)
        cs.append(c)
    return np.concatenate(ys, axis=2), np.stack(cs)


@functools.lru_cache(maxsize=None)
def lstm_torch_fp32(layer):
    import torch
    st = variant_state()
    name = "encoder" if layer == 0 else "decoder"
    m = torch.nn.LSTM(26 if layer == 0 else 512, VH, batch_first=True, bidirectional=True)
    m.load_state_dict({k[len(name) + 1:]: v for k, v in st.items() if k.startswith(name + ".")})
    with torch.no_grad():
        y, _ = m(torch.from_numpy(variant_inputs()[layer][CHECK_ROWS].astype(np.float32)))
    return y.numpy().astype(np.float64)


def run_lstm(layer, M, lo_x, lo_h, persist, poison, tiles, net=None):
    net = net or variant_net()
    x = np.ascontiguousarray(variant_inputs()[layer][:M])
    mt = -(-M // 128)
    y = np.empty((M, VT, 512), np.float32)
    c = np.empty((2, VH, M), np.float32)
    hi = np.empty(mt * VT * 16 * 4096, np.uint16) if tiles else None
    lo = np.empty(mt * VT * 16 * 4096, np.uint16) if tiles else None
    from pepper_b200 import _lib
    _lib.check(net.L.pb_test_variant_lstm_layer(net.h, layer, M, x.ctypes.data, lo_x, lo_h, persist, poison, y.ctypes.data,
                                                hi.ctypes.data if tiles else None, lo.ctypes.data if tiles else None,
                                                c.ctypes.data), "pb_test_variant_lstm_layer")
    return y, c, hi, lo


LSTM_CASES = [(0, 1, 0), (0, 1, 1), (1, 0, 0), (1, 0, 1), (1, 1, 0), (1, 1, 1)]     # (layer, lo_x, lo_h); layer 0 has no x lo


@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("layer,lo_x,lo_h", LSTM_CASES)
def test_lstm_layer(layer, lo_x, lo_h, M):
    tol = TOL_LSTM[layer]
    rows = rows_below(M)
    y, c, hi, lo = run_lstm(layer, M, lo_x, lo_h, persist=1, poison=1, tiles=True)
    assert np.isfinite(y).all() and np.isfinite(c).all()
    # 4. the per-step cross-check path: same wgmma sequence per k-tile, same epilogue arithmetic
    y0, c0, _, _ = run_lstm(layer, M, lo_x, lo_h, persist=0, poison=0, tiles=False)
    assert np.array_equal(y, y0) and np.array_equal(c, c0), np.abs(y - y0).max()
    del y0, c0
    # 5. output tiles
    check_reconstruct(y[rows].reshape(rows.size, -1).astype(np.float64), untile(hi, lo, rows, VT * 512))
    check_padding_unwritten(hi, lo, M, VT * 512)
    # 1. kernel vs model, each step on the h operands the kernel fed back (with two products the model's h_hi would
    # otherwise drift to the other side of an fp16 rounding boundary from the kernel's and both run on from there)
    fed = [p.reshape(rows.size, VT, 512) for p in untile_parts(hi, lo, rows, VT * 512)]
    del hi, lo
    x = variant_inputs()[layer][rows].astype(np.float64)

    def model(fx, fh):
        out = [lstm_dir(x, *lstm_params(layer, d), fx, fh, d == 1, False, forced=[p[:, :, d * VH:(d + 1) * VH] for p in fed])
               for d in range(2)]
        return np.concatenate([o[0] for o in out], axis=2), np.stack([o[1] for o in out])

    want, cw = model(lo_x, lo_h)
    err = np.abs(y[rows] - want).max()
    cerr = np.abs(c[:, :, rows] - cw.transpose(0, 2, 1)).max()
    print("MEASURE lstm layer %d lo_x %d lo_h %d M %d: |y - model| %.3g  |c - model| %.3g" % (layer, lo_x, lo_h, M, err, cerr))
    assert err <= tol, (err, tol)
    # 2. the model's own power to tell the flags apart, on the same rows and operands
    flips = [(lo_x, 1 - lo_h)] + ([(1 - lo_x, lo_h)] if layer == 1 else [])
    for fx, fh in flips:
        gap = np.abs(model(fx, fh)[0] - want).max()
        print("MEASURE lstm layer %d flags %d%d -> %d%d gap %.3g (%.1f tol)" % (layer, lo_x, lo_h, fx, fh, gap, gap / tol))
        assert gap >= 5 * tol, (fx, fh, gap, tol)
    # 3. against exact float64 with every product on, free running
    if lo_h and (lo_x or layer == 0):
        sel = np.searchsorted(CHECK_ROWS, rows)
        exact = lstm_model(layer, 1, 1, exact=True)[0][sel]
        e_kernel = np.abs(y[rows] - exact).max()
        e_torch = np.abs(lstm_torch_fp32(layer)[sel] - exact).max()
        print("MEASURE lstm layer %d M %d: kernel vs exact %.3g, torch fp32 vs exact %.3g" % (layer, M, e_kernel, e_torch))
        assert e_kernel <= FP32_FACTOR * e_torch, (e_kernel, e_torch)


# ------------------------------------------------------------------------------------------------ GRU
def gru_params(layer, d):
    st = polish_state()
    p = ("gru_encoder" if layer == 0 else "gru_decoder") + ".%s_l0" + ("_reverse" if d else "")
    return _f64(st[p % "weight_ih"]), _f64(st[p % "weight_hh"]), _f64(st[p % "bias_ih"]), _f64(st[p % "bias_hh"])


@functools.lru_cache(maxsize=None)
def gru_model(layer, lo_x, lo_h, exact=False):
    x0, x1, h0 = polish_inputs()
    x = (x0 if layer == 0 else x1)[CHECK_ROWS].astype(np.float64)
    h = h0[:, CHECK_ROWS].astype(np.float64)
    return np.concatenate([gru_dir(x, h[d], *gru_params(layer, d), lo_x, lo_h, d == 1, exact) for d in range(2)], axis=2)


@functools.lru_cache(maxsize=None)
def gru_torch_fp32(layer):
    import torch
    st = polish_state()
    name = "gru_encoder" if layer == 0 else "gru_decoder"
    m = torch.nn.GRU(10 if layer == 0 else 256, PH, batch_first=True, bidirectional=True)
    m.load_state_dict({k[len(name) + 1:]: v for k, v in st.items() if k.startswith(name + ".")})
    x0, x1, h0 = polish_inputs()
    with torch.no_grad():
        y, _ = m(torch.from_numpy((x0 if layer == 0 else x1)[CHECK_ROWS].astype(np.float32)),
                 torch.from_numpy(np.ascontiguousarray(h0[:, CHECK_ROWS])))
    return y.numpy().astype(np.float64)


GRU_CASES = [(0, 1, 0), (0, 1, 1), (1, 0, 0), (1, 0, 1), (1, 1, 0), (1, 1, 1)]


@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("layer,lo_x,lo_h", GRU_CASES)
def test_gru_layer(layer, lo_x, lo_h, M):
    tol = TOL_GRU[layer]
    rows = rows_below(M)
    x0, x1, h0 = polish_inputs()
    x = np.ascontiguousarray((x0 if layer == 0 else x1)[:M])
    h0m = np.ascontiguousarray(h0[:, :M])
    mt = -(-M // 128)
    hi = np.empty(mt * PT * 8 * 4096, np.uint16)
    lo = np.empty(mt * PT * 8 * 4096, np.uint16)
    net = polish_net()
    from pepper_b200 import _lib
    _lib.check(net.L.pb_test_polish_gru_layer(net.h, layer, M, x.ctypes.data, h0m.ctypes.data, lo_x, lo_h, 1, hi.ctypes.data,
                                              lo.ctypes.data), "pb_test_polish_gru_layer")
    check_padding_unwritten(hi, lo, M, PT * 256)
    allrows = np.arange(M) if M <= 1000 else np.concatenate([np.arange(256), np.arange(M - 256, M)])
    assert np.isfinite(untile(hi, lo, allrows, PT * 256)).all()
    fed = [p.reshape(rows.size, PT, 256) for p in untile_parts(hi, lo, rows, PT * 256)]
    y = fed[0] + fed[1]
    xs = (x0 if layer == 0 else x1)[rows].astype(np.float64)
    h0s = h0[:, rows].astype(np.float64)

    def model(fx, fh):
        # teacher forced like the LSTM: step t multiplies the h operands the kernel fed back from step t - 1
        return np.concatenate([gru_dir(xs, h0s[d], *gru_params(layer, d), fx, fh, d == 1, False,
                                       forced=[p[:, :, d * PH:(d + 1) * PH] for p in fed]) for d in range(2)], axis=2)

    want = model(lo_x, lo_h)
    err = np.abs(y - want).max()
    print("MEASURE gru layer %d lo_x %d lo_h %d M %d: |y - model| %.3g" % (layer, lo_x, lo_h, M, err))
    assert err <= tol, (err, tol)
    flips = [(lo_x, 1 - lo_h)] + ([(1 - lo_x, lo_h)] if layer == 1 else [])
    for fx, fh in flips:
        gap = np.abs(model(fx, fh) - want).max()
        print("MEASURE gru layer %d flags %d%d -> %d%d gap %.3g (%.1f tol)" % (layer, lo_x, lo_h, fx, fh, gap, gap / tol))
        assert gap >= 5 * tol, (fx, fh, gap, tol)
    if lo_h and (lo_x or layer == 0):
        sel = np.searchsorted(CHECK_ROWS, rows)
        exact = gru_model(layer, 1, 1, exact=True)[sel]
        e_kernel = np.abs(y - exact).max()
        e_torch = np.abs(gru_torch_fp32(layer)[sel] - exact).max()
        e_model = np.abs(gru_model(layer, 1, 1)[sel] - exact).max()
        print("MEASURE gru layer %d M %d: kernel vs exact %.3g, torch fp32 vs exact %.3g, model vs exact %.3g"
              % (layer, M, e_kernel, e_torch, e_model))
        # h is carried from step to step as its fp16 hi + lo, 22 significant bits against fp32's 24: over 100 steps of a
        # long-memory GRU that alone can exceed the float32 layer's error (the model shows it without any kernel noise)
        assert e_kernel <= FP32_FACTOR * max(e_torch, e_model), (e_kernel, e_torch, e_model)


# ------------------------------------------------------------------------------------------------ GEMM
def gemm_data(M, N, K, kind, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((M, K)).astype(np.float32)
    W = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    if kind == "wide":
        # rows of |a| up to 6e4, rows whose hi part is an fp16 subnormal (|a| < 2^-14), weights scaled by 1e-3
        A[1::3] = rng.uniform(-6e4, 6e4, size=A[1::3].shape).astype(np.float32)
        A[2::3] = rng.uniform(-6e-5, 6e-5, size=A[2::3].shape).astype(np.float32)
        W *= np.float32(1e-3)
        b *= np.float32(1e-3)
    return A, W, b


def gemm_model(A, W, b, K0, lo0, lo1, epi, exact=False):
    s = pow2_scale(W)
    A = A.astype(np.float64)
    if exact:
        acc = A @ W.astype(np.float64).T
    else:
        acc = SplitLinear(W[:, :K0], s)(A[:, :K0], lo0)
        if A.shape[1] > K0:
            acc = acc + SplitLinear(W[:, K0:], s)(A[:, K0:], lo1)
    y = acc + b.astype(np.float64)
    return selu(y) if epi == 1 else y


GEMM_CASES = [
    # M, N, K0, K1, epi, kind, max_ctas
    (1, 256, 32, 0, 0, "normal", 0),
    (127, 512, 512, 0, 1, "normal", 0),
    (129, 256, 16896, 0, 0, "normal", 7),          # linear_1's K
    (1000, 512, 256, 256, 0, "wide", 0),           # two K segments
    (1000, 512, 480, 32, 1, "normal", 1),
    (128 * 300, 512, 32, 0, 1, "normal", 1),       # 600 tiles on one CTA
    (128 * 300, 256, 32, 0, 0, "wide", 7),
    (128 * 300, 512, 32, 32, 0, "normal", 0),
    (257, 512, 16896, 0, 0, "wide", 1),
]


@pytest.mark.parametrize("M,N,K0,K1,epi,kind,max_ctas", GEMM_CASES)
@pytest.mark.parametrize("lo0,lo1", [(1, 1), (0, 1), (1, 0)])
def test_tc_gemm_layer(M, N, K0, K1, epi, kind, max_ctas, lo0, lo1):
    if K1 == 0 and lo1 == 0:
        pytest.skip("one segment: lo1 has no operand")
    from pepper_b200 import _lib
    L = _lib.lib()
    L.pb_test_tc_gemm_ex.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                     C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    K = K0 + K1
    A, W, b = gemm_data(M, N, K, kind, M + N + K + epi)
    A0, A1 = np.ascontiguousarray(A[:, :K0]), np.ascontiguousarray(A[:, K0:])
    mt = -(-M // 128)
    out = np.empty((M, N), np.float32)
    hi = np.empty(mt * N * 128, np.uint16)
    lo = np.empty(mt * N * 128, np.uint16)
    _lib.check(L.pb_test_tc_gemm_ex(M, N, epi, K0, A0.ctypes.data, lo0, K1, A1.ctypes.data if K1 else None, lo1, W.ctypes.data,
                                    b.ctypes.data, max_ctas, 1, out.ctypes.data, hi.ctypes.data, lo.ctypes.data), "gemm_ex")
    assert np.isfinite(out).all()
    check_padding_unwritten(hi, lo, M, N)
    rows = np.unique(np.concatenate([np.arange(min(M, 64)), np.arange(max(0, M - 64), M),
                                     np.random.default_rng(5).choice(M, min(M, 256), replace=False)]))
    check_reconstruct(out[rows].astype(np.float64), untile(hi, lo, rows, N))
    As = A[rows]
    want = gemm_model(As, W, b, K0, lo0, lo1, epi)
    # per element: the fp32 accumulation bound scales with sum_k |a_k w_k| (all products of the split)
    mag = np.abs(As.astype(np.float64)) @ np.abs(W.astype(np.float64)).T + np.abs(b)
    bound = tol_gemm(K) * mag + (2.0 ** -20 if epi == 1 else 0)
    ratio = (np.abs(out[rows] - want) / bound).max()
    print("MEASURE gemm %s: kernel vs model %.3g of tol" % ((M, N, K0, K1, epi, kind, max_ctas, lo0, lo1), ratio))
    assert ratio <= 1.0, ratio
    for f0, f1 in ([(1 - lo0, lo1)] + ([(lo0, 1 - lo1)] if K1 else [])):
        gap = (np.abs(gemm_model(As, W, b, K0, f0, f1, epi) - want) / bound).max()
        print("MEASURE gemm flags %d%d -> %d%d gap %.3g tol" % (lo0, lo1, f0, f1, gap))
        if K <= 4096:
            # at linear_1's K (16,896) the accumulation noise measured on H100 (62 x 2^-24 sum |a w|) is within 3x of
            # a dropped product's effect (165 x 2^-24 sum |a w| on this data): no max-norm bound separates them there
            assert gap >= 5, gap
    if lo0 and lo1 and epi == 0 and K <= 4096:
        # at K = 16,896 the wgmma accumulator's error (3.7e-6 of sum |a w| measured) is ~190x that of a blocked float32
        # CPU GEMM (1.9e-8): linear_1 is not fp32-equivalent, and assertion 1 (against the split model) is what holds there.
        # Below: rows whose activations are in the fp16 normal range (a row of |a| < 2^-14 keeps only
        # the bits of a above 2^-25: the split is exact to 2^-25 absolute, not 2^-22 relative, there)
        normal = np.abs(As).max(axis=1) >= 2.0 ** -14 * 4
        ex = gemm_model(As, W, b, K0, 1, 1, epi, exact=True)
        import torch
        t = torch.from_numpy(As) @ torch.from_numpy(W).T + torch.from_numpy(b)
        t = (torch.selu(t) if epi == 1 else t).numpy().astype(np.float64)
        e_k = (np.abs(out[rows] - ex) / mag)[normal].max()
        e_t = (np.abs(t - ex) / mag)[normal].max()
        print("MEASURE gemm %s: kernel vs exact %.3g, torch %.3g (relative to sum |a w|)" % ((M, N, K0, K1, epi, kind), e_k, e_t))
        assert e_k <= FP32_FACTOR * e_t, (e_k, e_t)
