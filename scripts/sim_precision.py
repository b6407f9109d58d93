"""CPU emulation of the tensor-core operand splits considered for the network kernels (round 2, VERDICT item 2).

Every GEMM of the two networks is re-evaluated with operands rounded the way a given scheme would feed them to
wgmma.mma_async (fp32 accumulate; products of 16-bit operands are exact in fp32), and the hidden states / probabilities are
compared with the fp32 CPU oracle.  Used to choose the scheme before spending GPU time; the GPU tests are the gate.

    python scripts/sim_precision.py variant|polish [n] [scheme,scheme,...] [--weights uniform|t3|outlier30|outlier100]

--weights (variant only) replaces the decoder LSTM's weights, at each matrix's std, with Student-t (3 dof) samples or puts one
weight per gate row at +-30 / +-100 std (tests/test_weight_distributions_gpu.py builds the same states for the GPU).

A variant scheme name ending in "+i8dec" runs the decoder LSTM on int8 slices (mode 2, k_lstm_layer_q8: 16-bit fixed-point
activations at the fixed scale 32,512, one per-column weight scale over [W_ih | W_hh], a0 x w0 dropped) and every other GEMM
with the scheme before it, e.g. "f16x3+i8dec".  A further "+i8lin1" runs linear_1 on int8 slices as well (mode 2, k_gemm_q8: the
decoder's h quantized to 1 / 32512 steps, one weight scale per output row, a0 x w0 dropped), e.g. "f16x3+i8dec+i8lin1".
--lin1 replaces linear_1's weights the way --weights replaces the decoder's (one weight per output row at +-3 .. +-100 std for
the outliers, so that the guard's threshold can be placed between passing and failing estimates; "edge": two
all-zero rows and two rows scaled by 1e-6), and each line then also prints the guard's estimate for linear_1 (head_err).
"""
import argparse
import sys
import os
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import nets  # noqa: E402  (a development script, not product code)

torch.set_num_threads(8)


def rn16(x, dt):
    return x.to(dt).to(torch.float64)


def split(x, dt):
    hi = rn16(x, dt)
    lo = rn16(x - hi, dt)
    return hi, lo


def q16(x, scale):
    """16-bit fixed point x * scale = 256 x1 + x0 as two int8 slices, x1 = floor((q + 128) / 256), x0 in [-128, 127]"""
    xi = torch.round(x * scale)
    x1 = torch.floor((xi + 128) / 256)
    return x1, xi - 256 * x1


def i8_joint(a, W, S):
    """a [B, K] in [-1, 1] times W [N, K] on int8 slices with exact accumulation and the a0 x w0 product dropped"""
    key = ("i8", id(W))
    if key not in S.cache:
        W64 = W.to(torch.float64)
        sw = 32512.0 / W64.abs().amax(1, keepdim=True).clamp_min(1e-30)
        S.cache[key] = (*q16(W64, sw), sw)
    w1, w0, sw = S.cache[key]
    a1, a0 = q16(a.clamp(-1, 1), 32512.0)
    acc = a1 @ w1.T * 65536 + (a1 @ w0.T + a0 @ w1.T) * 256
    return acc / 32512.0 / sw.T


class Scheme:
    """mm(a, W) with a [B,K] float64 activations, W [N,K] weights (fp32 values)."""

    def __init__(self, name):
        self.name = name
        self.cache = {}
        self.i8_dec = False
        self.i8_lin1 = False

    def wsplit(self, W, dt, scale=True):
        key = (id(W), dt)
        if key not in self.cache:
            W64 = W.to(torch.float64)
            s = 1.0
            if scale and dt == torch.float16:
                # per-tensor power-of-two scale so that max|w| lands in [2^-1, 1): keeps w_lo out of fp16 subnormals
                m = W64.abs().max().item()
                s = 2.0 ** (-np.ceil(np.log2(m))) if m > 0 else 1.0
            hi, lo = split(W64 * s, dt)
            self.cache[key] = (hi, lo, s)
        return self.cache[key]

    def mm(self, a, W, exact_a=False, slot=0):
        n = self.name
        if "/" in n:
            n = n.split("/")[slot]
        a = a.to(torch.float64)
        if n == "fp32":
            return (a.float() @ W.float().T).double()
        if n == "bf16x3":
            wh, wl, s = self.wsplit(W, torch.bfloat16)
            ah, al = split(a, torch.bfloat16)
            return ah @ wh.T + ah @ wl.T + al @ wh.T
        if n == "f16x3":
            wh, wl, s = self.wsplit(W, torch.float16)
            ah, al = split(a, torch.float16)
            return (ah @ wh.T + ah @ wl.T + al @ wh.T) / s
        if n == "f16x2":          # a_hi * (w_hi + w_lo)
            wh, wl, s = self.wsplit(W, torch.float16)
            ah = rn16(a, torch.float16)
            return (ah @ wh.T + ah @ wl.T) / s
        if n == "f16x2a":         # (a_hi + a_lo) * w_hi
            wh, wl, s = self.wsplit(W, torch.float16)
            ah, al = split(a, torch.float16)
            return (ah @ wh.T + al @ wh.T) / s
        if n == "f16x1":
            wh, wl, s = self.wsplit(W, torch.float16)
            ah = rn16(a, torch.float16)
            return (ah @ wh.T) / s
        if n == "bf16x2":
            wh, wl, s = self.wsplit(W, torch.bfloat16)
            ah = rn16(a, torch.bfloat16)
            return ah @ wh.T + ah @ wl.T
        raise ValueError(n)


def lstm_dir(S, x, Wih, Whh, b, reverse, slots=(0, 0)):
    B, T, _ = x.shape
    H = Whh.shape[1]
    h = torch.zeros(B, H, dtype=torch.float64)
    c = torch.zeros(B, H, dtype=torch.float64)
    out = torch.zeros(B, T, H, dtype=torch.float64)
    ts = range(T - 1, -1, -1) if reverse else range(T)
    for t in ts:
        if S.i8_dec and slots[0] == 1:
            key = ("cat", id(Wih), id(Whh))
            if key not in S.cache:
                S.cache[key] = torch.cat([Wih, Whh], 1)
            g = i8_joint(torch.cat([x[:, t].double(), h], 1), S.cache[key], S) + b
        else:
            g = S.mm(x[:, t], Wih, slot=slots[0]) + S.mm(h, Whh, slot=slots[1]) + b
        g = g.float()       # epilogue works in fp32
        i, f, gg, o = g.chunk(4, dim=1)
        c = (torch.sigmoid(f) * c.float() + torch.sigmoid(i) * torch.tanh(gg))
        h = (torch.sigmoid(o) * torch.tanh(c)).double()
        c = c.double()
        out[:, t] = h
    return out


def variant_forward(S, st, x):
    x = x.double()
    for layer in ("encoder", "decoder"):
        outs = []
        for suf, rev in (("", False), ("_reverse", True)):
            b = (st[f"{layer}.bias_ih_l0{suf}"] + st[f"{layer}.bias_hh_l0{suf}"]).double()
            outs.append(lstm_dir(S, x, st[f"{layer}.weight_ih_l0{suf}"], st[f"{layer}.weight_hh_l0{suf}"], b, rev,
                                 slots=(0, 0) if layer == "encoder" else (1, 2)))
        x = torch.cat(outs, dim=2)
    hid = x
    y = x.flatten(1, 2)
    for i in range(1, 6):
        W = st[f"linear_{i}.weight"]
        z = i8_joint(y, W, S) if i == 1 and S.i8_lin1 else S.mm(y, W, slot=3 if i == 1 else 4)
        y = torch.selu((z + st[f"linear_{i}.bias"].double()).float()).double()
    logits = y.float() @ st["output_layer_type.weight"].float().T + st["output_layer_type.bias"].float()
    return torch.softmax(logits, dim=1), hid


def gru_dir(S, x, h0, Wih, Whh, bih, bhh, reverse):
    B, T, _ = x.shape
    H = Whh.shape[1]
    h = h0.double()
    out = torch.zeros(B, T, H, dtype=torch.float64)
    ts = range(T - 1, -1, -1) if reverse else range(T)
    for t in ts:
        gi = (S.mm(x[:, t], Wih) + bih).float()
        gh = (S.mm(h, Whh) + bhh).float()
        ir, iz, in_ = gi.chunk(3, 1)
        hr, hz, hn = gh.chunk(3, 1)
        r = torch.sigmoid(ir + hr)
        z = torch.sigmoid(iz + hz)
        n = torch.tanh(in_ + r * hn)
        h = ((1 - z) * n + z * h.float()).double()
        out[:, t] = h
    return out, h


def polish_forward(S, st, images):
    B = images.shape[0]
    hidden = torch.zeros(B, 2, 128, dtype=torch.float64)
    acc = torch.zeros(B, 1000, 5)
    hids = []
    for i in range(0, 1000, 50):
        if i + 100 > 1000:
            break
        x = images[:, i:i + 100].double()
        hs = []
        outs = []
        for d, (suf, rev) in enumerate((("", False), ("_reverse", True))):
            o, h = gru_dir(S, x, hidden[:, d], st[f"gru_encoder.weight_ih_l0{suf}"], st[f"gru_encoder.weight_hh_l0{suf}"],
                           st[f"gru_encoder.bias_ih_l0{suf}"].double(), st[f"gru_encoder.bias_hh_l0{suf}"].double(), rev)
            outs.append(o); hs.append(h)
        x1 = torch.cat(outs, 2)
        outs2, hs2 = [], []
        for d, (suf, rev) in enumerate((("", False), ("_reverse", True))):
            o, h = gru_dir(S, x1, hs[d], st[f"gru_decoder.weight_ih_l0{suf}"], st[f"gru_decoder.weight_hh_l0{suf}"],
                           st[f"gru_decoder.bias_ih_l0{suf}"].double(), st[f"gru_decoder.bias_hh_l0{suf}"].double(), rev)
            outs2.append(o); hs2.append(h)
        y = torch.cat(outs2, 2).float()
        hidden = torch.stack(hs2, 1)
        hids.append(hidden.float().numpy())
        out = y @ st["dense1.weight"].float().T + st["dense1.bias"].float()
        acc[:, i:i + 100] += torch.softmax(out, 2)
    return acc.numpy(), np.stack(hids)


def reweight_decoder(st, dist, seed):
    """the decoder's W_ih / W_hh replaced as --weights says (uniform: unchanged)"""
    if dist == "uniform":
        return st
    st = dict(st)
    rng = np.random.default_rng([seed, 1])
    for suf in ("", "_reverse"):
        for i, part in enumerate(("ih", "hh")):
            name = f"decoder.weight_{part}_l0{suf}"
            W = st[name].numpy().astype(np.float64)
            if dist == "t3":
                X = rng.standard_t(3, size=W.shape)
                W = X * (W.std() / X.std())
            else:                 # outlier30 / outlier100: W_ih holds the even rows' outliers, W_hh the odd rows'
                k = float(dist[len("outlier"):])
                rows = np.arange(i, W.shape[0], 2)
                W = W.copy()
                W[rows, rng.integers(0, W.shape[1], rows.size)] = k * W.std() * rng.choice([-1.0, 1.0], rows.size)
            st[name] = torch.from_numpy(W.astype(np.float32))
    return st


def reweight_lin1(st, dist, seed):
    """linear_1's weight replaced as --lin1 says (uniform: unchanged)"""
    if dist == "uniform":
        return st
    st = dict(st)
    rng = np.random.default_rng([seed, 2])
    W = st["linear_1.weight"].numpy().astype(np.float64)
    if dist == "t3":
        X = rng.standard_t(3, size=W.shape)
        W = X * (W.std() / X.std())
    elif dist == "edge":
        W = W.copy()
        W[[5, 300]] = 0
        W[[7, 411]] *= 1e-6
    else:
        k = float(dist[len("outlier"):])
        W = W.copy()
        W[np.arange(W.shape[0]), rng.integers(0, W.shape[1], W.shape[0])] = k * W.std() * rng.choice([-1.0, 1.0], W.shape[0])
    st["linear_1.weight"] = torch.from_numpy(W.astype(np.float32))
    return st


def head_err(W):
    """the guard's weight-only estimate for linear_1 (nets_tc.cu pack_q8 with the activation rounding term), largest row"""
    W = W.to(torch.float64)
    sw = 32512.0 / torch.where(W.abs().amax(1, keepdim=True) > 0, W.abs().amax(1, keepdim=True), torch.tensor(32512.0, dtype=torch.float64))
    w1, w0 = q16(W, sw)
    e = ((256 * w1 + w0) / sw - W).pow(2).sum(1) + 128.0 ** 2 / 3 / 32512.0 ** 2 * (w0 / sw).pow(2).sum(1)
    e = e + W.pow(2).sum(1) / (12 * 32512.0 ** 2)
    return e.sqrt().max().item()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("which", choices=["variant", "polish"])
    ap.add_argument("n", type=int, nargs="?", default=256)
    ap.add_argument("schemes", nargs="?", default="bf16x3,f16x3,f16x2,f16x2a,f16x1,bf16x2")
    ap.add_argument("--weights", choices=["uniform", "t3", "outlier30", "outlier100"], default="uniform")
    ap.add_argument("--lin1", choices=["uniform", "t3", "outlier3", "outlier4", "outlier6", "outlier9", "outlier30", "outlier100", "edge"],
                    default="uniform")
    args = ap.parse_args()
    which, n, schemes, dist = args.which, args.n, args.schemes.split(","), args.weights
    if which == "variant":
        for seed in (1, 2):
            st = reweight_lin1(reweight_decoder(nets.make_variant_weights(seed), dist, seed), args.lin1, seed)
            he = head_err(st["linear_1.weight"])
            rng = np.random.default_rng(seed)
            x = rng.integers(-40, 41, size=(n, 33, 26)).astype(np.int8)
            x[:, :, 0] = rng.integers(1, 6, size=(n, 33))
            x[rng.random((n, 33, 26)) < 0.5] = 0
            want, whid = nets.variant_predict(st, x, threads=8, return_hidden=True)
            for name in schemes:
                S = Scheme(name.split("+")[0])
                S.i8_dec = "+i8dec" in name
                S.i8_lin1 = "+i8lin1" in name
                p, hid = variant_forward(S, st, torch.from_numpy(x.astype(np.float32)))
                eh = np.abs(hid.numpy() - whid).max()
                ep = np.abs(p.numpy() - want).max()
                srt = np.sort(want, 1)
                clear = (srt[:, -1] - srt[:, -2]) > 1e-4
                am = (p.numpy().argmax(1)[clear] != want.argmax(1)[clear]).sum()
                print(f"variant seed {seed} {dist} lin1 {args.lin1} {name:8s} max|dh| {eh:.2e}  max|dp| {ep:.2e}  "
                      f"argmax mismatches (clear) {am}  head_err {he:.2e}", flush=True)
    else:
        for seed in (4, 6):
            st = nets.make_polish_weights(seed)
            rng = np.random.default_rng(seed)
            x = np.zeros((n, 1000, 10), np.uint8)
            cov = rng.integers(0, 255, size=(n, 1000, 1))
            x[:] = (rng.random((n, 1000, 10)) < 0.25) * cov
            wb, wp, wh, wa = nets.polish_predict(st, x, threads=8)
            for name in schemes:
                S = Scheme(name)
                acc, hid = polish_forward(S, st, torch.from_numpy(x.astype(np.float32)))
                eh = np.abs(hid - wh).max()
                ea = np.abs(acc - wa).max()
                srt = np.sort(wa, 2)
                clear = (srt[:, :, -1] - srt[:, :, -2]) > 1e-4
                am = (acc.argmax(2)[clear] != wa.argmax(2)[clear]).sum()
                print(f"polish seed {seed} {name:8s} max|dh| {eh:.2e}  max|dacc| {ea:.2e}  argmax mismatches (clear) {am}", flush=True)


if __name__ == "__main__":
    main()
