"""Where the time of the LSTM layer kernels goes: per-phase %clock64 stamps of a PB_LSTM_TRACE build (tc_gemm.cuh), for
both variant LSTM layers of one VariantNet.predict chunk at each size (the encoder's k_lstm_layer_enc, or k_lstm_layer when
its h-part runs all three products, and the decoder's k_lstm_layer_q8, or k_lstm_layer in mode 1).

    python scripts/trace_lstm_layer.py [--sizes 8448 1408] [--lib TRACED.so] [--build-dir DIR] [--out FILE] [--raw FILE.npz]

Without --lib the traced library is built with `make EXTRA=-DPB_LSTM_TRACE` into --build-dir (default: a new temporary
directory), never into the tree.  CTAs 0, n/2 and n-1 are sampled; every phase is the median (and mean) over those CTAs,
their 8 consumer warps, steps 1..32 and the gate tiles, 4 in k_lstm_layer and 8 in k_lstm_layer_q8, or the 8 half gate tiles
of k_lstm_layer_enc (producer phases: over CTAs and steps; k_lstm_layer_q8's epilogue warpgroup: over its 4 warps).  The
hand-off rows of k_lstm_layer_q8 compare stamps of different warps of one SM (one %clock64).  Times are SM cycles; the
kernel's own clock (cycles over %globaltimer) is printed beside the card name, power limit and nvidia-smi's SM clock.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T = 33                  # PB_VARIANT_WINDOW: steps per layer
CTAS = 3                # LSTM_TRACE_CTAS
CTA_WORDS = 403 * T + 4  # lstm_trace_cta_words(T)


def build_traced(build_dir: str) -> str:
    os.makedirs(build_dir, exist_ok=True)
    out = os.path.join(build_dir, "libpepper_b200_trace.so")
    subprocess.run(["make", "-j8", "-C", os.path.join(ROOT, "pepper_b200", "csrc"), "BUILD=" + os.path.join(build_dir, "obj"),
                    "OUT=" + out, "EXTRA=-DPB_LSTM_TRACE"], check=True)
    return out


def gpu_info() -> dict:
    smi = shutil.which("nvidia-smi")
    if smi is None:
        return {}
    r = subprocess.run([smi, "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    f = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")] if r.returncode == 0 and r.stdout.strip() else []
    return dict(zip(("name", "power_limit", "sm_clock", "sm_clock_max"), f))


def phases(words: np.ndarray) -> dict:
    """One layer's stamps -> {phase: (median cycles, mean cycles, samples)} over the sampled CTAs that ran."""
    acc = {}

    def add(name, v):
        acc.setdefault(name, []).extend(np.asarray(v, dtype=np.float64).ravel().tolist())

    mhz = []
    for s in range(CTAS):
        w = words[s * CTA_WORDS:(s + 1) * CTA_WORDS].astype(np.int64)
        meta = w[275 * T:275 * T + 4]
        if meta[1] == 0:
            continue
        if meta[2] > meta[0]:
            mhz.append((meta[3] - meta[1]) / (meta[2] - meta[0]) * 1e3)
        tile = w[:256 * T].reshape(8, T, 8, 4)            # [warp][t][nt][start, first full, mma done, epilogue end]
        if not tile[:, :, 4:].any():                       # k_lstm_layer: 4 gate tiles per step
            tile = tile[:, :, :4]
        step = w[256 * T:272 * T].reshape(8, T, 2)         # [warp][t][fence returned, bar_h arrived]
        prod = w[272 * T:275 * T].reshape(T, 3)            # [t][bar_h wait start, wait end, first h copy issued]
        epi = w[275 * T + 4:403 * T + 4].reshape(4, T, 8, 4)  # [epilogue warp][t][nt][staged wait, cells done, h published, -]
        tl = tile[:, 1:]
        if epi.any():
            # k_lstm_layer_q8: consumers [start, first full, wg_wait<0>, staging stored]; the epilogue warpgroup runs the
            # cells of tile nt from the staging buffer under the k-loop of tile nt + 1.  "staged" is released when the last
            # consumer warp has stored (bar.sync defers its blocking, so the epilogue warps have no stamp of the release).
            el = epi[:, 1:]
            stored = tile[:, 1:, :, 3].max(axis=0)           # [t][nt] the last consumer warp's staging stored
            add("tile: start -> first bar_full", tl[..., 1] - tl[..., 0])
            add("tile: first bar_full -> wg_wait<0> (k-loop)", tl[..., 2] - tl[..., 1])
            add("tile: wg_wait<0> -> staging stored (hand-off)", tl[..., 3] - tl[..., 2])
            add("tile: staging stored -> next tile start", tl[:, :, 1:, 0] - tl[:, :, :-1, 3])
            add("tile period (start -> next start, same step)", tl[:, :, 1:, 0] - tl[:, :, :-1, 0])
            add("step period (tile 0 start -> next tile 0 start)", tile[:, 2:, 0, 0] - tile[:, 1:-1, 0, 0])
            add("epilogue: last consumer stored -> cells done", el[..., 1] - stored[None])
            add("epilogue: cells done -> next tile's staging stored (slack)", stored[None, :, 1:] - el[:, :, :-1, 1])
            add("step: tile 7 staged -> h published", el[:, :, 7, 2] - stored[None, :, 7])
            add("step: h published (last warp) -> producer bar_h passed", prod[2:, 1] - epi[:, 1:-1, 7, 2].max(axis=0))
            add("step: h published (last warp) -> next step's tile 0 k-loop end",
                tile[:, 2:, 0, 2].max(axis=0) - epi[:, 1:-1, 7, 2].max(axis=0))
            add("producer: bar_h wait", prod[1:, 1] - prod[1:, 0])
            add("producer: bar_h passed -> first h copy issued", prod[1:, 2] - prod[1:, 1])
            add("kernel (globaltimer, ns)", [meta[2] - meta[0]])
            continue
        if not prod.any():
            # k_lstm_layer_enc (no bar_h): per half tile [start, first full, last k-tile issued, end], the previous half's
            # epilogue running between the k-tiles; per step [half 7's epilogue done, h published (named barrier passed)]
            add("half: start -> first bar_full", tl[..., 1] - tl[..., 0])
            add("half: first bar_full -> last k-tile issued (previous half's epilogue under it)", tl[..., 2] - tl[..., 1])
            add("half, even: last k-tile issued -> end", tl[:, :, 0::2, 3] - tl[:, :, 0::2, 2])
            add("half, odd: last k-tile issued -> end (wg_wait<0>)", tl[:, :, 1::2, 3] - tl[:, :, 1::2, 2])
            add("half period (start -> next start, same step)", tl[:, :, 1:, 0] - tl[:, :, :-1, 0])
            add("step: half 7 epilogue done -> h published", step[:, 1:, 1] - step[:, 1:, 0])
            add("step period (half 0 start -> next half 0 start)", tile[:, 2:, 0, 0] - tile[:, 1:-1, 0, 0])
            add("kernel (globaltimer, ns)", [meta[2] - meta[0]])
            continue
        add("tile: start -> first bar_full", tl[..., 1] - tl[..., 0])
        add("tile: first bar_full -> wg_wait<0>", tl[..., 2] - tl[..., 1])
        add("tile: wg_wait<0> -> epilogue end", tl[..., 3] - tl[..., 2])
        add("tile: epilogue end -> next tile start", tl[:, :, 1:, 0] - tl[:, :, :-1, 3])
        add("tile period (start -> next start, same step)", tl[:, :, 1:, 0] - tl[:, :, :-1, 0])
        add("step: last epilogue end -> __threadfence returned", step[:, 1:, 0] - tile[:, 1:, -1, 3])
        add("step: __threadfence -> bar_h arrived", step[:, 1:, 1] - step[:, 1:, 0])
        add("step: bar_h arrived -> next step's first tile start", tile[:, 2:, 0, 0] - step[:, 1:-1, 1])
        add("step period (tile 0 start -> next tile 0 start)", tile[:, 2:, 0, 0] - tile[:, 1:-1, 0, 0])
        add("producer: bar_h wait", prod[1:, 1] - prod[1:, 0])
        add("producer: bar_h passed -> first h copy issued", prod[1:, 2] - prod[1:, 1])
        add("kernel (globaltimer, ns)", [meta[2] - meta[0]])
    out = {k: {"median": float(np.median(v)), "mean": float(np.mean(v)), "n": len(v)} for k, v in acc.items()}
    out["kernel_sm_mhz"] = float(np.median(mhz)) if mhz else None
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--sizes", type=int, nargs="+", default=[8448, 1408], help="candidates per predict chunk (<= 8448)")
    ap.add_argument("--lib", default=None, help="an existing PB_LSTM_TRACE build of libpepper_b200.so")
    ap.add_argument("--build-dir", default=None, help="where to build the traced library (default: a temporary directory)")
    ap.add_argument("--out", default=None, help="write the result as JSON here")
    ap.add_argument("--raw", default=None, help="write every size's stamps (both layers, uint64) as arrays of one .npz here")
    args = ap.parse_args()
    if any(n < 1 or n > 8448 for n in args.sizes):
        ap.error("--sizes must lie in 1..8448 (one network chunk)")

    if args.lib:
        lib_path = os.path.abspath(args.lib)
        if not os.path.exists(lib_path):
            sys.exit(f"--lib {lib_path} does not exist")
    else:
        lib_path = build_traced(args.build_dir or tempfile.mkdtemp(prefix="pb_lstm_trace_"))
    os.environ["PB_LIB_PATH"] = lib_path
    sys.path.insert(0, ROOT)
    from pepper_b200 import _lib

    L = _lib.lib()
    if not hasattr(L, "pb_lstm_trace_copy"):
        sys.exit(f"{lib_path} was not built with -DPB_LSTM_TRACE (no pb_lstm_trace_copy)")
    try:
        _lib.require_gpu()
    except _lib.PepperB200Error as e:
        sys.exit(f"trace_lstm_layer: {e}")

    import ctypes as C
    from oracle import nets
    from pepper_b200.variant import VariantNet

    net = VariantNet(nets.make_variant_weights(0), 0)
    rng = np.random.default_rng(0)
    res = {"lib": lib_path, "gpu_before": gpu_info(), "sizes": []}
    words = np.zeros(2 * CTAS * CTA_WORDS, dtype=np.uint64)
    raw = {}
    for n in args.sizes:
        x = rng.integers(-30, 31, size=(n, T, 26), dtype=np.int8)
        for _ in range(3):                                # warm-up; the trace holds the last call
            net.predict(x)
        _lib.check(L.pb_lstm_trace_copy(words.ctypes.data_as(C.c_void_p), C.c_int64(words.size)), "pb_lstm_trace_copy")
        raw[f"n{n}"] = words.copy()
        res["sizes"].append({"candidates": n, "ctas": 2 * ((n + 127) // 128),
                             "encoder": phases(words[:CTAS * CTA_WORDS]), "decoder": phases(words[CTAS * CTA_WORDS:])})
    res["gpu_after"] = gpu_info()
    net.close()

    g = res["gpu_before"]
    print(f"{g.get('name', '?')}, power limit {g.get('power_limit', '?')}, SM clock {g.get('sm_clock', '?')} "
          f"(after: {res['gpu_after'].get('sm_clock', '?')}), lib {lib_path}")
    for sz in res["sizes"]:
        print(f"\n{sz['candidates']} candidates, {sz['ctas']} CTAs; kernel SM clock: encoder "
              f"{sz['encoder']['kernel_sm_mhz']:.0f} MHz, decoder {sz['decoder']['kernel_sm_mhz']:.0f} MHz")
        print(f"{'phase (SM cycles; median / mean)':<56}{'encoder':>20}{'decoder':>20}")
        for k in dict.fromkeys(list(sz["encoder"]) + list(sz["decoder"])):
            if k == "kernel_sm_mhz":
                continue
            cols = "".join(f"{L[k]['median']:>11.0f} /{L[k]['mean']:>7.0f}" if k in L else f"{'-':>20}"
                           for L in (sz["encoder"], sz["decoder"]))
            print(f"{k:<56}{cols}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    if args.raw:
        np.savez(args.raw, **raw)


if __name__ == "__main__":
    main()
