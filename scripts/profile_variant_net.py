"""Per-kernel device time of VariantNet.predict (torch.profiler) at one or more chunk sizes, with the SM clock sampled by
nvidia-smi during the profiled calls.

Each k_lstm_layer CTA does the same work whatever the grid size, so a layer that takes longer at 8,448 candidates (132 CTAs)
than at 1,408 (22 CTAs) at the same clock is held back by something the CTAs share, such as L2 bandwidth for the weight tiles
every CTA streams.

    python scripts/profile_variant_net.py [--sizes 8448 1408] [--reps 5] [--mode 2] [--out FILE]     (PB_LIB_PATH selects the build)

In mode 2 the decoder layer is k_lstm_layer_q8 and linear_1 is k_gemm_q8 (int8 slices); --mode 1 profiles the fp16 hi/lo
decoder and linear_1 of the same build.  The first head launch of each predict is reported as linear_1, the other four as
head_gemm (linear_2 .. linear_5).
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def label(name: str) -> str:
    for key, short in (("k_lstm_layer", "lstm_layer"), ("k_tc_gemm_p", "head_gemm"), ("k_gemm_q8", "head_gemm"), ("k_tc_pack_images", "pack_images"),
                       ("k_variant_out", "out_softmax")):
        if key in name:
            return short
    return name[:40]


def profile_size(net, n: int, reps: int, rng) -> dict:
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    x = rng.integers(-30, 31, size=(n, 33, 26), dtype=np.int8)
    for _ in range(2):
        net.predict(x)
    torch.cuda.synchronize()
    smi = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-lms", "100"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                net.predict(x)
            torch.cuda.synchronize()
    finally:
        smi.terminate()
        rows = smi.communicate(timeout=5)[0].split()
    kernels = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA and "memcpy" not in e.name.lower()
                      and "memset" not in e.name.lower()), key=lambda e: e.time_range.start)
    per = {}
    n_lstm = n_head = 0
    for e in kernels:
        k = label(e.name)
        if k == "lstm_layer":                       # two launches per predict: encoder, then decoder
            k = ("encoder_" if n_lstm % 2 == 0 else "decoder_") + k
            n_lstm += 1
        elif k == "head_gemm":                      # five launches per chunk: linear_1, then linear_2 .. linear_5
            if n_head % 5 == 0:
                k = "linear_1"
            n_head += 1
        per.setdefault(k, []).append(e.time_range.elapsed_us() / 1e3)
    ms = {k: {"ms_per_predict": sum(v) / reps, "launches_per_predict": len(v) / reps} for k, v in per.items()}
    sm = [float(r) for r in rows if r.replace(".", "", 1).isdigit()]
    return {"candidates": n, "ctas_per_lstm_launch": 2 * ((n + 127) // 128), "kernels": ms,
            "sm_mhz_median": float(np.median(sm)) if sm else None, "sm_mhz_samples": len(sm)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[8448, 1408])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--mode", type=int, default=None, help="VariantNet.set_mode before profiling (default: the library's default)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from oracle import nets
    from pepper_b200.variant import VariantNet

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    net = VariantNet(nets.make_variant_weights(0), 0)
    if args.mode is not None:
        net.set_mode(args.mode)
    rng = np.random.default_rng(0)
    res = {"gpu": gpu, "mode": args.mode, "lib": os.environ.get("PB_LIB_PATH", "in-tree"), "sizes": [profile_size(net, n, args.reps, rng) for n in args.sizes]}
    net.close()
    txt = json.dumps(res, indent=1)
    print(txt)
    if args.out:
        with open(args.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
