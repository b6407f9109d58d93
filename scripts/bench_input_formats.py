"""The whole-genome variant call on the two input encodings: (BAM + BAI, plain FASTA) and (BAM + CSI, bgzip FASTA + GZI), the same
records and reference written both ways (the 64 Mb, 4-contig, 20x ONT workload of scripts/bench_call_genome.py).

call_genome runs on each encoding in turn, alternated `--rounds` times in one process, after one warm-up call each.  Reported per
encoding: wall time of each call; call_genome's own BAM-fetch (helper thread) and FASTA-fetch host time per group; then, outside
the timed calls, each group's BAM span through fetch_device (device time and host wall) with its record-start anchors and the
longest walk from one anchor, and each group's reference through the FASTA reader.  The card's name and power limit are read in
the same call.  The five VCFs of both encodings must decompress to the same text and the totals must agree.  Prints one JSON line.
    python scripts/bench_input_formats.py [--total-mb 64] [--rounds 3]"""
import argparse
import gzip
import json
import os
import subprocess
import sys
import tempfile
import time

from concurrent.futures import ProcessPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def log(msg: str) -> None:
    print("[bench_input_formats] " + msg, file=sys.stderr, flush=True)


def group_fetch_stats(bam: str, fa: str, jobs, batch: int) -> dict:
    """Every group's BAM span through fetch_device and its reference span through the FASTA reader, one at a time."""
    import numpy as np
    from pepper_b200.bamio import BamReader, FastaReader
    from pepper_b200.frontend import _FromFiles, variant_intervals, variant_rows
    r, f = BamReader(bam), FastaReader(fa)
    anchors, walks, bam_ms, fa_ms = [], [], [], []
    for c, n in jobs:
        iv = variant_intervals(0, n - 1)
        for i in range(0, len(iv), batch):
            g = iv[i:i + batch]
            t0 = time.perf_counter()
            r.fetch_device(c, *_FromFiles._group_span(g))
            bam_ms.append((time.perf_counter() - t0) * 1e3)
            a, w = r.fetch_device_anchors()
            anchors.append(a); walks.append(w)
            _, spans = variant_rows(g)
            t0 = time.perf_counter()
            f.fetch_array(c, min(s for s, _ in spans), max(e for _, e in spans))
            fa_ms.append((time.perf_counter() - t0) * 1e3)
    r.close(); f.close()
    q = lambda v: dict(median=round(float(np.median(v)), 3), max=round(float(np.max(v)), 3))     # noqa: E731
    return dict(groups=len(anchors), anchors_per_fetch=q(anchors), longest_walk=int(max(walks)), walk_per_anchor_max=q(walks),
                bam_fetch_device_ms=q(bam_ms), fasta_fetch_ms=q(fa_ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--total-mb", type=float, default=64.0)
    ap.add_argument("--coverage", type=float, default=20.0)
    ap.add_argument("--seed", type=int, default=41)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    a = ap.parse_args()
    from oracle import nets
    from pepper_b200 import synth, synth_files, _lib
    from pepper_b200.frontend import VariantFromFiles
    from pepper_b200.vcf import VCF_FILES
    _lib.require_gpu()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    shares = [("chr1", 0.34), ("chr2", 0.27), ("chr10", 0.22), ("chrX", 0.17)]
    tmp = tempfile.mkdtemp(prefix="bench_input_formats_")
    recs, fasta, lens = {}, [], []
    sizes = [int(a.total_mb * 1e6 * f) for _, f in shares]
    with ProcessPoolExecutor(max_workers=len(shares)) as pool:
        futs = [pool.submit(synth.simulate_contig_records, n, a.coverage, synth.ONT, a.seed + tid) for tid, n in enumerate(sizes)]
        for tid, ((c, _), n, fut) in enumerate(zip(shares, sizes, futs)):
            rec, genome = fut.result()
            recs[tid] = rec
            fasta.append((c, genome))
            lens.append((c, n))
    inputs = {}
    for tag, idx, gz in (("bai_plain", "bai", False), ("csi_bgzip", "csi", True)):
        bam, fa = os.path.join(tmp, tag + ".bam"), os.path.join(tmp, tag + ".fa" + (".gz" if gz else ""))
        synth_files.write_bam(bam, lens, recs, index=idx)
        synth_files.write_fasta(fa, fasta, bgzip=gz)
        inputs[tag] = (bam, fa)
    log("files written")
    state = nets.make_variant_weights(0)
    params = synth.ont_params()
    runs = {t: [] for t in inputs}
    outs = {}
    readers = {t: VariantFromFiles(*inputs[t], state) for t in inputs}
    try:
        for t, vf in readers.items():
            vf.call_genome(os.path.join(tmp, "warm_" + t), "sample", region="chr2:0-2000000", params=params)
        for k in range(a.rounds):
            for t, vf in readers.items():
                out = os.path.join(tmp, "%s_%d" % (t, k))
                t0 = time.perf_counter()
                totals = vf.call_genome(out, "sample", params=params, batch=a.batch)
                wall = time.perf_counter() - t0
                p = vf.last_genome_profile
                runs[t].append(dict(wall_s=round(wall, 3), bam_fetch_ms_per_group=round(p["bam_fetch"] / p["groups"], 3),
                                    fasta_fetch_ms_per_group=round(p["fasta_fetch"] / p["groups"], 3), groups=p["groups"]))
                outs.setdefault(t, (totals, out))
                log("%s round %d: %.2f s" % (t, k, wall))
    finally:
        for vf in readers.values():
            vf.close()
    files = {t: [gzip.decompress(open(os.path.join(o, n + ".vcf.gz"), "rb").read()) for n in VCF_FILES] for t, (_, o) in outs.items()}
    verified = outs["bai_plain"][0] == outs["csi_bgzip"][0] and files["bai_plain"] == files["csi_bgzip"]
    fetch = {t: group_fetch_stats(*inputs[t], lens, a.batch) for t in inputs}
    print(json.dumps(dict(card=card, total_mb=a.total_mb, coverage=a.coverage, rounds=runs, group_fetch=fetch,
                          totals=list(outs["bai_plain"][0]), verified=verified)))
    assert verified, "the two encodings gave different VCFs"


if __name__ == "__main__":
    main()
