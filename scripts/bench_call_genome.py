"""Whole-genome variant calling on one GPU: a seeded multi-contig BAM + FASTA (chr1, chr2, chr10, chrX: natural order differs from
the lexical order of the VCF) -> VariantFromFiles.call_genome -> the five bgzipped, tabix-indexed VCFs, in genomic bases/s.

The same job then goes through the host tail (call_stream -> D2H of the candidate columns -> find_site_records, i.e. the CUDA
selection + the array / Python site assembly -> format_vcf_line -> the same writer); both sets of files are compared byte for byte
after decompression.  Prints one JSON line.  Default size: 64 Mb in total (chr20), 20x ONT.
    python scripts/bench_call_genome.py [--total-mb 64] [--coverage 20]"""
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
    print("[bench_call_genome] " + msg, file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--total-mb", type=float, default=64.0)
    ap.add_argument("--coverage", type=float, default=20.0)
    ap.add_argument("--seed", type=int, default=41)
    a = ap.parse_args()
    from oracle import nets
    from pepper_b200 import synth, synth_files, _lib
    from pepper_b200.candidates import ONT_OPTIONS
    from pepper_b200.frontend import VariantFromFiles, variant_intervals
    from pepper_b200.vcf import VCF_FILES, find_site_records, host_tail_text, order_lines, write_vcfs
    _lib.require_gpu()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    shares = [("chr1", 0.34), ("chr2", 0.27), ("chr10", 0.22), ("chrX", 0.17)]
    tmp = tempfile.mkdtemp(prefix="bench_call_genome_")
    t0 = time.perf_counter()
    recs, fasta, lens = {}, [], []
    sizes = [int(a.total_mb * 1e6 * f) for _, f in shares]
    with ProcessPoolExecutor(max_workers=len(shares)) as pool:        # one contig per process
        futs = [pool.submit(synth.simulate_contig_records, n, a.coverage, synth.ONT, a.seed + tid) for tid, n in enumerate(sizes)]
        for tid, ((c, _), n, fut) in enumerate(zip(shares, sizes, futs)):
            rec, genome = fut.result()
            recs[tid] = rec
            fasta.append((c, genome))
            lens.append((c, n))
            log("simulated %s (%d bases, %d records)" % (c, n, rec.n_records))
    bam, fa = os.path.join(tmp, "g.bam"), os.path.join(tmp, "g.fa")
    synth_files.write_bam(bam, lens, recs)
    synth_files.write_fasta(fa, fasta)
    log("files written")
    gen_s = time.perf_counter() - t0
    bases = sum(n for _, n in lens)
    state = nets.make_variant_weights(0)
    params = synth.ont_params()
    with VariantFromFiles(bam, fa, state) as vf:
        vf.call_genome(os.path.join(tmp, "warm"), "sample", region="chr2:0-2000000", params=params)   # module load, first launches
        log("warm-up done")
        t0 = time.perf_counter()
        totals = vf.call_genome(os.path.join(tmp, "dev"), "sample", params=params)
        wall = time.perf_counter() - t0
        prof = dict(vf.last_genome_profile)
        log("call_genome: %.1f s" % wall)
        # the host tail over the same job
        job = vf.vcf_job()
        names = [c for c, _, _ in job]
        parts, t_calls, t_tail = [], 0.0, 0.0
        for cid, (c, s, e) in enumerate(job):
            iv = variant_intervals(s, e)
            t1 = time.perf_counter()
            calls = vf.call_stream(c, iv, params, 32)
            t2 = time.perf_counter()
            table = vf.genome_table(c, iv)
            recs_c = find_site_records(c, calls.positions, calls.region_of, calls.depths, calls.freqs, calls.keys_raw, calls.probs, table,
                                       ONT_OPTIONS)
            parts.append(host_tail_text(recs_c, cid))
            t3 = time.perf_counter()
            t_calls += t2 - t1; t_tail += t3 - t2
            log("host tail %s done" % c)
        t1 = time.perf_counter()
        text, lines = order_lines(parts, names)
        host_totals = write_vcfs(os.path.join(tmp, "host"), "sample", vf.fasta_contigs(), names, text, lines)
        t_write = time.perf_counter() - t1
    same = host_totals == totals and all(
        gzip.decompress(open(os.path.join(tmp, "dev", f + ".vcf.gz"), "rb").read())
        == gzip.decompress(open(os.path.join(tmp, "host", f + ".vcf.gz"), "rb").read()) for f in VCF_FILES)
    print(json.dumps(dict(
        metric="call_genome", value=bases / wall, unit="genomic bases/s", wall_s=round(wall, 3), genomic_bases=bases,
        contigs=[c for c, _ in lens], coverage=a.coverage, totals=totals,
        stage_ms=dict(sessions_host=prof["calls"], encoder_device=prof["encoder_device"], network_device=prof["network_device"],
                      vcf_pass=prof["vcf"], gather=None, writer_host=prof["write"]),
        host_tail_ms=dict(sessions_and_d2h=round(t_calls * 1e3, 2), select_assemble_format=round(t_tail * 1e3, 2),
                          writer=round(t_write * 1e3, 2)),
        verified=bool(same), card=card, gen_seconds=round(gen_s, 1),
        notes="one GPU: no gather (gather ms null); vcf_pass = host wall around the synchronous device VCF pass, uploads included")))


if __name__ == "__main__":
    main()
