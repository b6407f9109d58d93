"""Whole-genome variant calling on one GPU: a seeded multi-contig BAM + FASTA (chr1, chr2, chr10, chrX: natural order differs from
the lexical order of the VCF) -> VariantFromFiles.call_genome -> the five bgzipped, tabix-indexed VCFs, in genomic bases/s.

The same job then goes through the host tail (call_stream -> D2H of the candidate columns -> find_site_records, i.e. the CUDA
selection + the array / Python site assembly -> format_vcf_line -> the same writer); both sets of files are compared byte for byte
after decompression.  Prints one JSON line.  Default size: 64 Mb in total (chr20), 20x ONT.
    python scripts/bench_call_genome.py [--total-mb 64] [--coverage 20]

Under torchrun the ranks run dist.DistributedGenomeCaller on the same job instead (rank 0 simulates the files into a directory
every rank reads): rank 0 prints the JSON line with each stage's maximum over the ranks, and `verified` compares the decompressed
files with a one-GPU call_genome run on rank 0 outside the timed window.
    torchrun --nproc-per-node N scripts/bench_call_genome.py [--total-mb 64]

With --gvcf, one GPU runs dist.DistributedGenomeCaller over the job with and without the gVCF, alternating (--repeats each), and
reports both walls, the gVCF stages, the track bytes, the block and record lines and the compressed gVCF size; `verified` says
the five VCFs of every gVCF run equal those of the run without it after decompression.
    python scripts/bench_call_genome.py --gvcf [--total-mb 64] [--repeats 3]"""
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
    ap.add_argument("--gvcf", action="store_true")
    ap.add_argument("--repeats", type=int, default=3)
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
    if a.gvcf:
        return bench_gvcf(a, bam, fa, tmp, bases, state, params, card)
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


def bench_gvcf(a, bam, fa, tmp, bases, state, params, card):
    import numpy as np
    import torch
    from pepper_b200.cli import variant_capacity
    from pepper_b200.dist import DistributedGenomeCaller
    from pepper_b200.frontend import VariantGenomeSource
    from pepper_b200.pipeline import VariantCaller
    from pepper_b200.vcf import VCF_FILES
    caller = VariantCaller(state, 0)
    src = VariantGenomeSource(bam, fa, int(params["min_snp_baseq"]))
    cap = 4 * variant_capacity(bases, 1)        # room for the seeded random weights' candidates: no restart inside a timed run
    walls, phases, stats, outs = {False: [], True: []}, [], None, {}

    peaks = {False: 0, True: 0}

    def run(gvcf, out):
        dgc = DistributedGenomeCaller(None, 0, cap, "dynamic", distributed=False, caller=caller, gvcf=gvcf)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        dgc.call_source(src, out, "sample", params)
        torch.cuda.synchronize()
        w = time.perf_counter() - t0
        peaks[gvcf] = max(peaks[gvcf], int(torch.cuda.max_memory_allocated()))
        ph, st = dgc.phase_ms, getattr(dgc, "gvcf_stats", None)
        dgc.close()
        return w, ph, st
    try:
        run(False, os.path.join(tmp, "warm"))
        run(True, os.path.join(tmp, "warm_g"))
        log("warm-up done")
        for k in range(a.repeats):
            for gvcf in (False, True):
                out = os.path.join(tmp, "g%d_%d" % (k, gvcf))
                w, ph, st = run(gvcf, out)
                walls[gvcf].append(w)
                outs.setdefault(gvcf, []).append(out)
                if gvcf:
                    phases.append(ph); stats = st
                log("run %d gvcf=%s: %.2f s" % (k, gvcf, w))
    finally:
        src.close()
        caller.close()
    files = lambda d: [gzip.decompress(open(os.path.join(d, f + ".vcf.gz"), "rb").read()) for f in VCF_FILES]   # noqa: E731
    want = files(outs[False][0])
    same = all(files(d) == want for d in outs[False] + outs[True])
    g = os.path.join(outs[True][-1], "PEPPER_VARIANT.g.vcf.gz")
    med = lambda x: round(float(np.median(x)), 3)                               # noqa: E731
    stage = lambda k: round(float(np.median([p.get(k, 0.0) for p in phases])), 2)   # noqa: E731
    print(json.dumps(dict(
        metric="call_genome_gvcf", value=bases / med(walls[True]), unit="genomic bases/s", genomic_bases=bases, coverage=a.coverage,
        wall_s=dict(without_gvcf=[round(x, 3) for x in walls[False]], with_gvcf=[round(x, 3) for x in walls[True]],
                    median_without=med(walls[False]), median_with=med(walls[True])),
        gvcf_stage_ms=dict(exchange=stage("gvcf_exchange"), blocks_device=stage("gvcf_blocks"), records_device=stage("gvcf_records"),
                           merge_host=stage("gvcf_merge_host"), layout_device=stage("gvcf_layout"), compression=stage("gvcf_compress"),
                           gather=stage("gvcf_gather"), index_and_write=stage("gvcf_write")),
        track_bytes=stats["track_bytes"], block_lines=stats["block_lines"], record_lines=stats["record_lines"],
        gvcf_payload_bytes=stats["payload_bytes"], gvcf_file_bytes=os.path.getsize(g), verified=bool(same), card=card,
        peak_torch_allocated_bytes=dict(without_gvcf=peaks[False], with_gvcf=peaks[True]),     # the library's own buffers not included
        notes="medians over alternating runs in one process; stage times are host walls around synchronous device work")))


def main_distributed():
    import torch
    import torch.distributed as dist
    ap = argparse.ArgumentParser()
    ap.add_argument("--total-mb", type=float, default=64.0)
    ap.add_argument("--coverage", type=float, default=20.0)
    ap.add_argument("--seed", type=int, default=41)
    ap.add_argument("--dir", default=os.path.join(tempfile.gettempdir(), "bench_call_genome_dist"))
    a = ap.parse_args()
    rank, local = int(os.environ["RANK"]), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    world = dist.get_world_size()
    from oracle import nets
    from pepper_b200 import synth, synth_files, _lib
    from pepper_b200.dist import DistributedGenomeCaller
    from pepper_b200.frontend import VariantFromFiles
    from pepper_b200.vcf import VCF_FILES
    _lib.require_gpu()
    shares = [("chr1", 0.34), ("chr2", 0.27), ("chr10", 0.22), ("chrX", 0.17)]
    sizes = [int(a.total_mb * 1e6 * f) for _, f in shares]
    bam, fa = os.path.join(a.dir, "g.bam"), os.path.join(a.dir, "g.fa")
    if rank == 0:
        os.makedirs(a.dir, exist_ok=True)
        recs, fasta = {}, []
        with ProcessPoolExecutor(max_workers=len(shares)) as pool:
            futs = [pool.submit(synth.simulate_contig_records, n, a.coverage, synth.ONT, a.seed + tid) for tid, n in enumerate(sizes)]
            for tid, ((c, _), fut) in enumerate(zip(shares, futs)):
                recs[tid], g = fut.result()
                fasta.append((c, g))
        synth_files.write_bam(bam, [(c, n) for (c, _), n in zip(shares, sizes)], recs)
        synth_files.write_fasta(fa, fasta)
        log("files written")
    dist.barrier()
    state, params = nets.make_variant_weights(0), synth.ont_params()
    # session room: about one candidate per 15 genomic bases of this rank's share (84 bytes each)
    dgc = DistributedGenomeCaller(state, local, 84 * (sum(sizes) // 15 // world + (1 << 16)), "dynamic")
    dgc.call_genome(bam, fa, os.path.join(a.dir, "warm"), "sample", region="chr2:0-2000000", params=params)
    dist.barrier()
    t0 = time.perf_counter()
    totals = dgc.call_genome(bam, fa, os.path.join(a.dir, "dist"), "sample", params=params)
    dist.barrier()
    wall = time.perf_counter() - t0
    phases = [None] * world
    dist.all_gather_object(phases, dgc.phase_ms)
    extra = [None] * world
    dist.all_gather_object(extra, (dgc.payload_bytes, dgc.member_bytes))
    dgc.close()
    if rank == 0:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip().splitlines()[0]
        with VariantFromFiles(bam, fa, state) as vf:
            t1 = time.perf_counter()
            want = vf.call_genome(os.path.join(a.dir, "one"), "sample", params=params)
            one_wall = time.perf_counter() - t1
            one_prof = dict(vf.last_genome_profile)
        same = want == totals and all(
            gzip.decompress(open(os.path.join(a.dir, "dist", f + ".vcf.gz"), "rb").read())
            == gzip.decompress(open(os.path.join(a.dir, "one", f + ".vcf.gz"), "rb").read()) for f in VCF_FILES)
        stage = lambda k: round(max(p.get(k, 0.0) for p in phases), 2)      # noqa: E731
        pay, comp = sum(x for x, _ in extra), sum(y for _, y in extra)
        print(json.dumps(dict(
            metric="call_genome_distributed", value=sum(sizes) / wall, unit="genomic bases/s", wall_s=round(wall, 3), gpus=world,
            genomic_bases=sum(sizes), coverage=a.coverage, totals=totals,
            stage_ms=dict(sessions=stage("sessions"), vcf_pass=stage("vcf_pass"), edge_exchange=stage("edge_exchange"),
                          edge_pass=stage("edge"), layout=stage("layout"), compression=stage("compress"), gather=stage("gather"),
                          index_and_write=stage("write"), encoder_device=stage("encoder_device"), network_device=stage("network_device")),
            compressor=dict(payload_bytes=pay, member_bytes=comp, ratio=round(pay / max(1, comp), 2),
                            gb_per_s=round(pay / max(1e-9, stage("compress") / 1e3) / 1e9, 3)),
            one_gpu_call_genome=dict(wall_s=round(one_wall, 3), stage_ms=one_prof),
            verified=bool(same), card=card)))
    dist.destroy_process_group()


if __name__ == "__main__":
    if "WORLD_SIZE" in os.environ and "RANK" in os.environ:
        main_distributed()
    else:
        main()
