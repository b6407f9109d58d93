"""Whole-assembly polish throughput: a seeded multi-contig synthetic draft (default 5 Mb in 20 contigs, ONT 40x) written as BAM +
FASTA to a temporary directory, then make_images + call_consensus + the device stitch of every contig through
dist.DistributedPolisher (one streaming polish session per rank, one all-gather of the consensus bytes).  Launched like bench.py:
one process per GPU under RANK / WORLD_SIZE / LOCAL_RANK (torchrun), or plain `python` for one GPU.

Prints one JSON line: polished bases/s (consensus bytes of the whole assembly per wall second of the timed run) and draft
bases/s, per-rank encoder / network / wait / gather ms and groups, the card name and its power limit.  Rank 0 checks the
assembly against the single-GPU `polish_contig` of sampled contigs (`verified`).

`--fastq`: after the timed run above, the same assembly is polished `--reps` more times with and `--reps` times without
per-base qualities, the two modes alternating on one driver, and the line gains `fastq`: the wall time of every run, the
polished bases/s of each mode (total bases over total wall), and whether the FASTQ sequences equal the FASTA sequences.

`--vcf`: likewise with and without the edits VCF (edit events through the session and the all-gather, then the device record
pass, compression and index of DistributedPolisher.write_edits, inside the timed run); the line gains `vcf`: the wall times,
the polished bases/s of each mode, the records written, and whether the FASTA of the edits runs equals the plain FASTA.

    python scripts/bench_polish_assembly.py [--contigs 20] [--mb 5] [--coverage 40] [--group-regions 32] [--check 3]
                                            [--fastq] [--vcf] [--reps 3]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def power_limit_w(gpu: int):
    """Board power limit as nvidia-smi reports it (a read-only query); None where it is not available."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(gpu), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def write_draft(d: str, n_contigs: int, total: int, coverage: float, seed: int):
    """ctg1 .. ctgN of total / N bases each (natural and lexical orders differ from ctg10 on), reads simulated from them."""
    from pepper_b200 import synth, synth_files
    length = total // n_contigs
    names = ["ctg%d" % (k + 1) for k in range(n_contigs)]
    recs, genomes = {}, []
    for k, name in enumerate(names):
        rec, genome = synth.simulate_contig_records(length, coverage, synth.ONT, seed * 1000 + k)
        recs[k] = rec
        genomes.append((name, genome))
    bam, fa = os.path.join(d, "draft.bam"), os.path.join(d, "draft.fa")
    synth_files.write_bam(bam, [(n, g.shape[0]) for n, g in genomes], recs)
    synth_files.write_fasta(fa, genomes)
    return bam, fa, names, length


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--contigs", type=int, default=20)
    ap.add_argument("--mb", type=float, default=5.0)
    ap.add_argument("--coverage", type=float, default=40.0)
    ap.add_argument("--group-regions", type=int, default=32)
    ap.add_argument("--schedule", default="dynamic")
    ap.add_argument("--check", type=int, default=3, help="contigs compared with polish_contig on rank 0")
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--fastq", action="store_true", help="also time the assembly with per-base qualities, alternating with FASTA")
    ap.add_argument("--vcf", action="store_true", help="also time the assembly with the edits VCF, alternating with FASTA")
    ap.add_argument("--reps", type=int, default=3, help="--fastq / --vcf: runs of each mode")
    args = ap.parse_args()

    import torch
    import torch.distributed as dist
    from pepper_b200 import weights, _lib
    from pepper_b200.dist import DistributedPolisher
    from pepper_b200.frontend import PolishFileSource, PolishFromFiles

    rank, world, local = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    torch.cuda.set_device(local)
    _lib.require_gpu()
    tmp = tempfile.mkdtemp(prefix="pb_polish_asm_")
    try:
        t0 = time.time()
        bam, fa, names, length = write_draft(tmp, args.contigs, int(args.mb * 1e6), args.coverage, args.seed)
        gen_s = time.time() - t0
        state = weights.random_polish_state(0)
        draft = length * len(names)
        cap = int(2.5 * draft / world) + (4 << 20)            # this rank's consensus slice (bytes)
        # warm-up on one contig: library buffers, first kernel launches, NCCL communicator
        wsrc = PolishFileSource(bam, fa, contigs=names[:1], device=local)
        # events: at most one per image column plus one per image; the seeded random weights edit most draft bases
        dp = DistributedPolisher(state, local, cap, args.schedule, args.group_regions, capacity_events=cap)
        vcf_path = os.path.join(tmp, "edits.vcf.gz")
        for q, e in [(False, False)] + ([(True, False)] if args.fastq else []) + ([(False, True)] if args.vcf else []):
            dp.qualities, dp.edits = q, e
            dp.run(wsrc)
            if e and rank == 0:
                dp.write_edits(wsrc, vcf_path)
        dp.qualities = dp.edits = False
        wsrc.close()
        src = PolishFileSource(bam, fa, device=local)

        def timed(qualities: bool, edits: bool = False):
            dp.qualities, dp.edits = qualities, edits
            if world > 1:
                dist.barrier()
            torch.cuda.synchronize()
            t = time.perf_counter()
            n = dp.run(src)
            out = dp.assemble(src)
            if edits and rank == 0:
                dp.write_edits(src, vcf_path)
            return n, out, time.perf_counter() - t
        n, seqs, wall = timed(False)
        mine = dict(dp.phase_ms, consensus_bytes=n, images=dp.stats.get("images", 0))
        fastq = None
        if args.fastq:
            walls = {"fasta": [], "fastq": []}
            same = True
            for rep in range(args.reps):
                for q in ((True, False) if rep % 2 == 0 else (False, True)):
                    _, out, w = timed(q)
                    walls["fastq" if q else "fasta"].append(w)
                    same = same and ({c: s for c, (s, _) in out.items()} if q else out) == seqs
            bases = sum(len(s) for s in seqs.values())
            fastq = dict(reps=args.reps, wall_s={k: [round(w, 3) for w in v] for k, v in walls.items()},
                         polished_bases_per_s={k: round(bases * len(v) / sum(v), 1) for k, v in walls.items()},
                         fastq_sequences_equal_fasta=bool(same))
        vcf = None
        if args.vcf:
            import gzip
            walls = {"fasta": [], "vcf": []}
            same = True
            for rep_ in range(args.reps):
                for e in ((True, False) if rep_ % 2 == 0 else (False, True)):
                    _, out, w = timed(False, e)
                    walls["vcf" if e else "fasta"].append(w)
                    same = same and out == seqs
            bases = sum(len(s) for s in seqs.values())
            records = None
            if rank == 0:
                records = sum(1 for ln in gzip.decompress(open(vcf_path, "rb").read()).split(b"\n") if ln and not ln.startswith(b"#"))
            vcf = dict(reps=args.reps, wall_s={k: [round(w, 3) for w in v] for k, v in walls.items()},
                       polished_bases_per_s={k: round(bases * len(v) / sum(v), 1) for k, v in walls.items()},
                       records=records, vcf_fasta_equals_fasta=bool(same))
        per_rank = [None] * world
        if world > 1:
            dist.all_gather_object(per_rank, mine)
        else:
            per_rank = [mine]
        polished = sum(len(s) for s in seqs.values())
        groups_total = len(src.groups(args.group_regions))
        src.close()
        dp.close()
        verified = None
        if rank == 0:
            step = max(1, len(names) // max(1, args.check))
            sample = names[::step][:args.check]
            with PolishFromFiles(bam, fa, state, device=local) as pf:
                ok = all(pf.polish_contig(c) == seqs[c] for c in sample)
            verified = dict(contigs=sample, ok=bool(ok))
        if rank == 0:
            print(json.dumps(dict(
                metric="polish_assembly", world=world, contigs=len(names), draft_bases=draft, polished_bases=polished,
                coverage=args.coverage, group_regions=args.group_regions, schedule=args.schedule, groups=groups_total,
                wall_s=round(wall, 3), polished_bases_per_s=round(polished / wall, 1), draft_bases_per_s=round(draft / wall, 1),
                per_rank=[{k: (round(v, 2) if isinstance(v, float) else v) for k, v in r.items()} for r in per_rank],
                card=torch.cuda.get_device_name(local), power_limit_w=power_limit_w(local), synth_s=round(gen_s, 1),
                verified=verified, **({"fastq": fastq} if args.fastq else {}), **({"vcf": vcf} if args.vcf else {}))), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        if world > 1:
            dist.destroy_process_group()


if __name__ == "__main__":
    main()
