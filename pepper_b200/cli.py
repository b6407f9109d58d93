"""The command lines of the two pipelines, with the flags, defaults and platform presets of `pepper_variant call_variant` and
`pepper polish`:

    python -m pepper_b200 call_variant -b reads.bam -f ref.fa -m model.pkl -o out/ -s SAMPLE -t 16 --ont_r9_guppy5_sup
    python -m pepper_b200 call_variant_gvcf ... (call_variant's flags) [--gvcf_gq_binsize 5]   # + PEPPER_VARIANT.g.vcf.gz
    python -m pepper_b200 polish -b reads.bam -f draft.fa -m model.pkl -o out/asm -t 16 [--fastq]

Everything runs on the GPU (the device pipelines of frontend / dist).  With `-g`, one worker process per device of `-d_ids`
(default: every visible device) runs its rank of dist.DistributedGenomeCaller / dist.DistributedPolisher over NCCL and rank 0
writes the output; with one device, or without `-g`, the same drivers run in this process at world size 1.  Launched by
torchrun (WORLD_SIZE / RANK set), the command runs as that rank.

Flags of the reference that do not change its output (`-bs`, `-w`, `-per_gpu`, `--quantized`, `--no_quantized`,
`--region_bed`) are accepted and reported as having no effect."""
from __future__ import annotations

import argparse
import os
import sys
import time
from datetime import datetime

from . import presets


class CliError(Exception):
    """A one-line error the command reports before it exits with status 1."""


def log(msg: str, level: str = "INFO") -> None:
    sys.stderr.write("[%s] %s: %s\n" % (datetime.now().strftime("%m-%d-%Y %H:%M:%S"), level, msg))
    sys.stderr.flush()


# ----------------------------------------------------------------------------------------------------------- the parsers
def add_call_variant_arguments(p: argparse.ArgumentParser) -> argparse.ArgumentParser:
    """The options of `pepper_variant call_variant` (names, defaults and types of CallVariantsArguments.py)."""
    for names, help_ in ((("-b", "--bam"), "Coordinate-sorted, indexed BAM of the reads aligned to the reference."),
                         (("-f", "--fasta"), "Reference FASTA (indexed: .fai; bgzip-compressed: also .gzi)."),
                         (("-m", "--model_path"), "Trained PEPPER variant model (.pkl checkpoint)."),
                         (("-o", "--output_dir"), "Output directory."),
                         (("-s", "--sample_name"), "Sample name written to the VCFs.")):
        p.add_argument(*names, type=str, required=True, help=help_)
    p.add_argument("-t", "--threads", type=int, required=True, help="Host threads of the BAM readers.")
    p.add_argument("-d", "--downsample_rate", type=float, default=1.0, help="Fraction of the reads kept. Default is 1.0.")
    p.add_argument("-r", "--region", type=str, default=None,
                   help="Regions to call, contig[:start-end][,...]. Default: every contig common to the BAM and the FASTA, "
                        "decoy / alt / HLA / unplaced contigs excluded.")
    p.add_argument("--region_size", type=int, default=100000, help="Interval size the contigs are tiled with. Default is 100000.")
    p.add_argument("--region_bed", "-rb", type=str, default=None, help="Accepted; read only in training mode (no effect here).")
    p.add_argument("-hp", "--use_hp_info", default=False, action="store_true", help="Not supported: exits with an error.")
    p.add_argument("--include_supplementary", default=False, action="store_true", help="Use supplementary alignments.")
    for name, typ, help_ in (("--min_mapq", int, "Minimum mapping quality of a read."),
                             ("--min_snp_baseq", int, "Minimum base quality of a SNP base."),
                             ("--min_indel_baseq", int, "Minimum base quality of an indel base."),
                             ("--snp_frequency", float, "Minimum SNP frequency of a candidate site."),
                             ("--insert_frequency", float, "Minimum insert frequency of a candidate site."),
                             ("--delete_frequency", float, "Minimum delete frequency of a candidate site."),
                             ("--min_coverage_threshold", int, "Minimum coverage of a candidate site."),
                             ("--candidate_support_threshold", int, "Minimum reads supporting a candidate."),
                             ("--snp_candidate_frequency_threshold", float, "Minimum frequency of a SNP candidate."),
                             ("--indel_candidate_frequency_threshold", float, "Minimum frequency of an indel candidate.")):
        p.add_argument(name, type=typ, default=None, help=help_ + " Default: the preset's.")
    p.add_argument("--skip_indels", default=False, action="store_true", help="Skip indel candidates (always on with --clr).")
    p.add_argument("-bs", "--batch_size", type=int, default=512, help="Accepted (no effect: the network runs fixed-size chunks).")
    p.add_argument("-g", "--gpu", default=False, action="store_true",
                   help="One worker process per device of --device_ids. Without it the call runs on one GPU in this process.")
    p.add_argument("-per_gpu", "--callers_per_gpu", type=int, default=4, help="Accepted (no effect).")
    p.add_argument("-d_ids", "--device_ids", type=str, default=None, help="Comma list of CUDA devices for -g. Default: all visible.")
    p.add_argument("--quantized", default=False, action="store_true", help="Accepted (no effect).")
    p.add_argument("--no_quantized", dest="quantized", default=False, action="store_false", help="Accepted (no effect).")
    p.add_argument("-w", "--num_workers", type=int, default=0, help="Accepted (no effect).")
    p.add_argument("--allowed_multiallelics", type=int, default=None, help="Maximum alleles per site. Default: the preset's.")
    for name in ("snp_p_value", "insert_p_value", "delete_p_value", "snp_p_value_in_lc", "insert_p_value_in_lc",
                 "delete_p_value_in_lc", "snp_q_cutoff", "indel_q_cutoff", "snp_q_cutoff_in_lc", "indel_q_cutoff_in_lc",
                 "report_snp_above_freq", "report_indel_above_freq"):
        p.add_argument("--" + name, type=float, default=None, help="Candidate finding option. Default: the preset's.")
    group = p.add_mutually_exclusive_group(required=True)
    for name, help_ in (("ont_r9_guppy5_sup", "ONT R9.4.1 Guppy 5+ sup reads."), ("ont_r9_guppy4_hac", "ONT R9.4.1 Guppy HAC reads."),
                        ("ont_r10_q20", "ONT R10.4 Q20 reads."), ("hifi", "PacBio HiFi reads."), ("clr", "PacBio CLR reads.")):
        group.add_argument("--" + name, default=False, action="store_true", help="Preset: " + help_)
    return p


def add_polish_arguments(p: argparse.ArgumentParser) -> argparse.ArgumentParser:
    """The options of `pepper polish` (pepper.py), and --fastq."""
    for names, help_ in ((("-b", "--bam"), "Coordinate-sorted, indexed BAM of the reads aligned to the draft assembly."),
                         (("-f", "--fasta"), "Draft assembly FASTA (indexed: .fai)."),
                         (("-m", "--model_path"), "Trained PEPPER polish model (.pkl checkpoint)."),
                         (("-o", "--output_file"), "Output prefix: the polished assembly is <prefix>/_pepper_polished.fa.")):
        p.add_argument(*names, type=str, required=True, help=help_)
    p.add_argument("-t", "--threads", type=int, default=5, help="Host threads of the BAM readers. Default is 5.")
    p.add_argument("-r", "--region", type=str, help="Contigs to polish, contig[:start-end][,...]. Default: every common contig.")
    p.add_argument("-bs", "--batch_size", type=int, default=128, help="Accepted (no effect).")
    p.add_argument("-g", "--gpu", default=False, action="store_true",
                   help="One worker process per device of --device_ids. Without it the polish runs on one GPU in this process.")
    p.add_argument("-d_ids", "--device_ids", type=str, default=None, help="Comma list of CUDA devices for -g. Default: all visible.")
    p.add_argument("-w", "--num_workers", type=int, default=4, help="Accepted (no effect).")
    p.add_argument("--fastq", default=False, action="store_true",
                   help="Also write <prefix>/_pepper_polished.fastq: every polished base with its quality.")
    return p


def build_parser() -> argparse.ArgumentParser:
    parser = argparse.ArgumentParser(prog="python -m pepper_b200", description="PEPPER variant calling and polishing on the GPU.")
    sub = parser.add_subparsers(dest="sub_command")
    add_call_variant_arguments(sub.add_parser("call_variant", help="BAM + FASTA -> the five PEPPER_VARIANT VCFs."))
    add_polish_arguments(sub.add_parser("polish", help="BAM + draft FASTA -> polished FASTA (and FASTQ)."))
    g = add_call_variant_arguments(sub.add_parser("call_variant_gvcf", help="call_variant, and the gVCF PEPPER_VARIANT.g.vcf.gz."))
    g.add_argument("--gvcf_gq_binsize", type=int, default=5,
                   help="GQ band width of the gVCF's reference blocks: a block's positions share GQ // binsize. Default is 5.")
    return parser


VARIANT_COMMANDS = ("call_variant", "call_variant_gvcf")
NO_EFFECT = dict(call_variant=("batch_size", "num_workers", "callers_per_gpu", "quantized", "region_bed"),
                 polish=("batch_size", "num_workers"))
NO_EFFECT["call_variant_gvcf"] = NO_EFFECT["call_variant"]


def resolve(ns: argparse.Namespace) -> argparse.Namespace:
    """call_variant: the selected preset fills every option left unset (presets.resolve); ns.preset names it."""
    ns.preset = next(k for k in presets.PRESETS if getattr(ns, k))
    for k, v in presets.resolve(ns.preset, vars(ns)).items():
        setattr(ns, k, v)
    return ns


def no_effect_flags(parser: argparse.ArgumentParser, ns: argparse.Namespace) -> list[str]:
    """The options of NO_EFFECT the command line set to a value other than their default."""
    sub = next(a for a in parser._actions if isinstance(a, argparse._SubParsersAction)).choices[ns.sub_command]
    return [k for k in NO_EFFECT[ns.sub_command] if getattr(ns, k) != sub.get_default(k)]


# ----------------------------------------------------------------------------------------------------------- checks
MODEL_KIND = dict(call_variant="variant", call_variant_gvcf="variant", polish="polish")


def check_inputs(ns: argparse.Namespace) -> None:
    """The input checks of CallVariant.py / polish.py, with the indexes the readers need."""
    if not os.path.isfile(ns.bam):
        raise CliError("CAN NOT LOCATE BAM FILE: %s" % ns.bam)
    stem = ns.bam[:-4] if ns.bam.endswith(".bam") else ns.bam
    if not any(os.path.isfile(p + ext) for p in (ns.bam, stem) for ext in (".csi", ".bai")):
        raise CliError("CAN NOT LOCATE BAM INDEX: %s.bai or %s.csi (samtools index)" % (ns.bam, ns.bam))
    if not os.path.isfile(ns.fasta):
        raise CliError("CAN NOT LOCATE FASTA FILE: %s" % ns.fasta)
    if not os.path.isfile(ns.fasta + ".fai"):
        raise CliError("CAN NOT LOCATE FASTA INDEX: %s.fai (samtools faidx)" % ns.fasta)
    if not os.path.isfile(ns.model_path):
        raise CliError("CAN NOT LOCATE MODEL FILE: %s" % ns.model_path)
    if ns.threads <= 0:
        raise CliError("THREAD NEEDS TO BE >0.")
    if ns.batch_size <= 0:
        raise CliError("batch_size NEEDS TO BE >0.")
    if ns.num_workers < 0:
        raise CliError("num_workers NEEDS TO BE >=0.")
    if getattr(ns, "use_hp_info", False):
        raise CliError("-hp/--use_hp_info IS NOT SUPPORTED: the PEPPER variant model reads 33-feature images and has no "
                       "haplotype-aware (48-feature) counterpart to run.")
    if getattr(ns, "downsample_rate", 1.0) <= 0 or getattr(ns, "downsample_rate", 1.0) > 1:
        raise CliError("downsample_rate NEEDS TO BE IN (0, 1].")
    if getattr(ns, "region_size", 1) <= 0:
        raise CliError("region_size NEEDS TO BE >0.")
    if getattr(ns, "gvcf_gq_binsize", 1) <= 0:
        raise CliError("gvcf_gq_binsize NEEDS TO BE >0.")


def load_model(path: str, kind: str) -> dict:
    """weights.load_checkpoint, with every tensor's name and shape checked against the network the kernels run."""
    from .weights import load_checkpoint, random_variant_state, random_polish_state
    try:
        state = load_checkpoint(path)
    except Exception as ex:                                 # noqa: BLE001 — any unreadable file is a user error here
        raise CliError("CAN NOT READ MODEL FILE %s: %s" % (path, str(ex).splitlines()[0] if str(ex) else type(ex).__name__))
    want = {k: tuple(v.shape) for k, v in (random_variant_state(0) if kind == "variant" else random_polish_state(0)).items()}
    for k in want:
        if k not in state:
            raise CliError("MODEL %s IS NOT A PEPPER %s MODEL: tensor %s is missing" % (path, kind.upper(), k))
        got = tuple(getattr(state[k], "shape", ()))
        if got != want[k]:
            raise CliError("MODEL %s IS NOT A PEPPER %s MODEL: tensor %s has shape %s, expected %s"
                           % (path, kind.upper(), k, list(got), list(want[k])))
    extra = sorted(set(state) - set(want))
    if extra:
        raise CliError("MODEL %s IS NOT A PEPPER %s MODEL: unexpected tensor %s" % (path, kind.upper(), extra[0]))
    return state


def _device_ids(text: str) -> list[int]:
    try:
        return [int(i) for i in text.split(",")]
    except ValueError:
        raise CliError("--device_ids: INVALID VALUE %r" % text) from None


def device_list(ns: argparse.Namespace) -> list[int]:
    """The devices to run on: -d_ids (or every visible device) with -g; the first of -d_ids (or device 0) without it."""
    import torch
    n = torch.cuda.device_count()
    if n == 0:
        raise CliError("NO CUDA DEVICE IS VISIBLE: this build runs on the GPU only.")
    if ns.device_ids is None:
        ids = list(range(n)) if ns.gpu else [0]
    else:
        ids = _device_ids(ns.device_ids)
        bad = [i for i in ids if not 0 <= i < n]
        if bad or len(set(ids)) != len(ids):
            raise CliError("--device_ids: GPU DEVICE %s IS NOT AVAILABLE (%d visible)" % (bad[0] if bad else ids, n))
        ids = ids if ns.gpu else ids[:1]
    return ids


# ----------------------------------------------------------------------------------------------------------- the runs
def variant_capacity(bases: int, world: int) -> int:
    """Bytes of candidate records one rank's session may hold for a job of `bases` genomic bases: one candidate per 30 bases
    on one GPU, where an exhausted session restarts with twice the room (run_restarting); twice a rank's share of that on
    several GPUs, where it does not."""
    from .dist import RECORD_BYTES
    return RECORD_BYTES * (bases // (30 if world == 1 else 15 * world) + (1 << 16))


def polish_capacity(bases: int) -> int:
    """Consensus bytes (records with qualities) one rank may hold for an assembly of `bases` draft bases, as polish_assembly
    sizes it: one rank could hold the whole assembly."""
    return 2 * bases + (1 << 20)


def run_restarting(open_source, run, capacity, world: int, what: str):
    """run(source, cap) over a freshly opened source.  When the session's capacity is exhausted (PB_ERR_CAPACITY): on one GPU,
    again over a new source with twice the room (the fetch ring of the failed attempt may still hold claimed requests, so it is
    not reused); on several GPUs the run fails with a one-line message, since the ranks may be at different points of the job
    and a restart of one rank would pair its collectives with the others' of the failed attempt."""
    from ._lib import PepperB200Error
    from .abi import PB_ERR_CAPACITY
    cap = None
    while True:
        src = open_source()
        try:
            cap = cap or capacity(src)
            return run(src, cap)
        except PepperB200Error as ex:
            if ex.rc != PB_ERR_CAPACITY:
                raise
            if world > 1:
                raise CliError("THE %s CAPACITY OF ONE GPU (%d BYTES) IS EXHAUSTED ON %d GPUS; RUN ON ONE GPU, WHERE THE "
                               "CALL RESTARTS WITH MORE ROOM." % (what, cap, world)) from None
            log("THE %s CAPACITY (%d BYTES) IS EXHAUSTED: RESTARTING WITH %d BYTES." % (what, cap, 2 * cap))
            cap *= 2
        finally:
            src.close()


def run_call_variant(ns: argparse.Namespace, state: dict, device: int, distributed: bool):
    """This rank's part of the call (rank 0 writes the VCFs); returns the FindCandidates totals on every rank."""
    from .bamio import FastaReader
    from .dist import DistributedGenomeCaller
    from .exclude import excluded_contigs
    from .frontend import VariantGenomeSource
    from .gvcf import track_capacity
    from .pipeline import VariantCaller
    import torch.distributed as dist
    world, rank = (dist.get_world_size(), dist.get_rank()) if distributed else (1, 0)
    params = presets.image_params(vars(ns))
    exclude = []
    if not ns.region:
        fa = FastaReader(ns.fasta)
        try:
            exclude = excluded_contigs(fa.get_chromosome_names())
        finally:
            fa.close()
        if exclude and rank == 0:
            log("EXCLUDED CONTIGS (%d, DECOY / ALT / HLA / UNPLACED / VIRAL): %s%s"
                % (len(exclude), ", ".join(exclude[:10]), ", ..." if len(exclude) > 10 else ""))
    opened = []

    def open_source():
        try:
            src = VariantGenomeSource(ns.bam, ns.fasta, params["min_snp_baseq"], ns.region, exclude, ns.region_size, device,
                                      threads=ns.threads, **presets.read_filters(vars(ns)))
        except ValueError as ex:
            note = " (%d FASTA contigs excluded by name; give -r to call them)" % len(exclude) if exclude else ""
            raise CliError(str(ex) + note) from None
        if not opened and rank == 0:
            log("COMMON CONTIGS FOUND: %s" % src.names)
        opened.append(1)
        return src

    gvcf = ns.sub_command == "call_variant_gvcf"

    def run(src, cap):
        # the gVCF track grows with the candidate room: a restart doubles both
        bases = sum(e - s + 1 for s, e in src.intervals)
        track = track_capacity(bases, world) * (cap // variant_capacity(bases, world)) if gvcf else None
        dgc = DistributedGenomeCaller(None, device, cap, "dynamic", distributed=distributed, caller=caller, gvcf=gvcf,
                                      gvcf_binsize=getattr(ns, "gvcf_gq_binsize", 5), track_positions=track)
        try:
            return dgc.call_source(src, ns.output_dir, ns.sample_name, params, presets.candidate_options(vars(ns)),
                                   presets.vcf_options(vars(ns)))
        finally:
            dgc.close()
    caller = VariantCaller(state, device)
    try:
        return run_restarting(open_source, run, lambda src: variant_capacity(sum(e - s + 1 for s, e in src.intervals), world),
                              world, "CANDIDATE AND GVCF TRACK" if gvcf else "CANDIDATE")
    finally:
        caller.close()


def polish_output(prefix: str) -> str:
    """The directory of the polished files: `-o` as a directory (pepper polish.py:83), the files named as perform_stitch.py:53
    names them under it (<dir>/_pepper_polished.fa)."""
    return prefix if prefix.endswith("/") else prefix + "/"


def polish_contigs(ns: argparse.Namespace):
    """polish `-r` as the contig list of PolishFileSource (None: every common contig).  A contig may appear once: its
    polished sequence is one FASTA record."""
    from .frontend import parse_region
    if not ns.region:
        return None
    try:
        contigs = parse_region(ns.region)
    except ValueError as ex:
        raise CliError(str(ex)) from None
    names = [c for c, _ in contigs]
    dup = sorted({c for c in names if names.count(c) > 1})
    if dup:
        raise CliError("--region: CONTIG %s IS GIVEN MORE THAN ONCE; polish takes one span per contig." % dup[0])
    return contigs


def run_polish(ns: argparse.Namespace, state: dict, device: int, distributed: bool) -> dict:
    """This rank's part of the polish; returns {contig: sequence} or, with --fastq, {contig: (sequence, qualities)}."""
    from .dist import DistributedPolisher
    from .frontend import PolishFileSource
    from .pipeline import PolishCaller
    import torch.distributed as dist
    world = dist.get_world_size() if distributed else 1
    contigs = polish_contigs(ns)

    def open_source():
        try:
            src = PolishFileSource(ns.bam, ns.fasta, contigs, device, ns.threads)
        except KeyError as ex:
            raise CliError("--region: contig %s is not in the FASTA" % ex) from None
        except ValueError as ex:
            raise CliError(str(ex)) from None
        if not src.names:
            src.close()
            raise CliError("NO COMMON CONTIGS FOUND BETWEEN THE BAM FILE AND THE FASTA FILE.")
        return src

    def run(src, cap):
        dp = DistributedPolisher(None, device, cap, "dynamic", distributed=distributed, caller=caller, qualities=ns.fastq)
        try:
            dp.run(src)
            return dp.assemble(src)
        finally:
            dp.close()
    caller = PolishCaller(state, device)
    try:
        return run_restarting(open_source, run, lambda src: polish_capacity(sum(e - s + 1 for s, e in src.intervals)),
                              world, "CONSENSUS")
    finally:
        caller.close()


TOTALS = ("TOTAL CANDIDATES FOUND", "TOTAL VARIANTS IN PEPPER", "TOTAL VARIANTS SELECTED FOR RE-GENOTYPING",
          "TOTAL SNP VARIANTS SELECTED FOR RE-GENOTYPING", "TOTAL INDEL VARIANTS SELECTED FOR RE-GENOTYPING")


def finish(ns: argparse.Namespace, result, t0: float) -> None:
    """Rank 0's output: the totals lines of call_variant; the polished files of polish."""
    if ns.sub_command in VARIANT_COMMANDS:
        for label, n in zip(TOTALS, result):
            log("FINISHED PROCESSING, %s: %d" % (label, n))
        if ns.sub_command == "call_variant_gvcf":
            log("GVCF: %s" % os.path.join(ns.output_dir, "PEPPER_VARIANT.g.vcf.gz"))
    else:
        from .frontend import natural_key, write_polished_fasta, write_polished_fastq
        out = polish_output(ns.output_file)
        os.makedirs(out, exist_ok=True)
        seqs = {c: v[0] for c, v in result.items()} if ns.fastq else result
        for c in sorted(seqs, key=natural_key):
            log("FINISHED PROCESSING %s, POLISHED SEQUENCE LENGTH: %d." % (c, len(seqs[c])))
        write_polished_fasta(out + "_pepper_polished.fa", seqs)
        log("POLISHED ASSEMBLY: %s_pepper_polished.fa" % out)
        if ns.fastq:
            write_polished_fastq(out + "_pepper_polished.fastq", result)
            log("POLISHED ASSEMBLY WITH QUALITIES: %s_pepper_polished.fastq" % out)
    t = int(time.time() - t0)
    log("TOTAL ELAPSED TIME: %d Min %d Sec" % (t // 60, t % 60))


def _run(ns, state, device: int, distributed: bool):
    return (run_call_variant if ns.sub_command in VARIANT_COMMANDS else run_polish)(ns, state, device, distributed)


def _worker(rank: int, world: int, port: int, devices: list[int], ns, state, t0: float) -> None:
    """One rank of a multi-GPU run (torch.multiprocessing.spawn): NCCL over 127.0.0.1:port, device devices[rank]."""
    import torch
    import torch.distributed as dist
    device = devices[rank]
    torch.cuda.set_device(device)
    dist.init_process_group("nccl", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world,
                            device_id=torch.device("cuda", device))
    try:
        result = _run(ns, state, device, True)
        if rank == 0:
            finish(ns, result, t0)
    finally:
        dist.destroy_process_group()


def _free_port() -> int:
    import socket
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def execute(ns: argparse.Namespace, no_effect: list[str]) -> None:
    t0 = time.time()
    command = ns.sub_command
    if command in VARIANT_COMMANDS:
        resolve(ns)
        log("PRESET: --%s" % ns.preset)
        for k in presets.IMAGE_KEYS + presets.CANDIDATE_KEYS:
            log("%s: %s" % (k.upper(), getattr(ns, k)))
        log("CALL VARIANT MODULE SELECTED")
    else:
        log("POLISH MODULE SELECTED")
    check_inputs(ns)
    if command == "polish":
        polish_contigs(ns)
    for k in no_effect:
        log("--%s IS ACCEPTED AND HAS NO EFFECT HERE." % k)
    state = load_model(ns.model_path, MODEL_KIND[command])
    if command in VARIANT_COMMANDS:
        os.makedirs(ns.output_dir, exist_ok=True)
    import torch.distributed as dist
    if "WORLD_SIZE" in os.environ and "RANK" in os.environ:          # launched by torchrun: run as that rank
        import torch
        if not dist.is_initialized():
            local = int(os.environ.get("LOCAL_RANK", 0))
            device = local
            if ns.device_ids is not None:
                ids = _device_ids(ns.device_ids)
                if local >= len(ids):
                    raise CliError("--device_ids: %d DEVICES GIVEN FOR LOCAL RANK %d; give one device per local rank."
                                   % (len(ids), local))
                device = ids[local]
            torch.cuda.set_device(device)
            dist.init_process_group("nccl", device_id=torch.device("cuda", device))
            own = True
        else:
            device, own = torch.cuda.current_device(), False
        try:
            log("RANK %d OF %d ON GPU %d" % (dist.get_rank(), dist.get_world_size(), device))
            result = _run(ns, state, device, True)
            if dist.get_rank() == 0:
                finish(ns, result, t0)
        finally:
            if own:
                dist.destroy_process_group()
        return
    devices = device_list(ns)
    if len(devices) == 1:
        log("GPU %d, IN PROCESS" % devices[0])
        finish(ns, _run(ns, state, devices[0], False), t0)
        return
    import torch.multiprocessing as mp
    log("GPUS %s: ONE WORKER PROCESS PER GPU" % ",".join(map(str, devices)))
    try:
        mp.spawn(_worker, args=(len(devices), _free_port(), devices, ns, state, t0), nprocs=len(devices), join=True)
    except mp.ProcessRaisedException as ex:
        lines = [x for x in str(ex).strip().splitlines() if x.strip()]
        raise CliError("RANK %d FAILED: %s" % (ex.error_index, lines[-1] if lines else "unknown error")) from None
    except mp.ProcessExitedException as ex:
        raise CliError("RANK %d FAILED: %s" % (ex.error_index, ex)) from None


def main(argv: list[str] | None = None) -> int:
    """Runs one command; returns 0, or 1 after a one-line ERROR message on stderr."""
    argv = list(sys.argv[1:] if argv is None else argv)
    parser = build_parser()
    ns = parser.parse_args(argv)
    if ns.sub_command is None:
        parser.print_help(sys.stderr)
        log("NO SUBCOMMAND SELECTED. PLEASE SELECT ONE OF THE AVAILABLE SUB-COMMANDS.", "ERROR")
        return 1
    from ._lib import PepperB200Error
    try:
        execute(ns, no_effect_flags(parser, ns))
    except (CliError, PepperB200Error) as ex:              # PepperB200Error: a file the readers reject, a contig too long
        log(str(ex).strip().splitlines()[0] if str(ex).strip() else type(ex).__name__, "ERROR")
        return 1
    return 0
