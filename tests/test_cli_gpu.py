"""GPU: the command lines end to end (pepper_b200.cli) on synthetic BAM + FASTA files.

1. call_variant in process, every preset: the five VCFs hold the same bytes, once the BGZF members are inflated, as
   VariantFromFiles.call_genome's given the image thresholds, candidate / VCF options and read filters the preset maps to (the
   members themselves differ: the command compresses on the device, call_genome with zlib on the host), each with its index;
   the decoy contig of the files is left out; the five totals log lines carry call_genome's totals.  HiFi reads for --hifi, ONT
   reads otherwise.
2. `python -m pepper_b200 call_variant` as a subprocess exits 0 with the same files as the in-process command.
3. polish: the FASTA, and the FASTQ with --fastq, equal polish_assembly's; `-r contig:start-end` equals polish_contig(contig,
   start, end).
4. A session capacity too small for the job (forced through the command's capacity estimate): the in-process command
   restarts with more room, over a freshly opened source, until the job fits, and its VCFs, FASTA and FASTQ still equal
   call_genome's / polish_assembly's.
5. Two GPUs (skipped below 2): `-g -d_ids 0,1` gives the single-GPU files byte for byte for call_variant and polish, and
   leaves no child process behind."""
import gzip
import multiprocessing
import os
import subprocess
import sys

import pytest
import torch

from pepper_b200 import cli, presets, synth, synth_files

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DECOY = "chr1_KI270706v1_random"
CONTIGS = [("chr2", 160_000, 51), ("chr1", 210_000, 52), (DECOY, 30_000, 53)]


def _save(state: dict, path: str) -> str:
    torch.save({"model_state_dict": {"module." + k: torch.as_tensor(v) for k, v in state.items()}, "epochs": 1}, path)
    return path


@pytest.fixture(scope="module")
def genome(tmp_path_factory):
    from oracle import nets
    d = tmp_path_factory.mktemp("cli_genome")
    out = dict(dir=d, fa=str(d / "g.fa"), model=_save(nets.make_variant_weights(0), str(d / "variant.pkl")),
               state=nets.make_variant_weights(0))
    fasta = []
    for platform, tag in ((synth.ONT, "ont"), (synth.HIFI, "hifi")):
        recs = {}
        for tid, (c, n, seed) in enumerate(CONTIGS):
            recs[tid], g = synth.simulate_contig_records(n, 20, platform, seed)
            if tag == "ont":
                fasta.append((c, g))
        out[tag] = str(d / ("%s.bam" % tag))
        synth_files.write_bam(out[tag], [(c, n) for c, n, _ in CONTIGS], recs)
    synth_files.write_fasta(out["fa"], fasta)
    return out


def _files(d) -> list[bytes]:
    from pepper_b200.vcf import VCF_FILES
    return [gzip.decompress(open(os.path.join(d, n + ".vcf.gz"), "rb").read()) for n in VCF_FILES]


def _raw(d) -> list[bytes]:
    return [open(os.path.join(d, n), "rb").read() for n in sorted(os.listdir(d))]


def _argv(genome, preset: str, out: str) -> list[str]:
    bam = genome["hifi" if preset == "hifi" else "ont"]
    return ["call_variant", "-b", bam, "-f", genome["fa"], "-m", genome["model"], "-o", out, "-s", "SAMPLE", "-t", "4", "--" + preset]


def _call_genome(genome, preset: str, out: str) -> tuple:
    """VariantFromFiles.call_genome with the arguments the preset maps to."""
    from pepper_b200.frontend import VariantFromFiles
    ns = cli.resolve(cli.build_parser().parse_args(_argv(genome, preset, out)))
    o = vars(ns)
    with VariantFromFiles(ns.bam, ns.fasta, genome["state"]) as vf:
        return vf.call_genome(out, "SAMPLE", exclude=[DECOY], params=presets.image_params(o), options=presets.candidate_options(o),
                              vcf_options=presets.vcf_options(o), **presets.read_filters(o))


@pytest.mark.parametrize("preset", presets.PRESETS)
def test_call_variant_in_process_matches_call_genome(genome, preset, capsys):
    from pepper_b200.vcf import VCF_FILES
    d = genome["dir"]
    want = _call_genome(genome, preset, str(d / ("want_" + preset)))
    capsys.readouterr()
    out = str(d / ("cli_" + preset))
    assert cli.main(_argv(genome, preset, out)) == 0
    err = capsys.readouterr().err
    got = _files(out)
    assert got == _files(d / ("want_" + preset))
    assert all(DECOY.encode() not in body.split(b"#CHROM")[1] for body in got)
    for n in VCF_FILES:
        assert gzip.decompress(open(os.path.join(out, n + ".vcf.gz.tbi"), "rb").read())[:4] == b"TBI\x01"
    for label, n in zip(cli.TOTALS, want):
        assert "] INFO: FINISHED PROCESSING, %s: %d\n" % (label, n) in err, label
    assert want[0] > 0, want


def test_call_variant_subprocess(genome):
    d = genome["dir"]
    out = str(d / "sub_r10")
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "pepper_b200"] + _argv(genome, "ont_r10_q20", out), cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "FINISHED PROCESSING, TOTAL CANDIDATES FOUND" in r.stderr
    want = str(d / "sub_r10_want")
    _call_genome(genome, "ont_r10_q20", want)
    assert _files(out) == _files(want)


# -------------------------------------------------------------------------------------------------------------- polish
@pytest.fixture(scope="module")
def assembly(tmp_path_factory):
    from pepper_b200 import weights
    d = tmp_path_factory.mktemp("cli_asm")
    genomes, recs = {}, {}
    for k, (name, length) in enumerate([("ctg10", 9000), ("ctg2", 5200), ("bamonly", 4000), ("faonly", 3000)]):
        recs[name], genomes[name] = synth.simulate_contig_records(length, 20, synth.ONT, 80 + k)
    bam, fa = str(d / "a.bam"), str(d / "a.fa")
    in_bam = ["ctg10", "bamonly", "ctg2"]
    synth_files.write_bam(bam, [(c, genomes[c].shape[0]) for c in in_bam], {t: recs[c] for t, c in enumerate(in_bam)})
    synth_files.write_fasta(fa, [(c, genomes[c]) for c in ["faonly", "ctg2", "ctg10"]])
    state = weights.random_polish_state(1)
    return dict(dir=d, bam=bam, fa=fa, state=state, model=_save(state, str(d / "polish.pkl")))


def _polish_argv(a, prefix, *extra):
    return ["polish", "-b", a["bam"], "-f", a["fa"], "-m", a["model"], "-o", prefix] + list(extra)


def test_polish_matches_polish_assembly(assembly):
    from pepper_b200.frontend import PolishFromFiles, polished_fasta_text, polished_fastq_text
    d = assembly["dir"]
    with PolishFromFiles(assembly["bam"], assembly["fa"], assembly["state"]) as pf:
        want_fa = polished_fasta_text(pf.polish_assembly())
        want_fq = polished_fastq_text(pf.polish_assembly(fastq=True))
        want_span = ">ctg10\n%s\n" % pf.polish_contig("ctg10", 1500, 6200)
    assert want_fa.count(">") == 2 and len(want_fa) > 12000
    prefix = str(d / "plain")
    assert cli.main(_polish_argv(assembly, prefix)) == 0
    assert open(os.path.join(prefix, "_pepper_polished.fa")).read() == want_fa
    assert not os.path.exists(os.path.join(prefix, "_pepper_polished.fastq"))
    prefix = str(d / "fq")
    assert cli.main(_polish_argv(assembly, prefix, "--fastq")) == 0
    assert open(os.path.join(prefix, "_pepper_polished.fa")).read() == want_fa
    assert open(os.path.join(prefix, "_pepper_polished.fastq")).read() == want_fq
    prefix = str(d / "span")
    assert cli.main(_polish_argv(assembly, prefix, "-r", "ctg10:1500-6200")) == 0
    assert open(os.path.join(prefix, "_pepper_polished.fa")).read() == want_span


def test_exhausted_capacity_restarts_in_process(genome, assembly, monkeypatch, capsys):
    from pepper_b200.dist import RECORD_BYTES
    from pepper_b200.frontend import PolishFromFiles, polished_fasta_text, polished_fastq_text
    d = genome["dir"]
    want = _call_genome(genome, "ont_r9_guppy5_sup", str(d / "cap_want"))
    assert want[0] > 1024, want
    monkeypatch.setattr(cli, "variant_capacity", lambda bases, world: RECORD_BYTES * 128)
    capsys.readouterr()
    out = str(d / "cap_cli")
    assert cli.main(_argv(genome, "ont_r9_guppy5_sup", out)) == 0
    err = capsys.readouterr().err
    assert err.count("THE CANDIDATE CAPACITY (") >= 3, err[-3000:]
    assert _files(out) == _files(d / "cap_want")
    for label, n in zip(cli.TOTALS, want):
        assert "] INFO: FINISHED PROCESSING, %s: %d\n" % (label, n) in err, label
    with PolishFromFiles(assembly["bam"], assembly["fa"], assembly["state"]) as pf:
        want_fa = polished_fasta_text(pf.polish_assembly())
        want_fq = polished_fastq_text(pf.polish_assembly(fastq=True))
    monkeypatch.setattr(cli, "polish_capacity", lambda bases: 1024)
    prefix = str(assembly["dir"] / "cap")
    assert cli.main(_polish_argv(assembly, prefix, "--fastq")) == 0
    assert capsys.readouterr().err.count("THE CONSENSUS CAPACITY (") >= 2
    assert open(os.path.join(prefix, "_pepper_polished.fa")).read() == want_fa
    assert open(os.path.join(prefix, "_pepper_polished.fastq")).read() == want_fq


# ---------------------------------------------------------------------------------------------------------- two GPUs
def test_two_gpus_match_one_gpu(genome, assembly):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs: %d visible" % torch.cuda.device_count())
    d = genome["dir"]
    one, two = str(d / "g1"), str(d / "g2")
    assert cli.main(_argv(genome, "ont_r9_guppy5_sup", one)) == 0
    assert cli.main(_argv(genome, "ont_r9_guppy5_sup", two) + ["-g", "-d_ids", "0,1"]) == 0
    assert multiprocessing.active_children() == []
    assert _raw(one) == _raw(two) and len(_raw(one)) == 10
    one, two = str(assembly["dir"] / "p1"), str(assembly["dir"] / "p2")
    assert cli.main(_polish_argv(assembly, one, "--fastq")) == 0
    assert cli.main(_polish_argv(assembly, two, "--fastq", "-g", "-d_ids", "0,1")) == 0
    assert multiprocessing.active_children() == []
    assert _raw(one) == _raw(two)
