"""The command lines without a GPU (pepper_b200.cli, presets, exclude).

1. The call_variant and polish parsers have every option of the reference's (strings, dest, default, type, action, required:
   tests/golden/cli_contract.json, written by make_golden_cli.py from the reference's builders); polish adds --fastq only.
2. Each preset resolves an all-default command line to the reference's values; explicit flags win over a preset; zero or two
   presets are refused.
3. The r9 guppy5 preset maps to exactly synth.ont_params(), candidates.ONT_OPTIONS, vcf.VCF_OPTIONS_ONT and min_mapq 5;
   --hifi to synth.hifi_params().
4. The contig exclusion rule excludes every name of the reference's list (tests/golden/excluded_contigs.txt) and no primary
   chromosome (UCSC, Ensembl, GenBank or RefSeq naming) or synthetic contig name.
5. Missing BAM, index, FASTA or model, -t 0, -hp and a checkpoint of the wrong shape each exit 1 with a one-line message;
   a reference-format checkpoint with DataParallel names loads; polish -r with a contig given twice is refused.
6. The flags that have no effect are reported whenever argparse set them, abbreviated or with an attached value included."""
import argparse
import json
import os

import pytest
import torch

from pepper_b200 import cli, presets
from pepper_b200.exclude import is_excluded_contig

HERE = os.path.dirname(os.path.abspath(__file__))
with open(os.path.join(HERE, "golden", "cli_contract.json")) as _f:
    GOLD = json.load(_f)


def _sub(command: str) -> argparse.ArgumentParser:
    p = cli.build_parser()
    return next(a for a in p._actions if isinstance(a, argparse._SubParsersAction)).choices[command]


def _options(p) -> dict:
    return {a.dest + ":" + ",".join(a.option_strings): dict(option_strings=list(a.option_strings), dest=a.dest, default=a.default,
                                                            type=a.type.__name__ if a.type is not None else None,
                                                            action=type(a).__name__, required=bool(a.required))
            for a in p._actions if not isinstance(a, argparse._HelpAction)}


@pytest.mark.parametrize("command,extra", [("call_variant", set()), ("polish", {"fastq:--fastq"})])
def test_parser_matches_reference(command, extra):
    want = {o["dest"] + ":" + ",".join(o["option_strings"]): o for o in GOLD[command]["options"]}
    got = _options(_sub(command))
    assert set(got) - set(want) == extra
    for k, o in want.items():
        assert got.get(k) == o, k


def _parse(argv):
    return cli.build_parser().parse_args(["call_variant"] + GOLD["call_variant"]["required_argv"] + argv)


@pytest.mark.parametrize("preset", presets.PRESETS)
def test_preset_resolves_like_reference(preset):
    ns = cli.resolve(_parse(["--" + preset]))
    got = {k: v for k, v in vars(ns).items() if k not in ("sub_command", "preset")}
    assert got == GOLD["call_variant"]["presets"][preset]
    assert ns.preset == preset
    assert all(type(got[k]) is type(v) or {type(got[k]), type(v)} <= {int, float} for k, v in GOLD["call_variant"]["presets"][preset].items())


def test_explicit_flags_override_preset():
    ns = cli.resolve(_parse(["--clr", "--min_mapq", "0", "--snp_p_value", "0.5", "--allowed_multiallelics", "2",
                             "--min_snp_baseq", "7"]))
    assert (ns.min_mapq, ns.snp_p_value, ns.allowed_multiallelics, ns.min_snp_baseq) == (0, 0.5, 2, 7)
    assert ns.insert_p_value == 0.2 and ns.skip_indels is True
    ns = cli.resolve(_parse(["--hifi", "--skip_indels"]))
    assert ns.skip_indels is True and ns.min_snp_baseq == 10


@pytest.mark.parametrize("flags", [[], ["--hifi", "--clr"], ["--ont_r10_q20", "--ont_r9_guppy5_sup"]])
def test_zero_or_two_presets_are_refused(flags, capsys):
    with pytest.raises(SystemExit) as ei:
        _parse(flags)
    assert ei.value.code == 2
    assert "--ont_r9_guppy5_sup" in capsys.readouterr().err


def test_r9_guppy5_and_hifi_map_to_the_existing_tables():
    from pepper_b200.candidates import ONT_OPTIONS
    from pepper_b200.synth import hifi_params, ont_params
    from pepper_b200.vcf import VCF_OPTIONS_ONT
    o = vars(cli.resolve(_parse(["--ont_r9_guppy5_sup"])))
    assert presets.image_params(o) == ont_params()
    assert presets.candidate_options(o) == ONT_OPTIONS
    assert presets.vcf_options(o) == VCF_OPTIONS_ONT
    assert presets.read_filters(o) == dict(min_mapq=5, include_supplementary=False, downsample_rate=1.0)
    h = vars(cli.resolve(_parse(["--hifi"])))
    assert presets.image_params(h) == hifi_params()
    assert presets.read_filters(h)["min_mapq"] == 5
    assert presets.read_filters(vars(cli.resolve(_parse(["--ont_r10_q20"]))))["min_mapq"] == 1
    assert presets.image_params(vars(cli.resolve(_parse(["--clr"]))))["skip_indels"] == 1


def test_exclusion_rule_against_reference_list():
    with open(os.path.join(HERE, "golden", "excluded_contigs.txt")) as f:
        names = f.read().split()
    assert len(names) > 3000
    assert [n for n in names if not is_excluded_contig(n)] == []
    # primary chromosomes of both namings, and the contig names the synthetic BAM / FASTA files of the tests use
    kept = (["chr%d" % i for i in range(1, 23)] + ["chrX", "chrY", "chrM"] + [str(i) for i in range(1, 23)] + ["X", "Y", "MT"]
            + ["ctg", "ctg1", "ctg2", "ctg10", "ctgA", "ctgB", "chrA", "chrB", "chrEmpty", "c", "long", "short", "tiny", "M",
               "bamonly", "faonly", "chr3", "tig00000001", "contig_12"]
            # GRCh38 chromosomes in GenBank and RefSeq naming, and accessions outside the GRC scaffold prefixes
            + ["CM000663.2", "CM000686.2", "J01415.2", "NC_000001.11", "NC_012920.1", "CP000001.1"])
    assert [n for n in kept if is_excluded_contig(n)] == []


# ------------------------------------------------------------------------------------------------------------ errors
@pytest.fixture
def files(tmp_path):
    from pepper_b200 import weights
    p = {k: str(tmp_path / n) for k, n in (("bam", "r.bam"), ("fa", "r.fa"), ("model", "m.pkl"))}
    for path in (p["bam"], p["bam"] + ".bai", p["fa"], p["fa"] + ".fai"):
        open(path, "wb").close()
    torch.save({"model_state_dict": {k: torch.from_numpy(v) for k, v in weights.random_variant_state(0).items()}}, p["model"])
    p["out"] = str(tmp_path / "out")
    return p


def _cv(p, *extra):
    return ["call_variant", "-b", p["bam"], "-f", p["fa"], "-m", p["model"], "-o", p["out"], "-s", "S", "-t", "2",
            "--ont_r9_guppy5_sup"] + list(extra)


def _error_line(capsys) -> str:
    err = [ln for ln in capsys.readouterr().err.splitlines() if "ERROR" in ln]
    assert len(err) == 1, err
    assert "Traceback" not in err[0]
    return err[0]


@pytest.mark.parametrize("what,message", [("bam", "CAN NOT LOCATE BAM FILE"), ("bai", "CAN NOT LOCATE BAM INDEX"),
                                          ("fa", "CAN NOT LOCATE FASTA FILE"), ("model", "CAN NOT LOCATE MODEL FILE")])
def test_missing_input_exits_1(files, capsys, what, message):
    os.remove(files["bam"] + ".bai" if what == "bai" else files[what])
    assert cli.main(_cv(files)) == 1
    line = _error_line(capsys)
    assert message in line and "] ERROR: " in line


def test_threads_hp_and_polish_checks_exit_1(files, capsys):
    argv = _cv(files)
    argv[argv.index("-t") + 1] = "0"
    assert cli.main(argv) == 1
    assert "THREAD NEEDS TO BE >0" in _error_line(capsys)
    assert cli.main(_cv(files, "-hp")) == 1
    assert "use_hp_info IS NOT SUPPORTED" in _error_line(capsys)
    os.remove(files["fa"])
    assert cli.main(["polish", "-b", files["bam"], "-f", files["fa"], "-m", files["model"], "-o", files["out"]]) == 1
    assert "CAN NOT LOCATE FASTA FILE" in _error_line(capsys)


def test_wrong_checkpoint_exits_1_naming_the_tensor(files, capsys):
    from pepper_b200 import weights
    sd = weights.random_variant_state(0)
    sd["encoder.weight_ih_l0"] = sd["encoder.weight_ih_l0"][:, :1].repeat(48, 1)     # a 48-feature (HP) encoder
    torch.save({"model_state_dict": {k: torch.from_numpy(v) for k, v in sd.items()}}, files["model"])
    assert cli.main(_cv(files)) == 1
    line = _error_line(capsys)
    assert "encoder.weight_ih_l0" in line and "[1024, 48]" in line and "[1024, 26]" in line
    # a polish model given to call_variant
    torch.save({"model_state_dict": {k: torch.from_numpy(v) for k, v in weights.random_polish_state(0).items()}}, files["model"])
    assert cli.main(_cv(files)) == 1
    assert "IS NOT A PEPPER VARIANT MODEL" in _error_line(capsys)


def test_reference_checkpoint_with_module_prefix_loads(tmp_path):
    from pepper_b200 import weights
    sd = weights.random_variant_state(3)
    path = str(tmp_path / "m.pkl")
    torch.save({"model_state_dict": {"module." + k: torch.from_numpy(v) for k, v in sd.items()}, "epochs": 10}, path)
    got = cli.load_model(path, "variant")
    assert set(got) == set(sd)
    assert all(torch.equal(got[k], torch.from_numpy(v)) for k, v in sd.items())
    psd = weights.random_polish_state(1)
    torch.save({"model_state_dict": {"module." + k: torch.from_numpy(v) for k, v in psd.items()}}, path)
    assert set(cli.load_model(path, "polish")) == set(psd)


def test_no_effect_flags_are_reported():
    p = cli.build_parser()
    argv = ["call_variant", "-b", "x", "-f", "x", "-m", "x", "-o", "x", "-s", "x", "-t", "1", "--hifi"]
    assert cli.no_effect_flags(p, p.parse_args(argv)) == []
    for extra, dest in ((["-bs=64"], "batch_size"), (["--batch", "64"], "batch_size"), (["-w=2"], "num_workers"),
                        (["--quantized"], "quantized"), (["-rb", "r.bed"], "region_bed"), (["-per_gpu", "2"], "callers_per_gpu")):
        assert cli.no_effect_flags(p, p.parse_args(argv + extra)) == [dest], extra
    polish = ["polish", "-b", "x", "-f", "x", "-m", "x", "-o", "x"]
    assert cli.no_effect_flags(p, p.parse_args(polish)) == []
    assert cli.no_effect_flags(p, p.parse_args(polish + ["-w", "0", "-bs", "7"])) == ["batch_size", "num_workers"]


def test_polish_region_checks(files, capsys):
    base = ["polish", "-b", files["bam"], "-f", files["fa"], "-m", files["model"], "-o", files["out"], "-r"]
    assert cli.main(base + ["ctg1:0-1000,ctg1:5000-6000"]) == 1
    assert "CONTIG ctg1 IS GIVEN MORE THAN ONCE" in _error_line(capsys)
    assert cli.main(base + ["ctg1:5-1"]) == 1
    assert "--region: invalid value" in _error_line(capsys)
    ns = cli.build_parser().parse_args(base + ["ctg2,ctg1:10-20"])
    assert cli.polish_contigs(ns) == [("ctg2", None), ("ctg1", (10, 20))]


def test_polish_output_path_follows_reference():
    assert cli.polish_output("out/asm") + "_pepper_polished.fa" == "out/asm/_pepper_polished.fa"
    assert cli.polish_output("out/") == "out/"


class _Source:
    def __init__(self, log):
        self.log, self.closed = log, False
        log.append(self)

    def close(self):
        self.closed = True


def test_capacity_restarts_only_on_one_gpu(capsys):
    from pepper_b200._lib import PepperB200Error
    from pepper_b200.abi import PB_ERR_CAPACITY
    opened, caps = [], []

    def run(src, cap):
        caps.append(cap)
        if cap < 400:
            raise PepperB200Error("only 1 of 2 groups were run", PB_ERR_CAPACITY)
        return "done"
    # one GPU: a fresh source per attempt, twice the room each time, every source closed
    assert cli.run_restarting(lambda: _Source(opened), run, lambda src: 100, 1, "CANDIDATE") == "done"
    assert caps == [100, 200, 400] and len(opened) == 3 and all(s.closed for s in opened)
    assert capsys.readouterr().err.count("THE CANDIDATE CAPACITY (") == 2
    # several GPUs: no restart, a one-line error
    opened.clear(); caps.clear()
    with pytest.raises(cli.CliError, match="EXHAUSTED ON 2 GPUS"):
        cli.run_restarting(lambda: _Source(opened), run, lambda src: 100, 2, "CANDIDATE")
    assert caps == [100] and len(opened) == 1 and opened[0].closed

    def fail(src, cap):
        raise PepperB200Error("corrupt block", 3)
    with pytest.raises(PepperB200Error, match="corrupt"):
        cli.run_restarting(lambda: _Source(opened), fail, lambda src: 100, 1, "CANDIDATE")
