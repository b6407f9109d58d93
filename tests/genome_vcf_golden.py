"""Shared by the genome VCF tests: the reference-written golden of tests/golden/make_golden_genome_vcf.py, the product's inputs
built from it, and a parser that reads a written .vcf.gz back into comparable records."""
import gzip
import json
import os

import numpy as np

GOLD = os.path.join(os.path.dirname(__file__), "golden", "genome_vcf_seed29.npz")
SELECT_KEYS = ("snp_p_value", "insert_p_value", "delete_p_value", "snp_p_value_in_lc", "insert_p_value_in_lc", "delete_p_value_in_lc",
               "report_snp_above_freq", "report_indel_above_freq")


def load():
    """-> dict: options, names (FASTA order), genomes, the records in arrival order (contig id, positions, keys uint8 [n,64],
    depths, freqs, probs float32), one region per contig over the concatenated genomes, the written lines per file, the header
    contigs and the reference's totals."""
    from pepper_b200 import synth
    z = np.load(GOLD)
    names = [str(c) for c in z["fasta"]]
    genomes = [str(g) for g in z["genomes"]]
    n = len(z["positions"])
    keys = np.zeros((n, 64), np.uint8)
    for i, k in enumerate(z["keys"]):
        b = str(k).encode(); keys[i, :len(b)] = np.frombuffer(b, np.uint8)
    off = np.concatenate([[0], np.cumsum([len(g) for g in genomes])])
    tab = np.array([[0, len(g) - 1, 0, len(g) - 1, off[k], len(g), 0, 0] for k, g in enumerate(genomes)], np.int64)
    regions = synth.RegionTable(tab, np.frombuffer("".join(genomes).encode(), np.uint8).copy())
    contig = np.array([names.index(str(c)) for c in z["contigs"]], np.int32)
    written = {}
    for w in z["written"]:
        f, r = json.loads(str(w))
        written.setdefault(f, []).append(r)
    options = json.loads(str(z["options"]))
    return dict(options=options, select={k: options[k] for k in SELECT_KEYS}, names=names, genomes=genomes, contig=contig,
                positions=np.asarray(z["positions"], np.int64), keys=keys, key_str=[str(k) for k in z["keys"]],
                depths=np.asarray(z["depths"], np.uint8), freqs=np.asarray(z["freqs"], np.uint8),
                probs=np.asarray(z["probs"], np.float32), regions=regions, written=written,
                header_contigs=[tuple(x) for x in json.loads(str(z["header_contigs"]))], counts=tuple(int(x) for x in z["counts"]))


def _f32(text: str):
    return [np.float32(x) for x in text.split(",")]


def record_of_line(line: str) -> dict:
    f = line.split("\t")
    fmt = dict(zip(f[8].split(":"), f[9].split(":")))
    return dict(contig=f[0], start=int(f[1]) - 1, alleles=[f[3]] + f[4].split(","), qual=int(f[5]), filter=f[6],
                GT=[int(x) for x in fmt["GT"].split("/")], AP=_f32(fmt["AP"]), GQ=int(fmt["GQ"]), DP=int(fmt["DP"]),
                AD=[int(x) for x in fmt["AD"].split(",")], VAF=_f32(fmt["VAF"]), REP=fmt["REP"])


def record_of_golden(r: dict) -> dict:
    """The golden's new_record keywords as they come back from the file: floats through pysam's float32 "%g"."""
    return dict(contig=r["contig"], start=r["start"], alleles=list(r["alleles"]), qual=int(r["qual"]), filter=r["filter"], GT=list(r["GT"]),
                AP=[np.float32("%.6g" % np.float32(x)) for x in r["AP"]], GQ=int(r["GQ"]), DP=int(r["DP"]), AD=list(r["AD"]),
                VAF=[np.float32("%.6g" % np.float32(x)) for x in r["VAF"]], REP=r["REP"])


def read_vcf(path: str):
    """-> (header contigs [(name, length)], #CHROM line, records)"""
    text = gzip.decompress(open(path, "rb").read()).decode()
    contigs, chrom, recs = [], None, []
    for line in text.splitlines():
        if line.startswith("##contig=<ID="):
            body = line[len("##contig=<"):-1]
            kv = dict(x.split("=", 1) for x in body.split(","))
            contigs.append((kv["ID"], int(kv["length"])))
        elif line.startswith("#CHROM"):
            chrom = line
        elif not line.startswith("#"):
            recs.append(record_of_line(line))
    return contigs, chrom, recs


def check_against_golden(out_dir: str, g: dict, totals) -> None:
    from pepper_b200.vcf import VCF_FILES
    assert tuple(totals) == g["counts"]
    for name in VCF_FILES:
        contigs, chrom, recs = read_vcf(os.path.join(out_dir, name + ".vcf.gz"))
        assert contigs == g["header_contigs"], name
        assert chrom.split("\t")[-1] == "sample_b200"
        want = [record_of_golden(r) for r in g["written"].get(name, [])]
        assert len(recs) == len(want), name
        for a, b in zip(recs, want):
            assert a == b, (name, a, b)
