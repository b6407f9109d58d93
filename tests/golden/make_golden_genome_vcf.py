"""Pins the whole-genome VCF writer against the UNMODIFIED reference `find_candidates` (CandidateFinder.py:532-581) +
`VCFWriter` (VcfWriter.py:13-289) over several contigs, run with the stand-ins of make_golden_vcf.py: a fake h5py whose batches
carry each record's contig, a PEPPER_VARIANT whose FASTA_handler serves five contigs, and a pysam whose VariantHeader records the
declared contigs and whose VariantFile records every write and the file it went to.
    python tests/golden/make_golden_genome_vcf.py
Cases: FASTA order chr1, chr2, chr3, chr10, chrX (natural != lexical); chr2 has records of which none is selected, chr3 has none;
chr1's last site and chr10's first site share a position (the reference's `last_position` skip across contigs); multi-allelic
sites above allowed_multiallelics, deletions of several lengths at one site, het / hom-alt ties, batch-boundary duplicates."""
import json
import os
import sys
import types
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
L = 3000
P_SHARED = 1600
FASTA = ["chr1", "chr2", "chr3", "chr10", "chrX"]
rng = np.random.default_rng(29)
genomes = {c: "".join("ACGT"[i] for i in rng.integers(0, 4, L)) for c in FASTA}
genomes["chr1"] = genomes["chr1"][:400] + "AAAAAAAAA" + genomes["chr1"][409:]
genomes["chrX"] = genomes["chrX"][:700] + "TTTTTTT" + genomes["chrX"][707:]


def contig_records(c, lo, hi, n_pos):
    g = genomes[c]
    recs = []
    for p in np.sort(rng.choice(np.arange(lo, hi), size=n_pos, replace=False)):
        for _ in range(int(rng.choice([1, 1, 1, 2, 3, 5]))):
            t = int(rng.integers(1, 4))
            if c == "chr2":
                t = 1
            if t == 1:
                key = "1" + "ACGT"[rng.integers(0, 4)]
            elif t == 2:
                key = "2" + g[p] + "".join("ACGT"[i] for i in rng.integers(0, 4, rng.integers(1, 5)))
            else:
                key = "3" + g[p:p + int(rng.integers(2, 7))]
            d = int(rng.integers(4, 60))
            pr = rng.dirichlet([0.5, 0.6, 0.5])
            if rng.random() < 0.15:
                pr = np.array([0.2, 0.4, 0.4])              # ties between het and hom
            if c == "chr2":
                pr = np.array([0.95, 0.03, 0.02])            # never selected: every p-value rule fails, SNP frequency rule off
            recs.append((c, int(p), key, d, int(rng.integers(1, d + 1)), pr.astype(np.float32).astype(np.float64)))
    return recs


def forced(c, p):
    base = genomes[c][p]
    alt = "C" if base != "C" else "G"
    return (c, p, "1" + alt, 30, 20, np.array([0.05, 0.9, 0.05], np.float32).astype(np.float64))


per_contig = {"chr1": contig_records("chr1", 5, P_SHARED - 5, 90) + [forced("chr1", P_SHARED)],
              "chr2": contig_records("chr2", 5, L - 12, 30),
              "chr10": [forced("chr10", P_SHARED)] + contig_records("chr10", P_SHARED + 5, L - 12, 70),
              "chrX": contig_records("chrX", 5, L - 12, 90)}
batches = []
for c in ("chrX", "chr10", "chr1", "chr2"):                  # the prediction files come in any contig order
    recs = sorted(per_contig[c], key=lambda r: r[1])
    nb = 3
    cuts = [len(recs) * i // nb for i in range(nb + 1)]
    for b in range(nb):
        part = recs[cuts[b]:cuts[b + 1]]
        if b + 1 < nb:
            part = part + recs[cuts[b + 1]:cuts[b + 1] + 6]  # the next batch's first records again: duplicates
        batches.append(part)
options = dict(snp_p_value=0.1, insert_p_value=0.1, delete_p_value=0.1, snp_p_value_in_lc=0.3, insert_p_value_in_lc=0.35,
               delete_p_value_in_lc=0.25, report_snp_above_freq=0.0, report_indel_above_freq=0.6,
               allowed_multiallelics=3, snp_q_cutoff=15, indel_q_cutoff=10, snp_q_cutoff_in_lc=20, indel_q_cutoff_in_lc=12,
               threads=1)                                    # one worker chunk: the reference's arrival order is deterministic


class _L:
    def __init__(self, a):
        self.a = a

    def __getitem__(self, k):
        return self.a


def _batch_group(part):
    n = len(part)
    obj = np.empty((n, 1), dtype=object)
    for i, r in enumerate(part):
        obj[i, 0] = r[2]
    return {"contigs": _L(np.array([r[0].encode() for r in part])), "positions": _L(np.array([r[1] for r in part])),
            "depths": _L(np.array([r[3] for r in part])), "candidates": _L(obj),
            "candidate_frequency": _L(np.array([r[4] for r in part]).reshape(n, 1)), "base_prediction": _L(np.stack([r[5] for r in part]))}


class FakeH5:
    def __init__(self, name, mode="r"):
        self.d = {"predictions": {"batch_%d" % b: _batch_group(p) for b, p in enumerate(batches)}}

    def keys(self):
        return self.d.keys()

    def __getitem__(self, k):
        return self.d[k]

    def __enter__(self):
        return self

    def __exit__(self, *a):
        pass


class FASTA_handler:
    def __init__(self, path):
        pass

    def get_reference_sequence(self, contig, a, b):
        return genomes[contig][max(0, a):max(0, b)]

    def get_chromosome_names(self):
        return list(FASTA)

    def get_chromosome_sequence_length(self, c):
        return len(genomes[c])


class CandidateImagePrediction:
    def __init__(self, contig, position, depth, candidates, candidate_frequency, prediction_base, prediction_type):
        self.contig, self.position, self.depth = contig, position, depth
        self.candidates, self.candidate_frequency = candidates, candidate_frequency
        self.prediction_base, self.prediction_type = prediction_base, prediction_type


WRITTEN, HEADER_CONTIGS = [], []


class _Contigs:
    def add(self, name, length=None):
        HEADER_CONTIGS.append((name, length))


class _Header:
    def __init__(self):
        self.contigs = _Contigs()

    def add_meta(self, **kw):
        pass

    def add_sample(self, s):
        pass


class _VariantFile:
    def __init__(self, name, mode, header=None):
        self.name = os.path.basename(name)

    def new_record(self, **kw):
        return dict(kw)

    def write(self, rec):
        WRITTEN.append((self.name, rec))

    def close(self):
        pass


h5 = types.ModuleType("h5py"); h5.File = FakeH5
pv = types.ModuleType("pepper_variant.build.PEPPER_VARIANT")
pv.FASTA_handler = FASTA_handler; pv.CandidateImagePrediction = CandidateImagePrediction
build = types.ModuleType("pepper_variant.build"); build.PEPPER_VARIANT = pv
ps = types.ModuleType("pysam"); ps.VariantFile = _VariantFile; ps.VariantHeader = _Header; ps.tabix_index = lambda *a, **k: None
sys.modules.update({"h5py": h5, "pepper_variant.build": build, "pepper_variant.build.PEPPER_VARIANT": pv, "pysam": ps})
sys.path.insert(0, os.environ.get("PEPPER_REFERENCE", "/root/reference"))
from pepper_variant.modules.python import CandidateFinder as RefCF  # noqa: E402
from pepper_variant.modules.python import VcfWriter as RefVW  # noqa: E402

opt = types.SimpleNamespace(fasta="x", **options)
contigs, sites_phasing, sites_vc = RefCF.find_candidates(opt, "dir", [("f", "batch_%d" % b) for b in range(len(batches))])
w = RefVW.VCFWriter(contigs, "x", "sample", "out/", "PEPPER_VARIANT_FULL", "PEPPER_VARIANT_OUTPUT_PEPPER",
                    "PEPPER_VARIANT_OUTPUT_VARIANT_CALLING")
counts = w.write_vcf_records(sites_vc, opt)


def norm(o):
    if isinstance(o, dict):
        return {k: norm(v) for k, v in sorted(o.items())}
    if isinstance(o, (list, tuple)):
        return [norm(x) for x in o]
    if isinstance(o, (np.floating, float)):
        return float(o)
    if isinstance(o, np.integer):
        return int(o)
    if isinstance(o, (np.bool_, bool)):
        return bool(o)
    return o


written = [json.dumps([f[:-len(".vcf.gz")], norm(r)]) for f, r in WRITTEN]
recs = [r for b in batches for r in b]
chroms = [r["contig"] for f, r in WRITTEN if f.startswith("PEPPER_VARIANT_FULL")]
assert list(dict.fromkeys(chroms)) == ["chr1", "chr10", "chrX"], chroms
assert sum(1 for f, r in WRITTEN if f.startswith("PEPPER_VARIANT_FULL") and r["contig"] == "chr10" and r["start"] == P_SHARED) == 0
assert any(len(r["alleles"]) > 2 for _, r in WRITTEN)
np.savez_compressed(os.path.join(HERE, "genome_vcf_seed29.npz"), options=np.array(json.dumps(options)),
                    fasta=np.array(FASTA), genomes=np.array([genomes[c] for c in FASTA]),
                    batch_sizes=np.array([len(b) for b in batches]), contigs=np.array([r[0] for r in recs]),
                    positions=np.array([r[1] for r in recs]), keys=np.array([r[2] for r in recs]), depths=np.array([r[3] for r in recs]),
                    freqs=np.array([r[4] for r in recs]), probs=np.stack([r[5] for r in recs]), written=np.array(written),
                    header_contigs=np.array(json.dumps(HEADER_CONTIGS)), counts=np.array(counts))
print("genome vcf pinned: %d records in %d batches -> %d lines written to 5 files, totals %s" % (len(recs), len(batches), len(written), counts))
