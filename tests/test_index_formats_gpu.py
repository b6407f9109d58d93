"""GPU: CSI-indexed BAMs and bgzip-compressed FASTA through the whole-genome paths, and positions past 2^29.

1. fetch_device equals fetch on CSI-indexed files (depths 5 and 6, min_shift 12), a contig past 2^29 included.
2. (BAM + CSI, .fa.gz) and (BAM + BAI, .fa) of the same records and reference give the same call_genome files, totals and
   .tbi bytes, the same DistributedGenomeCaller files (world size 1, not distributed) and the same polished assembly.
3. Shift test: one reference and one read set placed at offset 100,000 of a short contig and at an offset X >= 2^29 (a multiple of
   the 100 kb interval) of a long, bgzipped, CSI-indexed contig.  call_genome over the two windows gives the same VCF lines once
   POS is shifted by X - 100,000 and the contig renamed, the long contig's VCFs carry .csi indexes, and polish_contig over the
   two windows returns the same sequence."""
import gzip
import os

import numpy as np
import pytest

from pepper_b200 import synth, synth_files

pytestmark = pytest.mark.gpu

FIELDS = ("pos", "seq_off", "cigar_off", "flag", "mapq", "seq", "qual", "cigar")
VCF_OPTS = dict(allowed_multiallelics=1, snp_q_cutoff=20, indel_q_cutoff=15, snp_q_cutoff_in_lc=20, indel_q_cutoff_in_lc=10)
X = 540_000_000                       # >= 2^29, a multiple of the 100 kb interval and of the 60-base FASTA line


def _shift(rec, by):
    return synth.RecordBatch(rec.pos + by, rec.seq_off, rec.cigar_off, rec.flag, rec.mapq, rec.seq, rec.qual, rec.cigar)


@pytest.fixture(scope="module")
def long_files(tmp_path_factory):
    """One BAM (CSI, depth 6) with a short and a long contig carrying the same reads at offsets 100,000 and X; a bgzipped FASTA
    whose contigs are N up to the offset, then the same sequence."""
    d = tmp_path_factory.mktemp("long")
    rec, genome = synth.simulate_contig_records(300_000, 20, synth.ONT, 81)
    n_line = np.frombuffer(b"N" * 60, np.uint8)
    contigs = [("short", 100_000 + genome.shape[0]), ("long", X + genome.shape[0])]
    bam, fa = str(d / "l.bam"), str(d / "l.fa.gz")
    synth_files.write_bam(bam, contigs, {0: _shift(rec, 100_000), 1: _shift(rec, X)}, index="csi")
    synth_files.write_fasta(fa, [("short", [(n_line, 100_000 // 60), (n_line[:100_000 % 60], 1), (genome, 1)]),
                                 ("long", [(n_line, X // 60), (genome, 1)])], bgzip=True)
    assert os.path.getsize(fa) < 4 << 20
    return dict(bam=bam, fa=fa, dir=d, n=genome.shape[0], rec=rec)


def test_fetch_device_equals_fetch_on_csi(long_files, tmp_path):
    from pepper_b200.bamio import BamReader
    rec0, _ = synth.simulate_contig_records(200_000, 10, synth.ONT, 11, contig_start=3000)
    paths = [long_files["bam"]]
    for tag, kw in [("c5", dict(index="csi")), ("c12", dict(index="csi", csi_min_shift=12, csi_depth=6))]:
        p = str(tmp_path / f"{tag}.bam")
        synth_files.write_bam(p, [("chrA", 210_000)], {0: rec0}, block_payload=20_000, **kw)
        paths.append(p)
    rng = np.random.default_rng(6)
    for p in paths:
        r = BamReader(p, 4)
        assert r.index_info()["format"] == "csi"
        for name, length in r.get_chromosome_sequence_names_with_length():
            lo = length - (long_files["n"] if p == long_files["bam"] else 200_000)
            qs = [(0, length), (lo, lo + 1), (length - 10, length + 10)] + \
                 [(int(b), int(b) + int(rng.choice([1, 3000, 40_000, 200_000]))) for b in rng.integers(lo, length, 12)]
            for beg, end in qs:
                want = r.fetch(name, beg, end).to_batch()
                got = r.fetch_device(name, beg, end).to_batch()
                for f in FIELDS:
                    assert np.array_equal(getattr(got, f), getattr(want, f)), (p, name, beg, end, f)
                anchors, walk = r.fetch_device_anchors()
                assert (anchors > 0 and walk > 0) or want.n_records == 0
        r.close()
    r = BamReader(long_files["bam"], 4)
    got = r.fetch_device("long", 0, X + long_files["n"]).to_batch()
    assert np.array_equal(got.pos, long_files["rec"].pos + X)


@pytest.fixture(scope="module")
def pair(tmp_path_factory):
    """The same records and reference written twice: (BAM + CSI, .fa.gz) and (BAM + BAI, .fa)."""
    d = tmp_path_factory.mktemp("pair")
    recs, fasta = {}, []
    for tid, (c, n, seed) in enumerate([("chr1", 230_000, 91), ("chr2", 120_000, 92), ("chr10", 90_000, 93)]):
        rec, genome = synth.simulate_contig_records(n, 20, synth.ONT, seed)
        recs[tid] = rec
        fasta.append((c, genome))
    out = {}
    for tag, idx, gz in (("new", "csi", True), ("old", "bai", False)):
        bam, fa = str(d / f"{tag}.bam"), str(d / (f"{tag}.fa" + (".gz" if gz else "")))
        synth_files.write_bam(bam, [(c, g.shape[0]) for c, g in fasta], recs, index=idx)
        synth_files.write_fasta(fa, fasta, bgzip=gz, block_lines=50)
        out[tag] = (bam, fa)
    return dict(d=d, **out)


def _files(d):
    from pepper_b200.vcf import VCF_FILES
    return [gzip.decompress(open(os.path.join(d, n + ".vcf.gz"), "rb").read()) for n in VCF_FILES]


def _tbis(d):
    from pepper_b200.vcf import VCF_FILES
    return [open(os.path.join(d, n + ".vcf.gz.tbi"), "rb").read() for n in VCF_FILES]


def test_csi_and_bgzip_inputs_give_the_same_outputs(pair):
    from oracle import nets
    from pepper_b200 import weights
    from pepper_b200.dist import DistributedGenomeCaller
    from pepper_b200.frontend import PolishFromFiles, VariantFromFiles
    state = nets.make_variant_weights(0)
    d = pair["d"]
    res = {}
    for tag in ("new", "old"):
        bam, fa = pair[tag]
        with VariantFromFiles(bam, fa, state) as vf:
            totals = vf.call_genome(str(d / f"one_{tag}"), "s", vcf_options=VCF_OPTS, batch=2)
            dgc = DistributedGenomeCaller(None, 0, 1 << 26, "static", group_regions=2, distributed=False, caller=vf.caller)
            dtot = dgc.call_genome(bam, fa, str(d / f"dist_{tag}"), "s", vcf_options=VCF_OPTS)
        with PolishFromFiles(bam, fa, weights.random_polish_state(1)) as pf:
            seqs = pf.polish_assembly()
        res[tag] = (totals, _files(d / f"one_{tag}"), _tbis(d / f"one_{tag}"), dtot, _files(d / f"dist_{tag}"), seqs)
    new, old = res["new"], res["old"]
    assert new[0] == old[0] and new[0][0] > 0
    assert new[1] == old[1] and new[2] == old[2]
    assert new[3] == old[3] == old[0] and new[4] == old[4] == old[1]
    assert new[5] == old[5] and sum(len(s) for s in old[5].values()) > 400_000


def _body(text: bytes, contig: str, shift: int) -> list[bytes]:
    out = []
    for line in text.split(b"\n"):
        if not line or line.startswith(b"#"):
            continue
        f = line.split(b"\t")
        assert f[0] == contig.encode()
        f[0] = b"C"
        f[1] = b"%d" % (int(f[1]) - shift)
        out.append(b"\t".join(f))
    return out


def test_positions_past_2_29_shift(long_files):
    from oracle import nets
    from pepper_b200 import weights
    from pepper_b200.frontend import PolishFromFiles, VariantFromFiles
    from pepper_b200.vcf import VCF_FILES
    bam, fa, d, n = long_files["bam"], long_files["fa"], long_files["dir"], long_files["n"]
    wins = {"short": 100_000, "long": X}
    got = {}
    with VariantFromFiles(bam, fa, nets.make_variant_weights(0)) as vf:
        for c, off in wins.items():
            out = str(d / f"vcf_{c}")
            got[c] = vf.call_genome(out, "s", region=f"{c}:{off}-{off + n - 1}", vcf_options=VCF_OPTS, batch=2), _files(out)
            ext = ".csi" if c == "long" else ".tbi"
            for name in VCF_FILES:
                assert os.path.exists(os.path.join(out, name + ".vcf.gz" + ext))
    assert got["short"][0] == got["long"][0] and got["short"][0][0] > 0
    for a, b in zip(got["short"][1], got["long"][1]):
        assert _body(a, "short", 100_000) == _body(b, "long", X)
    with PolishFromFiles(bam, fa, weights.random_polish_state(1)) as pf:
        seqs = {c: pf.polish_contig(c, off, off + n - 1) for c, off in wins.items()}
    assert seqs["short"] == seqs["long"] and len(seqs["short"]) > 250_000
