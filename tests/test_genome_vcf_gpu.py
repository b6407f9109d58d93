"""GPU: VCF text on the device.

1. The device "%.6g" (pb_test_format_g) equals Python's "%.6g" % float(np.float32(x)) on every float32 in [0.5, 1), every power
   of two down to 2^-149, every float32 in [1e-10, 1] whose exact value is a 7-significant-digit tie, both sides of 1e-4 and
   1e-5, 0, 1 and 10^6 seeded random values.
2. pb_variant_vcf_host on the records pinned against the unmodified reference (tests/golden/vcf_seed23.npz) gives the bytes
   format_vcf_line prints for the reference's records.
3. The same records spread over three contigs and six regions, in scrambled order, give the host tail's lines
   (find_site_records + format_vcf_line) contig by contig.
4. The reference-written multi-contig golden (tests/golden/genome_vcf_seed29.npz) through pb_variant_vcf_host + the writer.
5. The device QUAL against Python's on every float32 probability where QUAL steps.
6. call_genome from a multi-contig BAM + FASTA (natural order != lexical order, a FASTA-only contig, several session groups per
   contig), on both inflate paths, writes five VCFs that decompress to the host tail's files."""
import gzip
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _format_g(x):
    import ctypes as C
    from pepper_b200 import _lib
    L = _lib.lib()
    L.pb_test_format_g.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
    x = np.ascontiguousarray(x, np.float32)
    out = np.zeros(x.shape[0], "S16")
    _lib.check(L.pb_test_format_g(x.ctypes.data, x.shape[0], out.ctypes.data), "pb_test_format_g")
    return out


def _ties():
    """float32 values in [1e-10, 1] whose exact decimal value has 7 significant digits, the last a 5: N / 10^q = t / 2^q with
    N = t * 5^q odd, 10^6 <= N < 10^7 (q <= 10, else N / 10^q is not a binary fraction)."""
    out = []
    for q in range(0, 11):
        f = 5 ** q
        t = np.arange(-(-10 ** 6 // f), -(-10 ** 7 // f), dtype=np.int64)
        t = t[((t * f) % 10 == 5)]
        v = t.astype(np.float64) / 2.0 ** q
        v = v[(v >= 1e-10) & (v <= 1.0)]
        out.append(v[v.astype(np.float32).astype(np.float64) == v])
    return np.unique(np.concatenate(out)).astype(np.float32)


def test_format_g_matches_python():
    rng = np.random.default_rng(7)
    half = np.arange(np.float32(0.5).view(np.uint32), np.float32(1.0).view(np.uint32), dtype=np.uint32).view(np.float32)
    pows = (np.float32(2.0) ** -np.arange(0, 150)).astype(np.float32)
    ties = _ties()
    assert ties.shape[0] > 50 and np.float32(2.0 ** -9) in ties
    edges = []
    for c in (1e-4, 1e-5):
        b = np.float32(c).view(np.uint32)
        edges.append((b + np.arange(-300, 300)).astype(np.uint32).view(np.float32))
    x = np.concatenate([half, pows, ties, *edges, np.array([0, 1], np.float32), rng.random(10 ** 6).astype(np.float32)])
    got = _format_g(x)
    want = np.array([("%.6g" % v).encode() for v in x.astype(np.float64).tolist()], "S16")
    bad = np.flatnonzero(got != want)
    assert bad.shape[0] == 0, [(float(x[i]), got[i], want[i]) for i in bad[:5]]
    assert _format_g(np.array([2.0 ** -9], np.float32))[0] == b"0.00195312"


def _golden():
    from pepper_b200 import synth
    g = np.load(os.path.join(GOLD, "vcf_seed23.npz"))
    genome = str(g["genome"])
    options = json.loads(str(g["options"]))
    n = len(g["positions"])
    keys = np.zeros((n, 64), np.uint8)
    for i, k in enumerate(g["keys"]):
        b = str(k).encode(); keys[i, :len(b)] = np.frombuffer(b, np.uint8)
    ref = np.frombuffer(genome.encode(), np.uint8).copy()
    regions = synth.RegionTable(np.array([[0, len(genome) - 1, 0, len(genome) - 1, 0, len(genome), 0, 0]], np.int64), ref)
    sel = {k: options[k] for k in ("snp_p_value", "insert_p_value", "delete_p_value", "snp_p_value_in_lc", "insert_p_value_in_lc",
                                   "delete_p_value_in_lc", "report_snp_above_freq", "report_indel_above_freq")}
    return g, genome, keys, regions, sel, options


def test_vcf_host_matches_reference_records():
    from pepper_b200.vcf import format_vcf_line, vcf_text_host
    g, genome, keys, regions, sel, options = _golden()
    want = [json.loads(r) for r in g["records"]]
    n = len(g["positions"])
    text, lines = vcf_text_host(["ctg"], [0], g["positions"], np.zeros(n, np.int32), g["depths"], g["freqs"], keys,
                                g["probs"].astype(np.float32), regions, sel, options)
    assert text.tobytes().decode() == "".join(format_vcf_line(r) + "\n" for r in want)
    assert lines.shape[0] == len(want) and (lines["pos"] == [r["start"] for r in want]).all()
    assert (lines["ref_len"] == [len(r["alleles"][0]) for r in want]).all()
    assert [int(c) for c in lines["cls"]] == [0 if "pepper" in r["files"] else 1 if "variant_calling_snp" in r["files"] else 2 for r in want]


def test_vcf_host_multi_contig_matches_host_tail():
    from pepper_b200 import synth
    from pepper_b200.vcf import find_site_records, host_tail_text, vcf_text_host
    g, genome, keys, regions, sel, options = _golden()
    n = len(g["positions"])
    pos = np.asarray(g["positions"], np.int64)
    L = len(genome)
    # contig k = the same genome; regions cut each contig in two, overlapping by one base like the reference's tiling
    names = ["chrB", "chrA", "chr10"]
    contig = np.arange(n) % 3
    rows, cor = [], []
    for k in range(3):
        for (a, b) in ((0, L // 2), (L // 2, L - 1)):
            rows.append([max(0, a - 100), min(L - 1, b + 100), a, b, max(0, a - 100), min(L - 1, b + 100) - max(0, a - 100) + 1, 0, 0])
            cor.append(k)
    tab = np.array(rows, np.int64)
    rof = (contig * 2 + (pos >= L // 2)).astype(np.int32)
    order = np.random.default_rng(3).permutation(n)
    regs = synth.RegionTable(tab, regions.ref)
    probs = g["probs"].astype(np.float32)
    pos, rof, dep, frq, keys, probs, contig = (a[order] for a in (pos, rof, g["depths"], g["freqs"], keys, probs, contig))
    text, lines = vcf_text_host(names, cor, pos, rof, dep, frq, keys, probs, regs, sel, options)
    for k, c in enumerate(names):
        m = contig == k                 # the host tail sees each contig's records in the same arrival order
        recs = find_site_records(c, pos[m], rof[m], dep[m], frq[m], keys[m], probs[m], regs, sel, options)
        want_text, want_lines = host_tail_text(recs, k)
        mine = lines[lines["contig"] == k]
        got = b"".join(text[o:o + l].tobytes() for o, l in zip(mine["text_off"], mine["text_len"]))
        assert got == want_text.tobytes(), c
        assert (mine["cls"] == want_lines["cls"]).all() and (mine["ref_len"] == want_lines["ref_len"]).all()


@pytest.fixture(scope="module")
def genome_files(tmp_path_factory):
    from pepper_b200 import synth, synth_files
    d = tmp_path_factory.mktemp("genome_vcf")
    contigs = [("chr2", 150_000, 31), ("chr10", 120_000, 32), ("chr1", 230_000, 33)]
    recs, fasta = {}, []
    for tid, (c, n, seed) in enumerate(contigs):
        rec, genome = synth.simulate_contig_records(n, 20, synth.ONT, seed)
        recs[tid] = rec
        fasta.append((c, genome))
    fasta.append(("chr3", synth.make_reference(5000, 34)))                  # in the FASTA only
    bam, fa = str(d / "g.bam"), str(d / "g.fa")
    synth_files.write_bam(bam, [(c, n) for c, n, _ in contigs], recs)
    synth_files.write_fasta(fa, fasta)
    return dict(bam=bam, fa=fa, dir=d)


def _host_tail(vf, out_dir, params, batch):
    from pepper_b200.candidates import ONT_OPTIONS
    from pepper_b200.frontend import variant_intervals
    from pepper_b200.vcf import find_site_records, host_tail_text, order_lines, write_vcfs
    job = vf.vcf_job()
    names = [c for c, _, _ in job]
    parts = []
    for cid, (c, s, e) in enumerate(job):
        iv = variant_intervals(s, e)
        calls = vf.call_stream(c, iv, params, batch)
        table = vf.genome_table(c, iv)
        recs = find_site_records(c, calls.positions, calls.region_of, calls.depths, calls.freqs, calls.keys_raw, calls.probs, table,
                                 ONT_OPTIONS)
        parts.append(host_tail_text(recs, cid))
    text, lines = order_lines(parts, names)
    return write_vcfs(out_dir, "sample_b200", vf.fasta_contigs(), names, text, lines)


@pytest.mark.parametrize("gpu_inflate", [True, False])
def test_call_genome_matches_host_tail(genome_files, gpu_inflate):
    from oracle import nets
    from pepper_b200 import synth
    from pepper_b200.frontend import VariantFromFiles, variant_intervals
    from pepper_b200.vcf import VCF_FILES
    state = nets.make_variant_weights(0)
    params = synth.ont_params()
    d = genome_files["dir"]
    tag = "gpu" if gpu_inflate else "host"
    with VariantFromFiles(genome_files["bam"], genome_files["fa"], state, gpu_inflate=gpu_inflate) as vf:
        assert [c for c, _, _ in vf.vcf_job()] == ["chr1", "chr2", "chr10"]
        assert len(variant_intervals(0, 229_999)) == 3
        got = vf.call_genome(str(d / ("dev_" + tag)), "sample_b200", params=params, batch=2)
        want = _host_tail(vf, str(d / ("host_" + tag)), params, 2)
    assert got == want and got[0] > 100 and got[1] > 0 and got[2] > 0
    for name in VCF_FILES:
        a = gzip.decompress(open(d / ("dev_" + tag) / (name + ".vcf.gz"), "rb").read())
        b = gzip.decompress(open(d / ("host_" + tag) / (name + ".vcf.gz"), "rb").read())
        assert a == b, name
    body = [l.split("\t")[0] for l in a.decode().splitlines() if not l.startswith("#")]
    full = gzip.decompress(open(d / ("dev_" + tag) / (VCF_FILES[0] + ".vcf.gz"), "rb").read()).decode()
    chroms = [l.split("\t")[0] for l in full.splitlines() if not l.startswith("#")]
    assert list(dict.fromkeys(chroms)) == ["chr1", "chr10", "chr2"]        # lexical, as write_vcf_records sorts


def test_vcf_host_genome_matches_reference_writer(tmp_path):
    """The reference-written multi-contig golden (tests/golden/make_golden_genome_vcf.py): pb_variant_vcf_host over every record
    of the five contigs at once, then order_lines + write_vcfs, gives the files the reference wrote."""
    from pepper_b200.vcf import order_lines, vcf_text_host, write_vcfs
    from tests.genome_vcf_golden import load, check_against_golden
    g = load()
    names = g["names"]
    text, lines = vcf_text_host(names, np.arange(len(names)), g["positions"], g["contig"], g["depths"], g["freqs"], g["keys"],
                                g["probs"], g["regions"], g["select"], g["options"])
    text, lines = order_lines([(text, lines)], names)
    totals = write_vcfs(str(tmp_path), "sample_b200", [(c, len(s)) for c, s in zip(names, g["genomes"])], names, text, lines)
    check_against_golden(str(tmp_path), g, totals)


def test_qual_matches_python():
    """QUAL through the device log10 equals Python's int(-10 * math.log10(...)) on every float32 genotype probability in
    [0.19, 1] (every QUAL step from 1 to 90 lies there; below 0.19 QUAL is 1) and on 10^6 random values in [0, 0.19)."""
    import ctypes as C
    import math
    from pepper_b200 import _lib
    L = _lib.lib()
    L.pb_test_vcf_qual.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
    lo, hi = np.float32(0.19).view(np.uint32), np.float32(1.0).view(np.uint32)
    p = np.concatenate([np.arange(lo, hi + 1, dtype=np.uint32).view(np.float32),
                        (np.random.default_rng(5).random(10 ** 6) * 0.19).astype(np.float32)])
    got = np.zeros(p.shape[0], np.int32)
    _lib.check(L.pb_test_vcf_qual(p.ctypes.data, p.shape[0], got.ctypes.data), "pb_test_vcf_qual")
    want = np.fromiter((max(1, int(-10 * math.log10(max(0.000000001, 1.0 - x)))) for x in p.astype(np.float64).tolist()), np.int32, p.shape[0])
    bad = np.flatnonzero(got != want)
    assert bad.shape[0] == 0, [(float(p[i]), int(got[i]), int(want[i])) for i in bad[:5]]
