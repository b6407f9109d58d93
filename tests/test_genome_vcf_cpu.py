"""Whole-genome VCF output without a GPU:

1. The job plan of a genome-wide call: contigs common to the BAM and the FASTA in natural order, `exclude`, `-r/--region` parsing
   (comma lists, `contig:start-end` clamped to the contig, `chr1-3` expansion).
2. The writer against the unmodified reference (tests/golden/genome_vcf_seed29.npz, written by the reference's find_candidates +
   VCFWriter over five FASTA contigs): the golden's candidate records, selected per record by the oracle and assembled per contig
   by vcf.assemble_sites, go through host_tail_text -> order_lines -> write_vcfs.  Each of the five files parses back to exactly
   the records the reference wrote to it (floats as the float32 "%g" pysam prints), with the reference's header contigs and
   totals.
3. The same writer over the records of tests/golden/vcf_seed23.npz spread over four contigs: every BGZF member is valid, the file
   ends with the EOF block, and a tabix query over the .tbi finds each record in its own [pos, pos + len(REF)) and nothing
   outside it."""
import gzip
import json
import os
import struct
import zlib

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def test_variant_job_order_exclude_and_region():
    from pepper_b200.frontend import parse_region, variant_job
    fasta = [("chr1", 1000), ("chr10", 500), ("chr2", 300), ("chrM", 50), ("only_fa", 10)]
    bam = ["chr2", "chr10", "chr1", "chrM", "only_bam"]
    assert variant_job(fasta, bam) == [("chr1", 0, 999), ("chr2", 0, 299), ("chr10", 0, 499), ("chrM", 0, 49)]
    assert variant_job(fasta, bam, exclude=["chrM"]) == [("chr1", 0, 999), ("chr2", 0, 299), ("chr10", 0, 499)]
    assert variant_job(fasta, bam, "chr10:100-900,chr1") == [("chr10", 100, 499), ("chr1", 0, 999)]
    assert parse_region("chr1-3") == [("chr1", None), ("chr2", None), ("chr3", None)]
    assert parse_region("chr3-1:5-9") == [("chr1", (5, 9)), ("chr2", (5, 9)), ("chr3", (5, 9))]
    for bad in ("chr1:9-5", "chr1:1-2-3", "a:b:c"):
        with pytest.raises(ValueError):
            parse_region(bad)
    with pytest.raises(ValueError):
        variant_job(fasta, ["x"])
    with pytest.raises(ValueError):
        variant_job(fasta, bam, "chr7")


def test_writer_matches_reference_genome_golden(tmp_path):
    from oracle import find_candidates as ofc
    from pepper_b200.candidates import F_DV, F_REPEAT, F_SWAP
    from pepper_b200.vcf import assemble_sites, host_tail_text, order_lines, write_vcfs
    from tests.genome_vcf_golden import load, check_against_golden
    g = load()
    names, n = g["names"], g["positions"].shape[0]
    fetch = lambda c, a, b: g["genomes"][names.index(c)][max(0, a):max(0, b)]
    flags, geno = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
    for i in range(n):                 # the per-record selection the CUDA kernel makes, here from the oracle (no GPU)
        c = names[g["contig"][i]]
        _, d = ofc.select(g["options"], c, g["positions"][i:i + 1], g["depths"][i:i + 1], [g["key_str"][i]], g["freqs"][i:i + 1],
                          g["probs"][i:i + 1].astype(np.float64), fetch)
        geno[i] = int(np.argmax(g["probs"][i]))
        if d:
            swapped = g["key_str"][i][0] == "3" and d[0][3] == g["key_str"][i][1:]
            flags[i] = F_DV | (F_REPEAT if d[0][11] else 0) | (F_SWAP if swapped else 0)
    parts = []
    for k, c in enumerate(names):
        m = g["contig"] == k
        recs = assemble_sites(c, g["positions"][m], g["contig"][m], g["depths"][m], g["freqs"][m], g["keys"][m], g["probs"][m], flags[m],
                              geno[m], g["regions"], g["options"])
        parts.append(host_tail_text(recs, k))
    text, lines = order_lines(parts, names)
    fasta = [(c, len(s)) for c, s in zip(names, g["genomes"])]
    totals = write_vcfs(str(tmp_path), "sample_b200", fasta, names, text, lines, threads=2)
    check_against_golden(str(tmp_path), g, totals)


def _records():
    """The golden's records over chr1, chr2, chr10 and chrX (chr3 has none); chr10's first site sits at chr1's last position."""
    g = np.load(os.path.join(GOLD, "vcf_seed23.npz"))
    recs = [json.loads(r) for r in g["records"]]
    n = len(recs)
    cut = [0, n // 4, n // 2, 3 * n // 4, n]
    out = {}
    for k, c in enumerate(("chr1", "chr2", "chr10", "chrX")):
        out[c] = [dict(r, contig=c) for r in recs[cut[k]:cut[k + 1]]]
    first = dict(out["chr10"][0])
    out["chr10"][0] = dict(first, start=out["chr1"][-1]["start"])
    return out


def _expected(per_contig):
    """write_vcf_records over the same records: sorted by (contig, position), a site skipped when its position equals the last
    written one (VcfWriter.py:144-152)."""
    from pepper_b200.vcf import format_vcf_line
    files = {"full": [], "pepper": [], "variant_calling": [], "variant_calling_snp": [], "variant_calling_indel": []}
    last = -1
    for r in sorted((r for rs in per_contig.values() for r in rs), key=lambda r: (r["contig"], r["start"])):
        if r["start"] == last:
            continue
        last = r["start"]
        for f in r["files"]:
            files[f].append(format_vcf_line(r) + "\n")
    return files


def _bgzf_members(raw: bytes):
    off, out = 0, []
    while off < len(raw):
        assert raw[off:off + 4] == b"\x1f\x8b\x08\x04" and raw[off + 10:off + 14] == b"\x06\x00BC"
        bsize = struct.unpack_from("<H", raw, off + 16)[0] + 1
        blk = raw[off:off + bsize]
        data = zlib.decompress(blk[18:-8], -15)
        crc, isize = struct.unpack_from("<II", blk, bsize - 8)
        assert crc == zlib.crc32(data) and isize == len(data)
        out.append((off, data))
        off += bsize
    return out


def _tabix_query(tbi: bytes, gz: bytes, contig: str, beg: int, end: int):
    """Lines of `contig` overlapping [beg, end) by the index: bins on the reg2bin path, chunks cut by the linear index."""
    d = gzip.decompress(tbi)
    assert d[:4] == b"TBI\x01"
    n_ref, fmt, cs, cb, ce, meta, skip, l_nm = struct.unpack_from("<8i", d, 4)
    assert (fmt, cs, cb, ce, meta) == (2, 1, 2, 0, ord("#"))
    names = d[36:36 + l_nm].split(b"\0")[:-1]
    p = 36 + l_nm
    idx = []
    for _ in range(n_ref):
        (nb,) = struct.unpack_from("<i", d, p); p += 4
        bins = {}
        for _ in range(nb):
            b, nc = struct.unpack_from("<Ii", d, p); p += 8
            bins[b] = [struct.unpack_from("<QQ", d, p + 16 * k) for k in range(nc)]; p += 16 * nc
        (ni,) = struct.unpack_from("<i", d, p); p += 4
        lin = struct.unpack_from("<%dQ" % ni, d, p); p += 8 * ni
        idx.append((bins, lin))
    if contig.encode() not in names:
        return []
    bins, lin = idx[names.index(contig.encode())]
    want_bins = {0}
    for sh, base in ((26, 1), (23, 9), (20, 73), (17, 585), (14, 4681)):
        want_bins.update(range(base + (beg >> sh), base + ((end - 1) >> sh) + 1))
    min_off = lin[beg >> 14] if (beg >> 14) < len(lin) else 0
    members = {off: data for off, data in _bgzf_members(gz)}
    found = set()
    for b in want_bins & set(bins):
        for vb, ve in bins[b]:
            if ve <= min_off:
                continue
            co, uo = vb >> 16, vb & 0xffff
            buf = b""
            keys = sorted(members)
            k = keys.index(co)
            while len(buf) < (ve >> 16) - co + 65536 * 2 and k < len(keys):
                buf += members[keys[k]]; k += 1
            text = buf[uo:]
            stop_c, stop_u = ve >> 16, ve & 0xffff
            span = sum(len(members[x]) for x in keys if co <= x < stop_c) - uo + stop_u
            for line in text[:span].decode().splitlines():
                f = line.split("\t")
                s, e = int(f[1]) - 1, int(f[1]) - 1 + len(f[3])
                if f[0] == contig and s < end and e > beg:
                    found.add(line)
    return sorted(found)


def test_writer_files_match_reference_writer(tmp_path):
    from pepper_b200.synth_files import BGZF_EOF
    from pepper_b200.vcf import VCF_FILES, host_tail_text, order_lines, vcf_header, write_vcfs
    per_contig = _records()
    names = ["chr1", "chr2", "chr10", "chrX", "chr3"]
    fasta = [("chr1", 4000), ("chr2", 4000), ("chr3", 4000), ("chr10", 4000), ("chrX", 4000)]
    parts = [host_tail_text(per_contig[c], names.index(c)) for c in ("chrX", "chr10", "chr1", "chr2")]
    text, lines = order_lines(parts, names)
    totals = write_vcfs(str(tmp_path), "sample_b200", fasta, names, text, lines, threads=4)
    want = _expected(per_contig)
    head = vcf_header("sample_b200", fasta)
    assert head.count("##contig=") == 5 and head.index("ID=chr3,") < head.index("ID=chr10,")
    assert totals == tuple(len(want[k]) for k in ("full", "pepper", "variant_calling", "variant_calling_snp", "variant_calling_indel"))
    assert len(want["full"]) == sum(len(v) for v in per_contig.values()) - 1          # chr10's first site is skipped
    for name, key in zip(VCF_FILES, ("full", "pepper", "variant_calling", "variant_calling_snp", "variant_calling_indel")):
        raw = open(tmp_path / (name + ".vcf.gz"), "rb").read()
        assert raw.endswith(BGZF_EOF)
        assert gzip.decompress(raw).decode() == head + "".join(want[key]), name
        assert b"".join(d for _, d in _bgzf_members(raw)) == gzip.decompress(raw)
        if key not in ("full", "variant_calling_indel"):
            continue
        tbi = open(tmp_path / (name + ".vcf.gz.tbi"), "rb").read()
        assert tbi.endswith(BGZF_EOF)
        for line in want[key][::7]:
            f = line.rstrip("\n").split("\t")
            s = int(f[1]) - 1
            e = s + len(f[3])
            got = _tabix_query(tbi, raw, f[0], s, e)
            exp = sorted(x.rstrip("\n") for x in want[key] if x.split("\t")[0] == f[0]
                         and int(x.split("\t")[1]) - 1 < e and int(x.split("\t")[1]) - 1 + len(x.split("\t")[3]) > s)
            assert got == exp and line.rstrip("\n") in got
        assert _tabix_query(tbi, raw, "chr3", 0, 4000) == []
