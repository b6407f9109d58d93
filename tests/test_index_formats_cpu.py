"""CPU tests of the CSI index and bgzip-compressed FASTA readers (pepper_b200/csrc/bamio.cu) and of the writers behind them:

1. CSI fetch: the same records written with a .bai and with a .csi (depths 5 and 6, min_shift 14 and 12) come back from
   BamReader.fetch exactly as the htslib overlap rule picks them, on random queries and on bin / window / contig edges.
2. CSI layout: a CSI assembled here byte by byte from the CSIv1 specification is read back; a CSI at (14, 5) carries the same
   bins and chunks as the BAI of the same file.
3. bgzip FASTA: the .fa.gz decompresses to the plain file, and fetches on both agree, clamping and case included; plain gzip and
   a missing .gzi fail at open; the drop-in FASTA_handlers agree across the two encodings.
4. Reach: a BAI cannot address a contig longer than 2^29, so the planners refuse it; a VCF whose contig is longer gets a .csi in
   which every line's virtual offset lies in a chunk of its bins."""
import gzip
import os
import shutil
import struct
import zlib

import numpy as np
import pytest

from pepper_b200 import synth, synth_files

FIELDS = ("pos", "seq_off", "cigar_off", "flag", "mapq", "seq", "qual", "cigar")


def expected_fetch(rec, beg, end):
    rlen = np.array([synth_files.record_ref_len(rec.cigar[rec.cigar_off[r]:rec.cigar_off[r + 1]]) or 1 for r in range(rec.n_records)], np.int64)
    return np.nonzero((rec.pos < end) & (rec.pos + rlen > beg))[0]


def same_records(got, rec, idx):
    assert got.n_records == idx.shape[0]
    assert np.array_equal(got.pos, rec.pos[idx]) and np.array_equal(got.flag, rec.flag[idx]) and np.array_equal(got.mapq, rec.mapq[idx])
    so = rec.seq_off
    assert np.array_equal(got.qual, np.concatenate([rec.qual[so[i]:so[i + 1]] for i in idx]) if idx.shape[0] else np.zeros(0, np.uint8))
    co = rec.cigar_off
    assert np.array_equal(got.cigar, np.concatenate([rec.cigar[co[i]:co[i + 1]] for i in idx]) if idx.shape[0] else np.zeros(0, np.uint32))


@pytest.fixture(scope="module")
def bams(tmp_path_factory):
    d = tmp_path_factory.mktemp("csi")
    rec0, _ = synth.simulate_contig_records(200_000, 10, synth.ONT, 11, contig_start=3000)
    rec1, _ = synth.simulate_contig_records(70_000, 6, synth.HIFI, 12)
    contigs = [("chrA", 210_000), ("chrB", 70_000), ("chrE", 500)]
    out = {}
    for tag, kw in [("bai", dict(index="bai")), ("csi5", dict(index="csi")), ("csi6", dict(index="csi", csi_depth=6)),
                    ("csi12", dict(index="csi", csi_min_shift=12, csi_depth=6)), ("both", dict(index="both"))]:
        p = str(d / f"{tag}.bam")
        synth_files.write_bam(p, contigs, {0: rec0, 1: rec1}, block_payload=20_000, **kw)
        out[tag] = p
    return dict(paths=out, rec=[rec0, rec1], contigs=contigs, dir=d)


def edge_queries(length, min_shift, depth):
    q = [(0, 1), (0, length), (length - 1, length), (length, length + 10), (5, 5), (100, 99)]
    for l in range(1, depth + 1):
        w = 1 << (min_shift + 3 * (depth - l))
        for k in range(1, 4):
            if k * w < length:
                q += [(k * w - 1, k * w), (k * w, k * w + 1), (k * w - 1, k * w + 1), (k * w - 300, k * w + 300)]
    for k in range(1, length >> 14):
        q.append(((k << 14) - 1, (k << 14) + 1))
    return q


@pytest.mark.parametrize("tag", ["csi5", "csi6", "csi12", "both", "bai"])
def test_csi_fetch_matches_overlap_rule(bams, tag):
    from pepper_b200.bamio import BamReader
    r = BamReader(bams["paths"][tag], threads=3)
    info = r.index_info()
    want_fmt = "bai" if tag == "bai" else "csi"                 # a file with both indexes opens the CSI (htslib's order)
    assert info["format"] == want_fmt
    ms, depth = info["min_shift"], info["depth"]
    assert r.index_max_end == 1 << (ms + 3 * depth)
    rng = np.random.default_rng(3)
    n = 0
    for tid, (name, length) in enumerate(bams["contigs"][:2]):
        rec = bams["rec"][tid]
        qs = edge_queries(length, ms, depth) + [(int(b), int(b) + int(rng.choice([1, 17, 5000, 40_000, 150_000])))
                                                 for b in rng.integers(0, length, 40)]
        for beg, end in qs:
            got = r.fetch(name, beg, end).to_batch()
            same_records(got, rec, expected_fetch(rec, max(beg, 0), end) if end > beg else np.zeros(0, np.int64))
            n += got.n_records
    assert r.fetch("chrE", 0, 500).n_records == 0
    assert n > 1000
    r.close()


def test_index_lookup_forms(bams, tmp_path):
    """name.csi next to name.bam is found like name.bai; with no index at all the open names both forms it looked for."""
    from pepper_b200.bamio import BamReader
    from pepper_b200._lib import PepperB200Error
    src = bams["paths"]["csi6"]
    p = str(tmp_path / "x.bam")
    shutil.copy(src, p)
    with pytest.raises(PepperB200Error, match="csi"):
        BamReader(p)
    shutil.copy(src + ".csi", str(tmp_path / "x.csi"))
    r = BamReader(p)
    assert r.index_info() == dict(format="csi", min_shift=14, depth=6)
    same_records(r.fetch("chrB", 0, 70_000).to_batch(), bams["rec"][1], np.arange(bams["rec"][1].n_records))


# ------------------------------------------------------------------------------------------------------------ CSI layout
def _bgzf(data: bytes) -> bytes:
    """BGZF members written here from SAMv1 4.1 (not by the project's writer) + the EOF block."""
    out = b""
    for s in range(0, max(1, len(data)), 30_000):
        pl = data[s:s + 30_000]
        co = zlib.compressobj(6, zlib.DEFLATED, -15)
        c = co.compress(pl) + co.flush()
        out += (b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0" + struct.pack("<H", 18 + len(c) + 8 - 1) + c
                + struct.pack("<II", zlib.crc32(pl), len(pl)))
    return out + bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def _reg2bin(beg, end, min_shift, depth):
    """SAMv1 5.3 reg2bin in the binning (min_shift, depth)."""
    end -= 1
    for l in range(depth, 0, -1):
        s = min_shift + 3 * (depth - l)
        if beg >> s == end >> s:
            return ((1 << 3 * l) - 1) // 7 + (beg >> s)
    return 0


def _bam_records(path):
    """(tid, pos, end, virtual offset) of every record, from the file's BGZF blocks walked here."""
    raw = open(path, "rb").read()
    blocks, off = [], 0
    while off < len(raw):
        bs = struct.unpack_from("<H", raw, off + 16)[0] + 1
        blocks.append((off, zlib.decompress(raw[off + 18:off + bs - 8], -15)))
        off += bs
    ustart = np.cumsum([0] + [len(b) for _, b in blocks])
    stream = b"".join(b for _, b in blocks)

    def voff(u):
        k = int(np.searchsorted(ustart, u, side="right") - 1)
        return (blocks[k][0] << 16) | (u - int(ustart[k])) if k < len(blocks) else off << 16
    p = 8 + struct.unpack_from("<i", stream, 4)[0]
    n_ref = struct.unpack_from("<i", stream, p)[0]
    p += 4
    for _ in range(n_ref):
        p += 8 + struct.unpack_from("<i", stream, p)[0]
    out = []
    while p < len(stream):
        bs, tid, pos, l_name, _, _, n_cig = struct.unpack_from("<iiiBBHH", stream, p)
        cig = np.frombuffer(stream, "<u4", n_cig, p + 36 + l_name)
        rl = synth_files.record_ref_len(cig) or 1
        out.append((tid, pos, pos + rl, voff(p), voff(p + 4 + bs)))
        p += 4 + bs
    return out


def test_hand_built_csi_is_read_back(tmp_path):
    """Records on two contigs, min_shift 12 and depth 4: bins, loffsets and chunks computed here, one chunk per record."""
    from pepper_b200.bamio import BamReader
    recs = [dict(pos=p, seq="ACGT" * 5, cigar=[(0, 20)]) for p in (5, 4090, 4100, 40_000, 262_000, 262_140)]
    recs.append(dict(pos=300, seq="A" * 10, cigar=[(0, 5), (2, 70_000), (0, 5)]))     # a long deletion: a high-level bin
    recs = sorted(recs, key=lambda r: r["pos"])
    batch = synth.make_records(recs)
    bam = str(tmp_path / "h.bam")
    other = synth.make_records([dict(pos=5, seq="ACGT", cigar=[(0, 4)]), dict(pos=9, seq="ACGT", cigar=[(0, 4)])])
    synth_files.write_bam(bam, [("c0", 262_144), ("c1", 1000)], {0: batch, 1: other}, block_payload=90)
    os.remove(bam + ".bai")
    min_shift, depth = 12, 4
    body = b""
    rows = _bam_records(bam)
    for tid in (0, 1):
        mine = [r for r in rows if r[0] == tid]
        bins = {}
        for _, pos, end, vb, ve in mine:
            bins.setdefault(_reg2bin(pos, end, min_shift, depth), []).append((vb, ve))
        body += struct.pack("<i", len(bins))
        for b in sorted(bins):
            body += struct.pack("<IQi", b, 0, len(bins[b])) + b"".join(struct.pack("<QQ", *c) for c in bins[b])
    csi = b"CSI\x01" + struct.pack("<iii", min_shift, depth, 3) + b"aux" + struct.pack("<i", 2) + body + struct.pack("<Q", 0)
    open(bam + ".csi", "wb").write(_bgzf(csi))
    r = BamReader(bam, 2)
    assert r.index_info() == dict(format="csi", min_shift=12, depth=4) and r.index_max_end == 1 << 24
    for beg, end in [(0, 262_144), (0, 1), (4095, 4097), (4096, 4100), (70_000, 70_306), (70_306, 70_400), (262_139, 262_144),
                     (100_000, 100_001), (262_144, 1 << 30)]:
        same_records(r.fetch("c0", beg, end).to_batch(), batch, expected_fetch(batch, beg, end))
    assert r.fetch("c1", 0, 1000).n_records == 2
    # a truncated index is refused
    open(bam + ".csi", "wb").write(_bgzf(csi[:len(csi) - 40]))
    from pepper_b200._lib import PepperB200Error
    with pytest.raises(PepperB200Error, match="CSI"):
        BamReader(bam, 2)


def _parse_bai(data):
    n_ref = struct.unpack_from("<i", data, 4)[0]
    o, refs = 8, []
    for _ in range(n_ref):
        n_bin = struct.unpack_from("<i", data, o)[0]; o += 4
        bins = {}
        for _ in range(n_bin):
            b, nc = struct.unpack_from("<Ii", data, o); o += 8
            bins[b] = [struct.unpack_from("<QQ", data, o + 16 * k) for k in range(nc)]; o += 16 * nc
        n_intv = struct.unpack_from("<i", data, o)[0]; o += 4 + 8 * n_intv
        refs.append(bins)
    return refs


def _parse_csi(data):
    """CSIv1 read here: (min_shift, depth, aux, [{bin: (loffset, chunks)}])."""
    ms, depth, l_aux = struct.unpack_from("<iii", data, 4)
    aux = data[16:16 + l_aux]
    o = 16 + l_aux
    n_ref = struct.unpack_from("<i", data, o)[0]; o += 4
    refs = []
    for _ in range(n_ref):
        n_bin = struct.unpack_from("<i", data, o)[0]; o += 4
        bins = {}
        for _ in range(n_bin):
            b, loff, nc = struct.unpack_from("<IQi", data, o); o += 16
            bins[b] = (loff, [struct.unpack_from("<QQ", data, o + 16 * k) for k in range(nc)]); o += 16 * nc
        refs.append(bins)
    assert o in (len(data), len(data) - 8)
    return ms, depth, aux, refs


def test_csi_at_14_5_carries_the_bai_bins(bams):
    p = bams["paths"]["both"]
    bai = _parse_bai(open(p + ".bai", "rb").read())
    ms, depth, aux, csi = _parse_csi(gzip.decompress(open(p + ".csi", "rb").read()))
    assert (ms, depth, aux) == (14, 5, b"")
    assert len(bai) == len(csi) == 3
    for b, c in zip(bai, csi):
        assert {k: v for k, v in b.items()} == {k: v[1] for k, v in c.items()}
    # every record's virtual offset is at or past the loffset of each bin on its path (the shortcut the reader may take)
    for tid, pos, end, vb, _ in _bam_records(p):
        if tid > 1:
            continue
        for l in range(depth + 1):
            b = ((1 << 3 * l) - 1) // 7 + (pos >> (ms + 3 * (depth - l)))
            if b in csi[tid]:
                assert csi[tid][b][0] <= vb


# ---------------------------------------------------------------------------------------------------------- bgzip FASTA
@pytest.fixture(scope="module")
def fastas(tmp_path_factory):
    d = tmp_path_factory.mktemp("fagz")
    g = synth.make_reference(300_000, 21)
    g[1000:1300] = np.frombuffer((b"acgtn" * 60), np.uint8)                 # lower case is kept
    n_line = np.frombuffer(b"N" * 60, np.uint8)
    contigs = [("ctg1", g), ("ctg2", [(n_line, 3000), (g[:12_345], 1), (n_line[:7], 1), (g[5:70_005], 1)]),
               ("tiny", np.frombuffer(b"ACGTa", np.uint8))]
    fa, gz = str(d / "r.fa"), str(d / "r.fa.gz")
    synth_files.write_fasta(fa, contigs)
    synth_files.write_fasta(gz, contigs, bgzip=True, block_lines=97)       # small blocks: a fetch crosses many
    return dict(fa=fa, gz=gz, dir=d)


def test_bgzip_fasta_bytes_and_index(fastas):
    assert gzip.decompress(open(fastas["gz"], "rb").read()) == open(fastas["fa"], "rb").read()
    assert open(fastas["gz"] + ".fai").read() == open(fastas["fa"] + ".fai").read()
    n = struct.unpack_from("<Q", open(fastas["gz"] + ".gzi", "rb").read())[0]
    assert n > 50


def test_bgzip_fasta_fetch_equals_plain(fastas):
    from pepper_b200.bamio import FastaReader
    a, b = FastaReader(fastas["fa"]), FastaReader(fastas["gz"])
    assert a.get_chromosome_names() == b.get_chromosome_names() == ["ctg1", "ctg2", "tiny"]
    rng = np.random.default_rng(9)
    for c in ("ctg1", "ctg2", "tiny"):
        L = a.get_chromosome_sequence_length(c)
        assert b.get_chromosome_sequence_length(c) == L
        qs = [(0, 1), (0, L), (L - 1, L), (L - 3, L + 100), (-5, 3), (L + 10, L + 20), (7, 7), (59, 61)]
        qs += [(int(s), int(s) + int(rng.choice([1, 60, 61, 5821, 70_000]))) for s in rng.integers(0, L, 60)]
        for s, e in qs:
            assert np.array_equal(a.fetch_array(c, s, e), b.fetch_array(c, s, e)), (c, s, e)
    assert b.get_reference_sequence("ctg1", 1000, 1010) == "acgtnacgtn"
    from pepper_b200._lib import PepperB200Error
    with pytest.raises(PepperB200Error, match="NOT PRESENT"):
        b.fetch_array("nope", 0, 10)


def test_bgzip_fasta_concurrent_fetches(fastas):
    """Fetches on one handle from several threads (the streaming calls fetch from a helper thread and the main thread)."""
    from concurrent.futures import ThreadPoolExecutor
    from pepper_b200.bamio import FastaReader
    a, b = FastaReader(fastas["fa"]), FastaReader(fastas["gz"])
    qs = [(int(s), int(s) + 40_000) for s in np.random.default_rng(2).integers(0, 260_000, 64)]
    with ThreadPoolExecutor(8) as pool:
        got = list(pool.map(lambda q: b.fetch_array("ctg1", *q), qs))
    for q, g in zip(qs, got):
        assert np.array_equal(g, a.fetch_array("ctg1", *q))


def test_gzip_and_missing_gzi_fail_at_open(fastas, tmp_path):
    from pepper_b200.bamio import FastaReader
    from pepper_b200._lib import PepperB200Error
    plain = str(tmp_path / "p.fa.gz")
    open(plain, "wb").write(gzip.compress(open(fastas["fa"], "rb").read()))
    shutil.copy(fastas["fa"] + ".fai", plain + ".fai")
    with pytest.raises(PepperB200Error, match="gzip, not bgzip"):
        FastaReader(plain)
    nogzi = str(tmp_path / "n.fa.gz")
    shutil.copy(fastas["gz"], nogzi)
    shutil.copy(fastas["gz"] + ".fai", nogzi + ".fai")
    with pytest.raises(PepperB200Error, match=r"n\.fa\.gz\.gzi"):
        FastaReader(nogzi)


def test_dropin_fasta_handlers_agree(fastas):
    from pepper_b200.build import PEPPER, PEPPER_VARIANT
    for mod in (PEPPER, PEPPER_VARIANT):
        a, b = mod.FASTA_handler(fastas["fa"]), mod.FASTA_handler(fastas["gz"])
        assert a.get_chromosome_names() == b.get_chromosome_names()
        for c, s, e in [("ctg1", 990, 1320), ("ctg2", 179_990, 180_100), ("ctg2", 0, 50), ("tiny", 0, 5)]:
            assert a.get_reference_sequence(c, s, e) == b.get_reference_sequence(c, s, e)
            assert a.get_chromosome_sequence_length(c) == b.get_chromosome_sequence_length(c)


# --------------------------------------------------------------------------------------------------- reach and VCF index
def test_planners_refuse_contigs_past_the_bai_reach(tmp_path):
    from pepper_b200.bamio import BamReader
    from pepper_b200.frontend import genome_plan, polish_job, variant_job
    rec = synth.make_records([dict(pos=100, seq="ACGT", cigar=[(0, 4)])])
    big = (1 << 29) + 5
    for idx in ("bai", "csi"):
        bam = str(tmp_path / f"{idx}.bam")
        synth_files.write_bam(bam, [("long", big), ("short", 1000)], {0: rec}, index=idx)
        r = BamReader(bam, 1)
        fasta = [("long", big), ("short", 1000)]
        names = r.get_chromosome_sequence_names()
        reach = r.index_max_end
        if idx == "bai":
            assert reach == 1 << 29
            for call in (lambda: variant_job(fasta, names, max_end=reach), lambda: genome_plan(fasta, names, max_end=reach),
                         lambda: polish_job(fasta, names, max_end=reach)):
                with pytest.raises(ValueError, match="'long'"):
                    call()
            # a region that stays inside the reach is fine
            assert variant_job(fasta, names, "long:0-5000,short", max_end=reach) == [("long", 0, 5000), ("short", 0, 999)]
        else:
            assert reach == 1 << 32
            assert variant_job(fasta, names, max_end=reach)[0] == ("long", 0, big - 1)
            assert polish_job(fasta, names, max_end=reach)[0] == ["long", "short"]


def file_mask(name, lines):
    from pepper_b200.vcf import VCF_FILES, file_masks
    return file_masks(lines["cls"])[VCF_FILES.index(name)]


def test_vcf_of_a_long_contig_gets_a_csi(tmp_path):
    from pepper_b200.vcf import VCF_FILES, VCF_LINE, order_lines, write_vcfs
    rng = np.random.default_rng(4)
    names = ["chrL", "chrS"]
    L = (1 << 30) + 77
    parts = []
    for cid, (lo, hi, n) in enumerate([(0, L - 100, 3000), (1000, 60_000, 300)]):
        pos = np.sort(rng.choice(np.arange(lo, hi, 97), n, replace=False))
        pos[-1] = hi - 3 if cid == 0 else pos[-1]
        rl = np.where(rng.random(n) < 0.1, rng.integers(2, 50, n), 1)
        txt = [("%s\t%d\t.\t%s\tC\t5\tPASS\t.\tGT\t0/1\n" % (names[cid], p + 1, "A" * r)).encode() for p, r in zip(pos, rl)]
        lines = np.zeros(n, VCF_LINE)
        lines["pos"], lines["contig"], lines["ref_len"] = pos, cid, rl
        lines["cls"] = rng.integers(0, 3, n)
        lines["text_len"] = [len(t) for t in txt]
        lines["text_off"] = np.concatenate([[0], np.cumsum(lines["text_len"])[:-1]])
        parts.append((np.frombuffer(b"".join(txt), np.uint8), lines))
    text, lines = order_lines(parts, names)
    write_vcfs(str(tmp_path), "s", [("chrL", L), ("chrS", 70_000)], names, text, lines, threads=2)
    for name in VCF_FILES:
        path = str(tmp_path / (name + ".vcf.gz"))
        assert os.path.exists(path + ".csi") and not os.path.exists(path + ".tbi")
        ms, depth, aux, refs = _parse_csi(gzip.decompress(open(path + ".csi", "rb").read()))
        assert (ms, depth) == (14, 6)
        fmt, cs, cb, ce, meta, skip, l_nm = struct.unpack_from("<7i", aux)
        assert (fmt, cs, cb, ce, chr(meta), skip) == (2, 1, 2, 0, "#", 0)
        ref_names = aux[28:28 + l_nm].split(b"\0")[:-1]
        # every line: its virtual offset lies in a chunk of the bin of [pos, pos + len(REF))
        raw = open(path, "rb").read()
        off, bc, bu, stream = 0, [], [], b""
        while off < len(raw):
            bs = struct.unpack_from("<H", raw, off + 16)[0] + 1
            bc.append(off); bu.append(len(stream))
            stream += zlib.decompress(raw[off + 18:off + bs - 8], -15)
            off += bs
        n_lines = 0
        u = 0
        for t in stream.split(b"\n")[:-1]:
            if not t.startswith(b"#"):
                k = int(np.searchsorted(bu, u, side="right")) - 1
                v = (bc[k] << 16) | (u - bu[k])
                f = t.split(b"\t")
                pos = int(f[1]) - 1
                b = _reg2bin(pos, pos + len(f[3]), ms, depth)
                assert any(c0 <= v < c1 for c0, c1 in refs[ref_names.index(f[0])][b][1]), (name, t[:40])
                n_lines += 1
            u += len(t) + 1
        assert n_lines == int(file_mask(name, lines).sum())
    # all contigs short: the .tbi as before
    write_vcfs(str(tmp_path / "s"), "s", [("chrL", 1 << 29), ("chrS", 70_000)], names, text, lines[lines["contig"] == 1], threads=2)
    assert os.path.exists(str(tmp_path / "s" / (VCF_FILES[0] + ".vcf.gz.tbi")))
