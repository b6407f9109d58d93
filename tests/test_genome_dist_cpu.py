"""CPU: the pieces of the distributed genome call that need no GPU.

1. Group plan: groups never cross a contig; boundary positions for contigs of 1, 2 and many intervals; excluded and FASTA-only
   contigs are left out.
2. Index builder: the vectorised tabix index gives exactly the bytes of synth_files._bai_bytes on seeded random line sets
   (lines spanning several 16 kb windows, several contigs, member starts at line starts, the end-of-data offset).
3. Writer offsets: group parts compressed by host zlib, cut at group starts and mid-line, written by write_vcfs_from_parts,
   decompress to exactly what order_lines + write_vcfs give, including a `last_position` drop across "ranks"."""
import gzip
import struct

import numpy as np
import pytest


def _bai_tabix(names, tids, beg, end, ustart, uend, blk_u, blk_c, eof_c, total_u):
    """The per-line reference: spans per reference -> synth_files._bai_bytes."""
    from pepper_b200.synth_files import _bai_bytes
    u = np.concatenate([ustart, uend]).astype(np.int64)
    k = np.maximum(np.searchsorted(blk_u, u, side="right") - 1, 0)
    v = np.where(u >= total_u, np.int64(eof_c) << 16, (blk_c[k] << 16) | (u - blk_u[k]))
    voff = dict(zip(u.tolist(), v.tolist())).__getitem__
    spans = {}
    for t, b, e, us, ue in zip(tids.tolist(), beg.tolist(), end.tolist(), ustart.tolist(), uend.tolist()):
        spans.setdefault(t, []).append((b, e, us, ue))
    nm = b"".join(n.encode() + b"\0" for n in names)
    return b"TBI\x01" + struct.pack("<8i", len(names), 2, 1, 2, 0, ord("#"), 0, len(nm)) + nm + _bai_bytes(len(names), spans, voff)[8:]


@pytest.mark.parametrize("seed", range(6))
def test_vectorised_index_matches_bai_bytes(seed):
    from pepper_b200.vcf import _tabix
    rng = np.random.default_rng(seed)
    for _ in range(40):
        nt = int(rng.integers(1, 4))
        beg, tids = [], []
        for t in range(nt):
            b = np.unique(rng.integers(0, int(rng.choice([20_000, 300_000, 5_000_000])), int(rng.integers(1, 150))))
            beg.append(b); tids.append(np.full(b.shape[0], t))
        beg, tids = np.concatenate(beg), np.concatenate(tids)
        ref_len = np.where(rng.random(beg.shape[0]) < 0.1, rng.integers(1, 40_000, beg.shape[0]), rng.integers(1, 5, beg.shape[0]))
        end = beg + ref_len                                                          # some lines span several 16 kb windows
        tl = rng.integers(20, 200, beg.shape[0])
        us = 300 + np.concatenate([[0], np.cumsum(tl)[:-1]])
        ue = us + tl
        total = int(ue[-1])                                                          # the last line ends at the end of data
        blk = np.unique(np.concatenate([[0], rng.integers(1, total, int(rng.integers(1, 30))), us[rng.integers(0, us.shape[0], 3)]]))
        blk_c = np.cumsum(np.concatenate([[0], rng.integers(100, 5000, blk.shape[0])]))[:blk.shape[0]]
        eof = int(blk_c[-1]) + 1000
        names = ["c%d" % t for t in range(nt)]
        assert _tabix(names, tids, beg, end, us, ue, blk, blk_c, eof, total) == _bai_tabix(names, tids, beg, end, us, ue, blk, blk_c, eof, total)


def test_group_plan_and_boundaries():
    from pepper_b200.dist import plan_contig_groups
    from pepper_b200.frontend import genome_plan, group_boundaries
    fasta = [("chr2", 2501), ("chr10", 901), ("chr1", 4201), ("chrM", 1801), ("chr3", 1000)]      # chr3: in the FASTA only
    names, iv, first = genome_plan(fasta, ["chr2", "chr10", "chr1", "chrM"], exclude=("chrM",), interval_size=1000)
    assert names == ["chr1", "chr2", "chr10"]
    per = [first[k + 1] - first[k] for k in range(len(names))]
    assert per == [5, 3, 1]                                   # many intervals, several, one
    assert iv[:5] == [(0, 1000), (1000, 2000), (2000, 3000), (3000, 4000), (4000, 4200)]
    groups = plan_contig_groups(per, 2)
    assert groups == [(0, 2), (2, 4), (4, 5), (5, 7), (7, 8), (8, 9)]
    contig = np.repeat(np.arange(3), per)
    assert all(len(set(contig[g0:g1].tolist())) == 1 for g0, g1 in groups)
    bnd = group_boundaries(iv, first, groups)
    assert bnd.tolist() == [[-1, 2000], [2000, 4000], [4000, -1], [-1, 2000], [2000, -1], [-1, -1]]
    one = group_boundaries(iv, first, plan_contig_groups(per, 1))
    assert one[5:8].tolist() == [[-1, 1000], [1000, 2000], [2000, -1]]
    names2, iv2, first2 = genome_plan(fasta, ["chr2", "chr10", "chr1", "chrM"], region="chr2:500-1700,chr10", interval_size=1000)
    assert names2 == ["chr2", "chr10"] and iv2[:2] == [(500, 1500), (1500, 1700)]
    assert group_boundaries(iv2, first2, plan_contig_groups([2, 1], 1)).tolist() == [[-1, 1500], [1500, -1], [-1, -1]]


def _lines(rng, names, n_per):
    """Random VCF lines of each contig (one per site, increasing positions): (text, VCF_LINE) parts per contig."""
    from pepper_b200.vcf import VCF_LINE
    parts = []
    for cid, n in enumerate(n_per):
        pos = np.sort(rng.choice(np.arange(1000, 60_000), n, replace=False))
        rl = np.where(rng.random(n) < 0.1, rng.integers(2, 50, n), 1)
        txt = [("%s\t%d\t.\t%s\tC\t%d\tPASS\t.\tGT\t0/1%s\n" % (names[cid], p + 1, "A" * r, rng.integers(1, 60), "x" * int(rng.integers(0, 300)))).encode()
               for p, r in zip(pos, rl)]
        lines = np.zeros(n, VCF_LINE)
        lines["pos"], lines["contig"] = pos, cid
        lines["ref_len"] = rl
        lines["cls"] = rng.integers(0, 3, n)
        lines["text_len"] = [len(t) for t in txt]
        lines["text_off"] = np.concatenate([[0], np.cumsum(lines["text_len"])[:-1]])
        parts.append((np.frombuffer(b"".join(txt), np.uint8), lines))
    return parts


def test_writer_from_parts_matches_write_vcfs(tmp_path):
    from pepper_b200.dist import GT_FIRST, GT_LAST, GT_LINES, last_position_drops, genome_totals, GT_FIRST_CLS, GT_PEPPER, GT_SNP, GT_INDEL
    from pepper_b200.vcf import VCF_FILES, host_group_part, order_lines, write_vcfs, write_vcfs_from_parts
    rng = np.random.default_rng(5)
    names = ["chr2", "chr10", "chr1"]
    parts = _lines(rng, names, [400, 0, 300])
    # chr2's first line at chr10... chr1 (lexically first) ends where chr10 / chr2 begin: a last_position drop across "ranks"
    t1, l1 = parts[2]
    t0, l0 = parts[0]
    l0 = l0.copy(); l0["pos"][0] = l1["pos"][-1]
    l0["pos"][1:] = np.maximum(l0["pos"][1:], l0["pos"][0] + 1 + np.arange(l0.shape[0] - 1))
    parts[0] = (t0, l0)
    fasta = [(c, 70_000) for c in names]
    text, lines = order_lines(parts, names)
    want = write_vcfs(str(tmp_path / "want"), "s", fasta, names, text, lines)
    # groups: each contig cut into 3 groups; group g gets its own stream (cuts at group starts), members of 5,000 bytes (mid-line)
    gparts, group_contig, table = {}, [], []
    g = 0
    for cid, (t, l) in enumerate(parts):
        for piece in np.array_split(np.arange(l.shape[0]), 3):
            gl = l[piece]
            group_contig.append(cid)
            row = np.zeros(8, np.int64)
            row[0] = 1
            if gl.shape[0]:
                row[GT_LINES], row[GT_FIRST], row[GT_LAST], row[GT_FIRST_CLS] = gl.shape[0], gl["pos"][0], gl["pos"][-1], gl["cls"][0]
                row[GT_PEPPER], row[GT_SNP], row[GT_INDEL] = [(gl["cls"] == c).sum() for c in range(3)]
            table.append(row)
            gparts[g] = (t, gl)
            g += 1
    table = np.array(table)
    drop = last_position_drops(table, np.array(group_contig), names)
    assert drop.sum() == 1 and drop[0]
    assert genome_totals(table, drop) == want
    for g, (t, gl) in list(gparts.items()):
        gparts[g] = host_group_part(t, gl[1:] if drop[g] else gl, payload=5000)
    assert any(p.usizes[0].shape[0] > 1 for p in gparts.values())
    write_vcfs_from_parts(str(tmp_path / "got"), "s", fasta, names, group_contig, gparts)
    for name in VCF_FILES:
        a = gzip.decompress(open(tmp_path / "got" / (name + ".vcf.gz"), "rb").read())
        b = gzip.decompress(open(tmp_path / "want" / (name + ".vcf.gz"), "rb").read())
        assert a == b, name
