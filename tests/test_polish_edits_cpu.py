"""CPU: the polish edits VCF — the oracle's records (tests/polish_edits_oracle.py) rebuild the stitched sequence from any draft
on the golden stitch inputs, the record rules on hand-built winners tables, and the written file: header, text, a tabix query
over its .tbi for every record, and a .csi for a contig longer than 2^29."""
import gzip
import os

import numpy as np
import pytest

from pepper_b200.polish_edits import EDIT_LINE, edits_header, host_part, write_edits_vcf
from tests import polish_edits_oracle as E
from tests.test_genome_vcf_cpu import _tabix_query

HERE = os.path.dirname(os.path.abspath(__file__))


def _load(name):
    with np.load(os.path.join(HERE, "golden", name)) as z:
        return {k: z[k] for k in z.files}


def _contig_inputs():
    """(predictions, span) per contig of the golden inputs: stitch_seed11 and each contig of polish_fasta_seed5."""
    out = []
    g = _load("stitch_seed11.npz")
    out.append(((g["bases"], g["position"], g["index"], g["image_region"], g["chunk_id"], g["region_starts"], g["region_ends"]),
                (int(g["region_starts"].min()), int(g["region_ends"].max()))))
    f = _load("polish_fasta_seed5.npz")
    for c in range(len(f["contigs"])):
        regs = np.flatnonzero(f["region_contig"] == c)
        if not regs.shape[0]:
            continue
        sel = np.isin(f["image_region"], regs)
        out.append(((f["bases"][sel], f["position"][sel], f["index"][sel], f["image_region"][sel], f["chunk_id"][sel],
                     f["region_starts"], f["region_ends"]),
                    (int(f["region_starts"][regs].min()), int(f["region_ends"][regs].max()))))
    return out


def _draft(table, span, rng, identity: float):
    """A draft over [0, span end]: with probability `identity` the winner's base at (p, 0) (lower case now and then), else random."""
    s, e = span
    d = []
    for p in range(e + 1):
        w = table.get((p, 0))
        if w is not None and w[0] and rng.random() < identity:
            b = "ACGT"[w[0] - 1]
        else:
            b = "ACGTN"[rng.integers(0, 5)]
        d.append(b.lower() if rng.random() < 0.1 else b)
    return "".join(d)


@pytest.mark.parametrize("identity", [0.0, 0.97])
def test_records_rebuild_the_stitched_sequence(identity):
    rng = np.random.default_rng(7)
    for preds, span in _contig_inputs():
        ph = rng.integers(0, 101, preds[0].shape).astype(np.uint8)
        table = E.winners(preds[0], ph, *preds[1:])
        want = E.stitched(table)
        for _ in range(3):
            draft = _draft(table, span, rng, identity)
            recs = E.records(table, draft, span)
            assert E.apply(recs, draft, span) == want
            assert all(b[0] > a[0] + len(a[1]) - 1 for a, b in zip(recs, recs[1:]))          # sorted, not overlapping
            assert all(r[3] is None or 0 <= r[3] <= 100 for r in recs)


def _t(cols):
    """A winners table from {(pos, idx): label letter or '' (deleted)} with phred 10 + pos."""
    return {k: ("ACGT".index(v) + 1 if v else 0, 10 + k[0]) for k, v in cols.items()}


def _identity(draft, ps):
    return {(p, 0): draft[p] for p in ps}


def test_hand_built_cases():
    d = "ACGTACGTAC"
    span = (0, 9)
    # a deletion at the span start, anchored on the base after
    t = _t({**_identity(d, range(1, 10)), (0, 0): ""})
    assert E.records(t, d, span) == [(0, "AC", "C", 10, False)]
    # two such deletions sharing that anchor merge into one record
    t = _t({**_identity(d, [1] + list(range(3, 10))), (0, 0): "", (2, 0): ""})
    assert E.records(t, d, span) == [(0, "ACG", "C", 10, False)]
    # an insertion after an identity base
    t = _t({**_identity(d, range(10)), (4, 1): "T", (4, 2): "T"})
    assert E.records(t, d, span) == [(4, "A", "ATT", 14, False)]
    # a deleted base followed by inserted bases
    t = _t({**_identity(d, [p for p in range(10) if p != 5]), (5, 0): "", (5, 1): "G"})
    assert E.records(t, d, span) == [(5, "C", "G", 15, False)]
    # a run of substitutions is one record, QUAL the least phred
    t = _t({**_identity(d, range(10)), (3, 0): "A", (4, 0): "C", (5, 0): "A"})
    assert E.records(t, d, span) == [(3, "TAC", "ACA", 13, False)]
    # no image in mid-contig: UNCOVERED, QUAL '.'
    t = _t(_identity(d, [0, 1, 2, 7, 8, 9]))
    recs = E.records(t, d, span)
    assert recs == [(2, "GTACG", "G", None, True)] and E.line("c", recs[0]) == "c\t3\t.\tGTACG\tG\t.\t.\tUNCOVERED\n"
    # a -r span starting past 0: the buffer at its head is uncovered, anchored on the base after it
    t = _t(_identity(d, range(6, 10)))
    assert E.records(t, d, (3, 9)) == [(3, "TACG", "G", None, True)]
    assert E.apply(E.records(t, d, (3, 9)), d, (3, 9)) == "GTAC"
    # every base deleted: no anchor on either side (the contig's consensus is empty, so the writer leaves it out)
    t = _t({(p, 0): "" for p in range(10)})
    assert E.records(t, d, span) == [(0, "ACGTACGTAC", "", 10, False)]
    # lower-case draft bases are identities of upper-case labels
    t = _t(_identity(d, range(10)))
    assert E.records(t, d.lower(), span) == []


def test_header_text_and_tabix_query(tmp_path):
    rng = np.random.default_rng(11)
    contigs, parts, want = [], [], {}
    for k, (preds, span) in enumerate(_contig_inputs()[1:]):
        name = "ctg%d" % (k + 1)
        ph = rng.integers(0, 101, preds[0].shape).astype(np.uint8)
        table = E.winners(preds[0], ph, *preds[1:])
        draft = _draft(table, span, rng, 0.95)
        contigs.append((name, len(draft) + 5))
        recs = E.records(table, draft, span)
        text = "".join(E.line(name, r) for r in recs).encode()
        lines = np.zeros(len(recs), EDIT_LINE)
        lines["pos"] = [r[0] for r in recs]; lines["ref_len"] = [len(r[1]) for r in recs]
        lines["text_len"] = [len(E.line(name, r)) for r in recs]
        parts.append(host_part(name, text, lines))
        want[name] = (recs, text)
    path = str(tmp_path / "edits.vcf.gz")
    write_edits_vcf(path, contigs + [("empty", 100)], parts)
    raw = open(path, "rb").read()
    body = gzip.decompress(raw).decode()
    head = edits_header(contigs + [("empty", 100)])
    assert body.startswith(head) and body[len(head):] == "".join(t.decode() for _, t in want.values())
    assert head.splitlines()[0] == "##fileformat=VCFv4.2" and "##contig=<ID=empty,length=100>" in head
    assert head.splitlines()[-1] == "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO"
    tbi = open(path + ".tbi", "rb").read()
    n = 0
    for name, (recs, _) in want.items():
        for r in recs:
            got = _tabix_query(tbi, raw, name, r[0], r[0] + len(r[1]))
            assert E.line(name, r).rstrip("\n") in got
            n += 1
    assert n > 50


def test_long_contig_gets_a_csi(tmp_path):
    lines = np.zeros(1, EDIT_LINE)
    text = b"big\t600000001\t.\tA\tC\t20\t.\t.\n"
    lines["pos"], lines["ref_len"], lines["text_len"] = 600000000, 1, len(text)
    path = str(tmp_path / "e.vcf.gz")
    write_edits_vcf(path, [("big", (1 << 29) + 10 ** 8)], [host_part("big", text, lines)])
    assert os.path.exists(path + ".csi") and not os.path.exists(path + ".tbi")
    assert gzip.decompress(open(path, "rb").read()).decode().endswith(text.decode())
