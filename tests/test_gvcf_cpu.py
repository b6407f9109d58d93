"""CPU: the gVCF rules as the numpy oracle states them (PL / GQ, blocks, record lines), the header, the owned windows and the
running record-end mask of the genome driver."""
import numpy as np

from pepper_b200.gvcf import GVCF_SEGMENT, gvcf_header, model_terms
from pepper_b200.vcf import format_vcf_line, vcf_header
from tests import gvcf_oracle as O


def _track(nr, na):
    return (np.asarray(nr, np.uint32) | (np.asarray(na, np.uint32) << 16)).astype(np.uint32)


def _seg(rows):
    s = np.zeros(len(rows), GVCF_SEGMENT)
    for i, r in enumerate(rows):
        s[i] = tuple(r) + (0,)
    return s


def test_model_terms_match_oracle():
    assert model_terms() == (O.A, O.B, O.H)


def test_pl_gq_hand_picked():
    pl, gq = O.pl_gq([0, 30, 0, 15, 5000], [0, 0, 30, 15, 0])
    assert pl[0].tolist() == [0, 0, 0] and gq[0] == 0                  # zero depth
    assert pl[1].tolist() == [0, 90, 900] and gq[1] == 90               # all reference
    assert pl[2].tolist() == [900, 90, 0] and gq[2] == 0                # all alternative
    assert pl[3].tolist() == [360, 0, 360] and gq[3] == 0               # het
    assert pl[4][0] == 0 and gq[4] == 99                                # depth 5,000 caps at 99


def test_blocks_rules():
    ref = b"ACGTNACGTAcgtacgtACG"
    nr = [30] * 20
    nr[6] = 3                     # a low-GQ position splits its band
    na = [0] * 20
    nr[15] = na[15] = 0           # DP 0
    seg = _seg([(0, 1000, 10, 0, 0), (10, 1010, 10, 10, 0)])
    # a record at 1002 with REF length 2; a record at the block's end (1009) whose span crosses the interval boundary
    masks = [(2, 4), (9, 11)]
    got = O.blocks(_track(nr, na), seg, masks, ref, ["chrT"])
    spans = [(p, n) for _, p, n, _ in got]
    assert spans == [(1000, 2), (1004, 2), (1006, 1), (1007, 2), (1011, 4), (1015, 1), (1016, 4)]
    lines = [t for *_, t in got]
    assert lines[1].split("\t")[3] == "N"                              # the first base of the block is N
    assert lines[0] == "chrT\t1001\t.\tA\t<*>\t.\t.\tEND=1002\tGT:GQ:MIN_DP:PL\t0/0:90:30:0,90,900\n"
    assert lines[5].endswith("\t./.:0:0:0,0,0\n") and "END=1016" in lines[5]
    assert lines[4].split("\t")[3] == "G"                              # lower-case reference upper-cased


def test_blocks_overlapping_records_and_min_gq_first():
    nr = [40, 20, 20, 40, 40, 40]
    na = [0] * 6
    seg = _seg([(0, 50, 6, 0, 0)])
    got = O.blocks(_track(nr, na), seg, [], b"AAAAAA", ["c"], binsize=100)
    assert len(got) == 1 and got[0][3].endswith("0/0:60:20:0,60,600\n")
    got = O.blocks(_track(nr, na), seg, [(1, 3), (2, 5)], b"AAAAAA", ["c"], binsize=100)
    assert [(p, n) for _, p, n, _ in got] == [(50, 1), (55, 1)]


def test_record_line_rewrite_round_trip():
    rec = dict(contig="chr1", start=99, alleles=["AT", "A", "ATT"], qual=31, filter="PASS", GT=[1, 2], AP=[0.5, 0.25],
               GQ=30, DP=20, AD=[7, 8], VAF=[0.35, 0.4], REP=0)
    line = format_vcf_line(rec) + "\n"
    got = O.record_line(line)
    f = got.rstrip("\n").split("\t")
    assert f[4] == "A,ATT,<*>"
    assert f[9].split(":") == ["1/2", "0.5,0.25,.", "30", "20", "7,8,.", "0.35,0.4,.", "0"]
    assert len(got) == len(line) + 10
    assert O.strip_record(got) == line


def test_header():
    fc = [("chr1", 1000), ("chr2", 500)]
    h = gvcf_header("S", fc).split("\n")
    v = vcf_header("S", fc).split("\n")
    assert h[-2] == v[-2] and h[-2].startswith("#CHROM")
    assert [x for x in h if x not in v] == h[-6:-2]
    assert h[-6] == '##ALT=<ID=*,Description="Represents allele(s) other than observed.">'
    assert "ID=END,Number=1,Type=Integer" in h[-5] and "ID=MIN_DP,Number=1" in h[-4] and "ID=PL,Number=G" in h[-3]
    assert all(x in h for x in v)


def test_owned_ends_and_mask_until():
    from pepper_b200.dist import owned_ends, mask_until

    class S:
        intervals = [(0, 100), (100, 150), (10, 60), (60, 90)]
        _first = [0, 2, 2, 4]                 # an empty contig in the middle
    assert owned_ends(S).tolist() == [99, 150, 59, 90]
    assert mask_until(np.array([120, -1, 40, 70]), [0, 0, 1, 1]).tolist() == [-1, 120, -1, 40]
