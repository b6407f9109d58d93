"""Seeded synthetic genome / read generator (SURVEY.md §8d).

Produces *post-get_reads* read records (what ``BAM_handler::get_reads`` hands to the
encoders: reads trimmed to the padded region, first op a match, upper-case bases;
reference ``pepper_variant/modules/cpp/bam_handler.cpp:115-451``) directly in the
structure-of-arrays layout of ``include/pepper_b200.h`` (4-bit BAM sequence codes,
one quality byte per base, ``len<<4|op`` CIGAR words).

Nothing here depends on the oracle or on the reference; tests, ``bench.py`` and
``__graft_entry__.smoke()`` all draw their inputs from this module.
"""
from __future__ import annotations

from dataclasses import dataclass, field
import numpy as np

NT16 = "=ACMGRSVTWYHKDBN"
CODE_OF = {c: i for i, c in enumerate(NT16)}
ACGT_CODES = np.array([1, 2, 4, 8], dtype=np.uint8)

OP_M, OP_I, OP_D, OP_N, OP_S, OP_H, OP_P, OP_EQ, OP_X = range(9)


@dataclass
class ReadBatch:
    """SoA read batch == pb_reads_t."""
    pos: np.ndarray          # int64 [n]
    seq_off: np.ndarray      # int64 [n+1]  (bases)
    cigar_off: np.ndarray    # int64 [n+1]
    flags: np.ndarray        # uint8 [n]    bit0 = reverse
    mapq: np.ndarray         # uint8 [n]
    seq: np.ndarray          # uint8 [ceil(nbases/2)] packed, high nibble first
    qual: np.ndarray         # uint8 [nbases]
    cigar: np.ndarray        # uint32 [nops]

    @property
    def n_reads(self) -> int:
        return int(self.pos.shape[0])

    @property
    def n_bases(self) -> int:
        return int(self.seq_off[-1])

    def codes(self) -> np.ndarray:
        """Unpacked 4-bit codes, one per base."""
        n = self.n_bases
        out = np.empty(2 * self.seq.shape[0], dtype=np.uint8)
        out[0::2] = self.seq >> 4
        out[1::2] = self.seq & 15
        return out[:n]


@dataclass
class RegionTable:
    """Array-of-struct region table == pb_region_t[] (8 x int64 per region)."""
    table: np.ndarray                      # int64 [n_regions, 8]
    ref: np.ndarray                        # uint8 concatenated reference strings
    FIELDS = ("ref_start", "ref_end", "cand_start", "cand_end", "ref_off", "ref_len", "read_begin", "read_end")

    @property
    def n_regions(self) -> int:
        return int(self.table.shape[0])

    def col(self, name: str) -> np.ndarray:
        return self.table[:, self.FIELDS.index(name)]

    def genomic_bases(self) -> int:
        """TOTAL BASES as the reference logs it: sum(interval_end - interval_start)
        (pepper_variant ImageGenerationUI.py:316,323)."""
        return int((self.col("cand_end") - self.col("cand_start")).sum())


def pack_codes(codes: np.ndarray) -> np.ndarray:
    n = codes.shape[0]
    if n & 1:
        codes = np.concatenate([codes, np.zeros(1, dtype=np.uint8)])
    return ((codes[0::2] << 4) | codes[1::2]).astype(np.uint8)


def concat_batches(batches: list[ReadBatch]) -> ReadBatch:
    """Concatenate read batches (re-packing the 4-bit sequence at odd boundaries)."""
    pos = np.concatenate([b.pos for b in batches])
    flags = np.concatenate([b.flags for b in batches])
    mapq = np.concatenate([b.mapq for b in batches])
    qual = np.concatenate([b.qual for b in batches])
    cigar = np.concatenate([b.cigar for b in batches])
    codes = np.concatenate([b.codes() for b in batches])
    seq_off = [np.zeros(1, dtype=np.int64)]
    cig_off = [np.zeros(1, dtype=np.int64)]
    sb = 0
    cb = 0
    for b in batches:
        seq_off.append(b.seq_off[1:] + sb)
        cig_off.append(b.cigar_off[1:] + cb)
        sb += b.n_bases
        cb += int(b.cigar_off[-1])
    return ReadBatch(pos, np.concatenate(seq_off), np.concatenate(cig_off), flags, mapq,
                     pack_codes(codes), qual, cigar)


def make_batch(reads: list[dict]) -> ReadBatch:
    """Build a ReadBatch from explicit records (used by the hand-written KATs).
    Each record: pos, seq (str), qual (list[int] or int), cigar [(op,len),...], reverse, mapq."""
    pos, flags, mapq, codes, quals, cig = [], [], [], [], [], []
    seq_off, cig_off = [0], [0]
    for r in reads:
        s = r["seq"]
        q = r.get("qual", 30)
        if isinstance(q, int):
            q = [q] * len(s)
        assert len(q) == len(s)
        pos.append(r["pos"])
        flags.append(1 if r.get("reverse", False) else 0)
        mapq.append(r.get("mapq", 60))
        codes.extend(CODE_OF.get(c, 15) for c in s.upper())
        quals.extend(q)
        cig.extend((l << 4) | op for op, l in r["cigar"])
        seq_off.append(len(codes))
        cig_off.append(len(cig))
    return ReadBatch(np.array(pos, dtype=np.int64), np.array(seq_off, dtype=np.int64),
                     np.array(cig_off, dtype=np.int64), np.array(flags, dtype=np.uint8),
                     np.array(mapq, dtype=np.uint8), pack_codes(np.array(codes, dtype=np.uint8)),
                     np.array(quals, dtype=np.uint8), np.array(cig, dtype=np.uint32))


def make_reference(length: int, seed: int, hp_frac: float = 0.05, n_frac: float = 0.0) -> np.ndarray:
    """i.i.d. ACGT reference with homopolymer runs (len 5-15) covering ~hp_frac of it and
    optional N blocks; returned as ASCII uint8."""
    rng = np.random.default_rng(seed)
    ref = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, size=length)].copy()
    n_runs = int(length * hp_frac / 10)
    starts = rng.integers(0, max(1, length - 16), size=n_runs)
    lens = rng.integers(5, 16, size=n_runs)
    for s, l in zip(starts, lens):
        ref[s:s + l] = ref[s]
    if n_frac > 0:
        n_blocks = max(1, int(length * n_frac / 50))
        for s in rng.integers(0, max(1, length - 60), size=n_blocks):
            ref[s:s + 50] = ord("N")
    return ref


@dataclass
class Platform:
    name: str
    mean_len: float
    sigma: float
    min_len: int
    max_len: int
    p_mm: float
    p_ins: float
    p_del: float
    hp_mult: float
    indel_geo_p: float
    q_mean: float
    q_sd: float
    q_lo: int
    q_hi: int
    lognormal: bool


ONT = Platform("ont_r9", 9000.0, 0.6, 1000, 100000, 0.015, 0.012, 0.020, 3.0, 0.7, 18.0, 7.0, 1, 40, True)
HIFI = Platform("hifi", 15000.0, 2000.0, 1000, 30000, 0.0005, 0.001, 0.001, 3.0, 0.7, 35.0, 8.0, 2, 93, False)


def _truth_variants(rng, ref: np.ndarray, snp_rate=1e-3, indel_rate=1.25e-4):
    """Diploid truth: per-haplotype SNP alt code (0 = none), deletion length starting AFTER pos,
    insertion length AFTER pos.  60 % het."""
    L = ref.shape[0]
    hap_snp = np.zeros((2, L), dtype=np.uint8)
    hap_del = np.zeros((2, L), dtype=np.int32)
    hap_ins = np.zeros((2, L), dtype=np.int32)
    n_snp = rng.poisson(L * snp_rate)
    for p in rng.integers(0, L, size=n_snp):
        alt = ACGT_CODES[rng.integers(0, 4)]
        haps = (0, 1) if rng.random() > 0.6 else (int(rng.integers(0, 2)),)
        for h in haps:
            hap_snp[h, p] = alt
    n_indel = rng.poisson(L * indel_rate)
    for p in rng.integers(0, max(1, L - 12), size=n_indel):
        l = int(min(10, rng.geometric(0.4)))
        haps = (0, 1) if rng.random() > 0.6 else (int(rng.integers(0, 2)),)
        for h in haps:
            if rng.random() < 0.5:
                hap_del[h, p] = l
            else:
                hap_ins[h, p] = l
    return hap_snp, hap_del, hap_ins


def _ascii_to_code(ref: np.ndarray) -> np.ndarray:
    lut = np.full(256, 15, dtype=np.uint8)
    for c, i in CODE_OF.items():
        lut[ord(c)] = i
    return lut[ref]


def simulate_region_reads(ref: np.ndarray, ref_start: int, coverage: float, platform: Platform, seed: int,
                          p_soft_tail: float = 0.02, p_n_base: float = 1e-4, p_low_mapq: float = 0.01,
                          hp_mask: np.ndarray | None = None, truth=()) -> ReadBatch:
    """Reads over a padded region whose reference string is `ref` (positions ref_start..ref_start+len-1),
    each already trimmed to the region as get_reads would (first op M, inside [ref_start, ref_end]).  `truth`: variants placed
    on top of the random ones, (position, "snp" / "del" / "ins", alt base or length, haplotypes); the random draws are
    unchanged by it."""
    rng = np.random.default_rng(seed)
    L = ref.shape[0]
    refc = _ascii_to_code(ref)
    hap_snp, hap_del, hap_ins = _truth_variants(rng, ref)
    for p, kind, v, haps in truth:
        for h in haps:
            if kind == "snp":
                hap_snp[h, p - ref_start] = CODE_OF[v]
            else:
                (hap_del if kind == "del" else hap_ins)[h, p - ref_start] = int(v)
    if hp_mask is None:
        same = np.zeros(L, dtype=bool)
        same[1:] = ref[1:] == ref[:-1]
        run = same.copy()
        run[:-1] |= same[1:]
        hp_mask = run
    # how many reads: coverage * L / mean_len, with starts so that edges are covered evenly
    if platform.lognormal:
        draw_len = lambda n: np.clip(rng.lognormal(np.log(platform.mean_len), platform.sigma, n),
                                     platform.min_len, platform.max_len).astype(np.int64)
    else:
        draw_len = lambda n: np.clip(rng.normal(platform.mean_len, platform.sigma, n),
                                     platform.min_len, platform.max_len).astype(np.int64)
    exp_len = float(draw_len(2000).mean())
    n_reads = max(1, int(round(coverage * (L + exp_len) / exp_len)))
    lens = draw_len(n_reads)
    starts = rng.integers(-int(exp_len), L, size=n_reads)
    order = np.argsort(starts, kind="stable")
    starts, lens = starts[order], lens[order]

    pos_l, flag_l, mapq_l, code_l, qual_l, cig_l = [], [], [], [], [], []
    seq_off, cig_off = [0], [0]
    nb = 0
    nc = 0
    for s, ln in zip(starts, lens):
        a = max(0, int(s))
        b = min(L, int(s + ln))
        if b - a < 1:
            continue
        n = b - a
        hap = int(rng.integers(0, 2))
        mult = np.where(hp_mask[a:b], platform.hp_mult, 1.0)
        u = rng.random(n)
        mm = u < platform.p_mm
        u2 = rng.random(n)
        ins_len = np.where(u2 < platform.p_ins * mult, rng.geometric(platform.indel_geo_p, n), 0).astype(np.int64)
        u3 = rng.random(n)
        del_start = u3 < platform.p_del * mult
        del_len = np.where(del_start, rng.geometric(platform.indel_geo_p, n), 0).astype(np.int64)
        # haplotype truth
        ins_len = np.maximum(ins_len, hap_ins[hap, a:b])
        del_len = np.maximum(del_len, hap_del[hap, a:b])
        # deleted positions: a deletion "after pos i" removes i+1 .. i+len
        dmark = np.zeros(n + 1, dtype=np.int64)
        idx = np.nonzero(del_len)[0]
        if idx.size:
            st = np.minimum(idx + 1, n)
            en = np.minimum(idx + 1 + del_len[idx], n)
            np.add.at(dmark, st, 1)
            np.add.at(dmark, en, -1)
        deleted = np.cumsum(dmark[:n]) > 0
        deleted[0] = False                       # trimmed reads start on a match
        ins_len[deleted] = 0                     # keep I after kept bases only
        ins_len[n - 1] = ins_len[n - 1] if rng.random() < 0.5 else 0
        # bases at kept positions
        base = refc[a:b].copy()
        hs = hap_snp[hap, a:b]
        base = np.where(hs > 0, hs, base)
        alt = ACGT_CODES[rng.integers(0, 4, n)]
        base = np.where(mm, alt, base)           # may equal the ref base: then it is simply a match
        base = np.where(rng.random(n) < p_n_base, 15, base).astype(np.uint8)
        # token stream: per position one token (M or D) followed by ins_len I tokens
        cnt = 1 + ins_len
        tot = int(cnt.sum())
        first = np.cumsum(cnt) - cnt
        tok = np.full(tot, OP_I, dtype=np.uint8)
        tok[first] = np.where(deleted, OP_D, OP_M)
        codes = ACGT_CODES[rng.integers(0, 4, tot)]
        codes[first] = base
        keep = tok != OP_D
        read_codes = codes[keep]
        # run-length encode the tokens into a CIGAR
        chg = np.nonzero(np.diff(tok))[0] + 1
        run_st = np.concatenate([[0], chg])
        run_len = np.diff(np.concatenate([run_st, [tot]]))
        ops = tok[run_st].astype(np.uint32)
        cig = (run_len.astype(np.uint32) << 4) | ops
        # optional trailing soft clip (kept by get_reads when inside the region)
        if rng.random() < p_soft_tail and b < L:
            sl = int(rng.integers(1, 30))
            read_codes = np.concatenate([read_codes, ACGT_CODES[rng.integers(0, 4, sl)]])
            cig = np.concatenate([cig, np.array([(sl << 4) | OP_S], dtype=np.uint32)])
        m = read_codes.shape[0]
        q = np.clip(np.rint(rng.normal(platform.q_mean, platform.q_sd, m)), platform.q_lo, platform.q_hi).astype(np.uint8)
        pos_l.append(ref_start + a)
        flag_l.append(int(rng.random() < 0.5))
        mapq_l.append(int(rng.integers(0, 5)) if rng.random() < p_low_mapq else 60)
        code_l.append(read_codes)
        qual_l.append(q)
        cig_l.append(cig)
        nb += m
        nc += cig.shape[0]
        seq_off.append(nb)
        cig_off.append(nc)
    codes = np.concatenate(code_l) if code_l else np.zeros(0, dtype=np.uint8)
    return ReadBatch(np.array(pos_l, dtype=np.int64), np.array(seq_off, dtype=np.int64),
                     np.array(cig_off, dtype=np.int64), np.array(flag_l, dtype=np.uint8),
                     np.array(mapq_l, dtype=np.uint8), pack_codes(codes),
                     np.concatenate(qual_l) if qual_l else np.zeros(0, dtype=np.uint8),
                     np.concatenate(cig_l) if cig_l else np.zeros(0, dtype=np.uint32))


def make_variant_workload(n_regions: int, region_size: int, coverage: float, platform: Platform, seed: int,
                          safe_bases: int = 100, contig_start: int = 1_000_000, n_frac: float = 0.0):
    """Regions tiled as pepper_variant ImageGenerationUI.py:307-316 does (adjacent intervals share their
    boundary), each padded by REGION_SAFE_BASES (AlignmentSummarizer.py:181-182).
    Returns (ReadBatch, RegionTable)."""
    contig_len = n_regions * region_size + 2 * safe_bases
    genome = make_reference(contig_len, seed, n_frac=n_frac)
    batches, rows, refs = [], [], []
    rb = 0
    roff = 0
    for r in range(n_regions):
        s = contig_start + safe_bases + r * region_size      # interval start
        e = s + region_size                                   # interval end (shared with the next start)
        rs, re_ = s - safe_bases, e + safe_bases
        g0 = rs - contig_start
        ref = genome[g0:g0 + (re_ - rs + 1)]
        b = simulate_region_reads(ref, rs, coverage, platform, seed * 1000003 + r)
        batches.append(b)
        rows.append((rs, re_, s, e, roff, ref.shape[0], rb, rb + b.n_reads))
        refs.append(ref)
        rb += b.n_reads
        roff += ref.shape[0]
    reads = concat_batches(batches)
    return reads, RegionTable(np.array(rows, dtype=np.int64), np.concatenate(refs))


def make_polish_workload(n_regions: int, coverage: float, platform: Platform, seed: int,
                         chunk: int = 1000, overlap: int = 100, contig_start: int = 0):
    """Regions tiled as pepper ImageGenerationUI.py:269-272: (max(s,pos-100), min(e,pos+1000+100)).
    Returns (ReadBatch, RegionTable); the polish encoder takes no reference string."""
    contig_len = n_regions * chunk
    genome = make_reference(contig_len + 1, seed)
    batches, rows = [], []
    rb = 0
    for r in range(n_regions):
        p = contig_start + r * chunk
        rs = max(contig_start, p - overlap)
        re_ = min(contig_start + contig_len, p + chunk + overlap)
        ref = genome[rs - contig_start: re_ - contig_start + 1]
        b = simulate_region_reads(ref, rs, coverage, platform, seed * 1000003 + r)
        batches.append(b)
        rows.append((rs, re_, p, min(contig_start + contig_len, p + chunk), 0, 0, rb, rb + b.n_reads))
        rb += b.n_reads
    reads = concat_batches(batches)
    return reads, RegionTable(np.array(rows, dtype=np.int64), np.zeros(1, dtype=np.uint8))


def tile_workload(reads: ReadBatch, regions: RegionTable, times: int):
    """Replicate a workload `times` times (bench.py scales a generated block up to chr20 size with it;
    each copy is shifted along the contig so positions stay distinct)."""
    if times <= 1:
        return reads, regions
    span = int(regions.col("ref_end").max() - regions.col("ref_start").min() + 1)
    batches, tabs = [], []
    for t in range(times):
        b = ReadBatch(reads.pos + t * span, reads.seq_off, reads.cigar_off, reads.flags, reads.mapq,
                      reads.seq, reads.qual, reads.cigar)
        batches.append(b)
        tab = regions.table.copy()
        tab[:, 0:4] += t * span
        tab[:, 4] += t * regions.ref.shape[0] if regions.ref.shape[0] > 1 else 0
        tab[:, 6:8] += t * reads.n_reads
        tabs.append(tab)
    ref = np.tile(regions.ref, times) if regions.ref.shape[0] > 1 else regions.ref
    return concat_batches(batches), RegionTable(np.concatenate(tabs), ref)


def region_batch(reads: ReadBatch, regions: RegionTable, r: int):
    """The reads / table / reference of region r alone (re-based offsets)."""
    row = regions.table[r].copy()
    rb, re_ = int(row[6]), int(row[7])
    b0, b1 = int(reads.seq_off[rb]), int(reads.seq_off[re_])
    c0, c1 = int(reads.cigar_off[rb]), int(reads.cigar_off[re_])
    codes = reads.codes()[b0:b1]
    sub = ReadBatch(reads.pos[rb:re_].copy(), reads.seq_off[rb:re_ + 1] - b0, reads.cigar_off[rb:re_ + 1] - c0,
                    reads.flags[rb:re_].copy(), reads.mapq[rb:re_].copy(), pack_codes(codes), reads.qual[b0:b1].copy(),
                    reads.cigar[c0:c1].copy())
    ref = regions.ref[int(row[4]):int(row[4] + row[5])].copy() if regions.ref.shape[0] > 1 else regions.ref
    row[4] = 0
    row[6], row[7] = 0, re_ - rb
    return sub, RegionTable(row[None, :], ref)


def take_reads(reads: ReadBatch, indices) -> ReadBatch:
    """Gather reads in the given order (down-sampled / permuted read lists)."""
    idx = np.asarray(indices, dtype=np.int64)
    codes = reads.codes()
    lens = reads.seq_off[idx + 1] - reads.seq_off[idx]
    clens = reads.cigar_off[idx + 1] - reads.cigar_off[idx]
    seq_off = np.zeros(idx.shape[0] + 1, dtype=np.int64)
    cig_off = np.zeros(idx.shape[0] + 1, dtype=np.int64)
    np.cumsum(lens, out=seq_off[1:])
    np.cumsum(clens, out=cig_off[1:])
    pick = [np.arange(reads.seq_off[i], reads.seq_off[i + 1]) for i in idx]
    cpick = [np.arange(reads.cigar_off[i], reads.cigar_off[i + 1]) for i in idx]
    bi = np.concatenate(pick).astype(np.int64) if pick else np.zeros(0, dtype=np.int64)
    ci = np.concatenate(cpick).astype(np.int64) if cpick else np.zeros(0, dtype=np.int64)
    return ReadBatch(reads.pos[idx].copy(), seq_off, cig_off, reads.flags[idx].copy(), reads.mapq[idx].copy(),
                     pack_codes(codes[bi]), reads.qual[bi].copy(), reads.cigar[ci].copy())


def ont_params() -> dict:
    """--ont_r9_guppy5_sup image-generation thresholds, SetParameters.py:16-37."""
    return dict(min_snp_baseq=1, min_indel_baseq=1, snp_freq_threshold=0.10, insert_freq_threshold=0.15,
                delete_freq_threshold=0.15, min_coverage_threshold=3, snp_candidate_freq_threshold=0.10,
                indel_candidate_freq_threshold=0.10, candidate_support_threshold=2, skip_indels=0)


def hifi_params() -> dict:
    """--hifi thresholds, SetParameters.py:180-201."""
    return dict(min_snp_baseq=10, min_indel_baseq=10, snp_freq_threshold=0.10, insert_freq_threshold=0.12,
                delete_freq_threshold=0.10, min_coverage_threshold=2, snp_candidate_freq_threshold=0.10,
                indel_candidate_freq_threshold=0.10, candidate_support_threshold=2, skip_indels=0)


# ------------------------------------------------------------------ raw alignment records (input of get_reads, row a2)
FLAG_REVERSE, FLAG_UNMAP, FLAG_SECONDARY, FLAG_QCFAIL, FLAG_DUP, FLAG_SUPP = 16, 4, 256, 512, 1024, 2048


@dataclass
class RecordBatch:
    """SoA batch of alignment records as htslib hands them to BAM_handler::get_reads == pb_records_t
    (coordinate-sorted, one contig; BAM-native packing)."""
    pos: np.ndarray          # int64 [n]
    seq_off: np.ndarray      # int64 [n+1]
    cigar_off: np.ndarray    # int64 [n+1]
    flag: np.ndarray         # uint16 [n]   SAM FLAG
    mapq: np.ndarray         # uint8 [n]
    seq: np.ndarray          # uint8 packed
    qual: np.ndarray         # uint8 [nbases]
    cigar: np.ndarray        # uint32 [nops]

    @property
    def n_records(self) -> int:
        return int(self.pos.shape[0])

    @property
    def n_bases(self) -> int:
        return int(self.seq_off[-1])


def make_records(records: list[dict]) -> RecordBatch:
    """Explicit records for the hand-written KATs: pos, seq, qual, cigar [(op,len)...], flag, mapq."""
    b = make_batch([dict(r, reverse=False) for r in records])
    flag = np.array([r.get("flag", 0) for r in records], dtype=np.uint16)
    return RecordBatch(b.pos, b.seq_off, b.cigar_off, flag, b.mapq, b.seq, b.qual, b.cigar)


def simulate_contig_records(contig_len: int, coverage: float, platform: Platform, seed: int, contig_start: int = 0,
                            p_clip_head: float = 0.3, p_hard: float = 0.05, p_filtered: float = 0.06, truth=()):
    """Whole-contig alignment records: the read model of simulate_region_reads over the full contig, then decorated the
    way an aligner's output is — leading soft / hard clips, trailing hard clips, SAM FLAG bits (reverse, secondary,
    supplementary, duplicate, QC-fail, unmapped).  Returns (RecordBatch, genome uint8 ASCII)."""
    genome = make_reference(contig_len, seed)
    b = simulate_region_reads(genome, contig_start, coverage, platform, seed * 7919 + 13, truth=truth)
    rng = np.random.default_rng(seed + 991)
    codes = b.codes()
    pos, flag, code_l, qual_l, cig_l = [], [], [], [], []
    seq_off, cig_off = [0], [0]
    for r in range(b.n_reads):
        c = codes[b.seq_off[r]:b.seq_off[r + 1]]
        q = b.qual[b.seq_off[r]:b.seq_off[r + 1]]
        cg = b.cigar[b.cigar_off[r]:b.cigar_off[r + 1]]
        head = []
        if rng.random() < p_clip_head:
            sl = int(rng.integers(1, 40))
            c = np.concatenate([ACGT_CODES[rng.integers(0, 4, sl)], c])
            q = np.concatenate([rng.integers(2, 40, sl).astype(np.uint8), q])
            head.append((sl << 4) | OP_S)
        if rng.random() < p_hard:
            head.insert(0, (int(rng.integers(1, 500)) << 4) | OP_H)
        tail = [(int(rng.integers(1, 500)) << 4) | OP_H] if rng.random() < p_hard else []
        cg = np.concatenate([np.array(head, dtype=np.uint32), cg, np.array(tail, dtype=np.uint32)]).astype(np.uint32)
        f = FLAG_REVERSE if b.flags[r] & 1 else 0
        if rng.random() < p_filtered:
            f |= int(rng.choice([FLAG_UNMAP, FLAG_SECONDARY, FLAG_QCFAIL, FLAG_DUP, FLAG_SUPP]))
        pos.append(int(b.pos[r])); flag.append(f); code_l.append(c); qual_l.append(q); cig_l.append(cg)
        seq_off.append(seq_off[-1] + c.shape[0]); cig_off.append(cig_off[-1] + cg.shape[0])
    allc = np.concatenate(code_l) if code_l else np.zeros(0, dtype=np.uint8)
    rec = RecordBatch(np.array(pos, dtype=np.int64), np.array(seq_off, dtype=np.int64), np.array(cig_off, dtype=np.int64),
                      np.array(flag, dtype=np.uint16), b.mapq.copy(), pack_codes(allc),
                      np.concatenate(qual_l) if qual_l else np.zeros(0, dtype=np.uint8),
                      np.concatenate(cig_l) if cig_l else np.zeros(0, dtype=np.uint32))
    return rec, genome
