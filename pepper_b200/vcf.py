"""Site-level half of `pepper_variant find_candidates` (SURVEY 8f row f2) on the arrays the GPU path produces:

  * merge of the selected records per (contig, position) with the (ref, alt) de-duplication that removes the records adjacent
    intervals emit twice at their shared boundary      == CandidateFinder.py:547-581
  * per site: order by (genotype, genotype probability) descending, keep `allowed_multiallelics`, extend every allele to the
    longest reference allele, genotype / GQ / depth / supports                == VCFWriter.candidate_list_to_variant, VcfWriter.py:48-138
  * QUAL = max(1, int(-10 log10(max(1e-9, 1 - p)))), quality cut-offs, filter, which VCF a record goes to
                                                                              == VCFWriter.write_vcf_records, VcfWriter.py:140-218

The per-record decisions (genotype, repeat context, Margin / DeepVariant lists, delete ref/alt swap) come from the CUDA kernel
behind `candidates.select_flags`; everything here is array code over those flags (stable sort, unique, segmented min / any /
count via reduceat) plus one pass that formats the records.  Output: one dict per VCF record with the keyword arguments the
reference hands to pysam's `new_record` and `files`, the VCFs it is written to — a pysam writer consumes them unchanged."""
from __future__ import annotations

import ctypes as C
import math
import struct

import numpy as np

from . import _lib
from .abi import PB_ERR_CAPACITY
from .candidates import F_DV, F_REPEAT, F_SWAP, select_flags
from .synth import RegionTable

# --ont_r9_guppy5_sup defaults of find_candidates, pepper_variant/modules/argparse/SetParameters.py:40-65
VCF_OPTIONS_ONT = dict(allowed_multiallelics=4, snp_q_cutoff=20, indel_q_cutoff=15, snp_q_cutoff_in_lc=20, indel_q_cutoff_in_lc=10)
GT_OF = ([0, 0], [0, 1], [1, 1])


def _strlen(a: np.ndarray) -> np.ndarray:
    return np.char.str_len(a).astype(np.int64)


def assemble_sites(contig: str, positions, region_of, depths, freqs, keys_raw, probs, flags, geno, regions: RegionTable,
                   options: dict) -> list[dict]:
    """Records of ONE contig (arrays in the order the encoder produced them) -> VCF record dicts in position order."""
    sel = np.flatnonzero(np.asarray(flags) & F_DV)
    if sel.shape[0] == 0:
        return []
    pos = np.asarray(positions, dtype=np.int64)[sel]
    reg = np.asarray(region_of, dtype=np.int64)[sel]
    fl = np.asarray(flags)[sel]
    g = np.asarray(geno, dtype=np.int64)[sel]
    pb = np.asarray(probs, dtype=np.float32)[sel].astype(np.float64)
    dep = np.asarray(depths, dtype=np.int64)[sel]
    sup = np.asarray(freqs, dtype=np.int64)[sel]
    tab = regions.table
    ref_base = np.char.upper(regions.ref[tab[reg, 4] + pos - tab[reg, 0]].astype(np.uint8).view("S1"))
    kr = np.ascontiguousarray(np.asarray(keys_raw, dtype=np.uint8)[sel][:, 1:63]).view("S62")[:, 0]     # the allele = key[1:]
    swap = (fl & F_SWAP) != 0
    ref = np.where(swap, kr, ref_base.astype("S62"))
    alt = np.where(swap, ref_base.astype("S62"), kr)
    pv = pb[np.arange(pb.shape[0]), g]
    non_alt = np.maximum(pb[:, 1], pb[:, 2])
    rep = (fl & F_REPEAT) != 0

    # ---- sorted by position (stable), first record of every (position, ref, alt)                      CandidateFinder.py:547-574
    o = np.argsort(pos, kind="stable")
    st = np.zeros(o.shape[0], dtype=[("pos", np.int64), ("ref", "S62"), ("alt", "S62")])
    st["pos"], st["ref"], st["alt"] = pos[o], ref[o], alt[o]
    _, first = np.unique(st, return_index=True)
    o = o[np.sort(first)]
    pos, ref, alt, g, pv, pb, dep, sup, non_alt, rep = (a[o] for a in (pos, ref, alt, g, pv, pb, dep, sup, non_alt, rep))
    n = pos.shape[0]
    site = np.concatenate([[0], np.cumsum(pos[1:] != pos[:-1])])

    # ---- per site: by (genotype, probability) descending, ties in arrival order; keep allowed_multiallelics   VcfWriter.py:49-51
    o = np.lexsort((np.arange(n), -pv, -g, site))
    pos, ref, alt, g, pv, pb, dep, sup, non_alt, rep, site = (a[o] for a in (pos, ref, alt, g, pv, pb, dep, sup, non_alt, rep, site))
    start_all = np.flatnonzero(np.concatenate([[True], site[1:] != site[:-1]]))
    rank = np.arange(n) - np.repeat(start_all, np.diff(np.concatenate([start_all, [n]])))
    keep = rank < int(options["allowed_multiallelics"])
    pos, ref, alt, g, pv, pb, dep, sup, non_alt, rep, site = (a[keep] for a in (pos, ref, alt, g, pv, pb, dep, sup, non_alt, rep, site))
    n = pos.shape[0]
    s0 = np.flatnonzero(np.concatenate([[True], site[1:] != site[:-1]]))
    cnt = np.diff(np.concatenate([s0, [n]]))

    # ---- segmented reductions                                                                         VcfWriter.py:92-135
    s_depth = np.minimum.reduceat(dep, s0)
    s_rep = np.maximum.reduceat(rep.astype(np.int8), s0) > 0
    nz_min = np.minimum.reduceat(np.where(g != 0, pv, np.inf), s0)
    gt_qual = np.where(g[s0] != 0, nz_min, non_alt[s0])          # first of a site has the largest genotype: non-zero ones come first
    n_hom = np.add.reduceat((g == 2).astype(np.int64), s0)
    n_het = np.add.reduceat((g == 1).astype(np.int64), s0)
    rlen, alen = _strlen(ref), _strlen(alt)
    max_rlen = np.maximum.reduceat(rlen, s0)
    ragged = np.flatnonzero(np.minimum.reduceat(rlen, s0) != max_rlen)
    ref_s = [r.decode() for r in ref]
    alt_s = [a.decode() for a in alt]
    for k in ragged:                                             # extend to the longest reference allele        VcfWriter.py:53-74
        a, b = int(s0[k]), int(s0[k] + cnt[k])
        longest = ref_s[a + int(np.argmax(rlen[a:b]))]
        for i in range(a, b):
            need = len(longest) - len(ref_s[i])
            if need > 0:
                ref_s[i] += longest[-need:]
                alt_s[i] += longest[-need:]
    # ---- records                                                                                      VcfWriter.py:140-218
    out = []
    last_position = -1
    snp_cut, indel_cut = options["snp_q_cutoff"], options["indel_q_cutoff"]
    snp_cut_lc, indel_cut_lc = options["snp_q_cutoff_in_lc"], options["indel_q_cutoff_in_lc"]
    for k in range(s0.shape[0]):
        a, b = int(s0[k]), int(s0[k] + cnt[k])
        ref_start = int(pos[a])
        if ref_start == last_position:
            continue
        last_position = ref_start
        ref_seq = ref_s[a]
        alleles = alt_s[a:b]
        nh, nm = int(n_het[k]), int(n_hom[k])
        if nm == 1 and nh == 0:
            gt = [1, 1]
        elif nm == 0 and nh == 1:
            gt = [0, 1]
        elif nm == 0 and nh == 2:
            gt = [1, 2]
        else:
            gt = [0, 0]
        depth = int(s_depth[k])
        gp = float(gt_qual[k])
        qual = max(1, int(-10 * math.log10(max(0.000000001, 1.0 - gp))))
        in_rep = bool(s_rep[k])
        is_snp = max(len(ref_seq), max(len(x) for x in alleles)) == 1
        if is_snp:
            failed = (not in_rep and qual <= snp_cut) or (in_rep and qual <= snp_cut_lc)
        else:
            failed = (not in_rep and qual <= indel_cut) or (in_rep and qual <= indel_cut_lc)
        selected = gt == [0, 0] or failed
        ad = [int(x) for x in sup[a:b]]
        files = ["full"] + (["variant_calling_snp" if is_snp else "variant_calling_indel", "variant_calling"] if selected else ["pepper"])
        out.append(dict(contig=str(contig), start=ref_start, stop=ref_start + len(ref_seq), qual=qual,
                        filter="refCall" if gt == [0, 0] else "PASS", alleles=(ref_seq,) + tuple(alleles), GT=gt,
                        AP=[float(x) for x in non_alt[a:b]], GQ=qual, DP=depth, AD=ad, VAF=[round(x / max(1, depth), 3) for x in ad],
                        REP="1" if in_rep else "0", files=files))
    return out


def find_site_records(contig: str, positions, region_of, depths, freqs, keys_raw, probs, regions: RegionTable, options: dict,
                      vcf_options: dict | None = None) -> list[dict]:
    """predictions -> VCF records of one contig: the CUDA per-record selection + the site assembly."""
    flags, geno = select_flags(positions, region_of, depths, freqs, keys_raw, probs, regions, options)
    return assemble_sites(contig, positions, region_of, depths, freqs, keys_raw, probs, flags, geno, regions, vcf_options or VCF_OPTIONS_ONT)


def format_vcf_line(rec: dict, sample_fields=("GT", "AP", "GQ", "DP", "AD", "VAF", "REP")) -> str:
    """One VCF 4.2 data line for a record dict (text form of what pysam writes; positions are 1-based in VCF)."""
    def fmt(v):
        if isinstance(v, (list, tuple)):
            return ",".join(fmt(x) for x in v)
        if isinstance(v, float):
            return ("%.6g" % v)
        return str(v)
    sample = [("/".join(str(x) for x in rec["GT"]))] + [fmt(rec[f]) for f in sample_fields[1:]]
    return "\t".join([rec["contig"], str(rec["start"] + 1), ".", rec["alleles"][0], ",".join(rec["alleles"][1:]), str(rec["qual"]),
                      rec["filter"], ".", ":".join(sample_fields), ":".join(sample)])


# ---------------------------------------------------------------------------------------------------------------------------
# Whole-genome VCF output: the GPU turns each contig's records into VCF text (pb_variant_vcf_*); the writer below orders the lines
# as VCFWriter.write_vcf_records does, splits them into the reference's five files, and writes BGZF + a tabix index.

class PbVcfOptions(C.Structure):
    _fields_ = [("allowed_multiallelics", C.c_int32), ("reserved", C.c_int32), ("snp_q_cutoff", C.c_double),
                ("indel_q_cutoff", C.c_double), ("snp_q_cutoff_in_lc", C.c_double), ("indel_q_cutoff_in_lc", C.c_double)]


class PbVcfJob(C.Structure):
    _fields_ = [("contig_of_region", C.c_void_p), ("names", C.c_void_p), ("name_off", C.c_void_p), ("vaf_table", C.c_void_p),
                ("window", C.c_void_p)]


# pb_vcf_line_t; cls: 0 = pepper, 1 = variant-calling SNP, 2 = variant-calling indel
VCF_LINE = np.dtype([("pos", np.int64), ("text_off", np.int64), ("contig", np.int32), ("ref_len", np.int32), ("cls", np.int32),
                     ("text_len", np.int32)])
CLASS_PEPPER, CLASS_VC_SNP, CLASS_VC_INDEL = 0, 1, 2
VCF_FILES = ("PEPPER_VARIANT_FULL", "PEPPER_VARIANT_OUTPUT_PEPPER", "PEPPER_VARIANT_OUTPUT_VARIANT_CALLING",
             "PEPPER_VARIANT_OUTPUT_VARIANT_CALLING_SNPs", "PEPPER_VARIANT_OUTPUT_VARIANT_CALLING_INDEL")
_VAF_TABLE = None


def vaf_table() -> np.ndarray:
    """[256, 256, 8] NUL-padded text of round(ad / max(1, dp), 3) as format_vcf_line prints it, at [ad, dp] (AD and DP are the
    encoder's uint8 counts).  Python's rounding of that quotient is kept on the host rather than restated on the device."""
    global _VAF_TABLE
    if _VAF_TABLE is None:
        t = np.zeros((256, 256), dtype="S8")
        for ad in range(256):
            t[ad] = [("%.6g" % round(ad / max(1, dp), 3)).encode() for dp in range(256)]
        _VAF_TABLE = np.ascontiguousarray(t).view(np.uint8).reshape(256, 256, 8)
    return _VAF_TABLE


def vcf_options(options: dict) -> PbVcfOptions:
    return PbVcfOptions(int(options["allowed_multiallelics"]), 0, *(float(options[k]) for k in
                        ("snp_q_cutoff", "indel_q_cutoff", "snp_q_cutoff_in_lc", "indel_q_cutoff_in_lc")))


def _names_blob(names: list[str]):
    enc = [n.encode() for n in names]
    off = np.zeros(len(enc) + 1, np.int64)
    off[1:] = np.cumsum([len(e) for e in enc])
    return np.frombuffer(b"".join(enc) + b"\0", np.uint8).copy(), off


def vcf_text_host(names: list[str], contig_of_region, positions, region_of, depths, freqs, keys_raw, probs, regions: RegionTable,
                  options: dict, vcf_opts: dict | None = None, stream: int = 0):
    """pb_variant_vcf_host: records on the host (any order; region r belongs to contig names[contig_of_region[r]]) -> (text uint8,
    line table VCF_LINE) in (contig id, position) order."""
    from .candidates import PbCandidateOptions
    from .abi import regions_array, ALLELE_STRIDE
    _lib.require_gpu()
    L = _lib.lib()
    vp = C.c_void_p
    L.pb_variant_vcf_host.argtypes = [vp] * 6 + [C.c_int64, vp, C.c_int64, vp, C.c_int64, vp, vp, vp, C.c_int64, vp,
                                                 C.POINTER(PbCandidateOptions), C.POINTER(PbVcfOptions), vp, C.c_int64, vp, C.c_int64,
                                                 C.POINTER(C.c_int64), C.POINTER(C.c_int64), vp]
    n = int(len(positions))
    a = dict(pos=np.ascontiguousarray(positions, np.int64), rof=np.ascontiguousarray(region_of, np.int32),
             dep=np.ascontiguousarray(depths, np.uint8), frq=np.ascontiguousarray(freqs, np.uint8),
             keys=np.ascontiguousarray(keys_raw, np.uint8).reshape(n, ALLELE_STRIDE), pr=np.ascontiguousarray(probs, np.float32).reshape(n, 3))
    regs, keep = regions_array(regions)
    ref = np.ascontiguousarray(regions.ref, np.uint8)
    cor = np.ascontiguousarray(contig_of_region, np.int32)
    nm, off = _names_blob(names)
    vt = vaf_table()
    so, vo = PbCandidateOptions(**options), vcf_options(vcf_opts or VCF_OPTIONS_ONT)
    text_cap, lines_cap = max(1, 160 * n), max(1, n)
    while True:
        text = np.empty(text_cap, np.uint8)
        lines = np.empty(lines_cap, VCF_LINE)
        nt, nl = C.c_int64(0), C.c_int64(0)
        rc = L.pb_variant_vcf_host(a["pos"].ctypes.data, a["rof"].ctypes.data, a["dep"].ctypes.data, a["frq"].ctypes.data,
                                   a["keys"].ctypes.data, a["pr"].ctypes.data, n, C.cast(regs, vp), regions.n_regions, ref.ctypes.data,
                                   ref.shape[0], cor.ctypes.data, nm.ctypes.data, off.ctypes.data, len(names), vt.ctypes.data,
                                   C.byref(so), C.byref(vo), text.ctypes.data, text_cap, lines.ctypes.data, lines_cap,
                                   C.byref(nt), C.byref(nl), C.c_void_p(stream))
        if rc == PB_ERR_CAPACITY:
            text_cap, lines_cap = int(nt.value), int(nl.value)
            continue
        _lib.check(rc, "pb_variant_vcf_host")
        return text[:nt.value], lines[:nl.value]


def vcf_text_device(names: list[str], contig_of_region, cols, d_probs: int, n: int, d_regions: int, d_ref: int, options: dict,
                    vcf_opts: dict | None = None, device: int = 0, stream: int = 0, window: np.ndarray | None = None,
                    on_device: bool = False):
    """pb_variant_vcf_device over records already in HBM (`cols`: abi.PbCandidateColumns of device pointers) -> (text uint8, line
    table) on the host: only the VCF text and its line table leave the GPU.  `window` [n_regions, 2]: the positions [lo, hi]
    each region's records may form sites at (None: all).  `on_device`: the text and the line table stay on the device (uint8
    tensors)."""
    import torch
    from .candidates import PbCandidateOptions
    from .abi import PbCandidateColumns
    L = _lib.lib()
    vp = C.c_void_p
    L.pb_variant_vcf_device.argtypes = [C.POINTER(PbCandidateColumns), vp, C.c_int64, vp, vp, C.POINTER(PbVcfJob),
                                        C.POINTER(PbCandidateOptions), C.POINTER(PbVcfOptions), vp, C.c_int64, vp, C.c_int64,
                                        C.POINTER(C.c_int64), C.POINTER(C.c_int64), vp]
    dev = torch.device("cuda", device)
    nm, off = _names_blob(names)
    keep = [torch.from_numpy(x).to(dev) for x in (np.ascontiguousarray(contig_of_region, np.int32), nm, off, vaf_table().reshape(-1))]
    if window is not None:
        keep.append(torch.from_numpy(np.ascontiguousarray(window, np.int64).reshape(-1)).to(dev))
    job = PbVcfJob(*(t.data_ptr() for t in keep))
    so, vo = PbCandidateOptions(**options), vcf_options(vcf_opts or VCF_OPTIONS_ONT)
    text_cap, lines_cap = max(1, 160 * n), max(1, n)
    while True:
        text = torch.empty(text_cap, dtype=torch.uint8, device=dev)
        lines = torch.empty(lines_cap * VCF_LINE.itemsize, dtype=torch.uint8, device=dev)
        nt, nl = C.c_int64(0), C.c_int64(0)
        rc = L.pb_variant_vcf_device(C.byref(cols), vp(d_probs), n, vp(d_regions), vp(d_ref), C.byref(job), C.byref(so), C.byref(vo),
                                     vp(text.data_ptr()), text_cap, vp(lines.data_ptr()), lines_cap, C.byref(nt), C.byref(nl),
                                     vp(stream))
        if rc == PB_ERR_CAPACITY:
            text_cap, lines_cap = int(nt.value), int(nl.value)
            continue
        _lib.check(rc, "pb_variant_vcf_device")
        text, lines = text[:nt.value], lines[:nl.value * VCF_LINE.itemsize]
        return (text, lines) if on_device else (text.cpu().numpy(), lines.cpu().numpy().view(VCF_LINE))


def host_tail_text(records: list[dict], contig_id: int):
    """The host tail's records of one contig (assemble_sites) -> (text, line table) through format_vcf_line: the same form as the
    GPU's, so both go through one writer."""
    txt = [(format_vcf_line(r) + "\n").encode() for r in records]
    lines = np.zeros(len(records), VCF_LINE)
    lines["pos"] = [r["start"] for r in records]
    lines["contig"] = contig_id
    lines["ref_len"] = [len(r["alleles"][0]) for r in records]
    lines["cls"] = [CLASS_PEPPER if "pepper" in r["files"] else CLASS_VC_SNP if "variant_calling_snp" in r["files"] else CLASS_VC_INDEL
                    for r in records]
    lines["text_len"] = [len(t) for t in txt]
    lines["text_off"] = np.concatenate([[0], np.cumsum(lines["text_len"])[:-1]]) if len(txt) else []
    return np.frombuffer(b"".join(txt), np.uint8), lines


def vcf_header(sample_name: str, fasta_contigs: list[tuple[str, int]]) -> str:
    """The header VCFWriter.get_vcf_header declares (VcfWriter.py:220-289), each ID once, every FASTA contig in FAI order."""
    h = ["##fileformat=VCFv4.2"]
    for i, d in (("PASS", "All filters passed"), ("refCall", "Call is homozygous"), ("lowGQ", "Low genotype quality"),
                 ("lowQUAL", "Low variant call quality"), ("conflictPos", "Overlapping record")):
        h.append('##FILTER=<ID=%s,Description="%s">' % (i, d))
    for i, n, t, d in (("GT", "1", "String", "Genotype"), ("DP", "1", "Integer", "Depth"), ("AD", "A", "Integer", "Allele depth"),
                       ("VAF", "A", "Float", "Variant allele fractions."),
                       ("AP", "A", "Float", "Maximum variant allele probability for each allele."),
                       ("GQ", "1", "Float", "Genotype Quality"),
                       ("REP", "1", "String", "If set to 1 then variant site is considered to be ina LowCompexity repeat region")):
        h.append('##FORMAT=<ID=%s,Number=%s,Type=%s,Description="%s">' % (i, n, t, d))
    h += ["##contig=<ID=%s,length=%d>" % (c, n) for c, n in fasta_contigs]
    h.append("\t".join(["#CHROM", "POS", "ID", "REF", "ALT", "QUAL", "FILTER", "INFO", "FORMAT", sample_name]))
    return "\n".join(h) + "\n"


def order_lines(parts: list, names: list[str]):
    """(text, lines) parts -> one text + line table in the order of write_vcf_records: sorted by (contig NAME, position)
    (VcfWriter.py:144; lexical, so chr10 < chr2), and a site dropped when its position equals the previous written site's — the
    reference never resets `last_position` between contigs (VcfWriter.py:151-152)."""
    texts, tabs, base = [], [], 0
    for text, lines in parts:
        t = lines.copy()
        t["text_off"] += base
        base += text.shape[0]
        texts.append(text); tabs.append(t)
    text = np.concatenate(texts) if texts else np.zeros(0, np.uint8)
    lines = np.concatenate(tabs) if tabs else np.zeros(0, VCF_LINE)
    lex = np.empty(len(names), np.int64)
    lex[np.array(sorted(range(len(names)), key=lambda i: names[i]), dtype=np.int64)] = np.arange(len(names))
    lines = lines[np.lexsort((lines["pos"], lex[lines["contig"]]))]
    keep = np.ones(lines.shape[0], bool)
    keep[1:] = lines["pos"][1:] != lines["pos"][:-1]
    return text, lines[keep]


def _gather(text: np.ndarray, lines: np.ndarray) -> bytes:
    """The bytes of `lines`, in table order: one slice per run of lines that lie back to back in the text (the whole of a contig's
    part for the full file), so no per-byte index is built."""
    if lines.shape[0] == 0:
        return b""
    off, ln = lines["text_off"], lines["text_len"].astype(np.int64)
    brk = np.flatnonzero(off[1:] != off[:-1] + ln[:-1]) + 1
    first, last = np.concatenate([[0], brk]), np.concatenate([brk, [lines.shape[0]]]) - 1
    mv = memoryview(np.ascontiguousarray(text))
    return b"".join(mv[a:b] for a, b in zip(off[first].tolist(), (off[last] + ln[last]).tolist()))


BGZF_PAYLOAD = 0xff00


def _bgzf(data: bytes, pool, level: int = 6):
    """BGZF members of <= 65,280 bytes each (+ the EOF block) and the uncompressed start / compressed offset of each member."""
    from .synth_files import _bgzf_block, BGZF_EOF
    starts = list(range(0, len(data), BGZF_PAYLOAD))
    blocks = list(pool.map(lambda s: _bgzf_block(data[s:s + BGZF_PAYLOAD], level), starts))
    coff = np.concatenate([[0], np.cumsum([len(b) for b in blocks])]).astype(np.int64)
    return b"".join(blocks) + BGZF_EOF, np.array(starts, np.int64), coff


def vcf_csi_depth(fasta_contigs: list[tuple[str, int]], names: list[str]) -> int | None:
    """None when every contig of `names` fits a TBI (shorter than 2^29, the reach of BAI binning); otherwise the depth of the CSI
    that indexes the files instead: min_shift 14 and the smallest depth >= 5 that covers the longest contig (bcftools index)."""
    from .synth_files import csi_depth_for, BAI_MAX_END
    lengths = dict(fasta_contigs)
    longest = max([lengths.get(n, 0) for n in names] + [0])
    return None if longest <= BAI_MAX_END else csi_depth_for(longest)


def _tabix(names: list[str], tids: np.ndarray, beg: np.ndarray, end: np.ndarray, ustart: np.ndarray, uend: np.ndarray,
           blk_u: np.ndarray, blk_c: np.ndarray, eof_c: int, total_u: int, csi_depth: int | None = None) -> bytes:
    """TBI of a VCF (format 2, col_seq 1, col_beg 2, col_end 0, meta '#'): the per-reference bins / chunks / 16 kb linear index
    are those of a BAI (synth_files._bai_bytes) over [pos, pos + len(REF)) and the lines' virtual offsets.  With `csi_depth`, a
    CSI (min_shift 14) instead, whose aux holds the same configuration block, as `tabix --csi` writes; uncompressed either way."""
    blk_u, blk_c = np.asarray(blk_u, np.int64), np.asarray(blk_c, np.int64)

    def voff(u):
        u = np.asarray(u, np.int64)
        k = np.maximum(np.searchsorted(blk_u, u, side="right") - 1, 0)
        return np.where(u >= total_u, np.int64(eof_c) << 16, (blk_c[k] << 16) | (u - blk_u[k])).astype(np.uint64)
    tids = np.asarray(tids, np.int64)
    beg, end = np.asarray(beg, np.int64), np.asarray(end, np.int64)
    vb, ve = voff(ustart), voff(uend)
    nm = b"".join(n.encode() + b"\0" for n in names)
    if csi_depth is not None:
        from .synth_files import csi_bytes, csi_reference
        conf = struct.pack("<7i", 2, 1, 2, 0, ord("#"), 0, len(nm)) + nm
        refs = []
        for t in range(len(names)):
            sel = np.flatnonzero(tids == t)
            refs.append(csi_reference(beg[sel], end[sel], vb[sel], ve[sel], 14, csi_depth))
        return csi_bytes(14, csi_depth, conf, refs)
    out = [b"TBI\x01" + struct.pack("<8i", len(names), 2, 1, 2, 0, ord("#"), 0, len(nm)) + nm]
    for t in range(len(names)):
        sel = np.flatnonzero(tids == t)
        out.append(_index_reference(beg[sel], end[sel], vb[sel], ve[sel]))
    return b"".join(out)


def _index_reference(beg: np.ndarray, end: np.ndarray, vb: np.ndarray, ve: np.ndarray) -> bytes:
    """One reference's bins, chunks, pseudo-bin and 16 kb linear index: the bytes synth_files._bai_bytes writes for the spans
    (beg, end) with virtual offsets [vb, ve), lines in file order.  A chunk is a run of consecutive lines of one bin (the lines
    lie back to back, so _bai_bytes merges exactly those); a window's linear offset is the first line that covers it, and a
    window no line covers takes the previous window's."""
    from .synth_files import _reg2bin_v
    n = beg.shape[0]
    if n == 0:
        return struct.pack("<ii", 0, 0)
    bins = _reg2bin_v(beg, end)
    brk = np.flatnonzero(bins[1:] != bins[:-1]) + 1
    first, last = np.concatenate([[0], brk]), np.concatenate([brk, [n]]) - 1
    cbin, cvb, cve = bins[first], vb[first], ve[last]
    o = np.argsort(cbin, kind="stable")
    cbin, cvb, cve = cbin[o], cvb[o], cve[o]
    ub, ufirst, cnt = np.unique(cbin, return_index=True, return_counts=True)
    nb, nc = ub.shape[0], cbin.shape[0]
    words = np.zeros(2 * nb + 4 * nc, np.uint32)                 # per bin: bin, n_chunk, then (beg, end) as uint64 pairs
    bstart = 2 * np.arange(nb) + 4 * ufirst
    words[bstart], words[bstart + 1] = ub, cnt
    cpos = 2 * (np.repeat(np.arange(nb), cnt) + 1) + 4 * np.arange(nc)
    lo32 = np.uint64(0xffffffff)
    for k, v in enumerate((cvb & lo32, cvb >> np.uint64(32), cve & lo32, cve >> np.uint64(32))):
        words[cpos + k] = v
    meta = struct.pack("<Ii", 37450, 2) + struct.pack("<QQQQ", int(vb[0]), int(ve[-1]), n, 0)
    wa, wb = beg >> 14, (end - 1) >> 14
    n_win = int(wb.max()) + 1
    span = wb - wa + 1
    line = np.repeat(np.arange(n), span)
    win = np.repeat(wa, span) + np.arange(line.shape[0]) - np.repeat(np.cumsum(span) - span, span)
    none = np.iinfo(np.uint64).max
    lin = np.full(n_win, none, np.uint64)
    np.minimum.at(lin, win, vb[line])
    idx = np.maximum.accumulate(np.where(lin != none, np.arange(n_win), -1))
    lin = np.where(idx >= 0, lin[np.maximum(idx, 0)], np.uint64(0)).astype("<u8")
    return (struct.pack("<i", nb + 1) + words.astype("<u4").tobytes() + meta + struct.pack("<i", n_win) + lin.tobytes())


def write_vcfs(out_dir: str, sample_name: str, fasta_contigs: list[tuple[str, int]], names: list[str], text: np.ndarray,
               lines: np.ndarray, threads: int = 8) -> tuple[int, int, int, int, int]:
    """Ordered lines (order_lines) -> the five bgzipped, tabix-indexed VCFs of write_vcf_records under `out_dir`; returns its
    totals (full, pepper, variant calling, variant-calling SNPs, indels).  The index is a .tbi, or a .csi when a contig of `names`
    is longer than 2^29 (vcf_csi_depth)."""
    import os
    from concurrent.futures import ThreadPoolExecutor
    os.makedirs(out_dir, exist_ok=True)
    head = vcf_header(sample_name, fasta_contigs).encode()
    cls = lines["cls"]
    masks = (np.ones(cls.shape[0], bool), cls == CLASS_PEPPER, cls != CLASS_PEPPER, cls == CLASS_VC_SNP, cls == CLASS_VC_INDEL)
    depth = vcf_csi_depth(fasta_contigs, names)
    with ThreadPoolExecutor(max_workers=max(1, threads)) as pool:
        for name, mask in zip(VCF_FILES, masks):
            sel = lines[mask]
            body = _gather(text, sel)
            data = head + body
            gz, blk_u, blk_c = _bgzf(data, pool)
            path = os.path.join(out_dir, name + ".vcf.gz")
            with open(path, "wb") as f:
                f.write(gz)
            # tabix reference ids: contigs in the order their lines appear
            seen = list(dict.fromkeys(sel["contig"].tolist()))
            tid_of = {c: i for i, c in enumerate(seen)}
            us = len(head) + np.concatenate([[0], np.cumsum(sel["text_len"].astype(np.int64))])
            tbi = _tabix([names[c] for c in seen], np.array([tid_of[c] for c in sel["contig"].tolist()], np.int64), sel["pos"],
                         sel["pos"] + sel["ref_len"], us[:-1], us[1:], blk_u, blk_c, int(blk_c[-1]), len(data), depth)
            with open(path + (".tbi" if depth is None else ".csi"), "wb") as f:
                f.write(_bgzf(tbi, pool)[0])
    return tuple(int(m.sum()) for m in masks)


# ---------------------------------------------------------------------------------------------------------------------------
# Whole-genome output from BGZF members compressed elsewhere (each rank's GPU): the files are the header member, then every
# group's members in lexical contig order and group order, then the EOF block; only the members and a compact line table reach
# the writer.

# what the writer needs of a line: its position, REF length, class and length (its offset is the sum of the lengths before it)
GROUP_LINE = np.dtype([("pos", "<i8"), ("ref_len", "<i4"), ("cls", "<i4"), ("text_len", "<i4"), ("pad", "<i4")])


def file_masks(cls: np.ndarray) -> tuple:
    """The lines each of VCF_FILES takes, by class (write_vcfs)."""
    return (np.ones(cls.shape[0], bool), cls == CLASS_PEPPER, cls != CLASS_PEPPER, cls == CLASS_VC_SNP, cls == CLASS_VC_INDEL)


def member_cuts(stream_bytes: int, payload: int = BGZF_PAYLOAD) -> np.ndarray:
    """Payload sizes of the members one group stream is cut into (every member but the last is full; a member may end
    mid-line)."""
    n = -(-int(stream_bytes) // payload)
    cuts = np.full(n, payload, np.int64)
    if n:
        cuts[-1] = int(stream_bytes) - payload * (n - 1)
    return cuts


class GroupPart:
    """One group's share of the five files: its lines (GROUP_LINE, in file order) and, per file, the payload and compressed
    sizes of its members and their bytes."""

    def __init__(self, lines: np.ndarray, usizes: list, csizes: list, data: list):
        self.lines, self.usizes, self.csizes, self.data = lines, usizes, csizes, data


def group_line_table(lines: np.ndarray) -> np.ndarray:
    out = np.zeros(lines.shape[0], GROUP_LINE)
    for k in ("pos", "ref_len", "cls", "text_len"):
        out[k] = lines[k]
    return out


def host_group_part(text: np.ndarray, lines: np.ndarray, payload: int = BGZF_PAYLOAD, level: int = 1) -> GroupPart:
    """A GroupPart compressed on the host with zlib (the reference for the GPU compressor's parts)."""
    from .synth_files import _bgzf_block
    us, cs, data = [], [], []
    for m in file_masks(lines["cls"]):
        body = _gather(text, lines[m])
        cuts = member_cuts(len(body), payload)
        starts = np.concatenate([[0], np.cumsum(cuts)])
        blocks = [_bgzf_block(body[a:b], level) for a, b in zip(starts[:-1].tolist(), starts[1:].tolist())]
        us.append(cuts); cs.append(np.array([len(b) for b in blocks], np.int64)); data.append(b"".join(blocks))
    return GroupPart(group_line_table(lines), us, cs, data)


def write_vcfs_from_parts(out_dir: str, sample_name: str, fasta_contigs: list[tuple[str, int]], names: list[str],
                          group_contig: list[int], parts: dict) -> None:
    """The five bgzipped, tabix-indexed VCFs from compressed group parts: `parts` {group id: GroupPart}, group g of contig
    names[group_contig[g]]; the lines are final (the last_position drop already applied).  Same files as write_vcfs over the
    same lines, up to the DEFLATE bytes of the members."""
    import os
    from concurrent.futures import ThreadPoolExecutor
    os.makedirs(out_dir, exist_ok=True)
    head = vcf_header(sample_name, fasta_contigs).encode()
    lex = {c: i for i, c in enumerate(sorted(range(len(names)), key=lambda i: names[i]))}
    order = sorted(parts, key=lambda g: (lex[group_contig[g]], g))
    depth = vcf_csi_depth(fasta_contigs, names)
    with ThreadPoolExecutor(max_workers=8) as pool:
        for f, name in enumerate(VCF_FILES):
            pieces = []
            for g in order:
                p = parts[g]
                sel = p.lines[file_masks(p.lines["cls"])[f]]
                pieces.append((group_contig[g], p.usizes[f], p.csizes[f], p.data[f], sel["pos"], sel["pos"] + sel["ref_len"],
                               sel["text_len"]))
            write_indexed_members(os.path.join(out_dir, name + ".vcf.gz"), head, pieces, names, depth, pool)


def write_indexed_members(path: str, head: bytes, pieces: list, names: list[str], depth: int | None, pool) -> None:
    """One bgzipped file and its index from BGZF members compressed elsewhere: the header as its own members, then each piece
    (contig id, member payload sizes, member compressed sizes, member bytes, line begins, line ends, line lengths) in file
    order, then the EOF block; the .tbi (or, with `depth`, the .csi) indexes each line over [begin, end)."""
    from .synth_files import BGZF_EOF
    hgz, hu, hc = _bgzf(head, pool, 1)
    hgz = hgz[:-len(BGZF_EOF)]
    chunks, blk_u, blk_c = [hgz], [hu], [hc[:-1]]
    u, c = len(head), len(hgz)
    tids, beg, end, ulen, seen = [], [], [], [], {}
    for contig, usizes, csizes, data, b, e, tl in pieces:
        if usizes.shape[0]:
            blk_u.append(u + np.concatenate([[0], np.cumsum(usizes)[:-1]]))
            blk_c.append(c + np.concatenate([[0], np.cumsum(csizes)[:-1]]))
            chunks.append(data)
            u += int(usizes.sum()); c += int(csizes.sum())
        if b.shape[0]:
            tids.append(np.full(b.shape[0], seen.setdefault(contig, len(seen)), np.int64))
            beg.append(b); end.append(e); ulen.append(tl.astype(np.int64))
    with open(path, "wb") as fh:
        fh.write(b"".join(chunks) + BGZF_EOF)
    cat = (lambda a, dt: np.concatenate(a) if a else np.zeros(0, dt))     # noqa: E731
    ul = cat(ulen, np.int64)
    us = len(head) + np.concatenate([[0], np.cumsum(ul)])
    tbi = _tabix([names[k] for k in seen], cat(tids, np.int64), cat(beg, np.int64), cat(end, np.int64), us[:-1], us[1:],
                 np.concatenate(blk_u), np.concatenate(blk_c), c, u, depth)
    with open(path + (".tbi" if depth is None else ".csi"), "wb") as fh:
        fh.write(_bgzf(tbi, pool)[0])


def bgzf_compress_host(payload: np.ndarray, member_off: np.ndarray) -> tuple[bytes, np.ndarray]:
    """pb_bgzf_compress_host: payload bytes [member_off[k], member_off[k + 1]) -> BGZF member k; returns (members back to back,
    bytes of each member)."""
    _lib.require_gpu()
    L = _lib.lib()
    vp = C.c_void_p
    L.pb_bgzf_compress_host.argtypes = [vp, vp, C.c_int64, vp, C.c_int64, vp, C.POINTER(C.c_int64), vp]
    payload = np.ascontiguousarray(payload, np.uint8)
    off = np.ascontiguousarray(member_off, np.int64)
    n = off.shape[0] - 1
    sizes = np.zeros(max(1, n), np.int64)
    cap = max(64, int(off[-1] - off[0]) // 2 + 64 * n)
    while True:
        out = np.empty(cap, np.uint8)
        total = C.c_int64(0)
        rc = L.pb_bgzf_compress_host(payload.ctypes.data, off.ctypes.data, n, out.ctypes.data, cap, sizes.ctypes.data, C.byref(total), None)
        if rc == PB_ERR_CAPACITY:
            cap = int(total.value)
            continue
        _lib.check(rc, "pb_bgzf_compress_host")
        return out[:total.value].tobytes(), sizes[:n].copy()


def bgzf_compress_device(d_payload, member_off: np.ndarray, device: int = 0, stream: int = 0):
    """pb_bgzf_compress_device over a device byte tensor -> (members back to back as a device uint8 tensor, bytes of each
    member)."""
    import torch
    L = _lib.lib()
    vp = C.c_void_p
    L.pb_bgzf_compress_device.argtypes = [vp, vp, C.c_int64, vp, C.c_int64, vp, C.POINTER(C.c_int64), vp]
    off = np.ascontiguousarray(member_off, np.int64)
    n = off.shape[0] - 1
    sizes = np.zeros(max(1, n), np.int64)
    cap = max(64, int(off[-1] - off[0]) // 4 + 64 * n)
    while True:
        out = torch.empty(cap, dtype=torch.uint8, device=torch.device("cuda", device))
        total = C.c_int64(0)
        rc = L.pb_bgzf_compress_device(vp(d_payload.data_ptr()), off.ctypes.data, n, vp(out.data_ptr()), cap, sizes.ctypes.data,
                                       C.byref(total), vp(stream))
        if rc == PB_ERR_CAPACITY:
            cap = int(total.value)
            continue
        _lib.check(rc, "pb_bgzf_compress_device")
        return out[:total.value], sizes[:n].copy()


def gather_lines_device(d_text, d_lines, sel: np.ndarray, dst: np.ndarray, out, device: int = 0, stream: int = 0) -> None:
    """pb_vcf_gather_lines_device: line sel[i] of the device line table -> out[dst[i]:], on the device."""
    import torch
    L = _lib.lib()
    vp = C.c_void_p
    L.pb_vcf_gather_lines_device.argtypes = [vp, vp, vp, vp, C.c_int64, vp, vp]
    dev = torch.device("cuda", device)
    s = torch.from_numpy(np.ascontiguousarray(sel, np.int64)).to(dev)
    d = torch.from_numpy(np.ascontiguousarray(dst, np.int64)).to(dev)
    _lib.check(L.pb_vcf_gather_lines_device(vp(d_text.data_ptr()), vp(d_lines.data_ptr()), vp(s.data_ptr()), vp(d.data_ptr()),
                                            int(s.shape[0]), vp(out.data_ptr()), vp(stream)), "pb_vcf_gather_lines_device")
