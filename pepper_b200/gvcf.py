"""The gVCF of a genome call (DESIGN.md section 4, "gVCF"): every called position either in a record line (a
PEPPER_VARIANT_FULL line with the <*> allele) or in a reference block whose GQ / PL come from the binomial reference-confidence
model over the encoder's per-position (n_ref, n_alt) track.  The kernels are in csrc/gvcf.cu; dist.DistributedGenomeCaller runs
them per rank (gvcf=True) and rank 0 writes PEPPER_VARIANT.g.vcf.gz with its index."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from . import _lib
from .abi import PB_ERR_CAPACITY
from .vcf import VCF_LINE, vcf_header, _names_blob

GVCF_FILE = "PEPPER_VARIANT.g.vcf.gz"
GVCF_ERROR_RATE = 0.001               # e of the reference-confidence model
GVCF_GQ_BINSIZE = 5
CLASS_BLOCK = 3                        # PB_GVCF_CLASS_BLOCK
RECORD_EXTRA = 10                      # ",<*>" + three ",."
GVCF_HEADER_LINES = (
    '##ALT=<ID=*,Description="Represents allele(s) other than observed.">',
    '##INFO=<ID=END,Number=1,Type=Integer,Description="End position of the reference block (1-based, inclusive)">',
    '##FORMAT=<ID=MIN_DP,Number=1,Type=Integer,Description="Minimum DP observed within the reference block">',
    '##FORMAT=<ID=PL,Number=G,Type=Integer,Description="Phred-scaled genotype likelihoods rounded to the closest integer">')

# pb_gvcf_segment_t: one interval's owned window in the track
GVCF_SEGMENT = np.dtype([("toff", "<i8"), ("pos0", "<i8"), ("len", "<i8"), ("ref_off", "<i8"), ("contig", "<i4"), ("pad", "<i4")])
# a line of a rank's gathered gVCF part: 0-based POS, index end (exclusive), bytes
GVCF_LINE = np.dtype([("pos", "<i8"), ("end", "<i8"), ("text_len", "<i4"), ("pad", "<i4")])


class PbGvcfParams(C.Structure):
    _fields_ = [("a", C.c_double), ("b", C.c_double), ("h", C.c_double), ("binsize", C.c_int32), ("pad", C.c_int32)]


def model_terms(error_rate: float = GVCF_ERROR_RATE) -> tuple[float, float, float]:
    """(A, B, H) = (log10(1 - e), log10(e), log10(0.5)), computed once on the host; the kernels take them as doubles."""
    return math.log10(1.0 - error_rate), math.log10(error_rate), math.log10(0.5)


def gvcf_params(binsize: int = GVCF_GQ_BINSIZE) -> PbGvcfParams:
    if int(binsize) <= 0:
        raise ValueError("gvcf_gq_binsize must be > 0")
    return PbGvcfParams(*model_terms(), int(binsize), 0)


def gvcf_header(sample_name: str, fasta_contigs: list[tuple[str, int]]) -> str:
    """vcf_header's lines, with the <*> allele, END, MIN_DP and PL declared before the column line."""
    lines = vcf_header(sample_name, fasta_contigs).rstrip("\n").split("\n")
    return "\n".join(lines[:-1] + list(GVCF_HEADER_LINES) + lines[-1:]) + "\n"


def _bind(L):
    vp = C.c_void_p
    L.pb_gvcf_blocks_host.argtypes = [vp, C.c_int64, vp, C.c_int64, vp, C.c_int64, vp, C.c_int64, vp, vp, C.c_int64,
                                      C.POINTER(PbGvcfParams), vp, C.c_int64, vp, C.c_int64, C.POINTER(C.c_int64),
                                      C.POINTER(C.c_int64), vp]
    L.pb_gvcf_blocks_device.argtypes = [vp, C.c_int64, vp, C.c_int64, vp, C.c_int64, vp, vp, vp, C.c_int64, C.POINTER(PbGvcfParams),
                                        vp, C.c_int64, vp, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64), vp]
    L.pb_gvcf_records_device.argtypes = [vp, vp, C.c_int64, vp, vp, vp]
    return L


LINE_BOUND = 128                       # bytes of a block line beyond its contig name, at most


def _bounds(n_track: int, names: list[str]) -> tuple[int, int]:
    """(text bytes, lines) the block lines of `n_track` positions cannot exceed: at most one block per position."""
    return max(1, n_track * (max([len(n) for n in names] + [1]) + LINE_BOUND)), max(1, n_track)


def gvcf_blocks_host(track: np.ndarray, segments: np.ndarray, masks: np.ndarray, ref: np.ndarray, names: list[str],
                     binsize: int = GVCF_GQ_BINSIZE) -> tuple[np.ndarray, np.ndarray]:
    """pb_gvcf_blocks_host: the block lines of a track over host arrays -> (text uint8, VCF_LINE table) in track order.
    `segments` GVCF_SEGMENT (ref_off indexes `ref`), `masks` int64 [n][2] half-open track ranges."""
    _lib.require_gpu()
    L = _bind(_lib.lib())
    tr = np.ascontiguousarray(track, np.uint32)
    seg = np.ascontiguousarray(segments, GVCF_SEGMENT)
    msk = np.ascontiguousarray(masks, np.int64).reshape(-1, 2)
    rf = np.ascontiguousarray(ref, np.uint8)
    nm, off = _names_blob(names)
    p = gvcf_params(binsize)
    text_cap, lines_cap = _bounds(tr.shape[0], names)
    while True:
        text = np.empty(text_cap, np.uint8)
        lines = np.empty(lines_cap, VCF_LINE)
        nt, nl = C.c_int64(0), C.c_int64(0)
        rc = L.pb_gvcf_blocks_host(tr.ctypes.data, tr.shape[0], seg.ctypes.data, seg.shape[0], msk.ctypes.data, msk.shape[0],
                                   rf.ctypes.data, rf.shape[0], nm.ctypes.data, off.ctypes.data, len(names), C.byref(p),
                                   text.ctypes.data, text_cap, lines.ctypes.data, lines_cap, C.byref(nt), C.byref(nl), None)
        if rc == PB_ERR_CAPACITY:
            text_cap, lines_cap = max(1, int(nt.value)), max(1, int(nl.value))
            continue
        _lib.check(rc, "pb_gvcf_blocks_host")
        return text[:nt.value], lines[:nl.value]


def gvcf_blocks_device(d_track, n_track: int, segments: np.ndarray, masks: np.ndarray, d_ref: int, names: list[str],
                       binsize: int, device: int = 0):
    """pb_gvcf_blocks_device over a device track (torch tensor) and reference (pointer) -> (text, device uint8 tensor; VCF_LINE
    table, host).  The outputs are sized to their bounds (_bounds), so the pass runs once: call it over bounded batches."""
    import torch
    L = _bind(_lib.lib())
    vp = C.c_void_p
    seg = np.ascontiguousarray(segments, GVCF_SEGMENT)
    msk = np.ascontiguousarray(masks, np.int64).reshape(-1, 2)
    nm, off = _names_blob(names)
    p = gvcf_params(binsize)
    dev = torch.device("cuda", device)
    text_cap, lines_cap = _bounds(n_track, names)
    text = torch.empty(text_cap, dtype=torch.uint8, device=dev)
    lines = torch.empty(lines_cap * VCF_LINE.itemsize, dtype=torch.uint8, device=dev)
    nt, nl = C.c_int64(0), C.c_int64(0)
    _lib.check(L.pb_gvcf_blocks_device(vp(d_track.data_ptr()), int(n_track), seg.ctypes.data, seg.shape[0], msk.ctypes.data,
                                       msk.shape[0], vp(d_ref), nm.ctypes.data, off.ctypes.data, len(names), C.byref(p),
                                       vp(text.data_ptr()), text_cap, vp(lines.data_ptr()), lines_cap, C.byref(nt), C.byref(nl), None),
               "pb_gvcf_blocks_device")
    return text[:nt.value], lines[:nl.value * VCF_LINE.itemsize].cpu().numpy().view(VCF_LINE)


def gvcf_records_device(d_text, lines: np.ndarray, device: int = 0):
    """pb_gvcf_records_device: FULL lines (VCF_LINE rows into the device text) -> (device text of the record lines back to back,
    their VCF_LINE table)."""
    import torch
    L = _bind(_lib.lib())
    vp = C.c_void_p
    dev = torch.device("cuda", device)
    out_lines = np.array(lines, VCF_LINE, copy=True)
    out_lines["text_len"] += RECORD_EXTRA
    ln = out_lines["text_len"].astype(np.int64)
    out_lines["text_off"] = np.concatenate([[0], np.cumsum(ln)[:-1]]) if ln.shape[0] else ln
    out = torch.empty(max(1, int(ln.sum())), dtype=torch.uint8, device=dev)
    if lines.shape[0]:
        d_lines = torch.from_numpy(np.ascontiguousarray(lines, VCF_LINE).view(np.uint8).reshape(-1)).to(dev)
        d_off = torch.from_numpy(np.ascontiguousarray(out_lines["text_off"], np.int64)).to(dev)
        _lib.check(L.pb_gvcf_records_device(vp(d_text.data_ptr()), vp(d_lines.data_ptr()), int(lines.shape[0]), vp(d_off.data_ptr()),
                                            vp(out.data_ptr()), None), "pb_gvcf_records_device")
    return out[:int(ln.sum())], out_lines


def track_capacity(bases: int, world: int) -> int:
    """Track positions one rank's session may hold for a job of `bases` genomic bases (4 bytes each): the whole job on one GPU,
    where an exhausted track restarts with twice the room; twice a rank's share on several GPUs."""
    return int(bases) + 1 if world == 1 else 2 * (int(bases) // world) + (1 << 16)


def write_gvcf_from_parts(out_dir: str, sample_name: str, fasta_contigs: list[tuple[str, int]], names: list[str],
                          group_contig: list[int], parts: dict) -> str:
    """<out_dir>/PEPPER_VARIANT.g.vcf.gz and its .tbi / .csi from compressed group parts {group id: (GVCF_LINE table, member
    payload sizes, member compressed sizes, member bytes)}, groups in lexical contig order, then group order."""
    import os
    from concurrent.futures import ThreadPoolExecutor
    from .vcf import vcf_csi_depth, write_indexed_members
    os.makedirs(out_dir, exist_ok=True)
    head = gvcf_header(sample_name, fasta_contigs).encode()
    lex = {c: i for i, c in enumerate(sorted(range(len(names)), key=lambda i: names[i]))}
    pieces = []
    for g in sorted(parts, key=lambda g: (lex[group_contig[g]], g)):
        lines, us, cs, data = parts[g]
        pieces.append((group_contig[g], us, cs, data, lines["pos"], lines["end"], lines["text_len"]))
    path = os.path.join(out_dir, GVCF_FILE)
    with ThreadPoolExecutor(max_workers=8) as pool:
        write_indexed_members(path, head, pieces, names, vcf_csi_depth(fasta_contigs, names), pool)
    return path


def parse_gvcf_bytes(data) -> dict:
    """A rank's gathered gVCF bytes (dist.DistributedGenomeCaller.gvcf_pass) -> {group id: (GVCF_LINE, payload sizes,
    compressed sizes, member bytes)}."""
    buf = memoryview(np.ascontiguousarray(data, np.uint8))
    if len(buf) == 0:
        return {}
    meta_bytes, n_groups = (int(x) for x in np.frombuffer(buf[:16], np.int64))
    off, coff, out = 16, meta_bytes, {}
    for _ in range(n_groups):
        g, n_lines, n_members = (int(x) for x in np.frombuffer(buf[off:off + 24], np.int64))
        off += 24
        us = np.frombuffer(buf[off:off + 8 * n_members], np.int64).copy(); off += 8 * n_members
        cs = np.frombuffer(buf[off:off + 8 * n_members], np.int64).copy(); off += 8 * n_members
        lines = np.frombuffer(buf[off:off + GVCF_LINE.itemsize * n_lines], GVCF_LINE).copy()
        off += GVCF_LINE.itemsize * n_lines
        b = int(cs.sum())
        out[g] = (lines, us, cs, bytes(buf[coff:coff + b]))
        coff += b
    return out
