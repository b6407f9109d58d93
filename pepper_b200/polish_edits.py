"""Polish edits: the draft bases the stitch substituted, deleted or inserted, as a bgzipped, indexed sites-only VCF.

An edits session (pipeline.PolishStream(edits=True)) writes EDIT_EVENT records beside the consensus: one per winning image
column that is not an identity, and one coverage record per image.  `edits_vcf_device` turns the events of one contig and its
draft into VCF lines on the device (pb_polish_edits_vcf_device); `write_edits_vcf` writes the file and its .tbi (a .csi when a
contig is longer than 2^29, as vcf.vcf_csi_depth decides for the variant VCFs).  Applying the records to upper(draft[span])
gives the polished sequence (DESIGN.md section 4, "Polish edits")."""
from __future__ import annotations

import ctypes as C
import numpy as np

from . import _lib
from .abi import POLISH_SEQ_LEN, PB_ERR_CAPACITY

# pb_edit_event_t
EDIT_EVENT = np.dtype([("position", "<i8"), ("index", "<i4"), ("label", "u1"), ("phred", "u1"), ("draft", "u1"), ("kind", "u1")])
EDIT_COLUMN, EDIT_COVERAGE = 0, 1
# what the writer needs of a line: its 0-based POS, REF length and text bytes (pb_polish_edits_vcf_device's line table)
EDIT_LINE = np.dtype([("pos", "<i8"), ("ref_len", "<i8"), ("text_len", "<i8")])


def edits_header(fasta_contigs: list[tuple[str, int]]) -> str:
    h = ["##fileformat=VCFv4.2"]
    h += ["##contig=<ID=%s,length=%d>" % (c, n) for c, n in fasta_contigs]
    h.append('##INFO=<ID=UNCOVERED,Number=0,Type=Flag,Description="The record holds draft bases no image covered: the polished '
             'sequence has nothing for them">')
    h.append("\t".join(["#CHROM", "POS", "ID", "REF", "ALT", "QUAL", "FILTER", "INFO"]))
    return "\n".join(h) + "\n"


def split_events(ev: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """Events of a session -> (the column events, in order; int64 [n, 2] inclusive index-0 ranges the images won)."""
    cov = ev[ev["kind"] == EDIT_COVERAGE]
    ranges = np.stack([cov["position"], cov["position"] + cov["index"]], axis=1).astype(np.int64) if cov.shape[0] else np.zeros((0, 2), np.int64)
    return np.ascontiguousarray(ev[ev["kind"] == EDIT_COLUMN]), np.ascontiguousarray(ranges)


def events_by_contig(events: np.ndarray, segments: list[tuple[int, int]], group_contig: list[str], contigs: list[str]) -> dict:
    """Events `events` of the groups of `segments` ((group id, events), sorted by group id, laid out in that order) -> {contig:
    events in group order} (dist.assemble_contigs' cut, over event records)."""
    parts = {c: [] for c in contigs}
    off = 0
    for g, k in segments:
        parts[group_contig[g]].append(events[off:off + k])
        off += k
    return {c: np.concatenate(p) if p else np.zeros(0, EDIT_EVENT) for c, p in parts.items()}


def _bind(L):
    if getattr(L, "_edits_bound", False):
        return
    vp, i64 = C.c_void_p, C.c_int64
    L.pb_polish_edits_vcf_device.argtypes = [vp, i64, vp, i64, i64, i64, vp, C.c_char_p, vp, i64, vp, i64, C.POINTER(i64),
                                             C.POINTER(i64), vp]
    L.pb_test_polish_stitch_sink_edits.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, i64, i64, i64, vp, i64, C.POINTER(i64), vp, vp,
                                                   i64, C.POINTER(i64), vp, vp]
    L._edits_bound = True


def edits_vcf_device(d_columns, cover: np.ndarray, span: tuple[int, int], d_draft, contig: str, device: int = 0, stream: int = 0):
    """The VCF lines of one contig on the device: `d_columns` the contig's column events (a device uint8 tensor of EDIT_EVENT
    records, in group order), `cover` its coverage ranges, `span` = (first, last) draft position polished, `d_draft` the draft
    bases of the span (a device uint8 tensor).  Returns (text as a device uint8 tensor, EDIT_LINE table on the host)."""
    import torch
    L = _lib.lib()
    _bind(L)
    dev = torch.device("cuda", device)
    n_ev = d_columns.numel() // EDIT_EVENT.itemsize
    cov = np.ascontiguousarray(cover, np.int64)
    cap_lines = n_ev + cov.shape[0] + 2
    cap_text = cap_lines * (len(contig) + 48) + 4096
    while True:
        text = torch.empty(max(1, cap_text), dtype=torch.uint8, device=dev)
        lines = torch.empty((max(1, cap_lines), 3), dtype=torch.int64, device=dev)
        n_lines, n_text = C.c_int64(0), C.c_int64(0)
        rc = L.pb_polish_edits_vcf_device(C.c_void_p(d_columns.data_ptr() if n_ev else None), n_ev, cov.ctypes.data, cov.shape[0],
                                          int(span[0]), int(span[1]), C.c_void_p(d_draft.data_ptr()), contig.encode(),
                                          C.c_void_p(text.data_ptr()), cap_text, C.c_void_p(lines.data_ptr()), cap_lines,
                                          C.byref(n_lines), C.byref(n_text), C.c_void_p(stream))
        if rc == PB_ERR_CAPACITY:
            cap_lines, cap_text = int(n_lines.value), int(n_text.value)
            continue
        _lib.check(rc, "pb_polish_edits_vcf_device")
        break
    tab = lines[:n_lines.value].cpu().numpy()
    out = np.zeros(tab.shape[0], EDIT_LINE)
    out["pos"], out["ref_len"], out["text_len"] = tab[:, 0], tab[:, 1], tab[:, 2]
    return text[:n_text.value], out[out["text_len"] > 0]


class EditsPart:
    """One contig's share of the edits VCF: its lines (EDIT_LINE, in file order) and the BGZF members of its text, with the
    payload and compressed bytes of each."""

    def __init__(self, contig: str, lines: np.ndarray, usizes: np.ndarray, csizes: np.ndarray, data: bytes):
        self.contig, self.lines, self.usizes, self.csizes, self.data = contig, lines, usizes, csizes, data


def device_part(contig: str, d_text, lines: np.ndarray, device: int = 0) -> EditsPart:
    """An EditsPart compressed on the device (vcf.bgzf_compress_device)."""
    from .vcf import bgzf_compress_device, member_cuts
    cuts = member_cuts(d_text.numel())
    off = np.concatenate([[0], np.cumsum(cuts)]).astype(np.int64)
    if cuts.shape[0] == 0:
        return EditsPart(contig, lines, cuts, cuts.copy(), b"")
    members, sizes = bgzf_compress_device(d_text, off, device)
    return EditsPart(contig, lines, cuts, sizes, members.cpu().numpy().tobytes())


def host_part(contig: str, text: bytes, lines: np.ndarray, level: int = 1) -> EditsPart:
    """An EditsPart compressed on the host with zlib."""
    from .synth_files import _bgzf_block
    from .vcf import member_cuts
    cuts = member_cuts(len(text))
    starts = np.concatenate([[0], np.cumsum(cuts)]).tolist()
    blocks = [_bgzf_block(text[a:b], level) for a, b in zip(starts[:-1], starts[1:])]
    return EditsPart(contig, lines, cuts, np.array([len(b) for b in blocks], np.int64), b"".join(blocks))


def write_edits_vcf(path: str, fasta_contigs: list[tuple[str, int]], parts: list[EditsPart]) -> None:
    """The edits VCF at `path` (bgzipped: the header member, the parts' members in order, the EOF block) and its index at
    path + '.tbi', or '.csi' when a contig of the parts is longer than 2^29."""
    from concurrent.futures import ThreadPoolExecutor
    from .synth_files import BGZF_EOF
    from .vcf import _bgzf, _tabix, vcf_csi_depth
    head = edits_header(fasta_contigs).encode()
    names = [p.contig for p in parts if p.lines.shape[0]]
    depth = vcf_csi_depth(fasta_contigs, names)
    with ThreadPoolExecutor(max_workers=2) as pool:
        hgz, hu, hc = _bgzf(head, pool, 1)
        hgz = hgz[:-len(BGZF_EOF)]
        chunks, blk_u, blk_c = [hgz], [hu], [hc[:-1]]
        u, c = len(head), len(hgz)
        tids, beg, end, ulen = [], [], [], []
        for p in parts:
            if not p.lines.shape[0]:
                continue
            blk_u.append(u + np.concatenate([[0], np.cumsum(p.usizes)[:-1]]))
            blk_c.append(c + np.concatenate([[0], np.cumsum(p.csizes)[:-1]]))
            chunks.append(p.data)
            u += int(p.usizes.sum()); c += int(p.csizes.sum())
            tids.append(np.full(p.lines.shape[0], len(tids), np.int64))
            beg.append(p.lines["pos"]); end.append(p.lines["pos"] + p.lines["ref_len"]); ulen.append(p.lines["text_len"])
        with open(path, "wb") as fh:
            fh.write(b"".join(chunks) + BGZF_EOF)
        cat = (lambda a: np.concatenate(a).astype(np.int64) if a else np.zeros(0, np.int64))     # noqa: E731
        us = len(head) + np.concatenate([[0], np.cumsum(cat(ulen))])
        idx = _tabix(names, cat(tids), cat(beg), cat(end), us[:-1], us[1:], np.concatenate(blk_u), np.concatenate(blk_c), c, u, depth)
        with open(path + (".tbi" if depth is None else ".csi"), "wb") as fh:
            fh.write(_bgzf(idx, pool)[0])


def stitch_sink_edits_test(bases, phred, draft, position, index, image_region, chunk_id, region_starts, chunk: int,
                           capacity_events: int | None = None, stream: int = 0):
    """Diagnostics (pb_test_polish_stitch_sink_edits): pb_test_polish_stitch_sink with the event sink of an edits session;
    `draft` uint8 [n, 1000] holds each column's upper-cased draft base.  Returns (consensus str, bytes per region, events
    (EDIT_EVENT), events per region).  PepperB200Error(PB_ERR_CAPACITY) when `capacity_events` is too small."""
    _lib.require_gpu()
    L = _lib.lib()
    _bind(L)
    arr = lambda a, t: np.ascontiguousarray(a, dtype=t)          # noqa: E731
    b, q, d = arr(bases, np.uint8), arr(phred, np.uint8), arr(draft, np.uint8)
    p, i = arr(position, np.int64), arr(index, np.int32)
    r, c, s = arr(image_region, np.int32), arr(chunk_id, np.int32), arr(region_starts, np.int64)
    if not (q.shape == b.shape == d.shape):
        raise ValueError("bases, phred and draft must have one shape")
    cap = max(1, b.shape[0] * POLISH_SEQ_LEN)
    ecap = cap + b.shape[0] if capacity_events is None else int(capacity_events)
    out = np.empty(cap, np.uint8)
    ev = np.empty(max(1, ecap), EDIT_EVENT)
    per_region, ev_region = np.zeros(s.shape[0], np.int64), np.zeros(s.shape[0], np.int64)
    n, n_ev = C.c_int64(0), C.c_int64(0)
    _lib.check(L.pb_test_polish_stitch_sink_edits(b.ctypes.data, q.ctypes.data, d.ctypes.data, p.ctypes.data, i.ctypes.data, r.ctypes.data,
                                                  c.ctypes.data, s.ctypes.data, s.shape[0], b.shape[0], int(chunk), out.ctypes.data, cap,
                                                  C.byref(n), per_region.ctypes.data, ev.ctypes.data, ecap, C.byref(n_ev),
                                                  ev_region.ctypes.data, C.c_void_p(stream)), "pb_test_polish_stitch_sink_edits")
    return bytes(out[:n.value]).decode(), per_region, ev[:n_ev.value].copy(), ev_region
