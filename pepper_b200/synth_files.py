"""Writers for the file formats the readers of pepper_b200/csrc/bamio.cu consume: BAM (BGZF) + BAI, FASTA + FAI.
Written from the SAM/BAM specification (SAMv1 §4.1 BGZF, §4.2 BAM records, §5.2 BAI, §5.3 reg2bin) with Python's zlib;
used by tests and bench scripts to put the seeded synthetic records of synth.py on disk (there is no samtools / pysam in
the image and the reference ships no alignment files)."""
from __future__ import annotations

import os
import struct
import zlib
import numpy as np

from .synth import RecordBatch

BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def reg2bin(beg: int, end: int) -> int:
    end -= 1
    if beg >> 14 == end >> 14:
        return ((1 << 15) - 1) // 7 + (beg >> 14)
    if beg >> 17 == end >> 17:
        return ((1 << 12) - 1) // 7 + (beg >> 17)
    if beg >> 20 == end >> 20:
        return ((1 << 9) - 1) // 7 + (beg >> 20)
    if beg >> 23 == end >> 23:
        return ((1 << 6) - 1) // 7 + (beg >> 23)
    if beg >> 26 == end >> 26:
        return ((1 << 3) - 1) // 7 + (beg >> 26)
    return 0


def _bgzf_block(payload: bytes, level: int, deflate=None) -> bytes:
    """One BGZF member; `deflate(payload)` -> raw DEFLATE bytes replaces zlib at `level` when given."""
    if deflate is None:
        co = zlib.compressobj(level, zlib.DEFLATED, -15)
        data = co.compress(payload) + co.flush()
    else:
        data = deflate(payload)
    bsize = 18 + len(data) + 8
    assert bsize <= 65536
    return (b"\x1f\x8b\x08\x04" + b"\0\0\0\0" + b"\0\xff" + struct.pack("<H", 6) + b"BC" + struct.pack("<HH", 2, bsize - 1)
            + data + struct.pack("<II", zlib.crc32(payload) & 0xffffffff, len(payload)))


def record_ref_len(cigar_words: np.ndarray) -> int:
    ops = cigar_words & 15
    return int((cigar_words[np.isin(ops, [0, 2, 3, 7, 8])] >> 4).sum())


def write_bam(path: str, contigs: list[tuple[str, int]], batches: dict[int, RecordBatch], header_text: str | None = None,
              block_payload: int = 60000, level: int = 1, long_cigar_over: int = 65535, aux=b"", cg_first: bool = False,
              deflate=None) -> None:
    """`batches`: tid -> coordinate-sorted RecordBatch.  Writes `path` and `path + '.bai'`.  Records are cut into BGZF
    blocks every `block_payload` bytes regardless of record boundaries (records span blocks, as in real files).  CIGARs
    with more than `long_cigar_over` ops use the CG:B,I convention (SAMv1 4.2.2).  `aux`: the encoded aux tags of every
    record, or a function of the record's index in its batch that returns them; the CG tag goes after them, or before them
    with `cg_first`.  `deflate`: payload bytes -> raw DEFLATE stream of each BGZF block (default zlib at `level`); the
    index holds the virtual offsets of the blocks as written."""
    if header_text is None:
        header_text = "@HD\tVN:1.6\tSO:coordinate\n" + "".join(f"@SQ\tSN:{n}\tLN:{l}\n" for n, l in contigs) + \
            "@RG\tID:rg1\tSM:sample_b200\n"
    head = b"BAM\x01" + struct.pack("<i", len(header_text)) + header_text.encode() + struct.pack("<i", len(contigs))
    for n, l in contigs:
        head += struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", l)
    parts = [head]
    u = len(head)
    rec_spans = {}                                      # tid -> list of (beg, end, ustart, uend)
    for tid in sorted(batches):
        b = batches[tid]
        spans = []
        for r in range(b.n_records):
            so, se = int(b.seq_off[r]), int(b.seq_off[r + 1])
            l_seq = se - so
            cig = b.cigar[b.cigar_off[r]:b.cigar_off[r + 1]].astype("<u4")
            rlen = record_ref_len(cig) if cig.shape[0] else 0
            pos = int(b.pos[r])
            end = pos + (rlen if rlen > 0 else 1)
            name = f"r{tid}_{r}".encode() + b"\0"
            codes = _codes(b, so, se)
            if l_seq & 1:
                codes = np.concatenate([codes, np.zeros(1, np.uint8)])
            seq = ((codes[0::2] << 4) | codes[1::2]).astype(np.uint8).tobytes()
            qual = b.qual[so:se].tobytes()
            tags = aux(r) if callable(aux) else aux
            cig_field = cig
            if cig.shape[0] > long_cigar_over:
                cig_field = np.array([(l_seq << 4) | 4, (rlen << 4) | 3], dtype="<u4")
                cg = b"CGBI" + struct.pack("<i", cig.shape[0]) + cig.tobytes()
                tags = cg + tags if cg_first else tags + cg
            body = struct.pack("<iiBBHHHiiii", tid, pos, len(name), int(b.mapq[r]), reg2bin(pos, end), cig_field.shape[0],
                               int(b.flag[r]), l_seq, -1, -1, 0) + name + cig_field.tobytes() + seq + qual + tags
            rec = struct.pack("<i", len(body)) + body
            parts.append(rec)
            spans.append((pos, end, u, u + len(rec)))
            u += len(rec)
        rec_spans[tid] = spans
    stream = b"".join(parts)
    # cut into blocks
    ustart, coff, out = [], [], []
    c = 0
    for s in range(0, len(stream), block_payload):
        blk = _bgzf_block(stream[s:s + block_payload], level, deflate)
        ustart.append(s)
        coff.append(c)
        out.append(blk)
        c += len(blk)
    eof_coff = c
    out.append(BGZF_EOF)
    with open(path, "wb") as f:
        f.write(b"".join(out))
    ustart_a = np.array(ustart, dtype=np.int64)

    def voff(upos: int) -> int:
        if upos >= len(stream):
            return eof_coff << 16
        k = int(np.searchsorted(ustart_a, upos, side="right") - 1)
        return (coff[k] << 16) | (upos - ustart[k])
    with open(path + ".bai", "wb") as f:
        f.write(_bai_bytes(len(contigs), rec_spans, voff))


def _bai_bytes(n_contigs: int, rec_spans: dict, voff) -> bytes:
    """BAI (SAMv1 5.2) from per-contig record spans (pos, end, ustart, uend); `voff(upos)` -> virtual file offset."""
    bai = b"BAI\x01" + struct.pack("<i", n_contigs)
    for tid in range(n_contigs):
        spans = rec_spans.get(tid, [])
        bins: dict[int, list[list[int]]] = {}
        n_win = 0
        linear: dict[int, int] = {}
        for (pos, end, us, ue) in spans:
            vb, ve = voff(us), voff(ue)
            ch = bins.setdefault(reg2bin(pos, end), [])
            if ch and ch[-1][1] == vb:
                ch[-1][1] = ve
            else:
                ch.append([vb, ve])
            for w in range(pos >> 14, ((end - 1) >> 14) + 1):
                if w not in linear or vb < linear[w]:
                    linear[w] = vb
                n_win = max(n_win, w + 1)
        meta = None
        if spans:
            meta = [[voff(spans[0][2]), voff(spans[-1][3])], [len(spans), 0]]        # pseudo-bin 37450 (ignored by readers)
        bai += struct.pack("<i", len(bins) + (1 if meta else 0))
        for bn in sorted(bins):
            bai += struct.pack("<Ii", bn, len(bins[bn]))
            for vb, ve in bins[bn]:
                bai += struct.pack("<QQ", vb, ve)
        if meta:
            bai += struct.pack("<Ii", 37450, 2) + struct.pack("<QQQQ", meta[0][0], meta[0][1], meta[1][0], meta[1][1])
        bai += struct.pack("<i", n_win)
        last = 0
        parts = []
        for w in range(n_win):
            last = linear.get(w, last)
            parts.append(struct.pack("<Q", last))
        bai += b"".join(parts)
    return bai


def _reg2bin_v(beg: np.ndarray, end: np.ndarray) -> np.ndarray:
    e = end - 1
    conds = [(beg >> 14) == (e >> 14), (beg >> 17) == (e >> 17), (beg >> 20) == (e >> 20), (beg >> 23) == (e >> 23), (beg >> 26) == (e >> 26)]
    vals = [4681 + (beg >> 14), 585 + (beg >> 17), 73 + (beg >> 20), 9 + (beg >> 23), 1 + (beg >> 26)]
    return np.select(conds, vals, default=0).astype(np.int64)


_TILED = {}


def _compress_range(args):
    lo, hi, payload, level = args
    stream = _TILED["stream"]
    out, lens = [], []
    for k in range(lo, hi):
        blk = _bgzf_block(stream[k * payload:(k + 1) * payload].tobytes(), level)
        out.append(blk); lens.append(len(blk))
    return b"".join(out), lens


def write_bam_tiled(path: str, contig: str, rec: RecordBatch, span: int, times: int, block_payload: int = 60000, level: int = 1,
                    workers: int = 0) -> int:
    """A large coordinate-sorted BAM from ONE simulated block: the records of `rec` (positions inside [0, span)) are laid out
    `times` times along the contig, copy t shifted by t * span.  The uncompressed stream of the block is built once and tiled
    with numpy (position / bin fields patched per copy); BGZF blocks are compressed by a fork pool.  Returns the contig length.
    Same on-disk layout as write_bam (records span BGZF blocks; BAI with bins + 16 kb linear index)."""
    import multiprocessing as mp
    contig_len = span * times
    header_text = "@HD\tVN:1.6\tSO:coordinate\n" + f"@SQ\tSN:{contig}\tLN:{contig_len}\n" + "@RG\tID:rg1\tSM:sample_b200\n"
    head = b"BAM\x01" + struct.pack("<i", len(header_text)) + header_text.encode() + struct.pack("<i", 1)
    head += struct.pack("<i", len(contig) + 1) + contig.encode() + b"\0" + struct.pack("<i", contig_len)
    recs, rec_off, pos0, end0 = [], [], [], []
    u = 0
    for r in range(rec.n_records):
        so, se = int(rec.seq_off[r]), int(rec.seq_off[r + 1])
        l_seq = se - so
        cig = rec.cigar[rec.cigar_off[r]:rec.cigar_off[r + 1]].astype("<u4")
        rlen = record_ref_len(cig) if cig.shape[0] else 0
        pos = int(rec.pos[r])
        end = pos + (rlen if rlen > 0 else 1)
        name = f"r{r}".encode() + b"\0"
        codes = _codes(rec, so, se)
        if l_seq & 1:
            codes = np.concatenate([codes, np.zeros(1, np.uint8)])
        seq = ((codes[0::2] << 4) | codes[1::2]).astype(np.uint8).tobytes()
        body = struct.pack("<iiBBHHHiiii", 0, pos, len(name), int(rec.mapq[r]), 0, cig.shape[0], int(rec.flag[r]), l_seq, -1, -1, 0) + name + \
            cig.tobytes() + seq + rec.qual[so:se].tobytes()
        b = struct.pack("<i", len(body)) + body
        recs.append(b); rec_off.append(u); pos0.append(pos); end0.append(end)
        u += len(b)
    block = np.frombuffer(b"".join(recs), dtype=np.uint8)
    blen = block.shape[0]
    rec_off = np.array(rec_off, dtype=np.int64); pos0 = np.array(pos0, dtype=np.int64); end0 = np.array(end0, dtype=np.int64)
    assert pos0.shape[0] == 0 or (pos0.max() < span and np.all(np.diff(pos0) >= 0))
    stream = np.empty(len(head) + blen * times, dtype=np.uint8)
    stream[:len(head)] = np.frombuffer(head, dtype=np.uint8)
    stream[len(head):] = np.tile(block, times)
    shift = (np.arange(times, dtype=np.int64) * span)[:, None]
    pos = (pos0[None, :] + shift).ravel()
    end = (end0[None, :] + shift).ravel()
    off = (len(head) + rec_off[None, :] + (np.arange(times, dtype=np.int64) * blen)[:, None]).ravel()
    bins = _reg2bin_v(pos, end)
    for k in range(4):
        stream[off + 8 + k] = (pos >> (8 * k)) & 255
    for k in range(2):
        stream[off + 14 + k] = (bins >> (8 * k)) & 255
    n_blocks = (stream.shape[0] + block_payload - 1) // block_payload
    _TILED["stream"] = stream
    workers = workers or min(64, os.cpu_count() or 1)
    per = max(1, -(-n_blocks // (workers * 4)))
    tasks = [(lo, min(n_blocks, lo + per), block_payload, level) for lo in range(0, n_blocks, per)]
    if workers > 1 and len(tasks) > 1:
        with mp.get_context("fork").Pool(workers) as pool:
            parts = pool.map(_compress_range, tasks)
    else:
        parts = [_compress_range(t) for t in tasks]
    _TILED.clear()
    lens = np.array([l for _, ls in parts for l in ls], dtype=np.int64)
    coff = np.concatenate([[0], np.cumsum(lens)])
    with open(path, "wb") as f:
        for data, _ in parts:
            f.write(data)
        f.write(BGZF_EOF)
    eof_coff = int(coff[-1])
    total = stream.shape[0]

    def voff(upos: int) -> int:
        if upos >= total:
            return eof_coff << 16
        k = upos // block_payload
        return (int(coff[k]) << 16) | (upos - k * block_payload)
    rec_len = np.diff(np.concatenate([rec_off, [blen]]))
    uend = off + np.tile(rec_len, times)
    spans = list(zip(pos.tolist(), end.tolist(), off.tolist(), uend.tolist()))
    with open(path + ".bai", "wb") as f:
        f.write(_bai_bytes(1, {0: spans}, voff))
    return contig_len


def _codes(b: RecordBatch, so: int, se: int) -> np.ndarray:
    idx = np.arange(so, se)
    byte = b.seq[idx >> 1]
    return np.where(idx & 1, byte & 15, byte >> 4).astype(np.uint8)


def write_fasta(path: str, contigs: list[tuple[str, np.ndarray]], line: int = 60) -> None:
    """FASTA + .fai (name, length, offset, linebases, linewidth)."""
    off = 0
    fai = []
    with open(path, "wb") as f:
        for name, seq in contigs:
            hdr = f">{name} synthetic\n".encode()
            f.write(hdr)
            off += len(hdr)
            s = bytes(np.asarray(seq, dtype=np.uint8))
            fai.append(f"{name}\t{len(s)}\t{off}\t{line}\t{line + 1}\n")
            for i in range(0, len(s), line):
                f.write(s[i:i + line] + b"\n")
            off += len(s) + (len(s) + line - 1) // line
    with open(path + ".fai", "w") as f:
        f.write("".join(fai))
