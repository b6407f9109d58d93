"""Writers for the file formats the readers of pepper_b200/csrc/bamio.cu consume: BAM (BGZF) + BAI and / or CSI, FASTA + FAI,
plain or bgzip-compressed + GZI.  Written from the specifications (SAMv1 §4.1 BGZF, §4.2 BAM records, §5.2 BAI, §5.3 reg2bin;
CSIv1) with Python's zlib;
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


def csi_depth_for(max_len: int, min_shift: int = 14) -> int:
    """The smallest CSI depth >= 5 whose reach 2^(min_shift + 3 depth) covers positions [0, max_len)."""
    depth = 5
    while (1 << (min_shift + 3 * depth)) < max_len:
        depth += 1
    return depth


def write_bam(path: str, contigs: list[tuple[str, int]], batches: dict[int, RecordBatch], header_text: str | None = None,
              block_payload: int = 60000, level: int = 1, long_cigar_over: int = 65535, aux=b"", cg_first: bool = False,
              deflate=None, index: str = "bai", csi_depth: int | None = None, csi_min_shift: int = 14) -> None:
    """`batches`: tid -> coordinate-sorted RecordBatch.  Writes `path` and its index: `index` "bai" (`path + '.bai'`), "csi"
    (`path + '.csi'`, binning (`csi_min_shift`, `csi_depth`), the depth by default the smallest >= 5 that covers the contigs)
    or "both".  A record past 2^29 gets bin 4680 (no BAI bin can hold it; the readers ignore the field).  Records are cut into BGZF
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
            body = struct.pack("<iiBBHHHiiii", tid, pos, len(name), int(b.mapq[r]), reg2bin(pos, end) if end <= BAI_MAX_END else 4680, cig_field.shape[0],
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
    assert index in ("bai", "csi", "both"), index
    if index in ("bai", "both"):
        with open(path + ".bai", "wb") as f:
            f.write(_bai_bytes(len(contigs), rec_spans, voff))
    if index in ("csi", "both"):
        depth = csi_depth if csi_depth is not None else csi_depth_for(max([l for _, l in contigs] + [1]), csi_min_shift)
        refs = []
        for tid in range(len(contigs)):
            sp = np.array(rec_spans.get(tid, []), dtype=np.int64).reshape(-1, 4)
            vb = np.array([voff(int(u)) for u in sp[:, 2]], dtype=np.uint64)
            ve = np.array([voff(int(u)) for u in sp[:, 3]], dtype=np.uint64)
            refs.append(csi_reference(sp[:, 0], sp[:, 1], vb, ve, csi_min_shift, depth))
        with open(path + ".csi", "wb") as f:
            f.write(bgzf_bytes(csi_bytes(csi_min_shift, depth, b"", refs)))


BAI_MAX_END = 1 << 29


def bgzf_bytes(data: bytes, payload: int = 0xff00, level: int = 6) -> bytes:
    """`data` as BGZF members of `payload` bytes + the EOF block (how an index file is stored)."""
    return b"".join(_bgzf_block(data[s:s + payload], level) for s in range(0, len(data), payload)) + BGZF_EOF


def csi_bytes(min_shift: int, depth: int, aux: bytes, refs: list[bytes]) -> bytes:
    """The uncompressed CSI (CSIv1): magic, min_shift, depth, l_aux, aux, n_ref, then each reference's bytes (csi_reference)."""
    return b"CSI\x01" + struct.pack("<iii", min_shift, depth, len(aux)) + aux + struct.pack("<i", len(refs)) + b"".join(refs)


def csi_reference(beg: np.ndarray, end: np.ndarray, vb: np.ndarray, ve: np.ndarray, min_shift: int, depth: int) -> bytes:
    """One reference of a CSI from the spans [beg, end) of its records / lines, in file order, with virtual offsets [vb, ve):
    n_bin, then per bin (bin, loffset, n_chunk, chunks), the pseudo-bin last.  A chunk is a run of consecutive records of one bin
    (the BAI writers' rule).  A bin's loffset is the virtual offset of the first record, in file order, that ends past the bin's
    start: no record overlapping the bin lies before it."""
    beg, end = np.asarray(beg, np.int64), np.asarray(end, np.int64)
    vb, ve = np.asarray(vb, np.uint64), np.asarray(ve, np.uint64)
    n = beg.shape[0]
    if n == 0:
        return struct.pack("<i", 0)
    bins = _reg2bin_v(beg, end, min_shift, depth)
    brk = np.flatnonzero(bins[1:] != bins[:-1]) + 1
    first, last = np.concatenate([[0], brk]), np.concatenate([brk, [n]]) - 1
    o = np.argsort(bins[first], kind="stable")
    cbin, cvb, cve = bins[first][o], vb[first][o], ve[last][o]
    ub, ufirst, cnt = np.unique(cbin, return_index=True, return_counts=True)
    level = np.zeros(ub.shape[0], np.int64)
    for l in range(1, depth + 1):
        level[ub >= ((1 << (3 * l)) - 1) // 7] = l
    bin_start = (ub - ((1 << (3 * level)) - 1) // 7) << (min_shift + 3 * (depth - level))
    k = np.searchsorted(np.maximum.accumulate(end), bin_start, side="right")
    loff = vb[np.minimum(k, n - 1)]
    out = [struct.pack("<i", ub.shape[0] + 1)]
    for i in range(ub.shape[0]):
        a, c = int(ufirst[i]), int(cnt[i])
        ch = np.empty(2 * c, "<u8")
        ch[0::2], ch[1::2] = cvb[a:a + c], cve[a:a + c]
        out.append(struct.pack("<IQi", int(ub[i]), int(loff[i]), c) + ch.tobytes())
    pseudo = ((1 << (3 * (depth + 1))) - 1) // 7 + 1
    out.append(struct.pack("<IQi", pseudo, 0, 2) + struct.pack("<QQQQ", int(vb[0]), int(ve[-1]), n, 0))
    return b"".join(out)


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


def _reg2bin_v(beg: np.ndarray, end: np.ndarray, min_shift: int = 14, depth: int = 5) -> np.ndarray:
    """SAMv1 5.3 reg2bin for arrays, in the binning (min_shift, depth); (14, 5) is a BAI's."""
    e = end - 1
    shifts = [min_shift + 3 * (depth - l) for l in range(depth, 0, -1)]
    conds = [(beg >> s) == (e >> s) for s in shifts]
    vals = [((1 << (3 * l)) - 1) // 7 + (beg >> s) for l, s in zip(range(depth, 0, -1), shifts)]
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


def write_fasta(path: str, contigs: list, line: int = 60, bgzip: bool = False, block_lines: int | None = None) -> None:
    """FASTA + .fai (name, length, offset, linebases, linewidth).  `contigs`: (name, sequence) pairs; a sequence is a uint8 array
    or a list of (uint8 array, repeat count) pieces, so that a long, mostly-N contig never exists in memory.  With `bgzip`, the
    file is BGZF-compressed with a .gzi (a u64 count, then a (compressed, uncompressed) offset pair per block but the first) and
    the .fai keeps uncompressed offsets, as `bgzip -i` + `samtools faidx` write.  Each contig's sequence starts a block, and its
    blocks are cut every `block_lines` lines (default: the most whole lines in 65,280 bytes), so a run of identical lines gives
    identical blocks, compressed once."""
    fai, pieces = [], []                                  # pieces: (bytes, times) of the uncompressed file, in order
    off = 0
    for name, seq in contigs:
        hdr = f">{name} synthetic\n".encode()
        pieces += [(hdr, 1), (None, 0)]                    # None: end the BGZF block, so the sequence starts a block of its own
        off += len(hdr)
        parts = [(np.asarray(seq, dtype=np.uint8), 1)] if isinstance(seq, np.ndarray) else [(np.asarray(a, np.uint8), int(t)) for a, t in seq]
        n = sum(a.shape[0] * t for a, t in parts)
        fai.append(f"{name}\t{n}\t{off}\t{line}\t{line + 1}\n")
        col = 0                                            # bases already on the current line
        for a, t in parts:
            if a.shape[0] == 0 or t == 0:
                continue
            if col == 0 and a.shape[0] % line == 0 and t > 1:          # whole lines repeated: one laid-out copy, repeated
                pieces.append((_lines(bytes(a), line), t))
                continue
            for _ in range(t):
                b = bytes(a)
                if col:
                    take = min(line - col, len(b))
                    pieces.append((b[:take] + (b"\n" if col + take == line else b""), 1))
                    col = (col + take) % line
                    b = b[take:]
                if b:
                    full = len(b) // line * line
                    pieces.append((_lines(b[:full], line) + b[full:], 1))
                    col = len(b) - full
        if col:
            pieces.append((b"\n", 1))
        off += n + (n + line - 1) // line
    with open(path + ".fai", "w") as f:
        f.write("".join(fai))
    if not bgzip:
        with open(path, "wb") as f:
            for b, t in pieces:
                if b is not None:
                    f.write(b * t)
        return
    payload = (block_lines or (0xff00 // (line + 1))) * (line + 1)
    cache: dict[bytes, bytes] = {}
    gzi, coff, uoff = [], 0, 0
    with open(path, "wb") as f:
        pend = b""
        for chunk in _payload_chunks(pieces, payload):
            blk = cache.get(chunk)
            if blk is None:
                blk = _bgzf_block(chunk, 6)
                if len(cache) < 64:
                    cache[chunk] = blk
            if uoff:
                gzi.append((coff, uoff))
            f.write(blk)
            coff += len(blk); uoff += len(chunk)
        f.write(BGZF_EOF)
    with open(path + ".gzi", "wb") as f:
        f.write(struct.pack("<Q", len(gzi)) + b"".join(struct.pack("<QQ", c, u) for c, u in gzi))


def _lines(b: bytes, line: int) -> bytes:
    return b"".join(b[i:i + line] + b"\n" for i in range(0, len(b), line))


def _payload_chunks(pieces: list, payload: int):
    """The uncompressed stream of (bytes, times) pieces cut into `payload`-byte chunks, without building it: a piece repeated
    many times yields the same chunk again and again once the cut lines up with it."""
    buf = b""
    for b, t in pieces:
        if b is None and buf:
            yield buf
            buf = b""
        while t:
            if not buf and len(b) and payload % len(b) == 0 and t * len(b) >= payload:     # whole chunks of repeats
                per = payload // len(b)
                chunk = b * per
                for _ in range(t // per):
                    yield chunk
                t %= per
                continue
            if not buf and len(b) % payload == 0 and len(b):
                for _ in range(t):
                    for i in range(0, len(b), payload):
                        yield b[i:i + payload]
                t = 0
                continue
            buf += b
            t -= 1
            while len(buf) >= payload:
                yield buf[:payload]
                buf = buf[payload:]
    if buf:
        yield buf
