"""Host side of the polish path: batched SummaryGenerator + chunking + network wrappers.

* ``PolishEncoder.encode`` == many ``SummaryGenerator(...).generate_summary(...)`` calls
  (pepper/modules/python/AlignmentSummarizer.py:341-348);
* ``chunk_images`` == ``AlignmentSummarizer.chunk_images`` (pepper/.../AlignmentSummarizer.py:19-56);
* ``PolishNet.predict`` == the window loop of pepper/modules/python/models/predict_distributed_cpu.py:50-90.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
import numpy as np

from . import _lib
from .abi import HostReads, PbReads, PbRegion, regions_array, POLISH_FEATURES, POLISH_SEQ_LEN, PB_ERR_CAPACITY
from .synth import ReadBatch, RegionTable

SEQ_OVERLAP = 50      # pepper Options.py ImageSizeOptions.SEQ_OVERLAP
# one consensus base of a qualities sink (pb_polish_stream_begin_qual): the base letter and its FASTQ quality byte
QUAL_RECORD = np.dtype([("base", "u1"), ("qual", "u1")])


@dataclass
class PolishSummary:
    image: np.ndarray     # uint8 [cols,10]
    pos: np.ndarray       # int64 [cols]
    idx: np.ndarray       # int32 [cols]
    col_off: np.ndarray   # int64 [n_regions+1]


def _bind(L):
    if getattr(L, "_polish_bound", False):
        return
    vp = C.c_void_p
    L.pb_polish_encoder_create.argtypes = [C.POINTER(vp), C.c_int]
    L.pb_polish_encoder_destroy.argtypes = [vp]
    L.pb_polish_encode_host.argtypes = [vp, C.POINTER(PbReads), C.POINTER(PbRegion), C.c_int64, C.c_int64, vp, vp, vp, vp,
                                        C.POINTER(C.c_int64), vp]
    L.pb_polish_encoder_timings.argtypes = [vp, vp]
    L._polish_bound = True


class PolishEncoder:
    def __init__(self, device: int = 0):
        _lib.require_gpu()
        self.L = _lib.lib()
        _bind(self.L)
        self.h = C.c_void_p()
        _lib.check(self.L.pb_polish_encoder_create(C.byref(self.h), device), "pb_polish_encoder_create")

    def close(self):
        if self.h:
            self.L.pb_polish_encoder_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def encode(self, reads: ReadBatch, regions: RegionTable, capacity: int | None = None, stream: int = 0) -> PolishSummary:
        hr = HostReads(reads)
        regs, keep = regions_array(regions)
        n_regions = regions.n_regions
        if capacity is None:
            span = int((regions.col("ref_end") - regions.col("ref_start") + 1).sum())
            capacity = 2 * span + 1024
        while True:
            img = np.empty((capacity, POLISH_FEATURES), dtype=np.uint8)
            pos = np.empty(capacity, dtype=np.int64)
            idx = np.empty(capacity, dtype=np.int32)
            off = np.zeros(n_regions + 1, dtype=np.int64)
            n = C.c_int64(0)
            rc = self.L.pb_polish_encode_host(self.h, C.byref(hr.struct), regs, n_regions, capacity, img.ctypes.data,
                                              pos.ctypes.data, idx.ctypes.data, off.ctypes.data, C.byref(n),
                                              C.c_void_p(stream))
            if rc == PB_ERR_CAPACITY:
                capacity = int(n.value) + 16
                continue
            _lib.check(rc, "pb_polish_encode_host")
            k = int(n.value)
            return PolishSummary(img[:k], pos[:k], idx[:k], off)

    def timings(self) -> dict:
        ms = (C.c_float * 3)()
        _lib.check(self.L.pb_polish_encoder_timings(self.h, ms), "timings")
        return dict(zip(("prefix", "count", "columns"), [float(x) for x in ms]))


def chunk_images(summary: PolishSummary, chunk_size: int = POLISH_SEQ_LEN, chunk_overlap: int = SEQ_OVERLAP):
    """AlignmentSummarizer.chunk_images for every region of a batch (AlignmentSummarizer.py:19-56):
    chunks of `chunk_size` columns, the next chunk starting `chunk_overlap` before the previous end, the last
    chunk zero padded with positions (-1, -1).  Returns images uint8 [n,1000,10], position int64 [n,1000],
    index int64 [n,1000], chunk_ids int32 [n], region_of int32 [n]."""
    imgs, poss, idxs, cids, regs = [], [], [], [], []
    for r in range(summary.col_off.shape[0] - 1):
        c0, c1 = int(summary.col_off[r]), int(summary.col_off[r + 1])
        n = c1 - c0
        start, end, cid = 0, min(n, chunk_size), 0
        while True:
            img = np.zeros((chunk_size, POLISH_FEATURES), dtype=np.uint8)
            pos = np.full(chunk_size, -1, dtype=np.int64)
            idx = np.full(chunk_size, -1, dtype=np.int64)
            m = end - start
            img[:m] = summary.image[c0 + start:c0 + end]
            pos[:m] = summary.pos[c0 + start:c0 + end]
            idx[:m] = summary.idx[c0 + start:c0 + end]
            imgs.append(img); poss.append(pos); idxs.append(idx); cids.append(cid); regs.append(r)
            cid += 1
            if end == n:
                break
            start = end - chunk_overlap
            end = min(n, start + chunk_size)
    if not imgs:
        return (np.zeros((0, chunk_size, POLISH_FEATURES), np.uint8), np.zeros((0, chunk_size), np.int64),
                np.zeros((0, chunk_size), np.int64), np.zeros(0, np.int32), np.zeros(0, np.int32))
    return (np.stack(imgs), np.stack(poss), np.stack(idxs), np.array(cids, dtype=np.int32),
            np.array(regs, dtype=np.int32))


class PolishNet:
    """bi-GRU x2 + Linear with the 19-window loop on one GPU (pb_polish_net_*)."""

    def __init__(self, state: dict, device: int = 0):
        from .variant import _state_arrays
        _lib.require_gpu()
        self.L = L = _lib.lib()
        vp = C.c_void_p
        L.pb_polish_net_param_name.restype = C.c_char_p
        L.pb_polish_net_param_name.argtypes = [C.c_int]
        L.pb_polish_net_param_numel.restype = C.c_int64
        L.pb_polish_net_param_numel.argtypes = [C.c_int]
        L.pb_polish_net_create.argtypes = [C.POINTER(vp), C.c_int, C.POINTER(vp)]
        L.pb_polish_net_destroy.argtypes = [vp]
        L.pb_polish_net_forward_host.argtypes = [vp, vp, C.c_int64, vp, vp, vp, vp, vp]
        L.pb_polish_net_launches.argtypes = [vp, C.POINTER(C.c_int64)]
        n = 18
        arrs = _state_arrays(L, state, n, L.pb_polish_net_param_name, L.pb_polish_net_param_numel)
        ptrs = (vp * n)(*[a.ctypes.data for a in arrs])
        self.h = vp()
        _lib.check(L.pb_polish_net_create(C.byref(self.h), device, ptrs), "pb_polish_net_create")

    def close(self):
        if self.h:
            self.L.pb_polish_net_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def predict(self, images_u8: np.ndarray, debug: bool = False, stream: int = 0):
        """uint8 [N,1000,10] host -> bases uint8 [N,1000], phred uint8 [N,1000]
        (+ hidden float32 [19,N,2,128], acc float32 [N,1000,5] when debug)."""
        x = np.ascontiguousarray(images_u8, dtype=np.uint8)
        n = x.shape[0]
        bases = np.empty((n, POLISH_SEQ_LEN), dtype=np.uint8)
        phred = np.empty((n, POLISH_SEQ_LEN), dtype=np.uint8)
        hid = np.empty((19, n, 2, 128), dtype=np.float32) if debug else None
        acc = np.empty((n, POLISH_SEQ_LEN, 5), dtype=np.float32) if debug else None
        _lib.check(self.L.pb_polish_net_forward_host(self.h, x.ctypes.data, n, bases.ctypes.data, phred.ctypes.data,
                                                    hid.ctypes.data if debug else None,
                                                    acc.ctypes.data if debug else None, C.c_void_p(stream)),
                   "pb_polish_net_forward_host")
        return (bases, phred, hid, acc) if debug else (bases, phred)

    def set_lo_mask(self, mask: int) -> None:
        """Experiments only: bit set = that GEMM keeps its third product; bits: 0 encoder h, 1 decoder x, 2 decoder h; default 7."""
        self.L.pb_polish_net_set_lo_mask.argtypes = [C.c_void_p, C.c_int]
        _lib.check(self.L.pb_polish_net_set_lo_mask(self.h, mask), "pb_polish_net_set_lo_mask")

    def launches(self) -> int:
        n = C.c_int64(0)
        _lib.check(self.L.pb_polish_net_launches(self.h, C.byref(n)), "launches")
        return int(n.value)


def stitch(bases, position, index, image_region, chunk_id, region_starts, stream: int = 0) -> str:
    """Consensus sequence of one contig from the per-image predictions (== pepper Stitch.py:36-128), on the GPU.
    Images ordered by region then chunk id; regions sorted by start (the order PolishCaller.call returns)."""
    _lib.require_gpu()
    L = _lib.lib()
    vp = C.c_void_p
    L.pb_polish_stitch_host.argtypes = [vp, vp, vp, vp, vp, vp, C.c_int64, C.c_int64, vp, C.c_int64, C.POINTER(C.c_int64), vp]
    b = np.ascontiguousarray(bases, dtype=np.uint8)
    p = np.ascontiguousarray(position, dtype=np.int64)
    i = np.ascontiguousarray(index, dtype=np.int32)
    r = np.ascontiguousarray(image_region, dtype=np.int32)
    c = np.ascontiguousarray(chunk_id, dtype=np.int32)
    s = np.ascontiguousarray(region_starts, dtype=np.int64)
    n_img = b.shape[0]
    cap = max(1, n_img * POLISH_SEQ_LEN)
    out = np.empty(cap, dtype=np.uint8)
    n = C.c_int64(0)
    _lib.check(L.pb_polish_stitch_host(b.ctypes.data, p.ctypes.data, i.ctypes.data, r.ctypes.data, c.ctypes.data, s.ctypes.data,
                                       s.shape[0], n_img, out.ctypes.data, cap, C.byref(n), C.c_void_p(stream)), "pb_polish_stitch_host")
    return bytes(out[:int(n.value)]).decode()


def stitch_with_qualities(bases, phred, position, index, image_region, chunk_id, region_starts, stream: int = 0) -> tuple[str, str]:
    """`stitch` with the quality of every consensus base, on the GPU: (sequence, FASTQ quality string).  The QV of a base is
    the network phred of the image column whose base won the stitch, written as '!' + min(phred, 93); the sequence is what
    `stitch` returns."""
    _lib.require_gpu()
    L = _lib.lib()
    vp = C.c_void_p
    L.pb_polish_stitch_qual_host.argtypes = [vp, vp, vp, vp, vp, vp, vp, C.c_int64, C.c_int64, vp, vp, C.c_int64, C.POINTER(C.c_int64), vp]
    b = np.ascontiguousarray(bases, dtype=np.uint8)
    q = np.ascontiguousarray(phred, dtype=np.uint8)
    p = np.ascontiguousarray(position, dtype=np.int64)
    i = np.ascontiguousarray(index, dtype=np.int32)
    r = np.ascontiguousarray(image_region, dtype=np.int32)
    c = np.ascontiguousarray(chunk_id, dtype=np.int32)
    s = np.ascontiguousarray(region_starts, dtype=np.int64)
    if q.shape != b.shape:
        raise ValueError("phred shape %s != bases shape %s" % (q.shape, b.shape))
    n_img = b.shape[0]
    cap = max(1, n_img * POLISH_SEQ_LEN)
    out = np.empty(cap, dtype=np.uint8)
    qual = np.empty(cap, dtype=np.uint8)
    n = C.c_int64(0)
    _lib.check(L.pb_polish_stitch_qual_host(b.ctypes.data, q.ctypes.data, p.ctypes.data, i.ctypes.data, r.ctypes.data, c.ctypes.data,
                                            s.ctypes.data, s.shape[0], n_img, out.ctypes.data, qual.ctypes.data, cap, C.byref(n),
                                            C.c_void_p(stream)), "pb_polish_stitch_qual_host")
    k = int(n.value)
    return bytes(out[:k]).decode(), bytes(qual[:k]).decode()


def stitch_sink_test(bases, position, index, image_region, chunk_id, region_starts, chunk: int, stream: int = 0, phred=None):
    """Diagnostics (pb_test_polish_stitch_sink): the predictions of images in session order through the streaming session's
    stitch-to-sink kernel, `chunk` images per call.  Returns (consensus str, bytes per region int64 [n_regions]); given `phred`
    (pb_test_polish_stitch_sink_qual: the sink of a qualities session), ((consensus str, quality str), records per region)."""
    _lib.require_gpu()
    L = _lib.lib()
    vp = C.c_void_p
    b = np.ascontiguousarray(bases, dtype=np.uint8)
    p = np.ascontiguousarray(position, dtype=np.int64)
    i = np.ascontiguousarray(index, dtype=np.int32)
    r = np.ascontiguousarray(image_region, dtype=np.int32)
    c = np.ascontiguousarray(chunk_id, dtype=np.int32)
    s = np.ascontiguousarray(region_starts, dtype=np.int64)
    cap = max(1, b.shape[0] * POLISH_SEQ_LEN)
    per_region = np.zeros(s.shape[0], np.int64)
    n = C.c_int64(0)
    if phred is None:
        L.pb_test_polish_stitch_sink.argtypes = [vp, vp, vp, vp, vp, vp, C.c_int64, C.c_int64, C.c_int64, vp, C.c_int64,
                                                 C.POINTER(C.c_int64), vp, vp]
        out = np.empty(cap, dtype=np.uint8)
        _lib.check(L.pb_test_polish_stitch_sink(b.ctypes.data, p.ctypes.data, i.ctypes.data, r.ctypes.data, c.ctypes.data, s.ctypes.data,
                                                s.shape[0], b.shape[0], int(chunk), out.ctypes.data, cap, C.byref(n), per_region.ctypes.data,
                                                C.c_void_p(stream)), "pb_test_polish_stitch_sink")
        return bytes(out[:int(n.value)]).decode(), per_region
    L.pb_test_polish_stitch_sink_qual.argtypes = [vp, vp, vp, vp, vp, vp, vp, C.c_int64, C.c_int64, C.c_int64, vp, C.c_int64,
                                                  C.POINTER(C.c_int64), vp, vp]
    q = np.ascontiguousarray(phred, dtype=np.uint8)
    if q.shape != b.shape:
        raise ValueError("phred shape %s != bases shape %s" % (q.shape, b.shape))
    rec = np.empty(cap, dtype=QUAL_RECORD)
    _lib.check(L.pb_test_polish_stitch_sink_qual(b.ctypes.data, q.ctypes.data, p.ctypes.data, i.ctypes.data, r.ctypes.data, c.ctypes.data,
                                                 s.ctypes.data, s.shape[0], b.shape[0], int(chunk), rec.ctypes.data, cap, C.byref(n),
                                                 per_region.ctypes.data, C.c_void_p(stream)), "pb_test_polish_stitch_sink_qual")
    return split_records(rec[:int(n.value)]), per_region


def split_records(rec: np.ndarray) -> tuple[str, str]:
    """(base, qual) records of a qualities sink -> (sequence, quality string)."""
    return rec["base"].tobytes().decode(), rec["qual"].tobytes().decode()
