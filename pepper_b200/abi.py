"""ctypes mirror of include/pepper_b200.h (structs only; no library is loaded here)."""
from __future__ import annotations

import ctypes as C
import numpy as np

from .synth import ReadBatch, RecordBatch, RegionTable

WINDOW = 33
FEATURES = 26
ALLELE_STRIDE = 64
POLISH_FEATURES = 10
POLISH_SEQ_LEN = 1000

PB_OK = 0
PB_ERR_ARG = -1
PB_ERR_CUDA = -2
PB_ERR_CAPACITY = -3
PB_ERR_STATE = -4

# pb_variant_net_create runs the decoder in mode 2 only below this weight-only gate error estimate (pb_variant_net_q8_guard)
PB_VARIANT_Q8_MAX_GATE_ERR = 1e-4
# ... and linear_1 on int8 slices only below this one (pb_variant_net_q8_head_err)
PB_VARIANT_Q8_HEAD_MAX_ERR = 3e-5


class PbReads(C.Structure):
    _fields_ = [("n_reads", C.c_int64),
                ("pos", C.c_void_p), ("seq_off", C.c_void_p), ("cigar_off", C.c_void_p),
                ("flags", C.c_void_p), ("mapq", C.c_void_p),
                ("seq", C.c_void_p), ("qual", C.c_void_p), ("cigar", C.c_void_p)]


class PbRecords(C.Structure):
    _fields_ = [("n_records", C.c_int64),
                ("pos", C.c_void_p), ("seq_off", C.c_void_p), ("cigar_off", C.c_void_p),
                ("flag", C.c_void_p), ("mapq", C.c_void_p),
                ("seq", C.c_void_p), ("qual", C.c_void_p), ("cigar", C.c_void_p)]


class PbInterval(C.Structure):
    _fields_ = [("start", C.c_int64), ("stop", C.c_int64)]


class PbGetReadsOptions(C.Structure):
    _fields_ = [("include_supplementary", C.c_int32), ("min_mapq", C.c_int32), ("min_baseq", C.c_int32),
                ("reserved", C.c_int32)]


class PbRegion(C.Structure):
    _fields_ = [(n, C.c_int64) for n in RegionTable.FIELDS]


class PbVariantParams(C.Structure):
    _fields_ = [("min_snp_baseq", C.c_double), ("min_indel_baseq", C.c_double),
                ("snp_freq_threshold", C.c_double), ("insert_freq_threshold", C.c_double),
                ("delete_freq_threshold", C.c_double), ("min_coverage_threshold", C.c_double),
                ("snp_candidate_freq_threshold", C.c_double), ("indel_candidate_freq_threshold", C.c_double),
                ("candidate_support_threshold", C.c_double), ("skip_indels", C.c_int32), ("reserved", C.c_int32)]


class PbCandidateColumns(C.Structure):
    _fields_ = [("positions", C.c_void_p), ("region_of", C.c_void_p), ("depths", C.c_void_p), ("freqs", C.c_void_p),
                ("keys", C.c_void_p)]


# pb_pred_record_t: the 84-byte prediction record of one candidate (what a rank-0 writer needs, SURVEY 8e)
PRED_RECORD = np.dtype([("probs", np.float32, (3,)), ("position", np.int32), ("region", np.int32), ("depth", np.uint8),
                        ("freq", np.uint8), ("key", "S62")])
assert PRED_RECORD.itemsize == 84


def _c(a: np.ndarray, dtype) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=dtype)


class HostReads:
    """Keeps the numpy arrays alive and exposes a pb_reads_t pointing at them."""

    def __init__(self, b: ReadBatch, pin: bool = False):
        self._pin = pin
        self._pinned = []
        self.pos = _c(b.pos, np.int64)
        self.seq_off = _c(b.seq_off, np.int64)
        self.cigar_off = _c(b.cigar_off, np.int64)
        self.flags = _c(b.flags, np.uint8)
        self.mapq = _c(b.mapq, np.uint8)
        # one spare byte so an empty batch still has a valid pointer
        self.seq = _c(np.concatenate([b.seq, np.zeros(1, np.uint8)]), np.uint8)
        self.qual = _c(np.concatenate([b.qual, np.zeros(1, np.uint8)]), np.uint8)
        self.cigar = _c(np.concatenate([b.cigar, np.zeros(1, np.uint32)]), np.uint32)
        self.n_bases = int(b.seq_off[-1])
        self.n_ops = int(b.cigar_off[-1])
        if pin:
            # page-locked copies (torch is used only as the pinned allocator)
            import torch
            for name in ("pos", "seq_off", "cigar_off", "flags", "mapq", "seq", "qual", "cigar"):
                a = getattr(self, name)
                src = a.view(np.int32) if a.dtype == np.uint32 else a
                t = torch.from_numpy(src).pin_memory()
                self._pinned.append(t)
                v = t.numpy()
                setattr(self, name, v.view(np.uint32) if a.dtype == np.uint32 else v)
        self.nbytes = sum(getattr(self, n).nbytes for n in ("pos", "seq_off", "cigar_off", "flags", "mapq", "seq", "qual", "cigar"))
        self.struct = PbReads(b.n_reads, self.pos.ctypes.data, self.seq_off.ctypes.data,
                              self.cigar_off.ctypes.data, self.flags.ctypes.data, self.mapq.ctypes.data,
                              self.seq.ctypes.data, self.qual.ctypes.data, self.cigar.ctypes.data)


class HostRecords:
    """Keeps the numpy arrays alive and exposes a pb_records_t pointing at them."""

    def __init__(self, b: RecordBatch):
        self.pos = _c(b.pos, np.int64)
        self.seq_off = _c(b.seq_off, np.int64)
        self.cigar_off = _c(b.cigar_off, np.int64)
        self.flag = _c(b.flag, np.uint16)
        self.mapq = _c(b.mapq, np.uint8)
        self.seq = _c(np.concatenate([b.seq, np.zeros(1, np.uint8)]), np.uint8)
        self.qual = _c(np.concatenate([b.qual, np.zeros(1, np.uint8)]), np.uint8)
        self.cigar = _c(np.concatenate([b.cigar, np.zeros(1, np.uint32)]), np.uint32)
        self.nbytes = sum(getattr(self, n).nbytes for n in ("pos", "seq_off", "cigar_off", "flag", "mapq", "seq", "qual", "cigar"))
        self.struct = PbRecords(b.n_records, self.pos.ctypes.data, self.seq_off.ctypes.data, self.cigar_off.ctypes.data,
                                self.flag.ctypes.data, self.mapq.ctypes.data, self.seq.ctypes.data, self.qual.ctypes.data,
                                self.cigar.ctypes.data)


def intervals_array(intervals):
    """ctypes array of pb_interval_t from [(start, stop), ...]"""
    t = _c(np.asarray(intervals, dtype=np.int64).reshape(-1, 2), np.int64)
    return (PbInterval * t.shape[0]).from_buffer(t), t


def regions_array(tab: RegionTable):
    """ctypes array of pb_region_t sharing memory with a contiguous int64 copy of the table."""
    t = _c(tab.table, np.int64)
    arr = (PbRegion * t.shape[0]).from_buffer(t)
    return arr, t


def variant_params(**kw) -> PbVariantParams:
    p = PbVariantParams()
    for k, v in kw.items():
        setattr(p, k, v)
    return p
