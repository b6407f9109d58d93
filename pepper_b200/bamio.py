"""File readers under BAM_handler / FASTA_handler (SURVEY.md §8f row f4): ctypes front-end of the host-side BGZF / BAM /
BAI / CSI and FASTA / FAI (plain or bgzip + GZI) readers in libpepper_b200.so (pepper_b200/csrc/bamio.cu).  Reference: BAM_handler(path) and its
accessors (pepper/modules/src/dataio/bam_handler.cpp:6-113), FASTA_handler (fasta_handler.cpp:7-55)."""
from __future__ import annotations

import ctypes as C
import numpy as np

from . import _lib
from .abi import PbRecords
from .synth import RecordBatch


def _bind(L):
    if getattr(L, "_bamio_bound", False):
        return
    L.pb_bam_open.argtypes = [C.POINTER(C.c_void_p), C.c_char_p, C.c_int]
    L.pb_bam_close.argtypes = [C.c_void_p]
    L.pb_bam_n_contigs.argtypes = [C.c_void_p]
    L.pb_bam_contig_name.argtypes = [C.c_void_p, C.c_int]
    L.pb_bam_contig_name.restype = C.c_char_p
    L.pb_bam_contig_length.argtypes = [C.c_void_p, C.c_int]
    L.pb_bam_contig_length.restype = C.c_int64
    L.pb_bam_contig_id.argtypes = [C.c_void_p, C.c_char_p]
    L.pb_bam_header_text.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
    L.pb_bam_header_text.restype = C.c_void_p
    L.pb_bam_fetch.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.POINTER(PbRecords)]
    L.pb_bam_io_stats.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.pb_bam_index_max_end.argtypes = [C.c_void_p]
    L.pb_bam_index_max_end.restype = C.c_int64
    L.pb_bam_index_info.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.pb_bam_fetch_device_anchors.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.pb_bam_fetch_device.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_int, C.POINTER(PbRecords), C.c_void_p]
    L.pb_bam_fetch_device_timings.argtypes = [C.c_void_p, C.c_void_p]
    L.pb_bam_set_host_share.argtypes = [C.c_void_p, C.c_double]
    L.pb_bam_inflate_split.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.pb_inflate_blocks_host.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    L.pb_test_inflate_blocks.argtypes = L.pb_inflate_blocks_host.argtypes + [C.c_int]
    L.pb_fasta_open.argtypes = [C.POINTER(C.c_void_p), C.c_char_p]
    L.pb_fasta_close.argtypes = [C.c_void_p]
    L.pb_fasta_n_contigs.argtypes = [C.c_void_p]
    L.pb_fasta_contig_name.argtypes = [C.c_void_p, C.c_int]
    L.pb_fasta_contig_name.restype = C.c_char_p
    L.pb_fasta_contig_length.argtypes = [C.c_void_p, C.c_char_p]
    L.pb_fasta_contig_length.restype = C.c_int64
    L.pb_fasta_fetch.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]
    L._bamio_bound = True


class HostRecordsView:
    """pb_records_t whose pointers are reader-owned host buffers (valid until the reader's next fetch)."""
    on_host = True

    def __init__(self, struct: PbRecords, owner):
        self.struct = struct
        self._owner = owner

    @property
    def n_records(self) -> int:
        return int(self.struct.n_records)

    def to_batch(self) -> RecordBatch:
        s = self.struct
        n = int(s.n_records)

        def arr(ptr, count, dtype):
            if count == 0 or not ptr:
                return np.zeros(0, dtype=dtype)
            return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(np.ctypeslib.as_ctypes_type(dtype))), shape=(count,)).copy()
        seq_off = arr(s.seq_off, n + 1, np.int64) if n else np.zeros(1, np.int64)
        cigar_off = arr(s.cigar_off, n + 1, np.int64) if n else np.zeros(1, np.int64)
        nb, nc = int(seq_off[-1]), int(cigar_off[-1])
        return RecordBatch(arr(s.pos, n, np.int64), seq_off, cigar_off, arr(s.flag, n, np.uint16), arr(s.mapq, n, np.uint8),
                           arr(s.seq, (nb + 1) // 2, np.uint8), arr(s.qual, nb, np.uint8), arr(s.cigar, nc, np.uint32))


class DeviceRecordsView:
    """pb_records_t whose pointers are reader-owned DEVICE buffers (valid until the reader's next fetch_device): what
    ReadTrimmer.get_reads takes through pb_get_reads_plan_device."""
    on_host = False

    def __init__(self, struct: PbRecords, owner, device: int):
        self.struct = struct
        self._owner = owner
        self.device = device

    @property
    def n_records(self) -> int:
        return int(self.struct.n_records)

    def to_batch(self) -> RecordBatch:
        """Copy to the host (tests)."""
        s = self.struct
        n = int(s.n_records)
        L = _lib.lib()
        L.pb_memcpy_to_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]

        def arr(ptr, count, dtype):
            if count == 0 or not ptr:
                return np.zeros(0, dtype=dtype)
            out = np.empty(count, dtype=dtype)
            _lib.check(L.pb_memcpy_to_host(out.ctypes.data, C.c_void_p(ptr), out.nbytes), "pb_memcpy_to_host")
            return out
        seq_off = arr(s.seq_off, n + 1, np.int64)
        cigar_off = arr(s.cigar_off, n + 1, np.int64)
        nb, nc = int(seq_off[-1]), int(cigar_off[-1])
        return RecordBatch(arr(s.pos, n, np.int64), seq_off, cigar_off, arr(s.flag, n, np.uint16), arr(s.mapq, n, np.uint8),
                           arr(s.seq, (nb + 1) // 2, np.uint8), arr(s.qual, nb, np.uint8), arr(s.cigar, nc, np.uint32))


def inflate_blocks(streams: list[bytes], sizes: list[int], in_lens: list[int] | None = None, spec: int | None = None):
    """Raw DEFLATE streams through the GPU kernel (diagnostics / tests): returns (list of outputs, status array).
    The streams lie back to back in one buffer; `in_lens` (default: each stream's length) is the payload length the kernel is
    given for each, so a shorter one leaves the stream's remaining bytes in memory right after the payload.  `spec` 1 / 0
    selects the speculative / one-decoder symbol loop (pb_test_inflate_blocks); None leaves it to PB_INFLATE_SPEC."""
    _lib.require_gpu()
    L = _lib.lib()
    _bind(L)
    n = len(streams)
    comp = np.frombuffer(b"".join(streams) + b"\0" * 64, dtype=np.uint8).copy()
    full = np.array([len(s) for s in streams], dtype=np.int64)
    offs = np.concatenate([[0], np.cumsum(full[:-1])]).astype(np.int64) if n else np.zeros(0, np.int64)
    lens = np.array(full if in_lens is None else in_lens, dtype=np.int32)
    assert lens.shape == (n,) and np.all((lens >= 0) & (lens <= full))
    outl = np.array(sizes, dtype=np.int32)
    out = np.zeros(int(outl.sum()) + 1, dtype=np.uint8)
    status = np.zeros(max(n, 1), dtype=np.int32)
    args = (comp.ctypes.data, int(full.sum()), offs.ctypes.data, lens.ctypes.data, outl.ctypes.data, n, out.ctypes.data,
            status.ctypes.data, None)
    if spec is None:
        _lib.check(L.pb_inflate_blocks_host(*args), "pb_inflate_blocks_host")
    else:
        _lib.check(L.pb_test_inflate_blocks(*args, int(spec)), "pb_test_inflate_blocks")
    cuts = np.concatenate([[0], np.cumsum(outl)]).astype(np.int64)
    return [bytes(out[cuts[i]:cuts[i + 1]]) for i in range(n)], status[:n]


class BamReader:
    """BAM_handler(path) minus get_reads' trim (that runs on the GPU: pepper_b200.reads.ReadTrimmer)."""

    def __init__(self, path: str, threads: int = 0):
        self.L = _lib.lib()
        _bind(self.L)
        self.h = C.c_void_p()
        _lib.check(self.L.pb_bam_open(C.byref(self.h), path.encode(), threads), "pb_bam_open")
        self.path = path

    def close(self):
        if self.h:
            self.L.pb_bam_close(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:      # noqa: BLE001
            pass

    @property
    def index_max_end(self) -> int:
        """The index's reach: no fetch returns a record at or past it (2^29 for a BAI, 2^(min_shift + 3 depth) for a CSI)."""
        return int(self.L.pb_bam_index_max_end(self.h))

    def index_info(self) -> dict:
        """{"format": "csi" or "bai", "min_shift", "depth"} of the index the reader opened."""
        c, m, d = C.c_int(0), C.c_int(0), C.c_int(0)
        _lib.check(self.L.pb_bam_index_info(self.h, C.byref(c), C.byref(m), C.byref(d)), "pb_bam_index_info")
        return dict(format="csi" if c.value else "bai", min_shift=int(m.value), depth=int(d.value))

    def get_chromosome_sequence_names(self) -> list[str]:                      # bam_handler.cpp:103-113
        return [self.L.pb_bam_contig_name(self.h, i).decode() for i in range(self.L.pb_bam_n_contigs(self.h))]

    def get_chromosome_sequence_names_with_length(self) -> list[tuple[str, int]]:   # :88-101
        return [(self.L.pb_bam_contig_name(self.h, i).decode(), int(self.L.pb_bam_contig_length(self.h, i)))
                for i in range(self.L.pb_bam_n_contigs(self.h))]

    def header_text(self) -> str:
        n = C.c_int64(0)
        p = self.L.pb_bam_header_text(self.h, C.byref(n))
        return C.string_at(p, n.value).decode(errors="replace") if p else ""

    def get_sample_names(self) -> set[str]:                                    # :30-56 (@RG ... SM:<name>)
        out = set()
        for line in self.header_text().split("\n"):
            tok = line.split("\t")
            if tok and tok[0] == "@RG":
                for t in tok[1:]:
                    kv = t.split(":")
                    if kv[0] == "SM" and len(kv) > 1:
                        out.add(kv[1])
        return out

    def fetch(self, contig: str, beg: int, end: int) -> HostRecordsView:
        tid = self.L.pb_bam_contig_id(self.h, contig.encode())
        if tid < 0:
            raise _lib.PepperB200Error(f"contig {contig!r} is not in {self.path}")
        view = PbRecords()
        _lib.check(self.L.pb_bam_fetch(self.h, tid, beg, end, C.byref(view)), "pb_bam_fetch")
        return HostRecordsView(view, self)

    def fetch_device(self, contig: str, beg: int, end: int, device: int = 0, stream: int = 0) -> DeviceRecordsView:
        """The records of fetch(), produced on the GPU: only the compressed BGZF blocks cross PCIe (pb_bam_fetch_device)."""
        tid = self.L.pb_bam_contig_id(self.h, contig.encode())
        if tid < 0:
            raise _lib.PepperB200Error(f"contig {contig!r} is not in {self.path}")
        view = PbRecords()
        _lib.check(self.L.pb_bam_fetch_device(self.h, tid, beg, end, device, C.byref(view), C.c_void_p(stream)), "pb_bam_fetch_device")
        return DeviceRecordsView(view, self, device)

    def fetch_device_anchors(self) -> tuple[int, int]:
        """(known record starts, most records walked from one of them) of the last fetch_device: the walk runs one GPU thread per
        start, so the second number bounds the walk's length."""
        a, w = C.c_int64(0), C.c_int64(0)
        self.L.pb_bam_fetch_device_anchors(self.h, C.byref(a), C.byref(w))
        return int(a.value), int(w.value)

    def fetch_device_timings(self) -> dict:
        ms = (C.c_float * 3)()
        self.L.pb_bam_fetch_device_timings(self.h, ms)
        return dict(inflate_ms=float(ms[0]), chain_parse_ms=float(ms[1]), scatter_ms=float(ms[2]))

    def set_host_share(self, share: float) -> None:
        """Share (0..1) of the BGZF blocks fetch_device leaves to the host zlib pool while the kernel inflates the rest."""
        _lib.check(self.L.pb_bam_set_host_share(self.h, float(share)), "pb_bam_set_host_share")

    def inflate_split(self) -> tuple[int, int]:
        """(blocks inflated by the host pool, blocks inflated by the kernel) over all fetch_device calls."""
        a, b = C.c_int64(0), C.c_int64(0)
        self.L.pb_bam_inflate_split(self.h, C.byref(a), C.byref(b))
        return int(a.value), int(b.value)

    def io_stats(self) -> tuple[int, int]:
        a, b = C.c_int64(0), C.c_int64(0)
        self.L.pb_bam_io_stats(self.h, C.byref(a), C.byref(b))
        return int(a.value), int(b.value)


class FastaReader:
    """FASTA_handler(path) (fasta_handler.cpp)."""

    def __init__(self, path: str):
        self.L = _lib.lib()
        _bind(self.L)
        self.h = C.c_void_p()
        _lib.check(self.L.pb_fasta_open(C.byref(self.h), path.encode()), "pb_fasta_open")

    def close(self):
        if self.h:
            self.L.pb_fasta_close(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:      # noqa: BLE001
            pass

    def get_chromosome_names(self) -> list[str]:
        return [self.L.pb_fasta_contig_name(self.h, i).decode() for i in range(self.L.pb_fasta_n_contigs(self.h))]

    def get_chromosome_sequence_length(self, name: str) -> int:
        return int(self.L.pb_fasta_contig_length(self.h, name.encode()))

    def get_reference_sequence(self, region: str, start: int, stop: int) -> str:
        return self.fetch_array(region, start, stop).tobytes().decode()

    def fetch_array(self, region: str, start: int, stop: int) -> np.ndarray:
        cap = max(0, stop - start) + 1
        buf = np.zeros(cap, dtype=np.uint8)
        n = C.c_int64(0)
        rc = self.L.pb_fasta_fetch(self.h, region.encode(), start, stop, buf.ctypes.data, cap, C.byref(n))
        if rc == -3:
            buf = np.zeros(int(n.value), dtype=np.uint8)
            rc = self.L.pb_fasta_fetch(self.h, region.encode(), start, stop, buf.ctypes.data, buf.shape[0], C.byref(n))
        _lib.check(rc, "pb_fasta_fetch")
        return buf[:int(n.value)]
