"""Public API of the fused hot path: make_images + inference in one call.

``VariantCaller.call``  == `pepper_variant call_variant` steps 1+2 (CallVariant.py:12: generate_images ->
run_inference) for a batch of regions; returns what DataStorePredict.write_prediction stores
(pepper_variant/modules/python/DataStorePredict.py:49-66): contig positions, depths, candidate keys, candidate
frequencies and the float32 [N,3] genotype probabilities.

``PolishCaller.call``   == `pepper polish` steps 1+2 (polish.py:14: make_images -> call_consensus); returns what
pepper/modules/python/DataStorePredict.py:49-76 stores: per image position/index/bases/phred.

Both take HOST buffers (numpy) and do the host<->device copies themselves (pb_*_call_host); `call_device`
variants take torch CUDA tensors that already live in HBM (used by bench.py's device-resident leg).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
import numpy as np

from . import _lib
from .abi import (HostReads, PbReads, PbRegion, PbVariantParams, PbCandidateColumns, regions_array, variant_params, WINDOW,
                  FEATURES, ALLELE_STRIDE, POLISH_SEQ_LEN, PB_ERR_CAPACITY)
from .synth import ReadBatch, RegionTable
from .variant import VariantEncoder, VariantNet, _bind as _bind_variant
from .polish import PolishEncoder, PolishNet, _bind as _bind_polish


@dataclass
class VariantCalls:
    positions: np.ndarray    # int64 [N]
    depths: np.ndarray       # uint8 [N]
    freqs: np.ndarray        # uint8 [N]
    keys_raw: np.ndarray     # uint8 [N,64]
    region_of: np.ndarray    # int32 [N]
    probs: np.ndarray        # float32 [N,3]
    images: np.ndarray | None = None

    @property
    def keys(self):
        return [bytes(k).split(b"\0", 1)[0].decode() for k in self.keys_raw]

    def __len__(self):
        return int(self.positions.shape[0])


@dataclass
class PolishCalls:
    bases: np.ndarray        # uint8 [n_img,1000]
    phred: np.ndarray        # uint8 [n_img,1000]
    position: np.ndarray     # int64 [n_img,1000]
    index: np.ndarray        # int32 [n_img,1000]
    image_region: np.ndarray  # int32 [n_img]
    chunk_id: np.ndarray     # int32 [n_img]


def _bind_calls(L):
    if getattr(L, "_calls_bound", False):
        return
    vp = C.c_void_p
    L.pb_variant_call_host.argtypes = [vp, vp, C.POINTER(PbReads), C.POINTER(PbRegion), C.c_int64, vp, C.c_int64,
                                       C.POINTER(PbVariantParams), C.c_int64, vp, vp, vp, vp, vp, vp, vp,
                                       C.POINTER(C.c_int64), vp]
    L.pb_variant_call_device.argtypes = [vp, vp, C.POINTER(PbReads), vp, C.c_int64, C.POINTER(PbRegion), vp, C.c_int64,
                                         C.POINTER(PbVariantParams), C.c_int64, vp, vp, vp, vp, vp, vp, vp,
                                         C.POINTER(C.c_int64), vp]
    L.pb_variant_call_timings.argtypes = [vp, vp]
    L.pb_variant_stream_begin.argtypes = [vp, vp, C.POINTER(PbVariantParams), C.c_int64, vp, vp]
    L.pb_variant_stream_stage_host.argtypes = [vp, C.POINTER(PbReads), C.POINTER(PbRegion), C.c_int64, C.c_int64, vp, C.c_int32]
    L.pb_variant_stream_stage_device.argtypes = [vp, C.POINTER(PbReads), C.POINTER(PbRegion), C.c_int64, C.c_int64, vp, C.c_int32]
    L.pb_variant_stream_run.argtypes = [vp, vp, C.c_int, C.POINTER(C.c_int64)]
    L.pb_variant_stream_sync.argtypes = [vp]
    L.pb_variant_stream_end.argtypes = [vp, vp, C.POINTER(C.c_int64)]
    L.pb_variant_stream_stats.argtypes = [vp, vp, vp, C.POINTER(C.c_int64)]
    L.pb_variant_stream_columns.argtypes = [vp, C.POINTER(PbCandidateColumns), C.POINTER(vp), C.POINTER(vp)]
    L.pb_variant_stream_fetch.argtypes = [vp, C.c_int64, vp, vp, vp, vp, vp, vp, vp, vp]
    L.pb_variant_stream_track.argtypes = [vp, C.c_int64, vp]
    L.pb_variant_stream_owned.argtypes = [vp, vp, C.c_int64]
    L.pb_variant_stream_track_used.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.pb_polish_call_host.argtypes = [vp, vp, C.POINTER(PbReads), C.POINTER(PbRegion), C.c_int64, C.c_int64, vp, vp, vp, vp,
                                      vp, vp, C.POINTER(C.c_int64), vp]
    L.pb_polish_call_device.argtypes = [vp, vp, C.POINTER(PbReads), vp, C.c_int64, C.POINTER(PbRegion), C.c_int64, vp, vp,
                                        vp, vp, vp, vp, C.POINTER(C.c_int64), vp]
    L.pb_polish_call_timings.argtypes = [vp, vp]
    L.pb_polish_stream_begin.argtypes = [vp, vp, C.c_int64, vp, vp]
    L.pb_polish_stream_begin_qual.argtypes = [vp, vp, C.c_int64, vp, vp]
    L.pb_polish_stream_stage_device.argtypes = [vp, C.POINTER(PbReads), C.POINTER(PbRegion), C.c_int64, C.c_int64, C.c_int32]
    L.pb_polish_stream_run.argtypes = [vp, vp, C.c_int, C.POINTER(C.c_int64)]
    L.pb_polish_stream_sync.argtypes = [vp]
    L.pb_polish_stream_end.argtypes = [vp, vp, C.POINTER(C.c_int64)]
    L.pb_polish_stream_stats.argtypes = [vp, vp, vp]
    L.pb_polish_stream_group_bytes.argtypes = [vp, vp, C.c_int64]
    L.pb_polish_stream_edits.argtypes = [vp, C.c_int64, vp]
    L.pb_polish_stream_stage_device_draft.argtypes = [vp, C.POINTER(PbReads), C.POINTER(PbRegion), C.c_int64, C.c_int64, C.c_int32, vp]
    L.pb_polish_stream_event_total.argtypes = [vp, C.POINTER(C.c_int64)]
    L.pb_polish_stream_group_events.argtypes = [vp, vp, C.c_int64]
    L._calls_bound = True


class DeviceReads:
    """A ReadBatch (+ region table + reference) resident in HBM as torch tensors; builds the pb_reads_t whose
    pointers are device pointers."""

    def __init__(self, reads: ReadBatch, regions: RegionTable, device: int = 0):
        import torch
        dev = torch.device("cuda", device)
        hr = HostReads(reads)
        self._keep = []

        def up(a):
            t = torch.from_numpy(a).to(dev)
            self._keep.append(t)
            return t.data_ptr()
        self.struct = PbReads(reads.n_reads, up(hr.pos), up(hr.seq_off), up(hr.cigar_off), up(hr.flags), up(hr.mapq),
                              up(hr.seq), up(hr.qual), up(hr.cigar.view(np.int32)))
        self.h_regions, self._tab = regions_array(regions)
        self.d_regions = up(self._tab)
        ref = np.ascontiguousarray(regions.ref, dtype=np.uint8)
        self.d_ref = up(ref)
        self.ref_bytes = int(ref.shape[0])
        self.n_regions = regions.n_regions
        self.nbytes = sum(t.numel() * t.element_size() for t in self._keep)


class VariantCaller:
    def __init__(self, state: dict, device: int = 0):
        self.enc = VariantEncoder(device)
        self.net = VariantNet(state, device)
        self.L = _lib.lib()
        _bind_calls(self.L)
        self.device = device

    def close(self):
        self.enc.close()
        self.net.close()

    def call(self, reads: ReadBatch, regions: RegionTable, params: dict, capacity: int | None = None,
             want_images: bool = False, stream: int = 0, reuse_buffers: bool = False) -> VariantCalls:
        hr = HostReads(reads)
        return self.call_prepared(hr, regions, params, capacity, want_images, stream, reuse_buffers)

    def call_prepared(self, hr: HostReads, regions: RegionTable, params: dict, capacity: int | None = None,
                      want_images: bool = False, stream: int = 0, reuse_buffers: bool = False) -> VariantCalls:
        """`reuse_buffers=True`: results land in page-locked buffers owned by the caller object and the returned arrays are
        views of them (valid until the next call) — the streaming mode a pipeline worker uses; default: fresh arrays."""
        self._reuse = reuse_buffers
        regs, keep = regions_array(regions)
        ref = np.ascontiguousarray(regions.ref, dtype=np.uint8)
        p = variant_params(**params)
        if capacity is None:
            span = int((regions.col("cand_end") - regions.col("cand_start") + 1).sum())
            capacity = max(1024, span // 16)
        while True:
            img = self._out("images", (capacity, WINDOW, FEATURES), np.int8) if want_images else None
            pos = self._out("positions", (capacity,), np.int64)
            dep = self._out("depths", (capacity,), np.uint8)
            frq = self._out("freqs", (capacity,), np.uint8)
            keys = self._out("keys", (capacity, ALLELE_STRIDE), np.uint8)
            rof = self._out("region_of", (capacity,), np.int32)
            probs = self._out("probs", (capacity, 3), np.float32)
            n = C.c_int64(0)
            rc = self.L.pb_variant_call_host(self.enc.h, self.net.h, C.byref(hr.struct), regs, regions.n_regions,
                                             ref.ctypes.data, ref.shape[0], C.byref(p), capacity,
                                             img.ctypes.data if want_images else None, pos.ctypes.data, dep.ctypes.data,
                                             frq.ctypes.data, keys.ctypes.data, rof.ctypes.data, probs.ctypes.data,
                                             C.byref(n), C.c_void_p(stream))
            if rc == PB_ERR_CAPACITY:
                capacity = int(n.value) + 16
                continue
            _lib.check(rc, "pb_variant_call_host")
            k = int(n.value)
            return VariantCalls(pos[:k], dep[:k], frq[:k], keys[:k], rof[:k], probs[:k], img[:k] if want_images else None)

    def _out(self, name: str, shape, dtype):
        """Page-locked result buffers, reused across calls (the returned arrays are views: copy them to keep them past
        the next call)."""
        if not getattr(self, "_reuse", False):
            return np.empty(shape, dtype=dtype)
        import torch
        cache = self.__dict__.setdefault("_pinned", {})
        need = int(np.prod(shape)) * np.dtype(dtype).itemsize
        t = cache.get(name)
        if t is None or t.numel() < need:
            t = torch.empty(max(need, 1), dtype=torch.uint8).pin_memory()
            cache[name] = t
        return t.numpy()[:need].view(dtype).reshape(shape)

    def call_device(self, dreads: DeviceReads, params: dict, out: dict, stream: int = 0) -> int:
        """Everything in HBM.  `out` holds torch CUDA tensors: images int8 [cap,33,26], positions int64 [cap],
        depths/freqs uint8 [cap], keys uint8 [cap,64], region_of int32 [cap], probs float32 [cap,3]."""
        p = variant_params(**params)
        n = C.c_int64(0)
        cap = int(out["positions"].shape[0])
        rc = self.L.pb_variant_call_device(self.enc.h, self.net.h, C.byref(dreads.struct), dreads.d_regions,
                                           dreads.n_regions, dreads.h_regions, dreads.d_ref, dreads.ref_bytes, C.byref(p),
                                           cap, out["images"].data_ptr(), out["positions"].data_ptr(),
                                           out["depths"].data_ptr(), out["freqs"].data_ptr(), out["keys"].data_ptr(),
                                           out["region_of"].data_ptr(), out["probs"].data_ptr(), C.byref(n),
                                           C.c_void_p(stream))
        _lib.check(rc, "pb_variant_call_device")
        return int(n.value)

    def timings(self) -> dict:
        ms = (C.c_float * 2)()
        _lib.check(self.L.pb_variant_call_timings(self.enc.h, ms), "timings")
        d = dict(encode_ms=float(ms[0]), network_ms=float(ms[1]))
        d.update({"enc_" + k: v for k, v in self.enc.timings().items()})
        return d

    def stream(self, params: dict, capacity: int, d_records: int = 0, stream: int = 0) -> "VariantStream":
        """Streaming session over region groups (pb_variant_stream_*): see VariantStream."""
        return VariantStream(self, params, capacity, d_records, stream)


class TrackCapacityError(_lib.PepperB200Error):
    """A streaming session's gVCF track could not hold the next group (rc PB_ERR_CAPACITY)."""


class VariantStream:
    """One streaming session of a VariantCaller: region GROUPS are staged and run one after the other, the candidates
    accumulate on the device, the network runs over whole 9,472-candidate chunks as they fill.

        s = caller.stream(params, capacity, d_records=ptr)      # ptr: optional device buffer for 84-byte records
        s.stage_host(hr, regs, g0, g1, h_ref, region_id0)       # or stage_device(dreads, g0, g1, region_id0)
        while ...:
            s.run(last)                                         # kernels queued
            s.stage_host(...)                                   # next group's copies overlap them
            s.sync()
        n = s.end()
    """

    def __init__(self, caller: VariantCaller, params: dict, capacity: int, d_records: int = 0, stream: int = 0):
        self.c, self.L = caller, caller.L
        self.p = variant_params(**params)
        self.capacity = int(capacity)
        self._keep = []
        _lib.check(self.L.pb_variant_stream_begin(caller.enc.h, caller.net.h, C.byref(self.p), self.capacity,
                                                  C.c_void_p(d_records or None), C.c_void_p(stream)), "pb_variant_stream_begin")

    def stage_host(self, hr: HostReads, regs, g0: int, g1: int, h_ref: np.ndarray, region_id0: int = 0):
        """`regs` = ctypes array from abi.regions_array (the FULL table the group indices refer to)."""
        _lib.check(self.L.pb_variant_stream_stage_host(self.c.enc.h, C.byref(hr.struct), regs, g0, g1, h_ref.ctypes.data, region_id0),
                   "pb_variant_stream_stage_host")

    def stage_device(self, dreads: "DeviceReads", g0: int, g1: int, region_id0: int = 0):
        _lib.check(self.L.pb_variant_stream_stage_device(self.c.enc.h, C.byref(dreads.struct), dreads.h_regions, g0, g1,
                                                         C.c_void_p(dreads.d_ref), region_id0), "pb_variant_stream_stage_device")

    def track(self, capacity_positions: int, d_track: int):
        """Attaches a gVCF track (pb_variant_stream_track): uint32 device buffer [capacity_positions]; stage_device then takes
        each group's owned ends."""
        _lib.check(self.L.pb_variant_stream_track(self.c.enc.h, int(capacity_positions), C.c_void_p(d_track)), "pb_variant_stream_track")
        self.track_capacity = int(capacity_positions)

    def owned(self, owned_end):
        """The owned ends of the group staged last (pb_variant_stream_owned)."""
        a = np.ascontiguousarray(owned_end, np.int64)
        _lib.check(self.L.pb_variant_stream_owned(self.c.enc.h, a.ctypes.data, a.shape[0]), "pb_variant_stream_owned")

    def track_used(self) -> int:
        return self._track_counts()[0]

    def _track_counts(self) -> tuple[int, int]:
        n, need = C.c_int64(0), C.c_int64(0)
        _lib.check(self.L.pb_variant_stream_track_used(self.c.enc.h, C.byref(n), C.byref(need)), "pb_variant_stream_track_used")
        return int(n.value), int(need.value)

    def run(self, flush: bool = False) -> int:
        n = C.c_int64(0)
        rc = self.L.pb_variant_stream_run(self.c.enc.h, self.c.net.h, int(flush), C.byref(n))
        if rc == PB_ERR_CAPACITY and getattr(self, "track_capacity", None) is not None:
            used, need = self._track_counts()
            if need > self.track_capacity:
                raise TrackCapacityError("gVCF track capacity %d positions too small (need >= %d so far)"
                                         % (self.track_capacity, need), rc)
        if rc == PB_ERR_CAPACITY:
            raise _lib.PepperB200Error("stream capacity %d too small (need >= %d so far)" % (self.capacity, n.value), rc)
        _lib.check(rc, "pb_variant_stream_run")
        return int(n.value)

    def sync(self):
        _lib.check(self.L.pb_variant_stream_sync(self.c.enc.h), "pb_variant_stream_sync")

    def end(self) -> int:
        n = C.c_int64(0)
        _lib.check(self.L.pb_variant_stream_end(self.c.enc.h, self.c.net.h, C.byref(n)), "pb_variant_stream_end")
        return int(n.value)

    def stats(self) -> dict:
        ms = (C.c_float * 5)(); nl = (C.c_int64 * 2)(); g = C.c_int64(0)
        _lib.check(self.L.pb_variant_stream_stats(self.c.enc.h, ms, nl, C.byref(g)), "pb_variant_stream_stats")
        d = dict(zip(("enc_prefix", "enc_count", "enc_sites", "enc_alleles", "enc_windows"), [float(x) for x in ms]))
        d.update(encoder_launches=int(nl[0]), network_launches=int(nl[1]), groups=int(g.value))
        return d

    def fetch(self, n: int, want_images: bool = False, stream: int = 0) -> VariantCalls:
        img = np.empty((n, WINDOW, FEATURES), np.int8) if want_images else None
        pos = np.empty(n, np.int64); dep = np.empty(n, np.uint8); frq = np.empty(n, np.uint8)
        keys = np.empty((n, ALLELE_STRIDE), np.uint8); rof = np.empty(n, np.int32); probs = np.empty((n, 3), np.float32)
        _lib.check(self.L.pb_variant_stream_fetch(self.c.enc.h, n, img.ctypes.data if want_images else None, pos.ctypes.data,
                                                  dep.ctypes.data, frq.ctypes.data, keys.ctypes.data, rof.ctypes.data,
                                                  probs.ctypes.data, C.c_void_p(stream)), "pb_variant_stream_fetch")
        return VariantCalls(pos, dep, frq, keys, rof, probs, img)


class PolishCaller:
    def __init__(self, state: dict, device: int = 0):
        self.enc = PolishEncoder(device)
        self.net = PolishNet(state, device)
        self.L = _lib.lib()
        _bind_calls(self.L)

    def close(self):
        self.enc.close()
        self.net.close()

    def call(self, reads: ReadBatch, regions: RegionTable, capacity: int | None = None, stream: int = 0) -> PolishCalls:
        return self.call_prepared(HostReads(reads), regions, capacity, stream)

    def call_prepared(self, hr: HostReads, regions: RegionTable, capacity: int | None = None, stream: int = 0,
                      reuse_buffers: bool = False) -> PolishCalls:
        """`reuse_buffers=True`: results land in page-locked buffers owned by the caller object (views, valid until the next
        call) — the streaming mode of a pipeline worker; default: fresh arrays."""
        regs, keep = regions_array(regions)
        if capacity is None:
            span = int((regions.col("ref_end") - regions.col("ref_start") + 1).sum())
            capacity = 3 * (span // 950 + regions.n_regions) + 8
        while True:
            bases = self._out("bases", (capacity, POLISH_SEQ_LEN), np.uint8, reuse_buffers)
            phred = self._out("phred", (capacity, POLISH_SEQ_LEN), np.uint8, reuse_buffers)
            position = self._out("position", (capacity, POLISH_SEQ_LEN), np.int64, reuse_buffers)
            index = self._out("index", (capacity, POLISH_SEQ_LEN), np.int32, reuse_buffers)
            ireg = self._out("ireg", (capacity,), np.int32, reuse_buffers)
            cid = self._out("cid", (capacity,), np.int32, reuse_buffers)
            n = C.c_int64(0)
            rc = self.L.pb_polish_call_host(self.enc.h, self.net.h, C.byref(hr.struct), regs, regions.n_regions, capacity,
                                            bases.ctypes.data, phred.ctypes.data, position.ctypes.data, index.ctypes.data,
                                            ireg.ctypes.data, cid.ctypes.data, C.byref(n), C.c_void_p(stream))
            if rc == PB_ERR_CAPACITY:
                capacity = int(n.value) + 4
                continue
            _lib.check(rc, "pb_polish_call_host")
            k = int(n.value)
            return PolishCalls(bases[:k], phred[:k], position[:k], index[:k], ireg[:k], cid[:k])

    def _out(self, name: str, shape, dtype, reuse: bool):
        if not reuse:
            return np.empty(shape, dtype=dtype)
        import torch
        cache = self.__dict__.setdefault("_pinned", {})
        need = int(np.prod(shape)) * np.dtype(dtype).itemsize
        t = cache.get(name)
        if t is None or t.numel() < need:
            t = torch.empty(max(need, 1), dtype=torch.uint8).pin_memory()
            cache[name] = t
        return t.numpy()[:need].view(dtype).reshape(shape)

    def call_device(self, dreads: DeviceReads, out: dict, stream: int = 0) -> int:
        """Everything in HBM.  `out`: torch CUDA tensors bases/phred uint8 [cap,1000], position int64 [cap,1000],
        index int32 [cap,1000], image_region/chunk_id int32 [cap]."""
        n = C.c_int64(0)
        cap = int(out["bases"].shape[0])
        rc = self.L.pb_polish_call_device(self.enc.h, self.net.h, C.byref(dreads.struct), dreads.d_regions, dreads.n_regions,
                                          dreads.h_regions, cap, out["bases"].data_ptr(), out["phred"].data_ptr(),
                                          out["position"].data_ptr(), out["index"].data_ptr(), out["image_region"].data_ptr(),
                                          out["chunk_id"].data_ptr(), C.byref(n), C.c_void_p(stream))
        _lib.check(rc, "pb_polish_call_device")
        return int(n.value)

    def timings(self) -> dict:
        ms = (C.c_float * 2)()
        _lib.check(self.L.pb_polish_call_timings(self.enc.h, ms), "timings")
        d = dict(encode_ms=float(ms[0]), network_ms=float(ms[1]))
        d.update({"enc_" + k: v for k, v in self.enc.timings().items()})
        return d


    def stream(self, capacity_bytes: int, d_sink: int, stream: int = 0, qualities: bool = False, edits: bool = False,
               capacity_events: int = 0, d_events: int = 0) -> "PolishStream":
        """Streaming session over region groups with the stitch on the device (pb_polish_stream_*): see PolishStream."""
        return PolishStream(self, capacity_bytes, d_sink, stream, qualities, edits, capacity_events, d_events)


class PolishStream:
    """One streaming session of a PolishCaller: groups of WHOLE regions of one contig are staged and run one after the other;
    their images queue on the device, the network runs over whole 8,192-image chunks, and after each network call the stitch
    kernel appends the chunk's consensus bases to the device byte buffer `d_sink` (`capacity_bytes`).  A contig's consensus is
    the concatenation of its groups' bytes in group order.

        s = caller.stream(capacity_bytes, d_sink)
        s.stage_device(fetched, g0, g1, region_id0)
        while ...:
            s.run()                      # kernels queued; stage the next group while they run
            s.stage_device(...)
        n = s.end()                      # bytes written; PepperB200Error(PB_ERR_CAPACITY) when the sink was too small
        per_group = s.group_bytes()      # bytes of each group, in run order

    `qualities=True` (pb_polish_stream_begin_qual): the sink holds 2-byte polish.QUAL_RECORD records (base, FASTQ quality
    byte) in place of bytes, `d_sink` is 2 * `capacity_bytes` bytes, and every count of the session is in records.

    `edits=True` (pb_polish_stream_edits): the session also writes the edit events of every group (polish_edits.EDIT_EVENT:
    the winning columns that delete, substitute or insert, and one coverage record per image) to the device buffer `d_events`
    (`capacity_events` events); `group_events()` gives the events of each group.  Groups are staged with their reference
    (a FetchedReads), which the session holds until the group has been encoded."""

    def __init__(self, caller: PolishCaller, capacity_bytes: int, d_sink: int, stream: int = 0, qualities: bool = False,
                 edits: bool = False, capacity_events: int = 0, d_events: int = 0):
        from collections import deque
        self.c, self.L = caller, caller.L
        self.capacity = int(capacity_bytes)
        self.capacity_events = int(capacity_events)
        self.edits = bool(edits)
        self.groups = 0
        self._held = deque(maxlen=3)
        begin = self.L.pb_polish_stream_begin_qual if qualities else self.L.pb_polish_stream_begin
        _lib.check(begin(caller.enc.h, caller.net.h, self.capacity, C.c_void_p(d_sink or None), C.c_void_p(stream)),
                   "pb_polish_stream_begin_qual" if qualities else "pb_polish_stream_begin")
        if self.edits:
            _lib.check(self.L.pb_polish_stream_edits(caller.enc.h, self.capacity_events, C.c_void_p(d_events or None)),
                       "pb_polish_stream_edits")

    def stage_device(self, dreads, g0: int, g1: int, region_id0: int = 0):
        """`dreads`: DeviceReads / FetchedReads whose region table the group indices [g0, g1) refer to."""
        if not self.edits:
            _lib.check(self.L.pb_polish_stream_stage_device(self.c.enc.h, C.byref(dreads.struct), dreads.h_regions, g0, g1, region_id0),
                       "pb_polish_stream_stage_device")
            return
        # the group is encoded by the run after this stage, and the run after that synchronises with the encoder: the
        # reference (dreads' device tensors) must live until then
        self._held.append(dreads)
        _lib.check(self.L.pb_polish_stream_stage_device_draft(self.c.enc.h, C.byref(dreads.struct), dreads.h_regions, g0, g1,
                                                              region_id0, C.c_void_p(dreads.d_ref)),
                   "pb_polish_stream_stage_device_draft")

    def run(self, flush: bool = False) -> int:
        """Returns the encoded columns of the session so far: an upper bound of its consensus bytes."""
        n = C.c_int64(0)
        _lib.check(self.L.pb_polish_stream_run(self.c.enc.h, self.c.net.h, int(flush), C.byref(n)), "pb_polish_stream_run")
        self.groups += 1
        return int(n.value)

    def sync(self):
        _lib.check(self.L.pb_polish_stream_sync(self.c.enc.h), "pb_polish_stream_sync")

    def end(self) -> int:
        n = C.c_int64(0)
        rc = self.L.pb_polish_stream_end(self.c.enc.h, self.c.net.h, C.byref(n))
        self._held.clear()
        if rc == PB_ERR_CAPACITY and self.edits and n.value <= self.capacity:
            need = self.event_total()
            ex = _lib.PepperB200Error("edit event capacity %d too small (need %d events)" % (self.capacity_events, need), rc)
            ex.need, ex.need_events = int(n.value), need
            raise ex
        if rc == PB_ERR_CAPACITY:
            ex = _lib.PepperB200Error("consensus sink capacity %d too small (need %d bytes)" % (self.capacity, n.value), rc)
            ex.need = int(n.value)
            raise ex
        _lib.check(rc, "pb_polish_stream_end")
        return int(n.value)

    def group_bytes(self) -> np.ndarray:
        out = np.zeros(self.groups, np.int64)
        _lib.check(self.L.pb_polish_stream_group_bytes(self.c.enc.h, out.ctypes.data, self.groups), "pb_polish_stream_group_bytes")
        return out

    def event_total(self) -> int:
        """Edit events the session needed (an edits session, after end())."""
        n = C.c_int64(0)
        _lib.check(self.L.pb_polish_stream_event_total(self.c.enc.h, C.byref(n)), "pb_polish_stream_event_total")
        return int(n.value)

    def group_events(self) -> np.ndarray:
        out = np.zeros(self.groups, np.int64)
        _lib.check(self.L.pb_polish_stream_group_events(self.c.enc.h, out.ctypes.data, self.groups), "pb_polish_stream_group_events")
        return out

    def stats(self) -> dict:
        ms = (C.c_float * 2)(); n = (C.c_int64 * 4)()
        _lib.check(self.L.pb_polish_stream_stats(self.c.enc.h, ms, n), "pb_polish_stream_stats")
        return dict(encoder_ms=float(ms[0]), network_ms=float(ms[1]), groups=int(n[0]), images=int(n[1]), columns=int(n[2]),
                    network_launches=int(n[3]))


class FetchedReads:
    """Output of a batched ReadTrimmer.get_reads (reads in HBM, one query per region) + the region table: the object
    VariantCaller.call_device / PolishCaller.call_device take in place of DeviceReads.  read_begin / read_end of the
    table come from the trimmer."""

    def __init__(self, trimmed, regions: RegionTable, device: int = 0, stream=None):
        """`stream`: optional torch.cuda.Stream for the two small uploads (region table, reference strings), so that they do not
        queue behind kernels running on the default stream."""
        import contextlib
        import torch
        dev = torch.device("cuda", device)
        assert trimmed.read_begin.shape[0] == regions.n_regions
        tab = np.ascontiguousarray(regions.table, dtype=np.int64).copy()
        tab[:, 6] = trimmed.read_begin
        tab[:, 7] = trimmed.read_end
        self.table = tab
        self._trimmed = trimmed
        self.struct = trimmed.struct
        self.h_regions = (PbRegion * tab.shape[0]).from_buffer(tab)
        with (torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext()):
            self._keep = [torch.from_numpy(tab).to(dev), torch.from_numpy(np.ascontiguousarray(regions.ref, dtype=np.uint8)).to(dev)]
            if stream is not None:
                stream.synchronize()
        self.d_regions = self._keep[0].data_ptr()
        self.d_ref = self._keep[1].data_ptr()
        self.ref_bytes = int(self._keep[1].numel())
        self.n_regions = regions.n_regions
