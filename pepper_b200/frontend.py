"""File -> predictions in one call: the per-process loops of the reference's make_images + inference steps
(`pepper_variant ImageGenerationUI.generate_image_and_save_to_file` :191-251 + `AlignmentSummarizer.create_summary`
:181-236 + `predict_distributed_gpu.predict` :58-70;  `pepper ImageGenerationUI.image_generator` :191-236 +
`AlignmentSummarizer.create_summary` :296-356 + `predict_distributed_gpu.predict` :63-105) with every stage after the BGZF
inflate on the GPU: `pb_bam_fetch` -> batched `get_reads` (+ reservoir sampling) -> [SSW realignment] -> pileup encoder
-> recurrent network.  Nothing here is a CLI: intervals in, arrays out (what the reference writes to its HDF5 stores).
"""
from __future__ import annotations

import ctypes as C
import re
import time

import numpy as np

from . import _lib
from .bamio import BamReader, FastaReader
from ._lib import PepperB200Error
from .abi import PB_ERR_CAPACITY
from .pipeline import FetchedReads, PolishCaller, VariantCaller, PolishCalls, VariantCalls
from .reads import ReadTrimmer
from .realign import Realigner, ALIGNMENT_SAFE_BASES
from .synth import RegionTable

REGION_SAFE_BASES = 100              # ConsensCandidateFinder.REGION_SAFE_BASES (pepper_variant Options.py:2)
MIN_IMAGE_OVERLAP = 100              # ImageSizeOptions.MIN_IMAGE_OVERLAP (pepper Options.py:10)
VARIANT_MAX_READS = 5000             # AlingerOptions.MAX_READS_IN_REGION (pepper_variant Options.py:98)
# BAM fetches in flight in the streaming calls, and readers in rotation (FETCH_WORKERS being filled + the one whose records are
# being trimmed).  Measured on the chr20-scale files leg: 2 workers / 3 readers = 988 ms per step against 862 ms with 1 / 2 — the GPU
# is the bottleneck of that path, and two inflate kernels beside the network only slow the network down (DESIGN.md section 6).
FETCH_WORKERS = 1
FETCH_READERS = 2
POLISH_MAX_READS = 1500              # AlingerOptions.MAX_READS_IN_REGION (pepper Options.py:28)


def polish_intervals(interval_start: int, interval_end: int, max_size: int = 1000) -> list[tuple[int, int]]:
    """pepper ImageGenerationUI.py:269-272."""
    return [(max(interval_start, pos - MIN_IMAGE_OVERLAP), min(interval_end, pos + max_size + MIN_IMAGE_OVERLAP))
            for pos in range(interval_start, interval_end, max_size)]


def variant_intervals(interval_start: int, interval_end: int, region_size: int = 100_000) -> list[tuple[int, int]]:
    """pepper_variant ImageGenerationUI.py:307-316."""
    return [(max(interval_start, pos), min(interval_end, pos + region_size)) for pos in range(interval_start, interval_end, region_size)]


def variant_rows(intervals: list[tuple[int, int]]) -> tuple[list[list[int]], list[tuple[int, int]]]:
    """Region-table rows of variant intervals and the reference span of each: the interval widened by REGION_SAFE_BASES
    (AlignmentSummarizer.py:181-182), its reference get_reference_sequence(.., region_end + 1)."""
    rows = [[max(0, s - REGION_SAFE_BASES), e + REGION_SAFE_BASES, s, e, 0, 0, 0, 0] for s, e in intervals]
    return rows, [(r[0], r[1] + 1) for r in rows]


def polish_rows(regions_se: list[tuple[int, int]]) -> tuple[list[list[int]], list[tuple[int, int]]]:
    """Region-table rows of polish regions and the reference span of each (AlignmentSummarizer.py:164-170)."""
    return [[s, e, s, e, 0, 0, 0, 0] for s, e in regions_se], [(s, e + ALIGNMENT_SAFE_BASES) for s, e in regions_se]


class _FromFiles:
    """`gpu_inflate` (default): BGZF inflate, record walk and parse run on the GPU (pb_bam_fetch_device; only compressed blocks
    cross PCIe); False = the host thread-pool zlib path (pb_bam_fetch)."""

    def __init__(self, bam_path: str, fasta_path: str, device: int = 0, threads: int = 0, gpu_inflate: bool = True,
                 host_share: float | None = None):
        self.gpu_inflate = gpu_inflate
        self.host_share = host_share          # None = the reader's default (pb_bam_set_host_share)
        self.threads = threads
        self.bam = self._open_bam(bam_path)
        self.fasta = FastaReader(fasta_path)
        self.fasta_path = fasta_path
        self.trimmer = ReadTrimmer(device)
        self.device = device
        self._extra = []                      # further readers of the same file (one per fetch in flight)

    def _open_bam(self, path: str) -> BamReader:
        r = BamReader(path, self.threads)
        if self.host_share is not None:
            r.set_host_share(self.host_share)
        return r

    def _readers(self, n: int) -> list:
        """`n` readers of the BAM (each owns the host / device buffers of one fetch in flight)."""
        while 1 + len(self._extra) < n:
            self._extra.append(self._open_bam(self.bam.path))
        return [self.bam] + self._extra[:n - 1]

    @property
    def _bam2(self):
        return self._extra[0] if self._extra else None

    def inflate_split(self) -> tuple[int, int]:
        """(BGZF blocks inflated by the host pools, by the kernel) over all readers."""
        parts = [r.inflate_split() for r in [self.bam] + self._extra if r is not None]
        return sum(a for a, _ in parts), sum(b for _, b in parts)

    def close(self):
        """Releases the file readers (the extra readers of the streaming calls included) and the trimmer."""
        for r in [getattr(self, "bam", None)] + list(getattr(self, "_extra", [])):
            if r is not None and hasattr(r, "close"):
                r.close()
        self.bam, self._extra = None, []
        if getattr(self, "trimmer", None) is not None:
            self.trimmer.close()
            self.trimmer = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def fasta_contigs(self) -> list[tuple[str, int]]:
        return [(c, self.fasta.get_chromosome_sequence_length(c)) for c in self.fasta.get_chromosome_names()]

    def _fetch(self, reader, contig: str, beg: int, end: int):
        return reader.fetch_device(contig, beg, end, self.device) if self.gpu_inflate else reader.fetch(contig, beg, end)

    @staticmethod
    def _group_span(g: list[tuple[int, int]]) -> tuple[int, int]:
        """The BAM span one batch of intervals needs (each interval widened by REGION_SAFE_BASES, AlignmentSummarizer.py:181-182)."""
        return max(0, min(s for s, _ in g) - REGION_SAFE_BASES), max(e for _, e in g) + REGION_SAFE_BASES

    def _side_stream(self):
        import torch
        if getattr(self, "_side", None) is None:
            self._side = torch.cuda.Stream(device=self.device)        # get_reads of batch k+1 runs here, beside the network of batch k
        return self._side

    def _trim_variant(self, view, contig: str, g: list[tuple[int, int]], min_snp_baseq: int, include_supplementary: bool = False,
                      min_mapq: int = 0, max_reads: int = VARIANT_MAX_READS, downsample_rate: float = 1.0, prof: dict | None = None):
        """Reference strings + batched get_reads of one batch of variant intervals on the side stream (synchronous for the host):
        fetched records -> the FetchedReads the encoder consumes."""
        t1 = time.perf_counter()
        rows, spans = variant_rows(g)
        queries = [(r[0], r[1]) for r in rows]
        regions = self._ref_table(contig, rows, spans)
        t2 = time.perf_counter()
        side = self._side_stream()
        got = self.trimmer.get_reads(view, queries, include_supplementary, min_mapq, min_snp_baseq,
                                     max_reads=max_reads, downsample_rate=downsample_rate, stream=side.cuda_stream)
        fetched = FetchedReads(got, regions, self.device, stream=side)
        if prof is not None:
            prof["ref_table"] += t2 - t1; prof["get_reads"] += time.perf_counter() - t2
        return fetched

    def _ref_table(self, contig: str, rows: list[list[int]], spans: list[tuple[int, int]]) -> RegionTable:
        """Region table + reference strings: ONE faidx fetch of the covering span, the (overlapping) per-region strings are
        offsets into it (get_reference_sequence clamps at the contig end; so do the lengths here)."""
        lo, hi = min(a for a, _ in spans), max(b for _, b in spans)
        ref = self.fasta.fetch_array(contig, lo, hi)
        clen = self.fasta.get_chromosome_sequence_length(contig)
        for row, (a, b) in zip(rows, spans):
            row[4], row[5] = a - lo, max(0, min(b, clen) - a)
        return RegionTable(np.array(rows, dtype=np.int64).reshape(-1, 8), ref if ref.shape[0] else np.zeros(1, np.uint8))


class _FetchRing:
    """BAM fetches of a streaming call on a helper thread: FETCH_WORKERS fetches at once (the pread of one span beside the inflate
    of another), each on its own reader of `src`, FETCH_READERS readers in rotation, so that the records of the group being
    trimmed stay valid while later spans are read and inflated.  The caller keeps at most FETCH_READERS requests outstanding
    and waits for them in request order.  Given `prof`, the helper thread's fetch time is added to prof["fetch_thread"] and the
    caller's wait to prof["wait_fetch"] (seconds)."""

    def __init__(self, src: _FromFiles, prof: dict | None = None):
        from concurrent.futures import ThreadPoolExecutor
        self._src, self._prof = src, prof
        self._ring = src._readers(FETCH_READERS)
        self._pool = ThreadPoolExecutor(max_workers=FETCH_WORKERS)
        self._futs, self._issued = {}, 0

    def request(self, key, contig: str, beg: int, end: int) -> None:
        reader = self._ring[self._issued % FETCH_READERS]
        self._issued += 1
        self._futs[key] = self._pool.submit(self._fetch, reader, contig, beg, end)

    def _fetch(self, reader, contig: str, beg: int, end: int):
        t0 = time.perf_counter()
        view = self._src._fetch(reader, contig, beg, end)
        if self._prof is not None:
            self._prof["fetch_thread"] += time.perf_counter() - t0
        return view

    def wait(self, key):
        """The fetched view of request `key`."""
        t0 = time.perf_counter()
        view = self._futs.pop(key).result()            # a Future re-raises the worker's exception (bad contig, corrupt block) here
        if self._prof is not None:
            self._prof["wait_fetch"] += time.perf_counter() - t0
        return view

    def close(self):
        """Waits for the fetches still in flight, so that their readers are free again."""
        self._pool.shutdown(wait=True)
        self._futs = {}

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class VariantFromFiles(_FromFiles):
    """call_variant's make_images + run_inference for a list of intervals of one contig."""

    def __init__(self, bam_path: str, fasta_path: str, state: dict, device: int = 0, threads: int = 0, gpu_inflate: bool = True,
                 host_share: float | None = None):
        super().__init__(bam_path, fasta_path, device, threads, gpu_inflate, host_share)
        self.caller = VariantCaller(state, device)

    def call(self, contig: str, intervals: list[tuple[int, int]], params: dict, include_supplementary: bool = False,
             min_mapq: int = 0, downsample_rate: float = 1.0, max_reads: int = VARIANT_MAX_READS,
             capacity: int | None = None, want_images: bool = True, _view=None) -> tuple[VariantCalls, RegionTable]:
        import torch
        if not intervals:
            raise ValueError("no intervals")
        rows, spans = variant_rows(intervals)
        queries = [(r[0], r[1]) for r in rows]                                      # get_reads(chrom, region_start, region_end, ...)
        regions = self._ref_table(contig, rows, spans)
        view = _view if _view is not None else self._fetch(self.bam, contig, *self._group_span(intervals))
        got = self.trimmer.get_reads(view, queries, include_supplementary, min_mapq, int(params["min_snp_baseq"]),
                                     max_reads=max_reads, downsample_rate=downsample_rate)
        fetched = FetchedReads(got, regions, self.device)
        dev = torch.device("cuda", self.device)
        cap = capacity or max(1024, int(sum(e - s + 1 for s, e in intervals)) // 16)
        while True:
            out = dict(images=torch.empty((cap, 33, 26), dtype=torch.int8, device=dev), positions=torch.empty(cap, dtype=torch.int64, device=dev),
                       depths=torch.empty(cap, dtype=torch.uint8, device=dev), freqs=torch.empty(cap, dtype=torch.uint8, device=dev),
                       keys=torch.empty((cap, 64), dtype=torch.uint8, device=dev), region_of=torch.empty(cap, dtype=torch.int32, device=dev),
                       probs=torch.empty((cap, 3), dtype=torch.float32, device=dev))
            try:
                n = self.caller.call_device(fetched, params, out)
                break
            except PepperB200Error as ex:                  # candidate capacity too small: retry with twice the room
                if ex.rc != PB_ERR_CAPACITY:
                    raise
                cap *= 2
        h = {k: v[:n].cpu().numpy() for k, v in out.items() if want_images or k != "images"}
        return VariantCalls(h["positions"], h["depths"], h["freqs"], h["keys"], h["region_of"], h["probs"], h.get("images")), fetched_table(fetched, regions)


    def find_candidate_tuples(self, contig: str, intervals: list[tuple[int, int]], params: dict, options: dict | None = None, **kw):
        """make_images + run_inference + the per-record candidate selection of find_candidates (CandidateFinder.py:356-530):
        returns (margin_records, deepvariant_records) in the tuple layouts the reference's VcfWriter consumes."""
        from .candidates import find_candidates, ONT_OPTIONS
        calls, table = self.call(contig, intervals, params, want_images=False, **kw)
        return find_candidates(contig, calls.positions, calls.region_of, calls.depths, calls.freqs, calls.keys_raw, calls.probs, table,
                               options or ONT_OPTIONS)

    def find_candidates(self, contig: str, intervals: list[tuple[int, int]], params: dict, options: dict | None = None,
                        vcf_options: dict | None = None, **kw) -> list[dict]:
        """The whole `pepper_variant find_candidates` step for one contig: make_images + run_inference, the per-record selection
        (CUDA kernel), the (contig, position) merge with (ref, alt) de-duplication (CandidateFinder.py:547-581) and the per-site VCF
        record assembly (VcfWriter.py:48-218).  Returns one dict per VCF record (pysam `new_record` keywords + `files`)."""
        from .candidates import ONT_OPTIONS
        from .vcf import find_site_records
        calls, table = self.call(contig, intervals, params, want_images=False, **kw)
        return find_site_records(contig, calls.positions, calls.region_of, calls.depths, calls.freqs, calls.keys_raw, calls.probs, table,
                                 options or ONT_OPTIONS, vcf_options)

    def call_batches(self, contig: str, intervals: list[tuple[int, int]], params: dict, batch: int = 32, **kw):
        """Streaming form: yields (VariantCalls, RegionTable) per batch of `batch` intervals while a helper thread inflates the next
        batch's BAM span with a second reader (pb_bam_fetch runs outside the GIL), so the host inflate overlaps the GPU work."""
        from concurrent.futures import ThreadPoolExecutor
        readers = self._readers(2)
        groups = [intervals[i:i + batch] for i in range(0, len(intervals), batch)]

        def prefetch(k):
            return self._fetch(readers[k & 1], contig, *self._group_span(groups[k]))
        # a Future re-raises the worker's exception (bad contig, corrupt BGZF block) in the consumer
        with ThreadPoolExecutor(max_workers=1) as pool:
            fut = pool.submit(prefetch, 0)
            for k, g in enumerate(groups):
                view = fut.result()
                if k + 1 < len(groups):
                    fut = pool.submit(prefetch, k + 1)
                yield self.call(contig, g, params, _view=view, **kw)


    def call_stream(self, contig: str, intervals: list[tuple[int, int]], params: dict, batch: int = 32, capacity: int | None = None,
                    include_supplementary: bool = False, min_mapq: int = 0, downsample_rate: float = 1.0,
                    max_reads: int = VARIANT_MAX_READS, want_images: bool = False, _finish=None) -> VariantCalls:
        """The whole interval list as ONE streaming session (pipeline.VariantStream): batch k+1's BGZF blocks are read, copied and
        inflated (helper thread, second reader, its own CUDA stream) while batch k's get_reads / encoder / network kernels run;
        candidates accumulate on the device and the network runs over whole 9,472-candidate chunks across batch boundaries.
        `region_of` counts intervals from the start of the list.  `_finish(session, n)`, when given, replaces the D2H fetch of the
        candidates (they are still in the session's device buffers) and its result is returned."""
        if not intervals:
            raise ValueError("no intervals")
        groups = [intervals[i:i + batch] for i in range(0, len(intervals), batch)]
        cap = capacity or max(4096, int(sum(e - s + 1 for s, e in intervals)) // 30)
        prof = dict(wait_fetch=0.0, ref_table=0.0, get_reads=0.0, stage=0.0, run=0.0, sync=0.0, end_fetch=0.0, fetch_thread=0.0)
        while True:
            s = self.caller.stream(params, cap)
            try:
                with _FetchRing(self, prof) as ring:
                    # batch j + FETCH_READERS is requested on the reader of batch j as soon as j's records are trimmed
                    for k in range(min(FETCH_READERS, len(groups))):
                        ring.request(k, contig, *self._group_span(groups[k]))

                    def take(k):
                        fetched = self._trim_variant(ring.wait(k), contig, groups[k], int(params["min_snp_baseq"]), include_supplementary,
                                                     min_mapq, max_reads, downsample_rate, prof)
                        if k + FETCH_READERS < len(groups):
                            ring.request(k + FETCH_READERS, contig, *self._group_span(groups[k + FETCH_READERS]))
                        return fetched
                    nxt = take(0)
                    done = 0
                    for k, g in enumerate(groups):
                        fetched = nxt
                        t3 = time.perf_counter()
                        s.stage_device(fetched, 0, len(g), done)
                        t4 = time.perf_counter()
                        s.run(flush=False)                 # encoder done (host-synchronous), network of this batch queued
                        t5 = time.perf_counter()
                        if k + 1 < len(groups):            # while that network runs: the next batch's records -> trimmed reads
                            nxt = take(k + 1)
                        # no sync: run(k+1) builds its tables while network(k) runs; its encoder synchronises the stream before the
                        # trimmer's buffers (consumed by encoder(k+1)) are overwritten by the trim of batch k+2
                        prof["stage"] += t4 - t3; prof["run"] += t5 - t4
                        done += len(g)
                t0 = time.perf_counter()
                n = s.end()
                out = s.fetch(n, want_images=want_images) if _finish is None else _finish(s, n)
                prof["end_fetch"] = time.perf_counter() - t0
                self.last_profile = {k: round(v * 1e3, 2) for k, v in prof.items()}      # host wall time (ms) per stage of the last call
                return out
            except PepperB200Error as ex:
                if ex.rc != PB_ERR_CAPACITY:
                    raise
                cap *= 2


    def genome_table(self, contig: str, intervals: list[tuple[int, int]]) -> RegionTable:
        """The region table + reference of a whole interval list, rows as the streaming session's groups build them."""
        return self._ref_table(contig, *variant_rows(intervals))

    def vcf_job(self, region: str | None = None, exclude=()) -> list[tuple[str, int, int]]:
        return variant_job(self.fasta_contigs(), self.bam.get_chromosome_sequence_names(), region, exclude, self.bam.index_max_end)

    def call_genome(self, out_dir: str, sample_name: str, region: str | None = None, exclude=(), params: dict | None = None,
                    options: dict | None = None, vcf_options: dict | None = None, batch: int = 32, **kw) -> tuple:
        """`pepper_variant call_variant -b -f -o -s [-r]` on this GPU: make_images + run_inference for every contig of the job
        (variant_job), then per contig the candidate selection, site assembly and VCF text on the device over the session's
        candidate buffers (pb_variant_vcf_device; only the text and its line table come back), then write_vcfs.  Writes the five
        PEPPER_VARIANT_*.vcf.gz (+ .tbi) under `out_dir`; returns the totals of FindCandidates.py:185-189 (all, PEPPER, selected
        for re-genotyping, of them SNPs, indels)."""
        import time
        import torch
        from .abi import PbCandidateColumns, regions_array
        from .candidates import ONT_OPTIONS
        from .synth import ont_params
        from .vcf import order_lines, vcf_text_device, write_vcfs
        job = self.vcf_job(region, exclude)
        names = [c for c, _, _ in job]
        params = params or ont_params()
        parts = []
        prof = dict(calls=0.0, vcf=0.0, write=0.0, encoder_device=0.0, network_device=0.0, bam_fetch=0.0, fasta_fetch=0.0)
        n_groups = 0
        dev = torch.device("cuda", self.device)
        for cid, (contig, start, end) in enumerate(job):
            intervals = variant_intervals(start, end)
            if not intervals:
                continue
            t0 = time.perf_counter()
            table = self.genome_table(contig, intervals)
            prof["fasta_fetch"] += time.perf_counter() - t0

            def finish(s, n, table=table, cid=cid):
                dev_ms = self.caller.timings()                              # the session's encoder / network device time
                prof["encoder_device"] += dev_ms["encode_ms"] / 1e3; prof["network_device"] += dev_ms["network_ms"] / 1e3
                t0 = time.perf_counter()
                cols, d_probs = PbCandidateColumns(), C.c_void_p()
                _lib.check(s.L.pb_variant_stream_columns(self.caller.enc.h, C.byref(cols), C.byref(d_probs), None), "columns")
                d_regions = torch.from_numpy(regions_array(table)[1]).to(dev)
                d_ref = torch.from_numpy(np.ascontiguousarray(table.ref, np.uint8)).to(dev)
                out = vcf_text_device(names, np.full(table.n_regions, cid, np.int32), cols, d_probs.value or 0, n, d_regions.data_ptr(),
                                      d_ref.data_ptr(), options or ONT_OPTIONS, vcf_options, self.device)
                prof["vcf"] += time.perf_counter() - t0
                return out
            t0 = time.perf_counter()
            parts.append(self.call_stream(contig, intervals, params, batch, _finish=finish, **kw))
            prof["calls"] += time.perf_counter() - t0
            # the helper thread's BAM fetches and the groups' reference fetches (inside ref_table) of this contig's session
            prof["bam_fetch"] += self.last_profile["fetch_thread"] / 1e3; prof["fasta_fetch"] += self.last_profile["ref_table"] / 1e3
            n_groups += -(-len(intervals) // batch)
        t0 = time.perf_counter()
        text, lines = order_lines(parts, names)
        totals = write_vcfs(out_dir, sample_name, self.fasta_contigs(), names, text, lines)
        prof["write"] = time.perf_counter() - t0
        prof["calls"] -= prof["vcf"]
        # ms per stage of the last call: host wall of the sessions, of the VCF pass (synchronous) and of the writer; device time
        # of the encoder and the network; host time of the BAM fetches (helper thread) and of the FASTA fetches (the whole-contig
        # tables and each group's reference); "groups" is the number of groups (not a time)
        self.last_genome_profile = {k: round(v * 1e3, 2) for k, v in prof.items()}
        self.last_genome_profile["groups"] = n_groups
        return totals


class _GroupSource(_FromFiles):
    """The read source of the dist drivers: a job every rank opens as the same files (coordinate-sorted BAM + .bai, FASTA), laid
    out contig after contig — contig `names`, `intervals`, the first interval of each contig (+ the total) and `contig_of`, the
    contig id of each interval.  Groups (`groups`) are runs of whole intervals that never cross a contig.  A rank turns the
    groups it claims into trimmed device reads, so no rank reads, inflates or copies a block outside the groups it runs.
    `request(key, g0, g1)` starts the fetch of group [g0, g1)'s BAM span on the fetch ring (_FetchRing); `take(key, g0, g1)`
    waits for it and returns the group's FetchedReads.  A subclass sets the plan (`_set_plan`) and gives a group's BAM span
    (`_span`) and the trim of its fetched records (`_trim`)."""

    def __init__(self, bam_path: str, fasta_path: str, device: int, threads: int, gpu_inflate: bool, host_share: float | None):
        super().__init__(bam_path, fasta_path, device, threads, gpu_inflate, host_share)
        self._ring = _FetchRing(self)

    def _set_plan(self, names: list[str], intervals: list[tuple[int, int]], first: list[int]):
        self.names, self.intervals, self._first = list(names), list(intervals), list(first)
        self.contig_of = np.repeat(np.arange(len(self.names), dtype=np.int32), np.diff(self._first))

    @property
    def n_regions(self) -> int:
        return len(self.intervals)

    def regions_per_contig(self) -> list[int]:
        return np.diff(self._first).tolist()

    def groups(self, group_regions: int = 32) -> list[tuple[int, int]]:
        from .dist import plan_contig_groups
        return plan_contig_groups(self.regions_per_contig(), group_regions)

    def request(self, key, g0: int, g1: int) -> None:
        self._ring.request(key, self.names[self.contig_of[g0]], *self._span(self.intervals[g0:g1]))

    def take(self, key, g0: int, g1: int) -> FetchedReads:
        return self._trim(self._ring.wait(key), self.names[self.contig_of[g0]], self.intervals[g0:g1])

    def close(self):
        if getattr(self, "_ring", None) is not None:
            self._ring.close()
            self._ring = None
        super().close()


class _VariantSource(_GroupSource):
    """Groups of variant intervals: a group's BAM span is its intervals widened by REGION_SAFE_BASES, and its records are trimmed
    by get_reads with the filters of VariantFromFiles.call, on the side stream."""

    def __init__(self, bam_path: str, fasta_path: str, min_snp_baseq: int, device: int, threads: int, gpu_inflate: bool,
                 include_supplementary: bool, min_mapq: int, downsample_rate: float, max_reads: int, host_share: float | None):
        super().__init__(bam_path, fasta_path, device, threads, gpu_inflate, host_share)
        self._filters = (int(min_snp_baseq), include_supplementary, min_mapq, max_reads, downsample_rate)

    def _span(self, intervals: list[tuple[int, int]]) -> tuple[int, int]:
        return self._group_span(intervals)

    def _trim(self, view, contig: str, intervals: list[tuple[int, int]]) -> FetchedReads:
        return self._trim_variant(view, contig, intervals, *self._filters)


class VariantFileSource(_VariantSource):
    """The read source of dist.DistributedVariantCaller for a job given as FILES: the given intervals of one contig, so that
    make_images + run_inference of one contig shard over the ranks from the alignment file itself."""

    def __init__(self, bam_path: str, fasta_path: str, contig: str, intervals: list[tuple[int, int]], min_snp_baseq: int,
                 device: int = 0, threads: int = 0, gpu_inflate: bool = True, include_supplementary: bool = False, min_mapq: int = 0,
                 downsample_rate: float = 1.0, max_reads: int = VARIANT_MAX_READS, host_share: float | None = None):
        super().__init__(bam_path, fasta_path, min_snp_baseq, device, threads, gpu_inflate, include_supplementary, min_mapq,
                         downsample_rate, max_reads, host_share)
        self._set_plan([contig], intervals, [0, len(intervals)])


def genome_plan(fasta_contigs: list[tuple[str, int]], bam_contigs: list[str], region: str | None = None, exclude=(),
                interval_size: int = 100_000, max_end: int | None = None):
    """The job of a whole-genome call: the contigs of variant_job, each tiled with variant_intervals(start, end, interval_size),
    the intervals laid out contig after contig.  Returns (contig names, intervals, first interval of each contig + the total).
    `max_end`: the BAM index's reach (variant_job)."""
    job = variant_job(fasta_contigs, bam_contigs, region, exclude, max_end)
    intervals, first = [], []
    for _, s, e in job:
        first.append(len(intervals))
        intervals.extend(variant_intervals(s, e, interval_size))
    first.append(len(intervals))
    return [c for c, _, _ in job], intervals, first


def group_boundaries(intervals: list[tuple[int, int]], first: list[int], groups: list[tuple[int, int]]) -> np.ndarray:
    """[n_groups, 2] (left, right) boundary positions of each group, -1 where there is none: the start of its first interval
    unless that is the first of its contig, the end of its last interval unless that is the last of its contig.  Group g's right
    boundary is group g+1's left boundary; both groups' intervals emit candidates at that shared position."""
    firsts = set(first[:-1])
    lasts = {f - 1 for f in first[1:]}
    return np.array([[intervals[g0][0] if g0 not in firsts else -1, intervals[g1 - 1][1] if g1 - 1 not in lasts else -1]
                     for g0, g1 in groups], np.int64).reshape(-1, 2)


class VariantGenomeSource(_VariantSource):
    """The read source of dist.DistributedGenomeCaller: every contig of variant_job (the contigs call_genome processes, with the
    same `region` / `exclude` handling), each tiled with variant_intervals(start, end, interval_size).  Contig id k is the k-th
    contig of the job (call_genome's numbering)."""

    def __init__(self, bam_path: str, fasta_path: str, min_snp_baseq: int, region: str | None = None, exclude=(),
                 interval_size: int = 100_000, device: int = 0, threads: int = 0, gpu_inflate: bool = True,
                 include_supplementary: bool = False, min_mapq: int = 0, downsample_rate: float = 1.0,
                 max_reads: int = VARIANT_MAX_READS, host_share: float | None = None):
        super().__init__(bam_path, fasta_path, min_snp_baseq, device, threads, gpu_inflate, include_supplementary, min_mapq,
                         downsample_rate, max_reads, host_share)
        self._set_plan(*genome_plan(self.fasta_contigs(), self.bam.get_chromosome_sequence_names(), region, exclude, interval_size,
                                    self.bam.index_max_end))

    def boundaries(self, groups: list[tuple[int, int]]) -> np.ndarray:
        return group_boundaries(self.intervals, self._first, groups)

    def group_work(self, groups: list[tuple[int, int]]) -> np.ndarray:
        """Genomic bases per group: the work estimate the static schedule balances."""
        return np.array([self.intervals[g1 - 1][1] - self.intervals[g0][0] + 1 for g0, g1 in groups], dtype=np.int64)

    def table(self, regions) -> RegionTable:
        """The region table + reference of the given region ids, in rows as call_genome's genome_table builds them (the reference
        offsets point into one string); the other rows are zero."""
        rows = np.zeros((self.n_regions, 8), np.int64)
        refs, base = [], 0
        by_contig = {}
        for r in sorted(int(x) for x in regions):
            by_contig.setdefault(int(self.contig_of[r]), []).append(r)
        for k, rs in by_contig.items():
            t = self._ref_table(self.names[k], *variant_rows([self.intervals[r] for r in rs]))
            t.table[:, 4] += base
            rows[rs] = t.table
            refs.append(t.ref); base += t.ref.shape[0]
        return RegionTable(rows, np.concatenate(refs) if refs else np.zeros(1, np.uint8))


class PolishFromFiles(_FromFiles):
    """polish's make_images (with read realignment) + call_consensus for a list of regions of one contig."""

    def __init__(self, bam_path: str, fasta_path: str, state: dict, device: int = 0, threads: int = 0, gpu_inflate: bool = True,
                 host_share: float | None = None):
        super().__init__(bam_path, fasta_path, device, threads, gpu_inflate, host_share)
        self.caller = PolishCaller(state, device)
        self.realigner = Realigner(device)

    def call(self, contig: str, regions_se: list[tuple[int, int]], realign: bool = True, max_reads: int = POLISH_MAX_READS,
             capacity: int | None = None) -> tuple[PolishCalls, RegionTable]:
        import torch
        if not regions_se:
            raise ValueError("no regions")
        regions = self._ref_table(contig, *polish_rows(regions_se))
        view = self._fetch(self.bam, contig, min(r[0] for r in regions_se), max(r[1] for r in regions_se))
        got = self.trimmer.get_reads(view, regions_se, False, 0, 0, max_reads=max_reads, downsample_rate=1.0)   # :300-325
        fetched = FetchedReads(got, regions, self.device)
        if realign:
            fetched.struct = self.realigner.realign_device(fetched)                # :328-332
        dev = torch.device("cuda", self.device)
        cap = capacity or 3 * (sum(e - s + 1 for s, e in regions_se) // 950 + len(regions_se)) + 8
        while True:
            out = dict(bases=torch.empty((cap, 1000), dtype=torch.uint8, device=dev), phred=torch.empty((cap, 1000), dtype=torch.uint8, device=dev),
                       position=torch.empty((cap, 1000), dtype=torch.int64, device=dev), index=torch.empty((cap, 1000), dtype=torch.int32, device=dev),
                       image_region=torch.empty(cap, dtype=torch.int32, device=dev), chunk_id=torch.empty(cap, dtype=torch.int32, device=dev))
            try:
                n = self.caller.call_device(fetched, out)
                break
            except PepperB200Error as ex:
                if ex.rc != PB_ERR_CAPACITY:
                    raise
                cap *= 2
        h = {k: v[:n].cpu().numpy() for k, v in out.items()}
        return PolishCalls(h["bases"], h["phred"], h["position"], h["index"], h["image_region"], h["chunk_id"]), fetched_table(fetched, regions)

    def polish_contig(self, contig: str, start: int = 0, end: int | None = None, batch: int = 2000, realign: bool = True,
                      return_calls: bool = False, qualities: bool = False):
        """The whole polish path of one contig span: tiling (ImageGenerationUI.py:262-272: the span is [start, length - 1]),
        make_images + call_consensus in batches of `batch` regions, then the stitch (Stitch.py:36-128) -> polished sequence;
        `qualities`: (sequence, FASTQ quality string) (polish.stitch_with_qualities).  `return_calls`: (that, calls, regions)."""
        from .polish import stitch, stitch_with_qualities
        if end is None:
            end = self.fasta.get_chromosome_sequence_length(contig) - 1
        regs = polish_intervals(start, end)
        parts = []
        for i in range(0, len(regs), batch):
            calls, _ = self.call(contig, regs[i:i + batch], realign=realign)
            parts.append((calls, i))
        cat = lambda f: np.concatenate([getattr(c, f) for c, _ in parts])       # noqa: E731
        image_region = np.concatenate([c.image_region + off for c, off in parts]).astype(np.int32)
        allc = PolishCalls(cat("bases"), cat("phred"), cat("position"), cat("index"), image_region, cat("chunk_id"))
        starts = np.array([r[0] for r in regs], dtype=np.int64)
        if qualities:
            seq = stitch_with_qualities(allc.bases, allc.phred, allc.position, allc.index, allc.image_region, allc.chunk_id, starts)
        else:
            seq = stitch(allc.bases, allc.position, allc.index, allc.image_region, allc.chunk_id, starts)
        return (seq, allc, regs) if return_calls else seq

    def polish_assembly(self, out_path: str | None = None, contigs: list[str] | None = None, group_regions: int = 32,
                        capacity_bytes: int | None = None, realign: bool = True, fastq: bool = False, vcf_path: str | None = None,
                        capacity_events: int | None = None) -> dict:
        """`pepper polish` of a whole assembly on this GPU: every contig common to the BAM and the FASTA (or `contigs`),
        make_images + call_consensus + the stitch on the device through one streaming session (dist.DistributedPolisher at world
        size 1).  Returns {contig: polished sequence} and, given `out_path`, writes the FASTA perform_stitch writes.
        `fastq`: the quality of every base is carried through the stitch; returns {contig: (sequence, quality string)} and
        writes FASTQ (write_polished_fastq) to `out_path`.
        `vcf_path`: also writes the edits VCF there (bgzipped, with its .tbi or .csi; polish_edits): a record for every run of
        draft bases the stitch substituted, deleted or inserted after, with the least network phred of its columns as QUAL.
        The return value is the same.  `capacity_events`: the first size of the event sink (doubled until it fits)."""
        from .dist import DistributedPolisher
        src = PolishFileSource(self.bam.path, self.fasta_path, contigs, self.device, self.threads, self.gpu_inflate, realign,
                               host_share=self.host_share)
        try:
            span = sum(e - s + 1 for s, e in src.intervals)
            cap = capacity_bytes or 2 * span + (1 << 20)
            ecap = capacity_events or span // 32 + (1 << 16)
            while True:
                dp = DistributedPolisher(None, self.device, cap, "static", group_regions, distributed=False, caller=self.caller,
                                         qualities=fastq, edits=vcf_path is not None, capacity_events=ecap)
                try:
                    dp.run(src)
                    seqs = dp.assemble(src)
                    if vcf_path is not None:
                        dp.write_edits(src, vcf_path)
                    break
                except PepperB200Error as ex:        # consensus or events larger than their sink: restart the session larger
                    if ex.rc != PB_ERR_CAPACITY:
                        raise
                    if hasattr(ex, "need_events"):
                        ecap *= 2
                    else:
                        cap *= 2
                finally:
                    dp.close()
        finally:
            src.close()
        if out_path is not None:
            (write_polished_fastq if fastq else write_polished_fasta)(out_path, seqs)
        return seqs


def natural_key(string_: str) -> list:
    """Contig order of `pepper polish` (ImageGenerationUI.natural_key, pepper ImageGenerationUI.py:82-85; perform_stitch.py:12-14):
    digit runs compare as numbers, so ctg2 < ctg10."""
    return [int(s) if s.isdigit() else s for s in re.split(r"(\d+)", string_)]


def write_polished_fasta(path: str, seqs: dict) -> None:
    """What perform_stitch writes (perform_stitch.py:59,80-82): '>contig\n<sequence>\n' per contig, one line per sequence,
    contigs in natural order, contigs with an empty consensus left out."""
    with open(path, "w") as f:
        f.write(polished_fasta_text(seqs))


def polished_fasta_text(seqs: dict) -> str:
    return "".join(">%s\n%s\n" % (c, seqs[c]) for c in sorted(seqs, key=natural_key) if seqs[c])


def write_polished_fastq(path: str, records: dict) -> None:
    """The polished assembly with the quality of every base: '@contig\n<sequence>\n+\n<qualities>\n' per contig, no line
    wrapping, contigs in natural order, contigs with an empty consensus left out (the contigs and sequences of
    write_polished_fasta).  `records`: {contig: (sequence, quality string)}."""
    with open(path, "w") as f:
        f.write(polished_fastq_text(records))


def polished_fastq_text(records: dict) -> str:
    for c, (seq, qual) in records.items():
        if len(seq) != len(qual):
            raise ValueError("%s: %d bases but %d qualities" % (c, len(seq), len(qual)))
    return "".join("@%s\n%s\n+\n%s\n" % ((c,) + tuple(records[c])) for c in sorted(records, key=natural_key) if records[c][0])


def polish_job(fasta_contigs: list[tuple[str, int]], bam_contigs: list[str], contigs: list[str] | None = None,
               max_end: int | None = None):
    """The job of a whole-assembly polish: every contig common to the FASTA (name, length) and the BAM, in natural order
    (ImageGenerationUI.get_chromosome_list, pepper ImageGenerationUI.py:88-117), or `contigs`; each contig tiled with
    polish_intervals(0, length - 1) (a contig too short to tile has no region).  An entry of `contigs` may also be
    (contig, (start, end)) or (contig, None), as parse_region gives them: that contig is tiled over [max(0, start),
    min(end, length - 1)] (pepper ImageGenerationUI.py:257-272).  Returns (contigs, regions laid out contig after contig, first
    region of each contig + the total).  `max_end`: the BAM index's reach; a longer contig raises ValueError."""
    lengths = dict(fasta_contigs)
    if contigs is None:
        contigs = sorted(set(lengths) & set(bam_contigs), key=natural_key)
    spans = []
    for c in contigs:
        c, span = (c, None) if isinstance(c, str) else c
        s, e = span if span is not None else (0, lengths[c] - 1)
        spans.append((c, max(0, s), min(e, lengths[c] - 1)))
    check_reach([(c, e + 1) for c, _, e in spans], max_end)
    regions, first = [], []
    for _, s, e in spans:
        first.append(len(regions))
        regions.extend(polish_intervals(s, e))
    first.append(len(regions))
    return [c for c, _, _ in spans], regions, first


def parse_region(region: str) -> list[tuple[str, tuple[int, int] | None]]:
    """`-r/--region` of call_variant (ImageGenerationUI.get_chromosome_list, pepper_variant ImageGenerationUI.py:131-171): a comma
    list of `contig` or `contig:start-end`, where a name such as `chr1-3` expands to chr1, chr2, chr3."""
    out = []
    for name in [x.strip() for x in region.strip().split(",")]:
        span = None
        if ":" in name:
            parts = name.strip().split(":")
            if len(parts) != 2:
                raise ValueError("--region: invalid value %r" % name)
            name, rng = parts
            span = [int(x) for x in rng.strip().split("-")]
            if len(span) != 2 or not span[0] <= span[1]:
                raise ValueError("--region: invalid value %r" % rng)
            span = (span[0], span[1])
        pieces = name.split("-")
        if len(pieces) > 1:
            prefix = re.match(r"\D*", name).group(0)
            nums = sorted(int("".join(ch for ch in p if ch.isdigit())) for p in pieces)
            out += [(prefix + str(k), span) for k in range(nums[0], nums[-1] + 1)]
        else:
            out.append((name, span))
    return out


def check_reach(spans: list[tuple[str, int]], max_end: int | None) -> None:
    """Raise ValueError when a contig would be processed up to an end (exclusive) past `max_end`, the BAM index's reach: a fetch
    returns no read at or past it (a BAI addresses positions below 2^29), so that part of the contig would get no reads."""
    if max_end is None:
        return
    for c, end in spans:
        if end > max_end:
            raise ValueError("contig %r is processed up to position %d, but the BAM index only addresses positions below %d: "
                             "index the BAM with a CSI of enough depth (samtools index -c)" % (c, end, max_end))


def variant_job(fasta_contigs: list[tuple[str, int]], bam_contigs: list[str], region: str | None = None, exclude=(),
                max_end: int | None = None):
    """The contigs a genome-wide call_variant processes, as (contig, start, end) intervals to tile with variant_intervals
    (ImageGenerationUI.generate_images, pepper_variant ImageGenerationUI.py:283-316): without `region`, every contig common to the
    FASTA and the BAM and not in `exclude`, in natural order, over [0, length - 1]; with it, the listed contigs in the listed order,
    each span clamped to [0, length - 1].  `max_end`: the BAM index's reach; a span that ends past it raises ValueError."""
    lengths = dict(fasta_contigs)
    if region is None:
        common = sorted((set(lengths) & set(bam_contigs)) - set(exclude), key=natural_key)
        if not common:
            raise ValueError("no contig common to the BAM and the FASTA")
        job = [(c, 0, lengths[c] - 1) for c in common]
    else:
        job = []
        for c, span in parse_region(region):
            if c not in lengths:
                raise ValueError("--region: contig %r is not in the FASTA" % c)
            s, e = span if span is not None else (0, lengths[c] - 1)
            job.append((c, max(0, s), min(e, lengths[c] - 1)))
    check_reach([(c, e + 1) for c, _, e in job], max_end)
    return job


class PolishFileSource(_GroupSource):
    """The read source of dist.DistributedPolisher: a whole assembly, every contig common to both files in natural order
    (ImageGenerationUI.get_chromosome_list, pepper ImageGenerationUI.py:88-117) or the given `contigs`, each tiled with
    polish_intervals(0, length - 1), or over its span where `contigs` gives one (polish_job).  `take` runs get_reads with the filters of PolishFromFiles.call and the realignment on a
    side stream, so that a group's inflate, trim and realignment run beside the previous group's network."""

    def __init__(self, bam_path: str, fasta_path: str, contigs: list[str] | None = None, device: int = 0, threads: int = 0,
                 gpu_inflate: bool = True, realign: bool = True, max_reads: int = POLISH_MAX_READS, host_share: float | None = None):
        super().__init__(bam_path, fasta_path, device, threads, gpu_inflate, host_share)
        self._set_plan(*polish_job(self.fasta_contigs(), self.bam.get_chromosome_sequence_names(), contigs, self.bam.index_max_end))
        self.realign = realign
        self.realigner = Realigner(device) if realign else None
        self._max_reads = max_reads

    @property
    def contigs(self) -> list[str]:
        """The contigs of the assembly, in the order polished (the plan's `names`)."""
        return self.names

    def group_work(self, groups: list[tuple[int, int]]) -> np.ndarray:
        """Draft bases per group: the work estimate the static schedule balances."""
        return np.array([sum(e - s + 1 for s, e in self.intervals[g0:g1]) for g0, g1 in groups], dtype=np.int64)

    def _span(self, regs: list[tuple[int, int]]) -> tuple[int, int]:
        return min(s for s, _ in regs), max(e for _, e in regs)

    def _trim(self, view, contig: str, regs: list[tuple[int, int]]) -> FetchedReads:
        regions = self._ref_table(contig, *polish_rows(regs))
        side = self._side_stream()
        got = self.trimmer.get_reads(view, regs, False, 0, 0, max_reads=self._max_reads, downsample_rate=1.0, stream=side.cuda_stream)
        fetched = FetchedReads(got, regions, self.device, stream=side)
        if self.realign:
            fetched.struct = self.realigner.realign_device(fetched, stream=side.cuda_stream)     # synchronises the side stream
        return fetched

    def close(self):
        super().close()
        if getattr(self, "realigner", None) is not None:
            self.realigner.close()
            self.realigner = None


def fetched_table(fetched: FetchedReads, regions: RegionTable) -> RegionTable:
    """The region table with the read ranges get_reads produced (after down-sampling)."""
    return RegionTable(fetched.table.copy(), regions.ref)


# ---------------------------------------------------------------------------------------------- prediction stores
def write_variant_predictions(store, contig: str, calls: VariantCalls, batch_size: int = 512, first_batch: int = 0) -> int:
    """What run_inference leaves on disk: predictions/batch_<n>/... in batches of `batch_size` candidates
    (pepper_variant predict_distributed_gpu.py:58-70 -> DataStorePredict.write_prediction).  Returns the next batch number."""
    keys = calls.keys
    b = first_batch
    for lo in range(0, len(calls), batch_size):
        hi = min(len(calls), lo + batch_size)
        store.write_prediction(b, [contig] * (hi - lo), calls.positions[lo:hi], calls.depths[lo:hi], keys[lo:hi], calls.freqs[lo:hi],
                               calls.probs[lo:hi])
        b += 1
    return b


def write_polish_predictions(store, contig: str, calls: PolishCalls, regions_se: list[tuple[int, int]]) -> None:
    """What call_consensus leaves on disk: one predictions/<contig>/<contig>-<start>-<end>/<chunk> group per image
    (pepper predict_distributed_gpu.py:107-109 -> DataStorePredict.write_prediction)."""
    for i in range(calls.bases.shape[0]):
        rs, re_ = regions_se[int(calls.image_region[i])]
        store.write_prediction(contig, rs, re_, int(calls.chunk_id[i]), calls.position[i], calls.index[i], calls.bases[i], calls.phred[i])

