"""Multi-GPU product path of the variant hot path (SURVEY.md §8e; replaces the reference's file-chunk round robin over
processes / DataParallel, pepper_variant RunInference.py:70-72,104-106, ImageGenerationUI.py:307-316,
predict_distributed_gpu.py:41).

Regions (100 kb intervals) are independent units.  A job is cut into region GROUPS; every rank runs a streaming session
(`pipeline.VariantStream`) over the groups it owns and the network's head kernel writes each candidate's 84-byte prediction
record straight into this rank's slice of ONE gather buffer; a single fixed-capacity all-gather (no host round trip for the
ragged counts, which travel in a second tiny all-gather) then gives every rank the whole job's records.

Two schedules:
  * static  — contiguous blocks of groups balanced by aligned-base count (`shard_regions`): rank-major order == genomic order;
  * dynamic — ranks claim the next group from an atomic counter in the rendezvous store (`GroupClaimer`), so a GPU that runs
              slower under the board power cap simply takes fewer groups; genomic order is restored from the region ids the
              records carry (`order_records`).
Backend-agnostic (`nccl` on GPUs, `gloo` in the CPU tests)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .abi import PRED_RECORD

RECORD_BYTES = PRED_RECORD.itemsize
GVCF_BATCH = 1 << 22        # track positions per batch of the gVCF pass: bounds its device workspace (DESIGN.md section 4)


def shard_regions(work: np.ndarray, world: int) -> list[tuple[int, int]]:
    """Contiguous blocks [begin, end) of units per rank, balanced by `work` (e.g. aligned bases per region / group).
    Contiguity keeps rank-major order == genomic order after the gather."""
    n = int(work.shape[0])
    if n == 0:
        return [(0, 0)] * world
    csum = np.concatenate([[0], np.cumsum(work.astype(np.float64))])
    total = csum[-1]
    cuts = [0]
    for r in range(1, world):
        target = total * r / world
        k = int(np.searchsorted(csum, target, side="left"))
        k = min(max(k, cuts[-1]), n)
        # choose the nearer of k-1 / k to the target
        if k > cuts[-1] and abs(csum[k - 1] - target) <= abs(csum[min(k, n)] - target):
            k -= 1
        cuts.append(max(k, cuts[-1]))
    cuts.append(n)
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


def plan_groups(n_regions: int, group: int = 32) -> list[tuple[int, int]]:
    """Region groups [g0, g1) of a job: the hand-out unit (about 50 k candidates = 5 network chunks at ONT 30x)."""
    return [(g, min(n_regions, g + group)) for g in range(0, n_regions, group)]


def plan_groups_tapered(n_regions: int, group: int, world: int, min_group: int = 4) -> list[tuple[int, int]]:
    """Guided self-scheduling for the dynamic schedule: full `group`-sized groups, then shrinking ones (remaining / (2 world), at
    least `min_group`) so that the tail imbalance between ranks is a few regions, not one full group."""
    out, g = [], 0
    while g < n_regions:
        rem = n_regions - g
        size = max(min_group, min(group, -(-rem // (2 * max(1, world)))))
        out.append((g, min(n_regions, g + size)))
        g += size
    return out


def group_work(seq_off: np.ndarray, table: np.ndarray, groups: list[tuple[int, int]]) -> np.ndarray:
    """Aligned bases per group (the balance criterion of SURVEY 8e) from the reads' sequence offsets."""
    return np.array([int(seq_off[int(table[g1 - 1, 7])] - seq_off[int(table[g0, 6])]) for g0, g1 in groups], dtype=np.int64)


class GroupClaimer:
    """Hands out group indices.  `dynamic`: an atomic counter in the process group's rendezvous store (TCPStore.add is atomic;
    ~20 us per claim against ~20 ms of GPU work per group).  `static`: this rank's contiguous block."""

    def __init__(self, n_groups: int, rank: int, world: int, schedule: str = "dynamic", work: np.ndarray | None = None,
                 store=None, key: str = "pb_claim"):
        self.n, self.rank, self.world, self.schedule = n_groups, rank, world, schedule
        if schedule == "static" or world == 1:
            b, e = shard_regions(work if work is not None else np.ones(n_groups), world)[rank]
            self._it = iter(range(b, e))
            self.store = None
        elif schedule == "dynamic":
            if store is None:
                import torch.distributed as dist
                store = dist.distributed_c10d._get_default_store()
            self.store, self.key = store, key
            self._it = None
        else:
            raise ValueError("schedule must be 'static' or 'dynamic'")

    def next(self):
        if self._it is not None:
            return next(self._it, None)
        g = int(self.store.add(self.key, 1)) - 1
        return g if g < self.n else None

    def exhausted(self) -> bool:
        """Dynamic schedule: has every group been claimed?  (a rank that stopped claiming for lack of room checks this)"""
        if self._it is not None:
            return True
        return int(self.store.add(self.key, 0)) >= self.n


class GatherBuffer:
    """[world][capacity] records + [world] counts.  A record is `record` (a numpy dtype): the 84-byte prediction record of the
    variant path by default, one byte of polished consensus for the polish path (2 bytes, base and quality, with qualities).
    On NCCL the record tensor is allocated from NCCL's own allocator (ncclMemAlloc through torch.cuda.MemPool) when this torch
    build offers it, so the collective works on registered user buffers; otherwise a plain tensor."""

    def __init__(self, capacity: int, world: int, rank: int, device=None, max_groups: int = 0, record=PRED_RECORD):
        import torch
        self.capacity, self.world, self.rank = int(capacity), world, rank
        self.max_groups = int(max_groups)
        self.record = np.dtype(record)
        self.record_bytes = self.record.itemsize
        self.registered = False
        nbytes = world * self.capacity * self.record_bytes
        dev = device if device is not None else torch.device("cpu")
        self._dev = dev
        self.records = None
        if getattr(dev, "type", "cpu") == "cuda" and world > 1:
            try:
                import torch.distributed as dist
                backend = dist.distributed_c10d._get_default_group()._get_backend(dev)
                pool = torch.cuda.MemPool(backend.mem_allocator)
                with torch.cuda.use_mem_pool(pool):
                    self.records = torch.empty(nbytes, dtype=torch.uint8, device=dev)
                backend.register_mem_pool(pool)
                self._pool = pool
                self.registered = True
            except Exception:
                self.records = None
        if self.records is None:
            self.records = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        # per rank: [n_valid, (group id, records) x max_groups] — the ragged counts and, for the dynamic schedule, the order
        # in which the rank ran its groups (group id -1 = unused slot)
        self._w = 1 + 2 * self.max_groups
        self.meta = torch.zeros((world, self._w), dtype=torch.int64, device=dev)
        self._mine = torch.zeros(self._w, dtype=torch.int64, device=dev)
        self._mine_host = torch.zeros(self._w, dtype=torch.int64).pin_memory() if getattr(dev, "type", "cpu") == "cuda" else torch.zeros(self._w, dtype=torch.int64)

    @property
    def counts(self):
        return self.meta[:, 0]

    @property
    def slice_bytes(self) -> int:
        return self.capacity * self.record_bytes

    def my_slice(self):
        return self.records[self.rank * self.slice_bytes:(self.rank + 1) * self.slice_bytes]

    def my_ptr(self) -> int:
        return self.records.data_ptr() + self.rank * self.slice_bytes

    def set_mine(self, n_valid: int, segments=None):
        """This rank's row of the meta table: record count and the (group id, records) list in processing order."""
        if n_valid > self.capacity:
            raise ValueError("n_valid %d > capacity %d" % (n_valid, self.capacity))
        h = self._mine_host
        h.zero_()
        h[0] = n_valid
        if self.max_groups:
            h[1::2] = -1
            for i, (g, c) in enumerate(segments or []):
                h[1 + 2 * i], h[2 + 2 * i] = g, c
        self._mine.copy_(h, non_blocking=True)

    def gather_meta(self, group=None):
        import torch.distributed as dist
        if self.world == 1:
            self.meta[0].copy_(self._mine)
        else:
            dist.all_gather_into_tensor(self.meta.view(-1), self._mine, group=group)

    def gather_records(self, group=None):
        """In place: this rank's input is its own slice of the output."""
        import torch.distributed as dist
        if self.world > 1:
            dist.all_gather_into_tensor(self.records, self.my_slice(), group=group)

    def gather(self, n_valid: int, segments=None, group=None):
        """Both collectives are enqueued back to back; nothing is read on the host here."""
        self.set_mine(n_valid, segments)
        self.gather_meta(group)
        self.gather_records(group)

    def to_host(self, order: bool = True) -> np.ndarray:
        """The valid records of every rank on the host (one small host sync for the meta table, then asynchronous D2H copies
        straight into their FINAL place in one page-locked buffer — rank-major, or group by group in genomic order when the
        ranks reported their group segments — so no host-side re-ordering pass is needed).  The returned array is a view of
        that buffer (valid until the next to_host)."""
        import torch
        counts, segs = self._parse_meta()
        total = sum(counts)
        by_segment = order and bool(segs) and sum(k for _, _, k in segs) == total
        if by_segment:
            segs.sort()
            # merge neighbours that are contiguous in the source (a static schedule collapses to one copy per rank)
            plan = []
            for g, o, k in segs:
                if plan and plan[-1][0] + plan[-1][1] == o:
                    plan[-1][1] += k
                else:
                    plan.append([o, k])
        else:
            plan = [[r * self.capacity, counts[r]] for r in range(self.world)]
        cuda = self.records.is_cuda
        rb = self.record_bytes
        need = max(total, 1) * rb
        if getattr(self, "_host", None) is None or self._host.numel() < need:
            self._host = torch.empty(need + need // 8, dtype=torch.uint8)
            if cuda:
                self._host = self._host.pin_memory()
        dst = 0
        for o, k in plan:
            if k:
                self._host[dst * rb:(dst + k) * rb].copy_(self.records[o * rb:(o + k) * rb], non_blocking=True)
                dst += k
        if cuda:
            torch.cuda.current_stream(self.records.device).synchronize()
        rec = self._host.numpy()[:total * rb].view(self.record)
        reorder = order and not by_segment and self.record.names is not None and "region" in self.record.names
        return order_records(rec) if reorder else rec

    def segments(self) -> list[tuple[int, int]]:
        """(group id, records) of every group every rank ran, sorted by group id (after gather_meta)."""
        return sorted((g, k) for g, _, k in self._parse_meta()[1])

    def _parse_meta(self) -> tuple[list[int], list[tuple[int, int, int]]]:
        """The gathered meta table on the host: every rank's record count, and (group id, source record index in the gather
        buffer, records) of every group every rank ran, rank-major in run order."""
        meta = self.meta.cpu().numpy()
        counts, segs = [int(meta[r, 0]) for r in range(self.world)], []
        for r in range(self.world):
            off = r * self.capacity
            for i in range(self.max_groups):
                g, k = int(meta[r, 1 + 2 * i]), int(meta[r, 2 + 2 * i])
                if g < 0:
                    break
                segs.append((g, off, k))
                off += k
        return counts, segs

    def release(self):
        """Drops the NCCL-registered pool BEFORE the process group goes away (a registered MemPool destroyed after
        destroy_process_group aborts the process)."""
        self.records = None
        self.meta = None
        pool = getattr(self, "_pool", None)
        if pool is not None:
            try:
                import torch.distributed as dist
                backend = dist.distributed_c10d._get_default_group()._get_backend(self._dev)
                backend.deregister_mem_pool(pool)
            except Exception:
                pass
            self._pool = None
            del pool


def order_records(rec: np.ndarray) -> np.ndarray:
    """Genomic order = region id order (within a region the encoder's order is kept: stable sort)."""
    if rec.shape[0] == 0 or np.all(np.diff(rec["region"]) >= 0):
        return rec
    return rec[np.argsort(rec["region"], kind="stable")]


def records_from_calls(calls) -> np.ndarray:
    """A single-GPU VariantCalls as prediction records (the 1-rank answer the N-rank gather must reproduce)."""
    rec = np.zeros(len(calls), PRED_RECORD)
    rec["probs"] = calls.probs
    rec["position"] = calls.positions.astype(np.int32)
    rec["region"] = calls.region_of
    rec["depth"] = calls.depths
    rec["freq"] = calls.freqs
    rec["key"] = np.ascontiguousarray(calls.keys_raw[:, :62]).view("S62")[:, 0]
    return rec


def run_claimed(s, claimer: GroupClaimer, stage, request, depth: int, capacity: int, n_job: int, world: int) -> list[tuple[int, int]]:
    """The claim / stage / run loop of one streaming session (pipeline.VariantStream or PolishStream): claims up to `depth` groups
    ahead of the one being run (`request(j)`, optional, starts the fetch of claimed group j), stages group j with `stage(j)` and
    runs it while the next one is staged.  `s.run()` returns the session's running total of records (or an upper bound of it);
    returns (group, records) per group run, in run order."""
    from collections import deque
    segments, seen = [], 0
    # a rank stops claiming when its slice of the gather buffer could not hold the groups in flight plus the one it would
    # claim: under the dynamic schedule a rank that started early may otherwise take more than its capacity; what it leaves is
    # claimed by the others
    worst = max(1, capacity // max(4, 2 * n_job // max(1, world)))
    ahead = deque()

    def claim():
        while len(ahead) < depth and capacity - seen >= (len(ahead) + 2.2) * worst:
            j = claimer.next()
            if j is None:
                return
            if request is not None:
                request(j)
            ahead.append(j)
    claim()
    cur = ahead.popleft() if ahead else None
    if cur is not None:
        stage(cur)                        # (file source: takes this group's records before its reader is asked for another span)
    while cur is not None:
        claim()                           # claimed ahead: the next group's copies (or file fetch) overlap this group's kernels
        tot = s.run(flush=False)
        segments.append((cur, tot - seen))
        worst = max(worst, tot - seen)
        seen = tot
        cur = ahead.popleft() if ahead else None
        if cur is not None:
            stage(cur)                    # no sync: the next run() prepares its tables while this group's network runs
    return segments


def check_groups_ran(done: int, n_job: int, capacity: str, option: str) -> None:
    """Raises PB_ERR_CAPACITY unless the ranks together ran all `n_job` groups.  Under any schedule and world size, run_claimed
    stops claiming when a rank's `capacity` (named in the message, with the `option` that raises it) could not hold another
    group, so the groups it did not run would otherwise be missing from the result without a word."""
    if done != n_job:
        from ._lib import PepperB200Error
        from .abi import PB_ERR_CAPACITY
        raise PepperB200Error("only %d of %d groups were run: %s is exhausted — raise `%s`" % (done, n_job, capacity, option),
                              PB_ERR_CAPACITY)


class _RankDriver:
    """What the distributed drivers share: this process's rank in the default process group (world size 1 with
    `distributed=False` or without a process group), the caller it runs (closed with the driver unless it was given), a claim
    key per call, the claim / stage / run loop over a job's groups and the timed gather of the records into `buffer`."""

    _claim_prefix = "pb_claim"              # one per driver class: two drivers of one process group never share a claim counter

    def __init__(self, caller_cls, state: dict, device: int, schedule: str, group_regions: int, distributed: bool, caller):
        import torch
        import torch.distributed as dist
        on = distributed and dist.is_initialized()
        self.world = dist.get_world_size() if on else 1
        self.rank = dist.get_rank() if on else 0
        self._own_caller = caller is None
        self.caller = caller if caller is not None else caller_cls(state, device)
        self.device = torch.device("cuda", device)
        self.schedule, self.group_regions = schedule, group_regions
        self.buffer = None
        self._calls = 0
        self._ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        self.phase_ms, self.stats = {}, {}

    def close(self):
        """Call before destroy_process_group()."""
        if self.buffer is not None:
            self.buffer.release()
            self.buffer = None
        if self._own_caller:
            self.caller.close()

    def _claimer(self, n_job: int, work: np.ndarray | None) -> GroupClaimer:
        self._calls += 1
        return GroupClaimer(n_job, self.rank, self.world, self.schedule, work, key="%s_%d" % (self._claim_prefix, self._calls))

    def _gather_buffer(self, capacity: int, n_job: int, record=PRED_RECORD) -> GatherBuffer:
        if (self.buffer is None or self.buffer.max_groups < n_job or self.buffer.capacity != capacity
                or self.buffer.record != np.dtype(record)):
            if self.buffer is not None:
                self.buffer.release()
            self.buffer = GatherBuffer(capacity, self.world, self.rank, self.device, max_groups=n_job, record=record)
        return self.buffer

    def _run_job(self, s, claimer, groups: list[tuple[int, int]], capacity: int, source=None, stage=None, first=None,
                 world: int | None = None, owned=None) -> list[tuple[int, int]]:
        """run_claimed over the job's groups: group j covers regions groups[j] = [g0, g1) of the source and is staged with region
        ids from first[j] (default g0).  From a file source (frontend._GroupSource) the fetch of a claimed group starts on the
        source's fetch ring, one fetch per reader outstanding beside the group being run; otherwise `stage(j)` stages group j.
        `owned(j)`: the owned ends of group j's regions, given to a gVCF track session after each stage."""
        from .frontend import FETCH_READERS
        request, depth = None, 1
        if source is not None:
            def stage(j):
                g0, g1 = groups[j]
                s.stage_device(source.take(j, g0, g1), 0, g1 - g0, g0 if first is None else first[j])
                if owned is not None:
                    s.owned(owned(j))

            def request(j):
                source.request(j, *groups[j])
            depth = FETCH_READERS
        return run_claimed(s, claimer, stage, request, depth, capacity, len(groups), world or self.world)

    def _gather(self, s, n: int, segments: list[tuple[int, int]], n_job: int, capacity: str, option: str):
        """This rank's count and segments into the meta table, both all-gathers (timed: the wait for the slowest rank, then the
        transfer), then the check that the ranks together ran every group."""
        import torch
        t = self.caller.timings()
        self.stats = s.stats()
        self.buffer.set_mine(n, segments)
        self._ev[0].record()
        self.buffer.gather_meta()                 # tiny: completes when the slowest rank arrives -> the wait, not the transfer
        self._ev[1].record()
        self.buffer.gather_records()
        self._ev[2].record()
        torch.cuda.synchronize(self.device)
        self.phase_ms = dict(encoder_ms=t["encode_ms"], network_ms=t["network_ms"], wait_ms=self._ev[0].elapsed_time(self._ev[1]),
                             gather_ms=self._ev[1].elapsed_time(self._ev[2]), groups=len(segments))
        check_groups_ran(len(self.buffer.segments()), n_job, capacity, option)


class DistributedVariantCaller(_RankDriver):
    """make_images + run_inference of ONE job (a region list every rank can read) over all ranks of the default process group.

        dvc = DistributedVariantCaller(state, local_device, capacity)
        dvc.run(source, regions, params)        # source: abi.HostReads (pinned host buffers), pipeline.DeviceReads, or
                                                # frontend.VariantFileSource (BAM + FASTA every rank opens; regions=None)
        records = dvc.buffer.to_host()          # every rank holds the whole job's records after the gather

    `capacity`: the records of this rank's slice of the gather buffer; run() fails if the ranks together could not run every
    group.  `distributed=False` runs the same path on this process alone (world size 1)."""

    def __init__(self, state: dict, device: int, capacity: int, schedule: str = "dynamic", group_regions: int = 32,
                 distributed: bool = True, caller=None):
        from .pipeline import VariantCaller
        super().__init__(VariantCaller, state, device, schedule, group_regions, distributed, caller)
        self._capacity = capacity
        self.groups_done = 0

    def run(self, source, regions, params: dict, seq_off: np.ndarray | None = None, replicas: int = 1) -> int:
        """Returns this rank's candidate count; the gathered records are in self.buffer (device).
        `replicas` > 1 (benchmarks only): the job is `replicas` copies of the region list laid end to end — job group J is local
        group J mod G with region ids shifted by (J div G) * n_regions — so that a weak-scaling run can hand out N x the
        per-GPU block without holding N copies of it."""
        from .abi import HostReads, regions_array
        from .frontend import VariantFileSource
        from .pipeline import DeviceReads
        from_files = isinstance(source, VariantFileSource)
        n_reg = source.n_regions if from_files else regions.n_regions
        plain = plan_groups(n_reg, self.group_regions)
        dynamic = self.schedule == "dynamic" and self.world > 1
        last = plan_groups_tapered(n_reg, self.group_regions, self.world) if dynamic else plain
        # the job: `replicas` copies of the region list; only the last copy is cut into shrinking groups
        job = [(rep, g0, g1) for rep in range(replicas - 1) for (g0, g1) in plain] + [(replicas - 1, g0, g1) for (g0, g1) in last]
        work = None
        if seq_off is not None:
            w_plain, w_last = group_work(seq_off, regions.table, plain), group_work(seq_off, regions.table, last)
            work = np.concatenate([np.tile(w_plain, replicas - 1), w_last])
        n_job = len(job)
        cap = self._gather_buffer(self._capacity, n_job).capacity
        claimer = self._claimer(n_job, work)
        s = self.caller.stream(params, cap, d_records=self.buffer.my_ptr())
        groups = [(g0, g1) for _, g0, g1 in job]
        first = [rep * n_reg + g0 for rep, g0, _ in job]
        stage = None
        if isinstance(source, DeviceReads):
            def stage(j):
                s.stage_device(source, *groups[j], first[j])
        elif not from_files:
            assert isinstance(source, HostReads)
            regs, keep = regions_array(regions)
            ref = np.ascontiguousarray(regions.ref, dtype=np.uint8)

            def stage(j):
                s.stage_host(source, regs, *groups[j], ref, first[j])
        segments = self._run_job(s, claimer, groups, cap, source if from_files else None, stage, first)
        n = s.end()
        self.groups_done = len(segments)
        self._gather(s, n, segments, n_job, "every rank's record capacity (%d)" % cap, "capacity")
        return n


def plan_contig_groups(regions_per_contig: list[int], group: int = 32) -> list[tuple[int, int]]:
    """Groups [g0, g1) of a job whose regions are laid out contig after contig: runs of at most `group` whole regions that never
    cross a contig, so that each group's output belongs to one contig."""
    out, base = [], 0
    for n in regions_per_contig:
        out.extend((base + a, base + b) for a, b in plan_groups(int(n), group))
        base += int(n)
    return out


plan_polish_groups = plan_contig_groups          # the name the polish path first published; callers importing it keep working


class DistributedPolisher(_RankDriver):
    """make_images + call_consensus + stitch of ONE assembly (every contig of a frontend.PolishFileSource) over all ranks of the
    default process group.  Each rank runs a streaming polish session (pipeline.PolishStream) over the groups it claims; the
    stitch kernel writes the consensus bases straight into this rank's slice of one byte gather buffer, and a single all-gather
    of those bytes plus the (group id, bytes) table gives every rank the whole assembly.

        dp = DistributedPolisher(state, local_device, capacity_bytes)
        dp.run(source)                          # source: frontend.PolishFileSource (BAM + FASTA every rank opens)
        seqs = dp.assemble(source)              # {contig: polished sequence}, on every rank

    `capacity_bytes`: this rank's slice of the gather buffer; a rank stops claiming groups when the columns it has encoded (an
    upper bound of its consensus bytes) leave too little room, and run() fails if the ranks together could not run every
    group.  `distributed=False` runs the same path on this process alone (world size 1).

    `qualities=True`: the session writes 2-byte polish.QUAL_RECORD records (base, FASTQ quality byte) in place of bytes, still
    gathered by one all-gather; `capacity_bytes` then counts records (consensus bases) and assemble() returns
    {contig: (sequence, quality string)}.

    `edits=True`: the session also writes its edit events (polish_edits.EDIT_EVENT) into this rank's slice of a second, sparse
    gather buffer of `capacity_events` events, gathered by group like the consensus; `write_edits(source, path)` then writes
    the edits VCF.  A rank whose events overflow makes run() fail on every rank (PB_ERR_CAPACITY, `need_events` set)."""

    _claim_prefix = "pb_polish_claim"

    def __init__(self, state: dict, device: int, capacity_bytes: int, schedule: str = "dynamic", group_regions: int = 32,
                 distributed: bool = True, caller=None, qualities: bool = False, edits: bool = False, capacity_events: int = 0):
        from .pipeline import PolishCaller
        super().__init__(PolishCaller, state, device, schedule, group_regions, distributed, caller)
        self.capacity = int(capacity_bytes)
        self.qualities = bool(qualities)
        self.edits = bool(edits)
        self.capacity_events = int(capacity_events)
        self.edits_buffer = None

    def close(self):
        if self.edits_buffer is not None:
            self.edits_buffer.release()
            self.edits_buffer = None
        super().close()

    def run(self, source) -> int:
        """Returns this rank's consensus bytes (records with qualities); the gathered records of every rank are in self.buffer
        (device)."""
        from .polish import QUAL_RECORD
        groups = source.groups(self.group_regions)
        n_job = len(groups)
        self._gather_buffer(self.capacity, n_job, QUAL_RECORD if self.qualities else np.uint8)
        claimer = self._claimer(n_job, source.group_work(groups))
        d_events = 0
        if self.edits:
            from .polish_edits import EDIT_EVENT
            eb = self.edits_buffer
            if eb is None or eb.max_groups < n_job or eb.capacity != self.capacity_events:
                if eb is not None:
                    eb.release()
                self.edits_buffer = GatherBuffer(self.capacity_events, self.world, self.rank, self.device, max_groups=n_job,
                                                 record=EDIT_EVENT)
            d_events = self.edits_buffer.my_ptr()
        s = self.caller.stream(self.capacity, self.buffer.my_ptr(), qualities=self.qualities, edits=self.edits,
                               capacity_events=self.capacity_events, d_events=d_events)
        from ._lib import PepperB200Error
        segments = self._run_job(s, claimer, groups, self.capacity, source)
        need_events = 0
        try:
            n = s.end()
        except PepperB200Error as ex:
            if not hasattr(ex, "need_events"):
                raise
            # the other ranks still gather: this rank joins with the events that fit, and every rank fails after the gather
            n, need_events = ex.need, ex.need_events
        segments = [(g, int(k)) for (g, _), k in zip(segments, s.group_bytes())]
        self._gather(s, n, segments, n_job, "the consensus capacity (%d bytes per rank)" % self.capacity, "capacity_bytes")
        if self.edits:
            self._gather_events(s, segments, need_events)
        return n

    def _gather_events(self, s, segments: list[tuple[int, int]], need: int):
        """The events of every rank into edits_buffer, ordered by group like the consensus; fails on every rank when one rank's
        events did not fit."""
        import torch
        from ._lib import PepperB200Error
        from .abi import PB_ERR_CAPACITY
        ev_seg = [(g, int(k)) for (g, _), k in zip(segments, s.group_events())]
        ok = need == 0
        self.edits_buffer.gather(sum(k for _, k in ev_seg) if ok else 0, ev_seg if ok else [])
        worst = torch.tensor([need], dtype=torch.int64, device=self.device)
        if self.world > 1:
            import torch.distributed as dist
            dist.all_reduce(worst, op=dist.ReduceOp.MAX)
        need = int(worst.item())
        if need:
            ex = PepperB200Error("edit events overflow: %d events needed on one rank, capacity %d — raise `capacity_events`"
                                 % (need, self.capacity_events), PB_ERR_CAPACITY)
            ex.need_events = need
            raise ex

    def write_edits(self, source, path: str) -> None:
        """The edits VCF of the last run (polish_edits.write_edits_vcf) at `path`, with its index: the gathered events cut at the
        contig boundaries of the plan, turned into lines on the device contig by contig in the order of the polished FASTA, and
        compressed there.  Contigs whose consensus is empty are left out, as the FASTA leaves them out."""
        import torch
        from .frontend import natural_key
        from .polish_edits import events_by_contig, split_events, edits_vcf_device, device_part, write_edits_vcf
        groups = source.groups(self.group_regions)
        group_contig = [source.names[source.contig_of[g0]] for g0, _ in groups]
        seq_len = {c: 0 for c in source.names}
        for g, k in self.buffer.segments():
            seq_len[group_contig[g]] += k
        events = events_by_contig(self.edits_buffer.to_host(), self.edits_buffer.segments(), group_contig, source.names)
        first = dict(zip(source.names, source._first[:-1]))
        last = dict(zip(source.names, source._first[1:]))
        dev = torch.device("cuda", self.device.index)
        parts = []
        for c in sorted(source.names, key=natural_key):
            if not seq_len[c]:
                continue
            span = (source.intervals[first[c]][0], source.intervals[last[c] - 1][1])
            columns, cover = split_events(events[c])
            d_cols = torch.from_numpy(columns.view(np.uint8).reshape(-1)).to(dev)
            d_draft = torch.from_numpy(source.fasta.fetch_array(c, span[0], span[1] + 1)).to(dev)
            text, lines = edits_vcf_device(d_cols, cover, span, d_draft, c, self.device.index)
            parts.append(device_part(c, text, lines, self.device.index))
        write_edits_vcf(path, source.fasta_contigs(), parts)

    def assemble(self, source) -> dict:
        """{contig: polished sequence} of every contig of the source's plan (empty string: nothing survived), on every rank:
        the gathered bytes in group order, cut at the contig boundaries of the plan.  With qualities: {contig: (sequence,
        quality string)}."""
        groups = source.groups(self.group_regions)
        return assemble_contigs(self.buffer.to_host(), self.buffer.segments(), [source.names[source.contig_of[g0]] for g0, _ in groups],
                                source.names)


def assemble_contigs(data: np.ndarray, segments: list[tuple[int, int]], group_contig: list[str], contigs: list[str]) -> dict:
    """Consensus records `data` of the groups of `segments` ((group id, records), sorted by group id, laid out in that order) ->
    {contig: sequence} for every contig of `contigs` (group g belongs to contig group_contig[g]).  Records are bytes, or
    (base, qual) records (polish.QUAL_RECORD), which give {contig: (sequence, quality string)}."""
    spans = {c: [] for c in contigs}
    off = 0
    for g, k in segments:
        spans[group_contig[g]].append((off, off + k))
        off += k

    def cut(plane: bytes) -> dict:
        return {c: b"".join(plane[a:b] for a, b in sp).decode() for c, sp in spans.items()}
    if data.dtype.names is None:
        return cut(data.tobytes())
    seqs, quals = cut(data["base"].tobytes()), cut(data["qual"].tobytes())
    return {c: (seqs[c], quals[c]) for c in contigs}


# ---------------------------------------------------------------------------------------------------------------------------
# Whole-genome variant calling across ranks: BAM + FASTA in, the five indexed VCFs of `pepper_variant call_variant` out.

# the group table every rank publishes: per group [ran, lines, first position, last position, PEPPER lines, variant-calling
# SNP lines, indel lines, class of the first line]
GT_RAN, GT_LINES, GT_FIRST, GT_LAST, GT_PEPPER, GT_SNP, GT_INDEL, GT_FIRST_CLS = range(8)
NO_BOUNDARY = -1


class ListClaimer:
    """Hands out a fixed list of group ids: a rank's share given in advance (GroupClaimer's interface)."""

    def __init__(self, ids):
        self._it = iter([int(g) for g in ids])

    def next(self):
        return next(self._it, None)


class GenomeRankPart:
    """One rank's share of a genome call between the collectives: the groups it ran, the boundary records it held back
    (PRED_RECORD), its VCF text (device) and line table (host, VCF_LINE), each line's group, and the edge lines of the boundaries
    whose later group it owns."""

    def __init__(self):
        self.groups, self.held = [], np.zeros(0, PRED_RECORD)
        self.text, self.lines, self.line_group = None, None, np.zeros(0, np.int64)
        self.edges = {}
        self.meta, self.comp = b"", None
        self.phase_ms = {}
        # gVCF: the track (device) and its groups in run order; the written lines per group after the drops
        self.track, self.track_order, self.ref_table, self.d_ref = None, [], None, None
        self.written, self.all_lines, self.texts = {}, None, []
        self.track_overflow = None          # the message when this rank's gVCF track could not hold a group


def group_table_rows(part: GenomeRankPart, n_groups: int) -> np.ndarray:
    """This rank's rows of the group table (zeros for the groups it did not run), edge lines counted as their later group's
    first line."""
    from .vcf import CLASS_PEPPER, CLASS_VC_SNP, CLASS_VC_INDEL
    t = np.zeros((n_groups, 8), np.int64)
    for g in part.groups:
        pos, cls = group_lines(part, g)
        t[g, GT_RAN] = 1
        t[g, GT_LINES] = pos.shape[0]
        if pos.shape[0]:
            t[g, GT_FIRST], t[g, GT_LAST], t[g, GT_FIRST_CLS] = pos[0], pos[-1], cls[0]
            t[g, GT_PEPPER] = int((cls == CLASS_PEPPER).sum())
            t[g, GT_SNP] = int((cls == CLASS_VC_SNP).sum())
            t[g, GT_INDEL] = int((cls == CLASS_VC_INDEL).sum())
    return t


def group_lines(part: GenomeRankPart, g: int):
    """(positions, classes) of group g's lines in file order: its edge line, then the lines of its own VCF pass."""
    own = part.lines[part.line_group == g] if part.lines is not None else np.zeros(0)
    e = part.edges.get(g)
    pos = np.concatenate([e[1]["pos"] if e else np.zeros(0, np.int64), own["pos"] if own.shape[0] else np.zeros(0, np.int64)])
    cls = np.concatenate([e[1]["cls"] if e else np.zeros(0, np.int32), own["cls"] if own.shape[0] else np.zeros(0, np.int32)])
    return pos.astype(np.int64), cls.astype(np.int32)


def last_position_drops(table: np.ndarray, group_contig: np.ndarray, names: list[str]) -> np.ndarray:
    """Groups whose first line write_vcf_records skips (VcfWriter.py:151-152: `last_position` is never reset, so a contig's first
    line is dropped when its position equals that of the previous line in lexical contig order, whichever rank wrote it)."""
    lex = np.empty(len(names), np.int64)
    lex[np.array(sorted(range(len(names)), key=lambda i: names[i]), dtype=np.int64)] = np.arange(len(names))
    drop = np.zeros(table.shape[0], bool)
    prev = None
    for g in sorted(range(table.shape[0]), key=lambda g: (lex[group_contig[g]], g)):
        if table[g, GT_LINES] == 0:
            continue
        drop[g] = prev is not None and table[g, GT_FIRST] == prev
        prev = table[g, GT_LAST]
    return drop


def genome_totals(table: np.ndarray, drop: np.ndarray) -> tuple[int, int, int, int, int]:
    """The totals of FindCandidates.py:185-189 (all, PEPPER, variant calling, of them SNPs, indels) after the drops."""
    from .vcf import CLASS_PEPPER, CLASS_VC_SNP, CLASS_VC_INDEL
    fc = table[:, GT_FIRST_CLS]
    d = drop.astype(np.int64)
    pep = int(table[:, GT_PEPPER].sum() - (d * (fc == CLASS_PEPPER)).sum())
    snp = int(table[:, GT_SNP].sum() - (d * (fc == CLASS_VC_SNP)).sum())
    indel = int(table[:, GT_INDEL].sum() - (d * (fc == CLASS_VC_INDEL)).sum())
    return int(table[:, GT_LINES].sum() - d.sum()), pep, snp + indel, snp, indel


def parse_rank_bytes(data) -> dict:
    """A rank's gathered bytes (GenomeRankPart.meta + .comp) -> {group id: vcf.GroupPart}."""
    from .vcf import GROUP_LINE, GroupPart, member_cuts, file_masks
    buf = memoryview(np.ascontiguousarray(data, np.uint8))
    if len(buf) == 0:
        return {}
    head = np.frombuffer(buf[:16], np.int64)
    meta_bytes, n_groups = int(head[0]), int(head[1])
    off, coff = 16, meta_bytes
    out = {}
    for _ in range(n_groups):
        h = np.frombuffer(buf[off:off + 56], np.int64)
        off += 56
        g, n_lines, nm = int(h[0]), int(h[1]), [int(x) for x in h[2:7]]
        sizes = np.frombuffer(buf[off:off + 8 * sum(nm)], np.int64).copy()
        off += 8 * sum(nm)
        lines = np.frombuffer(buf[off:off + GROUP_LINE.itemsize * n_lines], GROUP_LINE).copy()
        off += GROUP_LINE.itemsize * n_lines
        us, cs, dat, k = [], [], [], 0
        for f, m in enumerate(file_masks(lines["cls"])):
            cs.append(sizes[k:k + nm[f]]); k += nm[f]
            us.append(member_cuts(int(lines["text_len"][m].astype(np.int64).sum())))
            assert us[-1].shape[0] == nm[f]
            b = int(cs[-1].sum())
            dat.append(bytes(buf[coff:coff + b])); coff += b
        out[g] = GroupPart(lines, us, cs, dat)
    return out


class DistributedGenomeCaller(_RankDriver):
    """`pepper_variant call_variant -b -f -o -s [-r]` of a whole genome over all ranks of the default process group.

        dgc = DistributedGenomeCaller(state, local_device, capacity_bytes)
        totals = dgc.call_genome(bam, fasta, out_dir, "sample")   # rank 0 writes the five PEPPER_VARIANT_*.vcf.gz + .tbi
        dgc.close()                                               # before destroy_process_group()

    Every rank runs one streaming session over the groups it claims (a session takes groups of any contig), then its own VCF
    pass over the session's device buffers with the records at its groups' boundary positions held back.  After the sessions:
    the held-back records are all-gathered and the owner of each boundary's later group writes that boundary's line (edge pass);
    the per-group (lines, first / last position) table is all-gathered and decides the `last_position` drops; each rank lays out
    its lines per file and group and compresses them to BGZF members on its GPU; rank 0 gathers the members + a compact line
    table and writes the files.  Returns the FindCandidates.py:185-189 totals on every rank.

    `capacity_bytes`: the candidate records one rank's session may hold (84 bytes each); run fails when the ranks together could
    not run every group.  `distributed=False` runs alone at world size 1.

    `gvcf=True`: the sessions also fill a track of (n_ref, n_alt) per owned position (4 bytes each, `track_positions` per rank,
    default gvcf.track_capacity); after the drops every rank builds the reference blocks and record lines of its groups on its
    GPU (gvcf_pass) and rank 0 also writes PEPPER_VARIANT.g.vcf.gz, blocks banded by GQ // `gvcf_binsize`."""

    _claim_prefix = "pb_genome_claim"

    def __init__(self, state: dict, device: int, capacity_bytes: int, schedule: str = "dynamic", group_regions: int = 32,
                 distributed: bool = True, caller=None, gvcf: bool = False, gvcf_binsize: int = 5, track_positions: int | None = None):
        from .pipeline import VariantCaller
        super().__init__(VariantCaller, state, device, schedule, group_regions, distributed, caller)
        self.device_id = device
        self.capacity = int(capacity_bytes)
        self.gvcf, self.gvcf_binsize, self.track_positions = bool(gvcf), int(gvcf_binsize), track_positions

    # ---------------------------------------------------------------- per-rank work
    def run_groups(self, src, claimer, params: dict, options: dict | None = None, vcf_options: dict | None = None,
                   world: int | None = None) -> GenomeRankPart:
        """The groups `claimer` hands out through one streaming session, the boundary records held back, and the VCF pass over
        the rest on the device."""
        import time
        import torch
        from .abi import PbCandidateColumns, regions_array, ALLELE_STRIDE
        from .candidates import ONT_OPTIONS
        from .vcf import vcf_text_device, VCF_LINE
        from ._lib import check
        groups = src.groups(self.group_regions)
        bnd = src.boundaries(groups)
        part = GenomeRankPart()
        cap = max(1, self.capacity // RECORD_BYTES)
        t0 = time.perf_counter()
        s = self.caller.stream(params, cap)
        owned = None
        if self.gvcf:
            from .gvcf import track_capacity
            tcap = self.track_positions or track_capacity(sum(e - b + 1 for b, e in src.intervals), world or self.world)
            part.track = torch.empty(max(1, int(tcap)), dtype=torch.int32, device=self.device)
            s.track(int(tcap), part.track.data_ptr())
            ends = owned_ends(src)

            def owned(j):
                return ends[groups[j][0]:groups[j][1]]
        from .pipeline import TrackCapacityError
        try:
            segments = self._run_job(s, claimer, groups, cap, src, world=world, owned=owned)
        except TrackCapacityError as ex:
            # the other ranks learn of it at the first collective (call_source), so that every rank fails there alike
            s.end()
            part.track_overflow = str(ex)
            return part
        n = s.end()
        part.groups = sorted(g for g, _ in segments)
        part.track_order = [g for g, _ in segments]
        part.phase_ms["sessions"] = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        if n > 0:
            cols, d_probs = PbCandidateColumns(), C.c_void_p()
            check(s.L.pb_variant_stream_columns(self.caller.enc.h, C.byref(cols), C.byref(d_probs), None), "columns")
            group_of = np.repeat(np.arange(len(groups)), [g1 - g0 for g0, g1 in groups])
            dev = self.device
            pos = _device_column(cols.positions, (n,), "<i8", dev)
            rof = _device_column(cols.region_of, (n,), "<i4", dev).long()
            gb = torch.from_numpy(bnd).to(dev)[torch.from_numpy(group_of).to(dev)[rof]]
            idx = torch.nonzero((pos == gb[:, 0]) | (pos == gb[:, 1])).squeeze(1)           # arrival order
            held = np.zeros(int(idx.shape[0]), PRED_RECORD)
            if held.shape[0]:
                held["position"] = pos[idx].cpu().numpy()
                held["region"] = rof[idx].cpu().numpy()
                held["depth"] = _device_column(cols.depths, (n,), "|u1", dev)[idx].cpu().numpy()
                held["freq"] = _device_column(cols.freqs, (n,), "|u1", dev)[idx].cpu().numpy()
                keys = _device_column(cols.keys, (n, ALLELE_STRIDE), "|u1", dev)[idx].cpu().numpy()
                held["key"] = np.ascontiguousarray(keys[:, :62]).view("S62")[:, 0]
                held["probs"] = _device_column(d_probs.value, (n, 3), "<f4", dev)[idx].cpu().numpy()
            part.held = held
            regs = [r for g in part.groups for r in range(*groups[g])]
            table = src.table(regs)
            window = np.empty((src.n_regions, 2), np.int64)
            window[:, 0] = np.where(bnd[group_of, 0] >= 0, bnd[group_of, 0] + 1, 0)
            window[:, 1] = np.where(bnd[group_of, 1] >= 0, bnd[group_of, 1] - 1, np.iinfo(np.int64).max)
            d_regions = torch.from_numpy(regions_array(table)[1]).to(dev)
            d_ref = torch.from_numpy(np.ascontiguousarray(table.ref, np.uint8)).to(dev)
            part.ref_table, part.d_ref = table, d_ref
            text, lines = vcf_text_device(src.names, src.contig_of, cols, d_probs.value or 0, n, d_regions.data_ptr(), d_ref.data_ptr(),
                                          options or ONT_OPTIONS, vcf_options, self.device_id, window=window, on_device=True)
            part.text, part.lines = text, lines.cpu().numpy().view(VCF_LINE)
            # a line's group: the first group of its contig whose last interval ends at or after the line
            gkey = np.array([(int(src.contig_of[g0]) << 40) | src.intervals[g1 - 1][1] for g0, g1 in groups], np.int64)
            part.line_group = np.searchsorted(gkey, (part.lines["contig"].astype(np.int64) << 40) | part.lines["pos"], side="left")
        part.phase_ms["vcf_pass"] = (time.perf_counter() - t0) * 1e3
        t = self.caller.timings()
        part.phase_ms["encoder_device"], part.phase_ms["network_device"] = t["encode_ms"], t["network_ms"]
        return part

    def edge_pass(self, part: GenomeRankPart, src, held: np.ndarray, options: dict | None = None, vcf_options: dict | None = None):
        """For each boundary whose later group this rank ran: the VCF pass over the earlier group's held-back records at that
        position followed by the later group's (arrival order within each) -> at most one line, the later group's first."""
        import time
        from .candidates import ONT_OPTIONS
        from .synth import RegionTable
        from .vcf import vcf_text_host
        from .abi import ALLELE_STRIDE
        t0 = time.perf_counter()
        groups = src.groups(self.group_regions)
        bnd = src.boundaries(groups)
        group_of = np.repeat(np.arange(len(groups)), [g1 - g0 for g0, g1 in groups])
        rg = group_of[held["region"]] if held.shape[0] else np.zeros(0, np.int64)
        part.edges = {}
        for g in part.groups:
            b = int(bnd[g, 0])
            if b < 0:
                continue
            sel = np.concatenate([np.flatnonzero((rg == g - 1) & (held["position"] == b)), np.flatnonzero((rg == g) & (held["position"] == b))])
            if sel.shape[0] == 0:
                continue
            rec = held[sel]
            regs = np.unique(rec["region"])
            tab = src.table(regs)
            keys = np.zeros((rec.shape[0], ALLELE_STRIDE), np.uint8)
            keys[:, :62] = np.ascontiguousarray(rec["key"]).view(np.uint8).reshape(-1, 62)
            cid = int(src.contig_of[regs[0]])
            text, lines = vcf_text_host(src.names, np.full(regs.shape[0], cid, np.int32), rec["position"].astype(np.int64),
                                        np.searchsorted(regs, rec["region"]).astype(np.int32), rec["depth"], rec["freq"], keys,
                                        rec["probs"], RegionTable(tab.table[regs], tab.ref), options or ONT_OPTIONS, vcf_options)
            if lines.shape[0]:
                part.edges[g] = (text, lines)
        part.phase_ms["edge"] = (time.perf_counter() - t0) * 1e3

    def compress(self, part: GenomeRankPart, src, table: np.ndarray):
        """Applies the `last_position` drops decided from the whole group table, lays out every file's lines per group on the
        device and compresses them to BGZF members (part.meta: the compact line table and member sizes; part.comp: the
        members, device).  Returns the totals."""
        import time
        import torch
        from .vcf import VCF_LINE, file_masks, member_cuts, group_line_table, gather_lines_device, bgzf_compress_device
        t0 = time.perf_counter()
        groups = src.groups(self.group_regions)
        group_contig = np.array([int(src.contig_of[g0]) for g0, _ in groups], np.int64)
        drop = last_position_drops(table, group_contig, src.names)
        totals = genome_totals(table, drop)
        # one text and line table: the VCF pass's, then the edge lines
        texts = [part.text] if part.text is not None else []
        tabs = [part.lines] if part.lines is not None else []
        base = int(part.text.shape[0]) if part.text is not None else 0
        edge_row = {}
        nrow = sum(t.shape[0] for t in tabs)
        for g, (text, lines) in sorted(part.edges.items()):
            t = lines.copy()
            t["text_off"] += base
            base += text.shape[0]
            texts.append(torch.from_numpy(text).to(self.device)); tabs.append(t)
            edge_row[g] = np.arange(nrow, nrow + t.shape[0]); nrow += t.shape[0]
        all_lines = np.concatenate(tabs) if tabs else np.zeros(0, VCF_LINE)
        sel, dst, member_off, meta = [], [], [0], [np.zeros(2, np.int64).tobytes()]
        pay = 0
        for g in part.groups:
            rows = np.concatenate([edge_row.get(g, np.zeros(0, np.int64)),
                                   np.flatnonzero(part.line_group == g) if part.lines is not None else np.zeros(0, np.int64)]).astype(np.int64)
            if drop[g]:
                rows = rows[1:]
            part.written[g] = rows
            gl = all_lines[rows]
            nm = []
            for m in file_masks(gl["cls"]):
                r = rows[m]
                ln = all_lines["text_len"][r].astype(np.int64)
                sel.append(r); dst.append(pay + np.concatenate([[0], np.cumsum(ln)[:-1]]) if r.shape[0] else np.zeros(0, np.int64))
                cuts = member_cuts(int(ln.sum()))
                member_off.extend((pay + np.cumsum(cuts)).tolist())
                pay += int(ln.sum())
                nm.append(cuts.shape[0])
            meta.append(np.array([g, gl.shape[0]] + nm, np.int64).tobytes())
            meta.append(None)                        # member sizes, filled in after the compression
            meta.append(group_line_table(gl).tobytes())
        part.all_lines, part.texts = all_lines, texts
        payload = torch.empty(max(1, pay), dtype=torch.uint8, device=self.device)
        if pay:
            text_all = torch.cat(texts) if len(texts) > 1 else texts[0]
            d_lines = torch.from_numpy(all_lines.view(np.uint8).reshape(-1)).to(self.device)
            gather_lines_device(text_all, d_lines, np.concatenate(sel), np.concatenate(dst), payload, self.device_id)
        t1 = time.perf_counter()
        comp, sizes = bgzf_compress_device(payload, np.array(member_off, np.int64), self.device_id)
        torch.cuda.synchronize(self.device)
        part.phase_ms["compress"] = (time.perf_counter() - t1) * 1e3
        part.phase_ms["layout"] = (t1 - t0) * 1e3
        k = 0
        for i in range(len(meta)):
            if meta[i] is None:
                nm = np.frombuffer(meta[i - 1], np.int64)[2:7]
                meta[i] = sizes[k:k + int(nm.sum())].tobytes()
                k += int(nm.sum())
        body = b"".join(meta)
        body = np.frombuffer(np.array([len(body), len(part.groups)], np.int64).tobytes() + body[16:], np.uint8).copy()
        part.meta, part.comp = body, comp
        part.payload_bytes = pay
        return totals

    # ---------------------------------------------------------------- the collectives
    def _all_gather_object(self, obj) -> list:
        if self.world == 1:
            return [obj]
        import torch.distributed as dist
        out = [None] * self.world
        dist.all_gather_object(out, obj)
        return out

    def _gather_bytes(self, part: GenomeRankPart, meta=None, comp=None) -> list | None:
        """Every rank's meta + members (part.meta / part.comp unless given) into one byte GatherBuffer (one all-gather); rank 0
        gets each rank's bytes."""
        import torch
        meta = part.meta if meta is None else meta
        comp = part.comp if comp is None else comp
        mine = int(meta.shape[0]) + int(comp.shape[0])
        cap = max(x for x in self._all_gather_object(mine))
        buf = GatherBuffer(max(1, cap), self.world, self.rank, self.device, record=np.uint8)
        try:
            sl = buf.my_slice()
            sl[:meta.shape[0]].copy_(torch.from_numpy(meta))
            sl[meta.shape[0]:mine].copy_(comp)
            buf.gather(mine)
            torch.cuda.synchronize(self.device)
            if self.rank != 0:
                return None
            counts = buf.meta[:, 0].cpu().numpy()
            return [buf.records[r * buf.slice_bytes:r * buf.slice_bytes + int(counts[r])].cpu().numpy() for r in range(self.world)]
        finally:
            buf.release()

    def call_genome(self, bam: str, fasta: str, out_dir: str, sample_name: str, region: str | None = None, exclude=(),
                    params: dict | None = None, options: dict | None = None, vcf_options: dict | None = None,
                    interval_size: int = 100_000, gpu_inflate: bool = True) -> tuple:
        """Rank 0 writes the five PEPPER_VARIANT_*.vcf.gz (and, with gvcf=True, PEPPER_VARIANT.g.vcf.gz) under out_dir."""
        from .frontend import VariantGenomeSource
        from .synth import ont_params
        params = params or ont_params()
        src = VariantGenomeSource(bam, fasta, int(params["min_snp_baseq"]), region, exclude, interval_size, self.device_id,
                                  gpu_inflate=gpu_inflate)
        try:
            return self.call_source(src, out_dir, sample_name, params, options, vcf_options)
        finally:
            src.close()

    def call_source(self, src, out_dir: str, sample_name: str, params: dict, options: dict | None = None,
                    vcf_options: dict | None = None) -> tuple:
        """call_genome over a read source the caller opened (frontend.VariantGenomeSource, with its own get_reads filters and
        BAM threads); every rank passes a source of the same job.  The source stays open."""
        import time
        from .vcf import write_vcfs_from_parts
        groups = src.groups(self.group_regions)
        part = self.run_groups(src, self._claimer(len(groups), src.group_work(groups)), params, options, vcf_options)
        t0 = time.perf_counter()
        held = self._all_gather_object((part.held, part.track_overflow))
        over = [(r, m) for r, (_, m) in enumerate(held) if m is not None]
        if over:
            from .pipeline import TrackCapacityError
            from .abi import PB_ERR_CAPACITY
            raise TrackCapacityError("rank %d: %s" % over[0], PB_ERR_CAPACITY)
        held = [h for h, _ in held]
        held = np.concatenate(held) if held else np.zeros(0, PRED_RECORD)
        part.phase_ms["edge_exchange"] = (time.perf_counter() - t0) * 1e3
        self.edge_pass(part, src, held, options, vcf_options)
        table = sum(self._all_gather_object(group_table_rows(part, len(groups))))
        check_groups_ran(int(table[:, GT_RAN].sum()), len(groups), "the session capacity (%d bytes per rank)" % self.capacity,
                         "capacity_bytes")
        totals = self.compress(part, src, table)
        t0 = time.perf_counter()
        got = self._gather_bytes(part)
        part.phase_ms["gather"] = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        if got is not None:
            parts = {}
            for data in got:
                parts.update(parse_rank_bytes(data))
            write_vcfs_from_parts(out_dir, sample_name, src.fasta_contigs(), src.names,
                                  [int(src.contig_of[g0]) for g0, _ in groups], parts)
        part.phase_ms["write"] = (time.perf_counter() - t0) * 1e3
        if self.gvcf:
            self._call_gvcf(part, src, out_dir, sample_name)
        part.phase_ms["groups"] = len(part.groups)
        self.phase_ms = {k: round(v, 2) for k, v in part.phase_ms.items()}
        self.payload_bytes, self.member_bytes = part.payload_bytes, int(part.comp.shape[0])
        return totals

    # ---------------------------------------------------------------- gVCF
    def _call_gvcf(self, part: GenomeRankPart, src, out_dir: str, sample_name: str):
        import time
        import torch
        from .gvcf import parse_gvcf_bytes, write_gvcf_from_parts
        groups = src.groups(self.group_regions)
        t0 = time.perf_counter()
        # each group's largest written record end (-1: none), then the running maximum of the earlier groups of its contig
        mine = np.full(len(groups), -1, np.int64)
        for g, rows in part.written.items():
            if rows.shape[0]:
                mine[g] = int((part.all_lines["pos"][rows] + part.all_lines["ref_len"][rows]).max())
        ends = np.maximum.reduce(self._all_gather_object(mine))
        part.phase_ms["gvcf_exchange"] = (time.perf_counter() - t0) * 1e3
        meta, comp = self.gvcf_pass(part, src, mask_until(ends, [int(src.contig_of[g0]) for g0, _ in groups]))
        t0 = time.perf_counter()
        # the members are on the host: one rank keeps them there, several all-gather them through their GPUs
        got = [np.concatenate([meta, comp])] if self.world == 1 else self._gather_bytes(part, meta, torch.from_numpy(comp))
        part.phase_ms["gvcf_gather"] = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        if got is not None:
            parts = {}
            for data in got:
                parts.update(parse_gvcf_bytes(data))
            write_gvcf_from_parts(out_dir, sample_name, src.fasta_contigs(), src.names, [int(src.contig_of[g0]) for g0, _ in groups],
                                  parts)
        part.phase_ms["gvcf_write"] = (time.perf_counter() - t0) * 1e3

    def gvcf_pass(self, part: GenomeRankPart, src, until: np.ndarray, batch_positions: int = GVCF_BATCH):
        """This rank's gVCF lines, in batches of whole groups of about `batch_positions` track positions (run order): per batch,
        the reference blocks of its track slice (positions inside a written record's span, or before `until[g]` of group g, are
        masked) and its written FULL lines with the <*> allele, merged by position per group, laid out on the device and
        compressed to BGZF members, which go to the host before the next batch.  Device memory beyond the track is bounded by
        the batch.  Returns (meta bytes, members) for the byte gather, both host arrays."""
        import time
        import torch
        from .gvcf import GVCF_SEGMENT, GVCF_LINE, gvcf_blocks_device, gvcf_records_device
        from .vcf import VCF_LINE, member_cuts, gather_lines_device, bgzf_compress_device
        groups = src.groups(self.group_regions)
        ends = owned_ends(src)
        regs = [r for g in part.track_order for r in range(*groups[g])]
        if part.ref_table is None and regs:
            part.ref_table = src.table(regs)
            part.d_ref = torch.from_numpy(np.ascontiguousarray(part.ref_table.ref, np.uint8)).to(self.device)
        gstart = np.array([(int(src.contig_of[g0]) << 40) | src.intervals[g0][0] for g0, _ in groups], np.int64)
        text_all = None
        if part.texts:
            text_all = torch.cat(part.texts) if len(part.texts) > 1 else part.texts[0]
        ms = dict(gvcf_blocks=0.0, gvcf_records=0.0, gvcf_merge_host=0.0, gvcf_layout=0.0, gvcf_compress=0.0)
        stats = dict(track_bytes=0, block_lines=0, record_lines=0, payload_bytes=0, compressed_bytes=0)
        heads, comps = [], []

        def flush(batch, t0):
            n = sum(t for _, t in batch)
            seg, masks, rec_rows, toff_g, t = [], [], [], {}, 0
            for g, _ in batch:
                g0, g1 = groups[g]
                p0, p1 = src.intervals[g0][0], int(ends[g1 - 1])
                toff_g[g] = t
                for r in range(g0, g1):
                    s0 = src.intervals[r][0]
                    row = part.ref_table.table[r]
                    seg.append((t, s0, int(ends[r]) - s0 + 1, int(row[4]) + s0 - int(row[0]), int(src.contig_of[r]), 0))
                    t += int(ends[r]) - s0 + 1
                rows = part.written.get(g, np.zeros(0, np.int64))
                rec_rows.append(rows)
                if until[g] > p0:
                    masks.append(np.array([[toff_g[g], toff_g[g] + min(int(until[g]), p1 + 1) - p0]], np.int64))
                if rows.shape[0]:
                    pos = part.all_lines["pos"][rows].astype(np.int64)
                    end = np.minimum(pos + part.all_lines["ref_len"][rows], p1 + 1)
                    masks.append(np.stack([toff_g[g] + pos - p0, toff_g[g] + end - p0], 1))
            seg = np.array(seg, GVCF_SEGMENT)
            masks = np.concatenate(masks) if masks else np.zeros((0, 2), np.int64)
            t1 = time.perf_counter()
            btext, blines = gvcf_blocks_device(part.track[t0:t0 + n], n, seg, masks, part.d_ref.data_ptr(), src.names,
                                               self.gvcf_binsize, self.device_id)
            t2 = time.perf_counter()
            rows = np.concatenate(rec_rows)
            if rows.shape[0]:
                rtext, rlines = gvcf_records_device(text_all, part.all_lines[rows], self.device_id)
            else:
                rtext, rlines = None, np.zeros(0, VCF_LINE)
            torch.cuda.synchronize(self.device)
            t3 = time.perf_counter()
            # merge: each line's group (blocks by position: the last group of the contig starting at or before it; records by
            # their rows), then position order inside each group, laid out back to back
            nb = blines.shape[0]
            lines = np.concatenate([blines, rlines])
            bgroup = np.searchsorted(gstart, (blines["contig"].astype(np.int64) << 40) | blines["pos"], side="right") - 1
            rgroup = np.repeat(np.array([g for g, _ in batch], np.int64), [r.shape[0] for r in rec_rows])
            lgroup = np.concatenate([bgroup, rgroup]).astype(np.int64)
            order = np.lexsort((lines["pos"], lgroup))
            ln = lines["text_len"].astype(np.int64)[order]
            dst = np.concatenate([[0], np.cumsum(ln)[:-1]]) if order.shape[0] else np.zeros(0, np.int64)
            ids = sorted(g for g, _ in batch)
            bounds = np.searchsorted(lgroup[order], np.array(ids + [np.iinfo(np.int64).max]), side="left")
            member_off, pay, batch_heads = [0], 0, []
            for i, g in enumerate(ids):
                sel = order[bounds[i]:bounds[i + 1]]
                nbytes = int(ln[bounds[i]:bounds[i + 1]].sum())
                cuts = member_cuts(nbytes)
                member_off.extend((pay + np.cumsum(cuts)).tolist())
                pay += nbytes
                gl = np.zeros(sel.shape[0], GVCF_LINE)
                gl["pos"], gl["end"], gl["text_len"] = lines["pos"][sel], lines["pos"][sel] + lines["ref_len"][sel], lines["text_len"][sel]
                batch_heads.append((g, gl, cuts))
            t4 = time.perf_counter()
            payload = torch.empty(max(1, pay), dtype=torch.uint8, device=self.device)
            isb = order < nb
            for mine, text, tab, shift in ((isb, btext, blines, 0), (~isb, rtext, rlines, nb)):
                if mine.any():
                    d_lines = torch.from_numpy(np.ascontiguousarray(tab).view(np.uint8).reshape(-1)).to(self.device)
                    gather_lines_device(text, d_lines, order[mine] - shift, dst[mine], payload, self.device_id)
            torch.cuda.synchronize(self.device)
            t5 = time.perf_counter()
            comp, sizes = bgzf_compress_device(payload, np.array(member_off, np.int64), self.device_id)
            comps.append(comp.cpu().numpy())
            t6 = time.perf_counter()
            k = 0
            for g, gl, cuts in batch_heads:
                heads.append((g, gl, cuts, sizes[k:k + cuts.shape[0]]))
                k += cuts.shape[0]
            ms["gvcf_blocks"] += (t2 - t1) * 1e3; ms["gvcf_records"] += (t3 - t2) * 1e3; ms["gvcf_merge_host"] += (t4 - t3) * 1e3
            ms["gvcf_layout"] += (t5 - t4) * 1e3; ms["gvcf_compress"] += (t6 - t5) * 1e3
            stats["track_bytes"] += 4 * n; stats["block_lines"] += nb; stats["record_lines"] += int(rlines.shape[0])
            stats["payload_bytes"] += pay; stats["compressed_bytes"] += int(comps[-1].shape[0])

        batch, t0, tb = [], 0, 0
        for g in part.track_order:
            g0, g1 = groups[g]
            n = int(ends[g1 - 1]) - src.intervals[g0][0] + 1
            batch.append((g, n))
            tb += n
            if tb >= batch_positions:
                flush(batch, t0)
                t0, batch, tb = t0 + tb, [], 0
        if batch:
            flush(batch, t0)
        meta = []
        for g, gl, cuts, sz in heads:
            meta += [np.array([g, gl.shape[0], cuts.shape[0]], np.int64).tobytes(), cuts.astype(np.int64).tobytes(),
                     sz.astype(np.int64).tobytes(), gl.tobytes()]
        body = b"".join(meta)
        meta = np.frombuffer(np.array([16 + len(body), len(heads)], np.int64).tobytes() + body, np.uint8).copy()
        part.phase_ms.update(ms)
        self.gvcf_stats = stats
        return meta, (np.concatenate(comps) if comps else np.zeros(0, np.uint8))


def owned_ends(src) -> np.ndarray:
    """The last position each interval owns: e - 1 for (s, e), e for the last interval of its contig's span."""
    ends = np.array([e - 1 for _, e in src.intervals], np.int64)
    first = np.array(src._first, np.int64)
    ends[(first[1:] - 1)[np.diff(first) > 0]] += 1
    return ends


def mask_until(ends: np.ndarray, group_contig: list[int]) -> np.ndarray:
    """Per group: the largest written record end (exclusive) of the earlier groups of its contig (-1 when none)."""
    out = np.full(len(group_contig), -1, np.int64)
    run, prev = -1, None
    for g, c in enumerate(group_contig):
        if c != prev:
            run, prev = -1, c
        out[g] = run
        run = max(run, int(ends[g]))
    return out


def _device_column(ptr: int, shape: tuple, typestr: str, device):
    """A torch view of a device array the library owns (valid while the session's buffers are)."""
    import torch

    class _A:
        pass
    a = _A()
    a.__cuda_array_interface__ = dict(shape=shape, typestr=typestr, data=(int(ptr), False), version=3)
    return torch.as_tensor(a, device=device)
