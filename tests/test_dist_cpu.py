"""CPU, world_size 2 over gloo: the host-side logic of the multi-GPU path (pepper_b200/dist.py) — group planning and static
sharding, the dynamic group claimer over the rendezvous store, the fixed-capacity in-place all-gather of 84-byte prediction
records with ragged counts, and the restoration of genomic order from the region ids."""
import os
import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from pepper_b200.abi import PRED_RECORD
from pepper_b200.dist import shard_regions, plan_groups, plan_groups_tapered, group_work, GroupClaimer, GatherBuffer, order_records, records_from_calls


def test_shard_regions_contiguous_and_balanced():
    rng = np.random.default_rng(0)
    work = rng.integers(1000, 5000, size=37)
    for world in (1, 2, 4, 8):
        blocks = shard_regions(work, world)
        assert blocks[0][0] == 0 and blocks[-1][1] == 37
        assert all(blocks[i][1] == blocks[i + 1][0] for i in range(world - 1))
        loads = [work[b:e].sum() for b, e in blocks]
        assert max(loads) <= work.sum() / world + work.max()
    assert shard_regions(np.zeros(0), 4) == [(0, 0)] * 4
    assert shard_regions(np.array([5, 5]), 4)[-1][1] == 2


def test_plan_groups_and_work():
    g = plan_groups(70, 32)
    assert g == [(0, 32), (32, 64), (64, 70)]
    assert plan_groups(0, 32) == []
    t = plan_groups_tapered(645, 32, 8)
    assert t[0] == (0, 32) and t[-1][1] == 645 and all(a[1] == b[0] for a, b in zip(t, t[1:]))
    sizes = [b - a for a, b in t]
    assert sizes == sorted(sizes, reverse=True) and sizes[-1] <= 8 and max(sizes) == 32        # shrinking tail
    assert plan_groups_tapered(10, 32, 2) == [(0, 4), (4, 8), (8, 10)]
    # 70 regions with 3 reads each, read i has i+1 bases
    table = np.zeros((70, 8), np.int64)
    table[:, 6] = np.arange(70) * 3
    table[:, 7] = table[:, 6] + 3
    seq_off = np.concatenate([[0], np.cumsum(np.arange(1, 211))])
    w = group_work(seq_off, table, g)
    assert w.sum() == seq_off[-1] and w[0] == seq_off[96]


def test_static_claimer_blocks():
    work = np.array([10, 10, 10, 10, 40, 40])
    got = []
    for r in range(2):
        c = GroupClaimer(6, r, 2, "static", work)
        mine = []
        while (g := c.next()) is not None:
            mine.append(g)
        got.append(mine)
    assert got[0] + got[1] == list(range(6)) and got[0] and got[1]


def test_capacity_stop_is_an_error_under_any_schedule():
    """run_claimed stops claiming when this rank's slice could not hold another group, under the static schedule and at world
    size 1 too; the meta table then lists fewer groups than the job has, and that is a capacity error, not a short result."""
    import pytest
    from pepper_b200._lib import PepperB200Error
    from pepper_b200.abi import PB_ERR_CAPACITY
    from pepper_b200.dist import check_groups_ran, run_claimed

    class Session:                                       # 100 records per group
        total = 0

        def run(self, flush=False):
            self.total += 100
            return self.total
    segments = run_claimed(Session(), GroupClaimer(10, 0, 1, "static"), lambda j: None, None, 1, 500, 10, 1)
    assert segments == [(0, 100), (1, 100), (2, 100), (3, 100)]
    buf = GatherBuffer(500, 1, 0, max_groups=10)
    buf.gather(400, segments)
    assert buf.segments() == segments
    with pytest.raises(PepperB200Error, match="groups were run") as ei:
        check_groups_ran(len(buf.segments()), 10, "the record capacity (500)", "capacity")
    assert ei.value.rc == PB_ERR_CAPACITY
    check_groups_ran(10, 10, "the record capacity (500)", "capacity")


def test_order_and_records_from_calls():
    class Calls:
        pass
    c = Calls()
    n = 7
    c.probs = np.arange(n * 3, dtype=np.float32).reshape(n, 3)
    c.positions = np.arange(n, dtype=np.int64) * 10
    c.region_of = np.array([2, 2, 0, 0, 1, 1, 1], np.int32)
    c.depths = np.arange(n, dtype=np.uint8)
    c.freqs = np.arange(n, dtype=np.uint8) + 1
    c.keys_raw = np.zeros((n, 64), np.uint8)
    for i in range(n):
        k = ("1" + "ACGT"[i % 4]).encode()
        c.keys_raw[i, :len(k)] = np.frombuffer(k, np.uint8)
    c.__class__.__len__ = lambda self: n
    rec = records_from_calls(c)
    assert rec.dtype == PRED_RECORD and rec["key"][2] == b"1G" and rec["position"][3] == 30
    o = order_records(rec)
    assert o["region"].tolist() == [0, 0, 1, 1, 1, 2, 2] and o["position"].tolist() == [20, 30, 40, 50, 60, 0, 10]
    assert order_records(o) is o


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    # dynamic claiming: every group exactly once over the two ranks
    c = GroupClaimer(25, rank, world, "dynamic", key="t1")
    mine = []
    while (g := c.next()) is not None:
        mine.append(g)
    # fixed-capacity gather with ragged counts: rank r contributes 5 + 3 r records of regions it "claimed"
    n = 5 + 3 * rank
    buf = GatherBuffer(16, world, rank)
    rec = np.zeros(n, PRED_RECORD)
    rec["region"] = np.arange(n) * world + rank          # interleaved region ids, as a dynamic schedule produces them
    rec["position"] = 1000 * rank + np.arange(n)
    rec["probs"][:, 0] = rank
    rec["key"] = b"2AC"
    buf.my_slice()[:n * PRED_RECORD.itemsize] = torch.from_numpy(rec.view(np.uint8))
    buf.gather(n)
    out = buf.to_host().copy()
    raw = buf.to_host(order=False).copy()
    q.put((rank, mine, out, raw, buf.counts.tolist()))
    dist.destroy_process_group()


def test_claimer_and_record_gather_gloo_world2():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    claimed = sorted(res[0][1] + res[1][1])
    assert claimed == list(range(25))
    for rank, mine, out, raw, counts in res:
        assert counts == [5, 8]
        assert raw["region"].tolist() == [0, 2, 4, 6, 8] + [1, 3, 5, 7, 9, 11, 13, 15]         # rank-major
        assert out["region"].tolist() == sorted(raw["region"].tolist())                          # genomic order restored
        assert np.all(out["key"] == b"2AC")
        r1 = out[out["probs"][:, 0] == 1]
        assert r1["position"].tolist() == list(range(1000, 1008))
    assert np.array_equal(res[0][2], res[1][2])                                                   # every rank holds the same job result
