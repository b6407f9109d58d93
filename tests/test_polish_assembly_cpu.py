"""CPU: the host side of whole-assembly polishing — the job plan (contigs common to BAM and FASTA in natural order, tiling,
groups of whole regions that never cross a contig), the polished FASTA against the reference's perform_stitch output
(tests/golden/polish_fasta_seed5.npz, made by make_golden_polish_fasta.py from the unmodified reference), and the gather of
per-group consensus bytes over a gloo world of 2 under a scrambled dynamic claim order."""
import os
import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import stitch as ostitch
from pepper_b200.dist import GatherBuffer, GroupClaimer, assemble_contigs, plan_contig_groups
from pepper_b200.frontend import natural_key, polish_intervals, polish_job, polished_fasta_text

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "polish_fasta_seed5.npz")


def _golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def test_natural_order_and_job_plan():
    assert sorted(["ctg10", "ctg2", "chrX", "ctg1"], key=natural_key) == ["chrX", "ctg1", "ctg2", "ctg10"]
    fasta = [("ctg10", 5000), ("ctg2", 2500), ("onlyfa", 3000), ("chrX", 1201), ("tiny", 1)]
    bam = ["tiny", "onlybam", "chrX", "ctg2", "ctg10"]
    contigs, regions, first = polish_job(fasta, bam)
    assert contigs == ["chrX", "ctg2", "ctg10", "tiny"]                 # common contigs only, natural order
    lengths = dict(fasta)
    for k, c in enumerate(contigs):
        assert regions[first[k]:first[k + 1]] == polish_intervals(0, lengths[c] - 1)
    assert first[-1] == len(regions) and first[3] == first[4]           # a 1-base contig is not tiled
    assert polish_intervals(0, 0) == []
    assert regions[:2] == [(0, 1100), (900, 1200)]
    # a given contig list is taken as given
    assert polish_job(fasta, bam, ["ctg10", "onlyfa"])[0] == ["ctg10", "onlyfa"]


def test_groups_never_cross_contigs():
    per_contig = [3, 1, 0, 70, 5]
    groups = plan_contig_groups(per_contig, 32)
    bounds = np.cumsum([0] + per_contig)
    assert groups[0][0] == 0 and groups[-1][1] == bounds[-1] and all(a[1] == b[0] for a, b in zip(groups, groups[1:]))
    for g0, g1 in groups:
        k = int(np.searchsorted(bounds, g0, side="right")) - 1
        assert bounds[k] <= g0 < g1 <= bounds[k + 1] and g1 - g0 <= 32
    assert plan_contig_groups(per_contig, 1) == [(r, r + 1) for r in range(bounds[-1])]


def _oracle_group_bytes(z, regions):
    """oracle/stitch.py over the images of some regions of one contig."""
    sel = np.isin(z["image_region"], regions)
    reg = z["image_region"][sel]
    local = np.searchsorted(np.array(sorted(regions)), reg)
    rs = [int(z["region_starts"][r]) for r in sorted(regions)]
    re_ = [int(z["region_ends"][r]) for r in sorted(regions)]
    return ostitch.stitch(z["bases"][sel], z["position"][sel], z["index"][sel], local, z["chunk_id"][sel], rs, re_)


def test_fasta_from_oracle_stitch_equals_reference_perform_stitch():
    z = _golden()
    contigs = [str(c) for c in z["contigs"]]
    assert sorted(contigs, key=natural_key) == contigs and sorted(contigs) != contigs
    assert int(z["chunk_id"].max()) >= 10
    seqs = {}
    for k, c in enumerate(contigs):
        seqs[c] = _oracle_group_bytes(z, np.nonzero(z["region_contig"] == k)[0].tolist())
    assert seqs["ctg7"] == "" and ">ctg7" not in str(z["fasta"])
    assert polished_fasta_text(seqs) == str(z["fasta"])
    # per-region stitches concatenated in region order give the same contigs
    for k, c in enumerate(contigs):
        regs = np.nonzero(z["region_contig"] == k)[0].tolist()
        assert "".join(_oracle_group_bytes(z, [r]) for r in regs) == seqs[c]


def test_write_polished_fasta(tmp_path):
    from pepper_b200.frontend import write_polished_fasta
    p = str(tmp_path / "asm.fa")
    write_polished_fasta(p, {"ctg10": "AC", "ctg2": "G", "empty": "", "chrX": "TTT"})
    assert open(p).read() == ">chrX\nTTT\n>ctg2\nG\n>ctg10\nAC\n"


def _worker(rank, world, port, q):
    import random
    import time
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    z = _golden()
    contigs = [str(c) for c in z["contigs"]]
    per_contig = [int((z["region_contig"] == k).sum()) for k in range(len(contigs))]
    groups = plan_contig_groups(per_contig, 1)
    group_contig = [contigs[int(z["region_contig"][g0])] for g0, _ in groups]
    buf = GatherBuffer(40000, world, rank, max_groups=len(groups), record=np.uint8)
    c = GroupClaimer(len(groups), rank, world, "dynamic", key="polish")
    rnd = random.Random(rank)
    off, segments = 0, []
    while (g := c.next()) is not None:
        time.sleep(rnd.random() * 0.05)                      # scrambles which rank takes which group
        b = _oracle_group_bytes(z, list(range(*groups[g]))).encode()
        buf.my_slice()[off:off + len(b)] = torch.from_numpy(np.frombuffer(b, np.uint8).copy())
        off += len(b)
        segments.append((g, len(b)))
    buf.gather(off, segments)
    seqs = assemble_contigs(buf.to_host(), buf.segments(), group_contig, contigs)
    q.put((rank, [g for g, _ in segments], polished_fasta_text(seqs)))
    dist.destroy_process_group()


def test_byte_segments_gather_gloo_world2():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000) + 7
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    z = _golden()
    claimed = sorted(res[0][1] + res[1][1])
    assert claimed == list(range(len(z["region_starts"])))          # every group exactly once
    assert res[0][1] and res[1][1]
    for _, _, text in res:
        assert text == str(z["fasta"])
