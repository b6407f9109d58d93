"""GPU: polished FASTQ — the quality of every consensus base carried through the device stitch, the streaming session's sink
and the all-gather.

1. The one-shot stitch with qualities (pb_polish_stitch_qual_host) equals the quality oracle (tests/stitch_quality_oracle.py) on
   the golden and many-chunk inputs with phred 0..100, and its sequence is byte-identical to the plain stitch.
2. The stitch-to-sink kernel with qualities, fed 1, 7 or all images per call, equals the oracle on polish_fasta_seed5.npz with
   synthetic phred, with the per-region record counts of the plain sink.
3. From BAM + FASTA: polish_assembly(fastq=True) has the sequences of polish_assembly(), the qualities of the oracle over the
   phred of polish_contig, and writes FASTQ that reads back to the same records; a too-small sink restarts to the same result.
4. Two ranks (skipped below 2 GPUs): DistributedPolisher(qualities=True) gives the 1-rank records on both ranks under both
   schedules; every group runs once."""
import os
import numpy as np
import pytest

from pepper_b200 import synth, synth_files
from tests.stitch_quality_oracle import stitch_with_qualities as oracle_stitch_q
from tests.test_stitch import _many_chunks

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _load(name):
    with np.load(os.path.join(HERE, "golden", name)) as z:
        return {k: z[k] for k in z.files}


def _phred(shape, seed):
    """Random phred over the network's whole range, with 94..100 (clamped to '~') in every image."""
    ph = np.random.default_rng(seed).integers(0, 101, shape).astype(np.uint8)
    ph[:, :20] = np.arange(81, 101, dtype=np.uint8)
    return ph


def test_stitch_with_qualities_equals_oracle():
    from pepper_b200.polish import stitch, stitch_with_qualities
    g = _load("stitch_seed11.npz")
    ph = _phred(g["bases"].shape, 1)
    args = (g["position"], g["index"], g["image_region"], g["chunk_id"])
    got = stitch_with_qualities(g["bases"], ph, *args, g["region_starts"])
    assert got == oracle_stitch_q(g["bases"], ph, *args, g["region_starts"], g["region_ends"])
    assert got[0] == str(g["consensus"]) == stitch(g["bases"], *args, g["region_starts"])
    imgs = _many_chunks(5)
    b = np.stack([i[4] for i in imgs]); p = np.stack([i[2] for i in imgs]); x = np.stack([i[3] for i in imgs])
    r = np.zeros(len(imgs), np.int32); c = np.arange(len(imgs), dtype=np.int32)
    ph = _phred(b.shape, 2)
    got = stitch_with_qualities(b, ph, p, x, r, c, [300])
    assert got == oracle_stitch_q(b, ph, p, x, r, c, [300], [9299])
    assert got[0] == stitch(b, p, x, r, c, [300]) and len(got[1]) == len(got[0]) > 5000
    assert "~" in got[1] and max(got[1]) == "~"


def test_stitch_sink_with_qualities_at_any_chunk_size():
    from pepper_b200.polish import stitch_sink_test
    g = _load("polish_fasta_seed5.npz")
    ph = _phred(g["bases"].shape, 3)
    contigs = [str(c) for c in g["contigs"]]
    want = {}
    for k, c in enumerate(contigs):
        regs = np.nonzero(g["region_contig"] == k)[0]
        sel = np.isin(g["image_region"], regs)
        want[c] = oracle_stitch_q(g["bases"][sel], ph[sel], g["position"][sel], g["index"][sel],
                                  np.searchsorted(regs, g["image_region"][sel]), g["chunk_id"][sel], g["region_starts"][regs],
                                  g["region_ends"][regs])
    n = g["bases"].shape[0]
    args = (g["bases"], g["position"], g["index"], g["image_region"], g["chunk_id"], g["region_starts"])
    for chunk in (1, 7, n):
        (seq, qual), per_region = stitch_sink_test(*args, chunk, phred=ph)
        plain, plain_per_region = stitch_sink_test(*args, chunk)
        assert seq == plain and np.array_equal(per_region, plain_per_region), chunk
        got, off = {}, 0
        for k, c in enumerate(contigs):
            m = int(per_region[g["region_contig"] == k].sum())
            got[c] = (seq[off:off + m], qual[off:off + m])
            off += m
        assert got == want, chunk


@pytest.fixture(scope="module")
def assembly_files(tmp_path_factory):
    d = tmp_path_factory.mktemp("asmq")
    genomes, recs = {}, {}
    for k, (name, length) in enumerate([("ctg10", 9000), ("ctg2", 5200), ("bamonly", 4000), ("faonly", 3000)]):
        rec, genome = synth.simulate_contig_records(length, 20, synth.ONT, 70 + k)
        genomes[name], recs[name] = genome, rec
    bam, fa = str(d / "a.bam"), str(d / "a.fa")
    in_bam = ["ctg10", "bamonly", "ctg2"]
    synth_files.write_bam(bam, [(c, genomes[c].shape[0]) for c in in_bam], {t: recs[c] for t, c in enumerate(in_bam)})
    synth_files.write_fasta(fa, [(c, genomes[c]) for c in ["faonly", "ctg2", "ctg10"]])
    return bam, fa


def _read_fastq(path):
    lines = open(path).read().split("\n")
    assert lines[-1] == "" and (len(lines) - 1) % 4 == 0
    out, names = {}, []
    for k in range(0, len(lines) - 1, 4):
        name, seq, plus, qual = lines[k:k + 4]
        assert name[0] == "@" and plus == "+"
        out[name[1:]] = (seq, qual)
        names.append(name[1:])
    return out, names


def test_polish_assembly_fastq_from_files(assembly_files, tmp_path):
    from pepper_b200 import weights
    from pepper_b200.frontend import PolishFromFiles
    bam, fa = assembly_files
    with PolishFromFiles(bam, fa, weights.random_polish_state(1)) as pf:
        fasta = pf.polish_assembly()
        out = str(tmp_path / "asm.fq")
        got = pf.polish_assembly(out, fastq=True)
        assert set(got) == set(fasta) == {"ctg2", "ctg10"}
        for c in fasta:
            seq, qual = got[c]
            assert seq == fasta[c] and len(qual) == len(seq) > 4000
            (pseq, pqual), calls, regs = pf.polish_contig(c, return_calls=True, qualities=True)
            want = oracle_stitch_q(calls.bases, calls.phred, calls.position, calls.index, calls.image_region, calls.chunk_id,
                                   [s for s, _ in regs], [e for _, e in regs])
            assert (seq, qual) == want == (pseq, pqual), c
        back, names = _read_fastq(out)
        assert back == got and names == ["ctg2", "ctg10"]
        # a sink too small for the records: the session restarts larger and gives the same records
        assert pf.polish_assembly(fastq=True, capacity_bytes=1000) == got


def _rank_main(rank, world, port, q, paths):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from pepper_b200 import weights
    from pepper_b200.dist import DistributedPolisher
    from pepper_b200.frontend import PolishFileSource
    bam, fa = paths
    out = {}
    for schedule in ("static", "dynamic"):
        src = PolishFileSource(bam, fa, device=rank)
        dp = DistributedPolisher(weights.random_polish_state(1), rank, 64 << 10, schedule, group_regions=2, qualities=True)
        dp.run(src)
        out[schedule] = (dp.assemble(src), dp.phase_ms["groups"], len(src.groups(2)))
        dp.close()
        src.close()
    q.put((rank, out))
    dist.destroy_process_group()


def test_two_rank_fastq_equals_one_rank(assembly_files):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    from pepper_b200 import weights
    from pepper_b200.frontend import PolishFromFiles
    bam, fa = assembly_files
    with PolishFromFiles(bam, fa, weights.random_polish_state(1)) as pf:
        want = pf.polish_assembly(fastq=True)
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() % 2000) + 13
    procs = [ctx.Process(target=_rank_main, args=(r, world, port, q, (bam, fa))) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=600) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
    for schedule in ("static", "dynamic"):
        assert all(res[r][schedule][0] == want for r in range(world)), schedule
        assert sum(res[r][schedule][1] for r in range(world)) == res[0][schedule][2]        # every group of the plan run once
