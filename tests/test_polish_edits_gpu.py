"""GPU: the polish edits VCF — the edit events of the stitch-to-sink kernel, the device record pass and the written file.

1. The edits sink, fed 1, 7 or all images per call, gives the oracle's events (the non-identity winners and the index-0 ranges
   each image won) on polish_fasta_seed5.npz with a synthetic draft, and the consensus and per-region counts of the plain sink.
2. The record pass (pb_polish_edits_vcf_device) gives the oracle's lines on those events, for drafts of any identity.
3. From BAM + FASTA (one contig with a stretch no read covers): polish_assembly(vcf_path=...) returns and writes the FASTA of
   polish_assembly(); the VCF applied to each draft gives the polished sequence and equals the oracle over polish_contig's
   calls; a too-small event sink restarts to the same bytes; fastq=True works with it.
4. Two ranks (skipped below 2 GPUs): the decompressed VCF equals the one-rank VCF under both schedules."""
import gzip
import os
import numpy as np
import pytest

from pepper_b200 import synth, synth_files
from tests import polish_edits_oracle as E

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _load(name):
    with np.load(os.path.join(HERE, "golden", name)) as z:
        return {k: z[k] for k in z.files}


def _golden_contigs(identity, seed):
    """polish_fasta_seed5 with random phred and, per contig, a draft of the given identity: (g, phred, {contig k: (table, draft,
    span)}, per-column draft bytes)."""
    g = _load("polish_fasta_seed5.npz")
    rng = np.random.default_rng(seed)
    ph = rng.integers(0, 101, g["bases"].shape).astype(np.uint8)
    col_draft = np.zeros(g["bases"].shape, np.uint8)
    out = {}
    for k in range(len(g["contigs"])):
        regs = np.flatnonzero(g["region_contig"] == k)
        if not regs.shape[0]:
            continue
        sel = np.flatnonzero(np.isin(g["image_region"], regs))
        args = (g["bases"][sel], ph[sel], g["position"][sel], g["index"][sel], np.searchsorted(regs, g["image_region"][sel]),
                g["chunk_id"][sel], g["region_starts"][regs], g["region_ends"][regs])
        table = E.winners(*args)
        span = (int(g["region_starts"][regs].min()), int(g["region_ends"][regs].max()))
        d = []
        for p in range(span[1] + 1):
            w = table.get((p, 0))
            d.append("ACGT"[w[0] - 1] if (w is not None and w[0] and rng.random() < identity) else "ACGTN"[rng.integers(0, 5)])
        draft = "".join(d)
        pos = g["position"][sel]
        col_draft[sel] = np.where(pos >= 0, np.frombuffer(draft.encode(), np.uint8)[np.clip(pos, 0, None)], 0)
        out[k] = (table, draft, span)
    return g, ph, out, col_draft


def _oracle_events(table, draft):
    """The column events (position, index, label, phred, draft) of a winners table, in (position, index) order."""
    ev = []
    for (p, k), (b, q) in sorted(table.items()):
        if (k == 0 and (b == 0 or "ACGT"[b - 1] != draft[p])) or (k >= 1 and b != 0):
            ev.append((p, k, b, q, ord(draft[p])))
    return ev


@pytest.mark.parametrize("chunk", [1, 7, 0])
def test_edits_sink_gives_the_oracle_events(chunk):
    from pepper_b200.polish import stitch_sink_test
    from pepper_b200.polish_edits import stitch_sink_edits_test, split_events
    g, ph, contigs, col_draft = _golden_contigs(0.9, 5)
    n = g["bases"].shape[0]
    chunk = chunk or n
    args = (g["bases"], g["position"], g["index"], g["image_region"], g["chunk_id"], g["region_starts"])
    seq, per_region, ev, ev_region = stitch_sink_edits_test(g["bases"], ph, col_draft, *args[1:], chunk)
    plain, plain_per_region = stitch_sink_test(*args, chunk)
    assert seq == plain and np.array_equal(per_region, plain_per_region)
    off = 0
    for k, (table, draft, span) in contigs.items():
        m = int(ev_region[g["region_contig"] == k].sum())
        cols, cover = split_events(ev[off:off + m])
        off += m
        got = [(int(e["position"]), int(e["index"]), int(e["label"]), int(e["phred"]), int(e["draft"])) for e in cols]
        assert got == _oracle_events(table, draft), (chunk, k)
        won = sorted(p for (p, i) in table if i == 0)
        covered = sorted(p for a, b in cover.tolist() for p in range(a, b + 1))
        assert covered == won, (chunk, k)
    assert off == ev.shape[0]
    with pytest.raises(Exception):
        stitch_sink_edits_test(g["bases"], ph, col_draft, *args[1:], chunk, capacity_events=5)


@pytest.mark.parametrize("identity", [0.0, 0.97])
def test_record_pass_gives_the_oracle_lines(identity):
    import torch
    from pepper_b200.polish_edits import EDIT_EVENT, edits_vcf_device
    _, _, contigs, _ = _golden_contigs(identity, 9)
    dev = torch.device("cuda", 0)
    for k, (table, draft, span) in contigs.items():
        ev = _oracle_events(table, draft)
        cols = np.zeros(len(ev), EDIT_EVENT)
        for i, (p, x, b, q, d) in enumerate(ev):
            cols[i] = (p, x, b, q, d, 0)
        won = sorted(p for (p, i) in table if i == 0)
        cover = np.array([[p, p] for p in won], np.int64).reshape(-1, 2)
        d_cols = torch.from_numpy(cols.view(np.uint8).reshape(-1)).to(dev)
        d_draft = torch.from_numpy(np.frombuffer(draft[span[0]:].encode(), np.uint8).copy()).to(dev)
        text, lines = edits_vcf_device(d_cols, cover, span, d_draft, "ctg%d" % k)
        want = E.records(table, draft, span)
        assert bytes(text.cpu().numpy()).decode() == "".join(E.line("ctg%d" % k, r) for r in want), k
        assert lines["pos"].tolist() == [r[0] for r in want] and lines["ref_len"].tolist() == [len(r[1]) for r in want]


@pytest.fixture(scope="module")
def assembly_files(tmp_path_factory):
    """ctg10 and ctg2 simulated at 20x; ctg3 has 2,500 draft bases past the last read."""
    d = tmp_path_factory.mktemp("asme")
    genomes, recs = {}, {}
    for k, (name, length) in enumerate([("ctg10", 9000), ("ctg2", 5200), ("ctg3", 4000)]):
        rec, genome = synth.simulate_contig_records(length, 20, synth.ONT, 80 + k)
        genomes[name], recs[name] = genome, rec
    tail = np.frombuffer(b"ACGT", np.uint8)[np.random.default_rng(3).integers(0, 4, 2500)]
    genomes["ctg3"] = np.concatenate([genomes["ctg3"], tail])
    bam, fa = str(d / "a.bam"), str(d / "a.fa")
    names = ["ctg10", "ctg2", "ctg3"]
    synth_files.write_bam(bam, [(c, genomes[c].shape[0]) for c in names], {t: recs[c] for t, c in enumerate(names)})
    synth_files.write_fasta(fa, [(c, genomes[c]) for c in names])
    return bam, fa, {c: genomes[c].tobytes().decode() for c in names}


def _read_vcf(path):
    text = gzip.decompress(open(path, "rb").read()).decode()
    head = [ln for ln in text.splitlines() if ln.startswith("#")]
    recs = {}
    for ln in text.splitlines():
        if ln.startswith("#"):
            continue
        f = ln.split("\t")
        recs.setdefault(f[0], []).append((int(f[1]) - 1, f[3], f[4], None if f[5] == "." else int(f[5]), f[7] == "UNCOVERED"))
    return head, recs, text


def test_polish_assembly_vcf_from_files(assembly_files, tmp_path):
    from pepper_b200 import weights
    from pepper_b200.frontend import PolishFromFiles
    bam, fa, drafts = assembly_files
    with PolishFromFiles(bam, fa, weights.random_polish_state(1)) as pf:
        fa_plain = str(tmp_path / "plain.fa")
        want = pf.polish_assembly(fa_plain)
        fa_vcf, vcf = str(tmp_path / "v.fa"), str(tmp_path / "e.vcf.gz")
        got = pf.polish_assembly(fa_vcf, vcf_path=vcf)
        assert got == want and open(fa_vcf).read() == open(fa_plain).read()
        assert os.path.exists(vcf + ".tbi")
        head, recs, text = _read_vcf(vcf)
        assert head[0] == "##fileformat=VCFv4.2" and head[-1] == "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO"
        n = 0
        for c, seq in want.items():
            if not seq:
                continue
            span = (0, len(drafts[c]) - 1)
            assert E.apply(recs.get(c, []), drafts[c], span) == seq, c
            _, calls, regs = pf.polish_contig(c, return_calls=True)
            table = E.winners(calls.bases, calls.phred, calls.position, calls.index, calls.image_region, calls.chunk_id,
                              [s for s, _ in regs], [e for _, e in regs])
            assert recs.get(c, []) == E.records(table, drafts[c], span), c
            n += len(recs.get(c, []))
        assert n > 10
        # an event sink too small: the session restarts larger and writes the same bytes
        vcf2 = str(tmp_path / "e2.vcf.gz")
        assert pf.polish_assembly(vcf_path=vcf2, capacity_events=16) == want
        assert _read_vcf(vcf2)[2] == text
        # with FASTQ
        vcf3 = str(tmp_path / "e3.vcf.gz")
        fq = pf.polish_assembly(str(tmp_path / "a.fq"), fastq=True, vcf_path=vcf3)
        assert {c: s for c, (s, _) in fq.items()} == want and _read_vcf(vcf3)[2] == text


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
    bam, fa, out_dir = paths
    out = {}
    for schedule in ("static", "dynamic"):
        src = PolishFileSource(bam, fa, device=rank)
        dp = DistributedPolisher(weights.random_polish_state(1), rank, 64 << 10, schedule, group_regions=2, edits=True,
                                 capacity_events=1 << 16)
        dp.run(src)
        path = os.path.join(out_dir, "r%d_%s.vcf.gz" % (rank, schedule))
        dp.write_edits(src, path)
        out[schedule] = (gzip.decompress(open(path, "rb").read()).decode(), dp.phase_ms["groups"], len(src.groups(2)))
        dp.close()
        src.close()
    q.put((rank, out))
    dist.destroy_process_group()


def test_two_rank_vcf_equals_one_rank(assembly_files, tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    from pepper_b200 import weights
    from pepper_b200.frontend import PolishFromFiles
    bam, fa, _ = assembly_files
    vcf = str(tmp_path / "one.vcf.gz")
    with PolishFromFiles(bam, fa, weights.random_polish_state(1)) as pf:
        pf.polish_assembly(vcf_path=vcf)
    want = gzip.decompress(open(vcf, "rb").read()).decode()
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() % 2000) + 17
    procs = [ctx.Process(target=_rank_main, args=(r, world, port, q, (bam, fa, str(tmp_path)))) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=600) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
    for schedule in ("static", "dynamic"):
        assert all(res[r][schedule][0] == want for r in range(world)), schedule
        assert sum(res[r][schedule][1] for r in range(world)) == res[0][schedule][2]
