"""CPU: polished FASTQ — the stitch with per-base qualities (tests/stitch_quality_oracle.py) against oracle/stitch.py, which
image each QV comes from, the clamp of phred to FASTQ's quality alphabet, the FASTQ text, and the gather of (base, qual) records
over a gloo world of 2 under a scrambled dynamic claim order."""
import os
import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import stitch as ostitch
from pepper_b200.dist import GatherBuffer, GroupClaimer, assemble_contigs, plan_contig_groups
from pepper_b200.frontend import polished_fasta_text, polished_fastq_text, write_polished_fastq
from pepper_b200.polish import QUAL_RECORD
from tests.stitch_quality_oracle import qv_char, stitch_with_qualities
from tests.test_stitch import _many_chunks

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "polish_fasta_seed5.npz")


def _load(name):
    with np.load(os.path.join(HERE, "golden", name)) as z:
        return {k: z[k] for k in z.files}


def test_oracle_sequence_equals_stitch_on_golden_and_many_chunks():
    rng = np.random.default_rng(3)
    g = _load("stitch_seed11.npz")
    ph = rng.integers(0, 101, g["bases"].shape).astype(np.uint8)
    seq, qual = stitch_with_qualities(g["bases"], ph, g["position"], g["index"], g["image_region"], g["chunk_id"], g["region_starts"],
                                      g["region_ends"])
    assert seq == str(g["consensus"]) and len(qual) == len(seq)
    imgs = _many_chunks(5)
    b = np.stack([i[4] for i in imgs]); p = np.stack([i[2] for i in imgs]); x = np.stack([i[3] for i in imgs])
    r = np.zeros(len(imgs), np.int32); c = np.arange(len(imgs), dtype=np.int32)
    ph = rng.integers(0, 101, b.shape).astype(np.uint8)
    seq, qual = stitch_with_qualities(b, ph, p, x, r, c, [300], [9299])
    assert seq == ostitch.stitch(b, p, x, r, c, [300], [9299]) and len(qual) == len(seq) and len(seq) > 5000
    assert set(qual) <= {chr(k) for k in range(33, 127)}


def _tiled(regions, seed):
    """Images of whole regions (start, end), chunked 1000 / 50 like the encoder does: a random column layout with inserts,
    random labels 0..4.  Returns bases, position, index, image_region, chunk_id, region_starts, region_ends."""
    rng = np.random.default_rng(seed)
    B, P, X, R, C = [], [], [], [], []
    for ri, (st, en) in enumerate(regions):
        cols = [(q, k) for q in range(st, en + 1) for k in range(1 + int(rng.random() < 0.3))]
        n, start, end, cid = len(cols), 0, min(len(cols), 1000), 0
        while True:
            pos = np.full(1000, -1, np.int64); idx = np.full(1000, -1, np.int64)
            m = end - start
            pos[:m] = [t[0] for t in cols[start:end]]; idx[:m] = [t[1] for t in cols[start:end]]
            B.append(rng.integers(0, 5, 1000).astype(np.uint8)); P.append(pos); X.append(idx); R.append(ri); C.append(cid)
            cid += 1
            if end == n:
                break
            start = end - 50
            end = min(n, start + 1000)
    return (np.stack(B), np.stack(P), np.stack(X), np.array(R, np.int32), np.array(C, np.int32),
            [s for s, _ in regions], [e for _, e in regions])


def test_every_qv_comes_from_the_winning_image():
    """Each image carries its own phred (10 + image number); label-0 columns carry phred 0 and the dropped region-buffer columns
    phred 1, so a QV names the image it came from, and '!' / '"' would betray a dropped column."""
    regions = [(0, 8000), (7800, 10500)]
    b, p, x, r, c, rs, re_ = _tiled(regions, 11)
    assert int(c.max()) >= 10
    ph = (10 + np.arange(b.shape[0], dtype=np.int64))[:, None].repeat(1000, 1)
    for i in range(b.shape[0]):
        st = rs[r[i]]
        ph[i, (st > 0) & (p[i] <= st + ostitch.BUFFER) & (p[i] >= 0)] = 1
    ph[b == 0] = 0
    ph = ph.astype(np.uint8)
    seq, qual = stitch_with_qualities(b, ph, p, x, r, c, rs, re_)
    assert seq == ostitch.stitch(b, p, x, r, c, rs, re_) and len(qual) == len(seq)
    assert "!" not in qual and '"' not in qual
    # independently: the image whose chunk id sorts last as a string among those holding a key is the one the QV names
    holders = {}
    for i in range(b.shape[0]):
        st = rs[r[i]]
        for col in range(1000):
            pos, idx = int(p[i, col]), int(x[i, col])
            if pos < 0 or idx < 0 or (st > 0 and pos <= st + ostitch.BUFFER):
                continue
            holders.setdefault((pos, idx), []).append((str(int(c[i])), i, col))
    want_seq, want_qual, overlap_9_10 = [], [], 0
    for key in sorted(holders):
        h = holders[key]
        _, i, col = max(h)
        if len(h) > 1 and {s for s, _, _ in h} == {"9", "10"} and r[i] == 0:
            assert c[i] == 9                                   # chunk 9 over chunk 10: "9" > "10"
            overlap_9_10 += 1
        if b[i, col]:
            want_seq.append("ACGT"[b[i, col] - 1]); want_qual.append(qv_char(ph[i, col]))
    assert overlap_9_10 == 50
    assert seq == "".join(want_seq) and qual == "".join(want_qual)


def test_qv_clamp():
    assert [qv_char(q) for q in (0, 92, 93, 94, 100)] == ["!", "}", "~", "~", "~"]
    pos = np.full((1, 1000), -1, np.int64); pos[0, :5] = np.arange(5)
    idx = np.full((1, 1000), -1, np.int64); idx[0, :5] = 0
    b = np.zeros((1, 1000), np.uint8); b[0, :5] = [1, 2, 3, 4, 1]
    ph = np.zeros((1, 1000), np.uint8); ph[0, :5] = [0, 92, 93, 94, 100]
    assert stitch_with_qualities(b, ph, pos, idx, [0], [0], [0], [4]) == ("ACGTA", "!}~~~")


def test_fastq_text(tmp_path):
    recs = {"ctg10": ("AC", "!#"), "ctg2": ("G", "~"), "empty": ("", ""), "chrX": ("TTT", "+5?")}
    want = "@chrX\nTTT\n+\n+5?\n@ctg2\nG\n+\n~\n@ctg10\nAC\n+\n!#\n"
    assert polished_fastq_text(recs) == want
    p = str(tmp_path / "asm.fq")
    write_polished_fastq(p, recs)
    lines = open(p).read().split("\n")
    assert lines[-1] == "" and (len(lines) - 1) % 4 == 0
    for k in range(0, len(lines) - 1, 4):
        name, seq, plus, qual = lines[k:k + 4]
        assert name[0] == "@" and plus == "+" and len(seq) == len(qual) == len(recs[name[1:]][0])
    # the sequence lines are the FASTA's
    fa = polished_fasta_text({c: s for c, (s, _) in recs.items()}).split("\n")
    assert lines[1::4] == fa[1::2]
    with pytest.raises(ValueError):
        polished_fastq_text({"a": ("AC", "!")})


def _synthetic_phred(z):
    return np.random.default_rng(17).integers(0, 101, z["bases"].shape).astype(np.uint8)


def _oracle_group(z, ph, regions):
    sel = np.isin(z["image_region"], regions)
    local = np.searchsorted(np.array(sorted(regions)), z["image_region"][sel])
    rs = [int(z["region_starts"][r]) for r in sorted(regions)]
    re_ = [int(z["region_ends"][r]) for r in sorted(regions)]
    return stitch_with_qualities(z["bases"][sel], ph[sel], z["position"][sel], z["index"][sel], local, z["chunk_id"][sel], rs, re_)


def _worker(rank, world, port, q):
    import random
    import time
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    z = _load("polish_fasta_seed5.npz")
    ph = _synthetic_phred(z)
    contigs = [str(c) for c in z["contigs"]]
    per_contig = [int((z["region_contig"] == k).sum()) for k in range(len(contigs))]
    groups = plan_contig_groups(per_contig, 1)
    group_contig = [contigs[int(z["region_contig"][g0])] for g0, _ in groups]
    buf = GatherBuffer(20000, world, rank, max_groups=len(groups), record=QUAL_RECORD)
    c = GroupClaimer(len(groups), rank, world, "dynamic", key="polish_fastq")
    rnd = random.Random(rank)
    off, segments = 0, []
    while (g := c.next()) is not None:
        time.sleep(rnd.random() * 0.05)                      # scrambles which rank takes which group
        seq, qual = _oracle_group(z, ph, list(range(*groups[g])))
        rec = np.empty(len(seq), QUAL_RECORD)
        rec["base"] = np.frombuffer(seq.encode(), np.uint8); rec["qual"] = np.frombuffer(qual.encode(), np.uint8)
        buf.my_slice()[2 * off:2 * (off + len(seq))] = torch.from_numpy(rec.view(np.uint8).copy())
        off += len(seq)
        segments.append((g, len(seq)))
    buf.gather(off, segments)
    out = assemble_contigs(buf.to_host(), buf.segments(), group_contig, contigs)
    q.put((rank, [g for g, _ in segments], out))
    dist.destroy_process_group()


def test_qual_record_gather_gloo_world2():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000) + 11
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    z = _load("polish_fasta_seed5.npz")
    ph = _synthetic_phred(z)
    contigs = [str(c) for c in z["contigs"]]
    want = {c: _oracle_group(z, ph, np.nonzero(z["region_contig"] == k)[0].tolist()) for k, c in enumerate(contigs)}
    assert sorted(res[0][1] + res[1][1]) == list(range(len(z["region_starts"])))      # every group exactly once
    assert res[0][1] and res[1][1]
    for _, _, got in res:
        assert got == want
        assert polished_fasta_text({c: s for c, (s, _) in got.items()}) == str(z["fasta"])
