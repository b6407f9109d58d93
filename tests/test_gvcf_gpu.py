"""GPU: the gVCF.

1. The block pass (pb_gvcf_blocks_host) gives the numpy oracle's lines on seeded random tracks: segments of every length
   (empty ones included), overlapping masks, blocks across tile boundaries, positions past 2^31.
2. The session's track equals the counts of the port oracle's count matrix on the 12 variant KATs and seeded ONT / HiFi
   regions (depth below 125, where the matrix clamp cannot bite).
3. A genome call with the gVCF over a multi-contig BAM + FASTA (variants planted on interval boundaries, a deletion across a
   group boundary, an N block, an interval with no reads): the five VCFs are byte-identical to a call without it; blocks never overlap each other or a
   record, and with the record spans cover every called position; the record lines stripped of their suffixes are FULL's body;
   the blocks are the oracle's over the pass's inputs; the index finds the lines.  Played ranks, with the pass in batches of
   two groups, give the same gVCF.
4. `python -m pepper_b200 call_variant_gvcf` writes the six files; an exhausted track restarts in process."""
import gzip
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import gvcf_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _segments(lengths, pos0, contigs):
    from pepper_b200.gvcf import GVCF_SEGMENT
    s = np.zeros(len(lengths), GVCF_SEGMENT)
    t = 0
    for i, n in enumerate(lengths):
        s[i] = (t, pos0[i], n, t + 7, contigs[i], 0)
        t += n
    return s, t


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_block_pass_matches_oracle(seed):
    from pepper_b200.gvcf import gvcf_blocks_host
    rng = np.random.default_rng(seed)
    lengths = [int(x) for x in rng.integers(0, 5000, 12)] + [0, 4097]
    pos0 = [int(x) for x in rng.integers(0, 1 << 33, len(lengths))]
    pos0[0] = (1 << 31) - 100                                          # a block across 2^31
    contigs = [int(x) for x in rng.integers(0, 3, len(lengths))]
    seg, T = _segments(lengths, pos0, contigs)
    depth = rng.integers(0, 45, T)
    depth[rng.integers(0, T, T // 50)] = 0
    alt = rng.binomial(depth, rng.choice([0.0, 0.01, 0.5, 1.0], T))
    track = (depth - alt).astype(np.uint32) | (alt.astype(np.uint32) << 16)
    starts = rng.integers(-5, T, 300)
    masks = np.stack([starts, starts + rng.integers(0, 40, 300)], 1).astype(np.int64)
    ref = np.frombuffer(bytes(rng.choice(list(b"ACGTacgtNNR"), T + 16)), np.uint8)
    names = ["chrA", "contig_2", "c3"]
    for binsize in (5, 1, 30):
        text, lines = gvcf_blocks_host(track, seg, masks, ref, names, binsize)
        want = O.blocks(track, seg, masks, ref.tobytes(), names, binsize)
        assert text.tobytes().decode() == "".join(w[3] for w in want)
        assert lines["pos"].tolist() == [w[1] for w in want]
        assert lines["ref_len"].tolist() == [w[2] for w in want]
        assert lines["contig"].tolist() == [w[0] for w in want]
        assert len(want) > 100


def _session_track(caller, reads, regions, params):
    """The track of one session over `regions` (each region owns its whole candidate range), one group per region."""
    import torch
    from pepper_b200.abi import HostReads, regions_array
    hr = HostReads(reads)
    regs, _keep = regions_array(regions)
    t = regions.table
    n = int((t[:, 3] - t[:, 2] + 1).sum())
    track = torch.zeros(n, dtype=torch.int32, device="cuda:0")
    s = caller.stream(params, 1 << 16)
    s.track(n, track.data_ptr())
    h_ref = np.ascontiguousarray(regions.ref, np.uint8)
    for r in range(regions.n_regions):
        s.stage_host(hr, regs, r, r + 1, h_ref, r)
        s.owned([int(t[r, 3])])
        s.run(flush=r + 1 == regions.n_regions)
        s.sync()
    s.end()
    assert s.track_used() == n
    return track.cpu().numpy().view(np.uint32)


def _oracle_track(oracle, reads, regions, params):
    want = oracle.variant_encode(reads, regions, params, "port", debug=True)
    out, ok = [], []
    for r in range(regions.n_regions):
        rs, _, cs, ce, roff, rlen = (int(x) for x in regions.table[r, :6])
        m = want["debug"][r][0]
        for p in range(cs, ce + 1):
            x = p - rs
            c = chr(regions.ref[roff + x]) if x < rlen else "N"
            nr, na = O.counts_from_columns(c, m[x, 8:15], m[x, 19:26])
            out.append(nr | (na << 16))
            # the port clamps columns 11-24 of its matrix at 125: depth there is compared only below that
            ok.append(bool(np.abs(m[x, 11:25]).max() < 125))
    return np.array(out, np.uint32), np.array(ok, bool)


def test_track_matches_port_counts(oracle_built):
    from oracle import nets
    from pepper_b200 import synth
    from pepper_b200.pipeline import VariantCaller
    from tests import kats
    caller = VariantCaller(nets.make_variant_weights(0), 0)
    try:
        cases = [(n, r, g, p) for n, r, g, p in kats.variant_kats()]
        for platform, params, seed in ((synth.ONT, synth.ont_params(), 3), (synth.HIFI, synth.hifi_params(), 4)):
            reads, regions = synth.make_variant_workload(3, 6000, 30, platform, seed=seed, n_frac=0.01)
            cases.append(("synth%d" % seed, reads, regions, params))
        compared = 0
        for name, reads, regions, params in cases:
            got = _session_track(caller, reads, regions, params)
            want, ok = _oracle_track(oracle_built, reads, regions, params)
            bad = np.flatnonzero((got != want) & ok)
            assert bad.size == 0, (name, bad[:10], got[bad[:4]], want[bad[:4]])
            compared += int(ok.sum())
        assert compared > 30_000, compared
    finally:
        caller.close()


# ---------------------------------------------------------------------------------------------------- the genome call
CONTIGS = [("chr2", 250_000, 41), ("chr10", 210_000, 42), ("chr1", 300_000, 43)]
GAP = 195_000
VCF_OPTS = dict(allowed_multiallelics=1, snp_q_cutoff=20, indel_q_cutoff=15, snp_q_cutoff_in_lc=20, indel_q_cutoff_in_lc=10)


def _planted(length):
    out = []
    for b in range(100_000, length, 100_000):
        out += [(b, "snp", "A" if b % 200_000 else "C", (0,)), (b, "ins", 3, (1,)), (b + 1, "snp", "G", (0, 1)),
                (b - 2, "del", 5, (0, 1))]                             # a deletion across the group boundary
    return out


@pytest.fixture(scope="module")
def genome_files(tmp_path_factory):
    from pepper_b200 import synth, synth_files
    d = tmp_path_factory.mktemp("gvcf_genome")
    recs, fasta = {}, []
    for tid, (c, n, seed) in enumerate(CONTIGS):
        rec, genome = synth.simulate_contig_records(n, 20, synth.ONT, seed, truth=_planted(n))
        recs[tid] = rec
        if c == "chr10":
            genome = genome.copy()
            genome[150_000:150_300] = ord("N")                            # an N block: no counted base
        if c == "chr1":
            # a zero-coverage gap: reads reaching past GAP get mapping quality 0, which the callers' min_mapq 1 drops, so the
            # last interval [200,000, 300,000] has no reads at all
            rec.mapq = rec.mapq.copy()
            for r in range(rec.n_records):
                if int(rec.pos[r]) + synth_files.record_ref_len(rec.cigar[rec.cigar_off[r]:rec.cigar_off[r + 1]]) > GAP:
                    rec.mapq[r] = 0
        fasta.append((c, genome))
    bam, fa = str(d / "g.bam"), str(d / "g.fa")
    synth_files.write_bam(bam, [(c, n) for c, n, _ in CONTIGS], recs)
    synth_files.write_fasta(fa, fasta)
    return dict(bam=bam, fa=fa, dir=d)


def _body(path):
    text = gzip.decompress(open(path, "rb").read()).decode()
    return [x + "\n" for x in text.split("\n") if x and not x.startswith("#")]


def _query(tbi: bytes, gz: bytes, contig: str, beg: int):
    """Lines of `contig` whose POS is `beg` (0-based), found through the index: the bins of [beg, beg + 1) on the reg2bin path,
    their chunks read member by member to the chunk's end."""
    import struct
    from tests.test_genome_vcf_cpu import _bgzf_members
    d = gzip.decompress(tbi)
    assert d[:4] == b"TBI\x01"
    n_ref, l_nm = struct.unpack_from("<i", d, 4)[0], struct.unpack_from("<i", d, 32)[0]
    names = d[36:36 + l_nm].split(b"\0")[:-1]
    p, idx = 36 + l_nm, []
    for _ in range(n_ref):
        (nb,) = struct.unpack_from("<i", d, p); p += 4
        bins = {}
        for _ in range(nb):
            b, nc = struct.unpack_from("<Ii", d, p); p += 8
            bins[b] = [struct.unpack_from("<QQ", d, p + 16 * k) for k in range(nc)]; p += 16 * nc
        (ni,) = struct.unpack_from("<i", d, p); p += 4 + 8 * ni
        idx.append(bins)
    bins = idx[names.index(contig.encode())]
    want = {0} | {base + (beg >> sh) for sh, base in ((26, 1), (23, 9), (20, 73), (17, 585), (14, 4681))}
    members = dict(_bgzf_members(gz))
    keys = sorted(members)
    found = []
    for b in want & set(bins):
        for vb, ve in bins[b]:
            k = keys.index(vb >> 16)
            buf = b""
            while k < len(keys) and keys[k] <= (ve >> 16):
                buf += members[keys[k]]; k += 1
            span = sum(len(members[x]) for x in keys if (vb >> 16) <= x < (ve >> 16)) - (vb & 0xffff) + (ve & 0xffff)
            for line in buf[vb & 0xffff:][:span].decode().splitlines():
                f = line.split("\t")
                if f[0] == contig and int(f[1]) - 1 == beg:
                    found.append(line)
    return found


def lines_ref(src, contig, pos):
    from pepper_b200.bamio import FastaReader
    fa = FastaReader(src.fasta_path)
    try:
        c = fa.get_reference_sequence(contig, pos, pos + 1).upper()
    finally:
        fa.close()
    return c if c in ("A", "C", "G", "T") else "N"


def _check_gvcf(out_dir, src):
    g = os.path.join(out_dir, "PEPPER_VARIANT.g.vcf.gz")
    lines = _body(g)
    recs = [x for x in lines if x.split("\t")[4] != "<*>"]
    blocks = [x for x in lines if x.split("\t")[4] == "<*>"]
    assert [O.strip_record(x) for x in recs] == _body(os.path.join(out_dir, "PEPPER_VARIANT_FULL.vcf.gz"))
    assert len(blocks) > 100 and any(":./.:" in x or "\t./.:" in x for x in blocks)
    for k, c in enumerate(src.names):
        first, last = src._first[k], src._first[k + 1]
        s0, e0 = src.intervals[first][0], src.intervals[last - 1][1]
        block_cov = np.zeros(e0 - s0 + 1, np.int32)
        rec_cov = np.zeros(e0 - s0 + 1, np.int32)
        prev = -1
        for x in lines:
            f = x.split("\t")
            if f[0] != c:
                continue
            p = int(f[1]) - 1
            assert p > prev                                            # POS order, one line per POS
            prev = p
            if f[4] == "<*>":
                end = int(f[7][4:])
                block_cov[p - s0:end - s0] += 1
            else:
                rec_cov[max(p - s0, 0):p - s0 + len(f[3])] += 1
        assert block_cov.max() <= 1 and not (block_cov & (rec_cov > 0)).any(), c
        assert ((block_cov > 0) | (rec_cov > 0)).all(), (c, np.flatnonzero((block_cov == 0) & (rec_cov == 0))[:10])
    # the interval without reads (chr1's last): one no-call block over its whole owned window
    s_gap, e_gap = src.intervals[src._first[src.names.index("chr1") + 1] - 1]
    assert s_gap == 200_000 and s_gap > GAP
    assert "chr1\t%d\t.\t%s\t<*>\t.\t.\tEND=%d\tGT:GQ:MIN_DP:PL\t./.:0:0:0,0,0\n" % (
        s_gap + 1, lines_ref(src, "chr1", s_gap), e_gap + 1) in lines
    tbi = open(g + ".tbi", "rb").read()
    gz = open(g, "rb").read()
    rng = np.random.default_rng(0)
    for x in [lines[i] for i in rng.choice(len(lines), 12, replace=False)]:
        f = x.split("\t")
        assert x.rstrip("\n") in _query(tbi, gz, f[0], int(f[1]) - 1), x


def test_genome_gvcf(genome_files, monkeypatch):
    from oracle import nets
    from pepper_b200 import gvcf, synth
    from pepper_b200.dist import DistributedGenomeCaller
    from pepper_b200.frontend import VariantGenomeSource
    from pepper_b200.pipeline import VariantCaller
    params = synth.ont_params()
    d = genome_files["dir"]
    seen = []
    real = gvcf.gvcf_blocks_device

    def spy(d_track, n_track, segments, masks, d_ref, names, binsize, device=0):
        text, lines = real(d_track, n_track, segments, masks, d_ref, names, binsize, device)
        seen.append((d_track[:n_track].cpu().numpy().view(np.uint32), segments.copy(), masks.copy(), d_ref, names, binsize,
                     text.cpu().numpy().tobytes().decode()))
        return text, lines
    monkeypatch.setattr(gvcf, "gvcf_blocks_device", spy)
    caller = VariantCaller(nets.make_variant_weights(0), 0)
    try:
        src = VariantGenomeSource(genome_files["bam"], genome_files["fa"], int(params["min_snp_baseq"]), min_mapq=1)
        try:
            outs = {}
            for tag, kw in (("plain", {}), ("gvcf", dict(gvcf=True))):
                dgc = DistributedGenomeCaller(None, 0, 1 << 26, "static", group_regions=1, distributed=False, caller=caller, **kw)
                outs[tag] = str(d / tag)
                dgc.call_source(src, outs[tag], "S", params, None, VCF_OPTS)
                dgc.close()
            from pepper_b200.vcf import VCF_FILES
            for n in VCF_FILES:
                a, b = (open(os.path.join(outs[t], n + ".vcf.gz"), "rb").read() for t in ("plain", "gvcf"))
                assert a == b, n
            _check_gvcf(outs["gvcf"], src)
            # the blocks of the pass equal the oracle's over the same inputs
            track, seg, masks, d_ref, names, binsize, text = seen[-1]
            import torch
            n_ref = int((seg["ref_off"] + seg["len"]).max())
            from pepper_b200.dist import _device_column
            ref_bytes = _device_column(d_ref, (n_ref,), "|u1", torch.device("cuda", 0)).cpu().numpy().tobytes()
            assert text == "".join(w[3] for w in O.blocks(track, seg, masks, ref_bytes, names, binsize))
            # played ranks: interleaved shares, one rank owning everything, a rank with none
            want = gzip.decompress(open(os.path.join(outs["gvcf"], "PEPPER_VARIANT.g.vcf.gz"), "rb").read())
            n = len(src.groups(1))
            dgc = DistributedGenomeCaller(None, 0, 1 << 26, "static", group_regions=1, distributed=False, caller=caller, gvcf=True)
            for k, shares in enumerate(([list(range(0, n, 2)), list(range(1, n, 2))], [list(range(n))], [list(range(n)), []])):
                out = str(d / ("play%d" % k))
                _play(dgc, src, shares, params, out)
                assert gzip.decompress(open(os.path.join(out, "PEPPER_VARIANT.g.vcf.gz"), "rb").read()) == want, k
        finally:
            src.close()
    finally:
        caller.close()


def _play(dgc, src, shares, params, out_dir):
    """The per-rank work of each share in one process, the collectives replaced by concatenation, sums and maxima."""
    from pepper_b200.dist import ListClaimer, group_table_rows, mask_until
    from pepper_b200.gvcf import parse_gvcf_bytes, write_gvcf_from_parts
    groups = src.groups(dgc.group_regions)
    gc = [int(src.contig_of[g0]) for g0, _ in groups]
    parts = [dgc.run_groups(src, ListClaimer(ids), params, None, VCF_OPTS, world=len(shares)) for ids in shares]
    held = np.concatenate([p.held for p in parts])
    for p in parts:
        dgc.edge_pass(p, src, held, None, VCF_OPTS)
    table = sum(group_table_rows(p, len(groups)) for p in parts)
    for p in parts:
        dgc.compress(p, src, table)
    ends = np.full(len(groups), -1, np.int64)
    for p in parts:
        for g, rows in p.written.items():
            if rows.shape[0]:
                ends[g] = int((p.all_lines["pos"][rows] + p.all_lines["ref_len"][rows]).max())
    got = {}
    for p in parts:
        # batches of two 100 kb groups: the batched pass must give the one-batch call's file
        meta, comp = dgc.gvcf_pass(p, src, mask_until(ends, gc), batch_positions=150_000)
        got.update(parse_gvcf_bytes(np.concatenate([meta, comp])))
    write_gvcf_from_parts(out_dir, "S", src.fasta_contigs(), src.names, gc, got)


def test_call_variant_gvcf_command(genome_files, monkeypatch, capsys):
    import torch
    from oracle import nets
    from pepper_b200 import cli, gvcf
    d = genome_files["dir"]
    model = str(d / "variant.pkl")
    state = nets.make_variant_weights(0)
    torch.save({"model_state_dict": {"module." + k: torch.as_tensor(v) for k, v in state.items()}, "epochs": 1}, model)
    argv = ["call_variant_gvcf", "-b", genome_files["bam"], "-f", genome_files["fa"], "-m", model, "-s", "SAMPLE", "-t", "4",
            "--ont_r9_guppy5_sup", "--gvcf_gq_binsize", "10"]
    out = str(d / "cli_sub")
    r = subprocess.run([sys.executable, "-m", "pepper_b200"] + argv + ["-o", out], cwd=ROOT, env=dict(os.environ, PYTHONPATH=ROOT),
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    names = sorted(os.listdir(out))
    assert "PEPPER_VARIANT.g.vcf.gz" in names and "PEPPER_VARIANT.g.vcf.gz.tbi" in names
    assert sum(n.endswith(".vcf.gz") for n in names) == 6
    # an exhausted track restarts in process with twice the room, to the same files
    monkeypatch.setattr(gvcf, "track_capacity", lambda bases, world: 150_000)
    small = str(d / "cli_small")
    assert cli.main(argv + ["-o", small]) == 0
    err = capsys.readouterr().err
    assert "IS EXHAUSTED: RESTARTING WITH" in err
    for n in names:
        if n.endswith(".vcf.gz"):
            assert gzip.decompress(open(os.path.join(out, n), "rb").read()) == gzip.decompress(open(os.path.join(small, n), "rb").read()), n


def _rank_main(rank, world, port, q, bam, fa, out_dir):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from oracle import nets
    from pepper_b200 import synth
    from pepper_b200.dist import DistributedGenomeCaller
    dgc = DistributedGenomeCaller(nets.make_variant_weights(0), rank, 1 << 26, "dynamic", group_regions=1, gvcf=True)
    dgc.call_genome(bam, fa, out_dir, "S", params=synth.ont_params(), vcf_options=VCF_OPTS)
    dgc.close()
    dist.destroy_process_group()
    q.put(rank)


@pytest.mark.skipif(not __import__("torch").cuda.is_available() or __import__("torch").cuda.device_count() < 2,
                    reason="needs 2 GPUs")
def test_two_nccl_ranks(genome_files):
    import socket
    import torch.multiprocessing as mp
    from oracle import nets
    from pepper_b200 import synth
    from pepper_b200.dist import DistributedGenomeCaller
    d = genome_files["dir"]
    one = str(d / "nccl_one")
    dgc = DistributedGenomeCaller(nets.make_variant_weights(0), 0, 1 << 26, "static", group_regions=1, distributed=False, gvcf=True)
    dgc.call_genome(genome_files["bam"], genome_files["fa"], one, "S", params=synth.ont_params(), vcf_options=VCF_OPTS)
    dgc.close()
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    two = str(d / "nccl_two")
    mp.spawn(_rank_main, args=(2, port, q, genome_files["bam"], genome_files["fa"], two), nprocs=2, join=True)
    a, b = (gzip.decompress(open(os.path.join(x, "PEPPER_VARIANT.g.vcf.gz"), "rb").read()) for x in (one, two))
    assert a == b
