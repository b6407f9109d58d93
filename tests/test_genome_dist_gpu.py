"""GPU: the whole-genome variant call split across ranks.

1. The BGZF compressor (pb_bgzf_compress_host) round-trips empty, 1-byte, random (stored), one-byte-run, distance-32,768 /
   32,769 repeat, all-byte-value and VCF-text payloads through zlib, gzip (CRC + ISIZE) and the project's GPU inflate; on VCF
   text it stays within 1.25x of zlib level 1.
2. One process plays the ranks of dist.DistributedGenomeCaller (interleaved groups, so every boundary crosses ranks; one rank
   owning everything; a rank with no group) over a multi-contig BAM + FASTA with variants planted at interval boundaries: the
   five decompressed files and the totals equal VariantFromFiles.call_genome's, on both inflate paths.
3. Two NCCL ranks, static and dynamic schedules, give the same files (skipped below 2 GPUs)."""
import ctypes as C
import gzip
import os
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _vcf_text() -> bytes:
    from tests.genome_vcf_golden import load
    from pepper_b200.vcf import vcf_text_host
    g = load()
    text, _ = vcf_text_host(g["names"], np.arange(len(g["names"])), g["positions"], g["contig"], g["depths"], g["freqs"], g["keys"],
                            g["probs"], g["regions"], g["select"], g["options"])
    return text.tobytes()


def _payloads():
    rng = np.random.default_rng(11)
    block = rng.integers(0, 256, 32_769, dtype=np.uint8).tobytes()
    return dict(empty=b"", one=b"x", random=rng.integers(0, 256, 65_280, dtype=np.uint8).tobytes(), run=b"a" * 65_280,
                d32768=block[:32_768] * 2, d32769=block[:32_769] + block[:32_769][:65_280 - 32_769],
                bytes256=bytes(range(256)) * 40, vcf=_vcf_text())


def _inflate_gpu(raws: list[bytes], sizes: list[int]) -> list[bytes]:
    from pepper_b200 import _lib
    L = _lib.lib()
    vp = C.c_void_p
    L.pb_inflate_blocks_host.argtypes = [vp, C.c_int64, vp, vp, vp, C.c_int64, vp, vp, vp]
    comp = np.frombuffer(b"".join(raws) + b"\0" * 8, np.uint8).copy()
    in_off = np.concatenate([[0], np.cumsum([len(r) for r in raws])[:-1]]).astype(np.int64)
    in_len = np.array([len(r) for r in raws], np.int32)
    out_len = np.array(sizes, np.int32)
    out = np.zeros(max(1, int(out_len.sum())), np.uint8)
    status = np.zeros(len(raws), np.int32)
    _lib.check(L.pb_inflate_blocks_host(comp.ctypes.data, len(comp) - 8, in_off.ctypes.data, in_len.ctypes.data, out_len.ctypes.data,
                                        len(raws), out.ctypes.data, status.ctypes.data, None), "pb_inflate_blocks_host")
    assert not status.any(), status
    o = np.concatenate([[0], np.cumsum(out_len)]).tolist()
    return [out[a:b].tobytes() for a, b in zip(o[:-1], o[1:])]


@pytest.mark.parametrize("name", ["empty", "one", "random", "run", "d32768", "d32769", "bytes256", "vcf"])
def test_compressor_round_trip(name):
    from pepper_b200.synth_files import _bgzf_block
    from pepper_b200.vcf import BGZF_PAYLOAD, bgzf_compress_host
    data = _payloads()[name]
    cuts = list(range(0, len(data), BGZF_PAYLOAD)) + [len(data)] if data else [0, 0]
    off = np.array(cuts, np.int64)
    members, sizes = bgzf_compress_host(np.frombuffer(data, np.uint8), off)
    assert sizes.shape[0] == off.shape[0] - 1 and int(sizes.sum()) == len(members)
    raws, payloads, pos = [], [], 0
    for k, sz in enumerate(sizes.tolist()):
        m = members[pos:pos + sz]
        pos += sz
        assert m[:4] == b"\x1f\x8b\x08\x04" and m[12:16] == b"BC\x02\x00"
        assert int.from_bytes(m[16:18], "little") == sz - 1 and sz <= 65_536
        p = data[off[k]:off[k + 1]]
        assert zlib.decompress(m[18:-8], -15) == p
        raws.append(m[18:-8]); payloads.append(p)
    assert gzip.decompress(members) == data                     # checks every member's CRC32 and ISIZE
    if data:
        assert _inflate_gpu(raws, [len(p) for p in payloads]) == payloads
    if name == "random":
        assert sizes[0] == 18 + 5 + 65_280 + 8                    # stored
    if name == "vcf":
        zl1 = sum(len(_bgzf_block(p, 1)) for p in payloads)
        zl6 = sum(len(_bgzf_block(p, 6)) for p in payloads)
        print("vcf text %d bytes: gpu %d, zlib-1 %d, zlib-6 %d" % (len(data), len(members), zl1, zl6))
        assert len(members) <= 1.25 * zl1, (len(members), zl1)


# ---------------------------------------------------------------------------------------------------- the genome call
CONTIGS = [("chr2", 250_000, 41), ("chr10", 210_000, 42), ("chr1", 300_000, 43)]


def _planted(length):
    """Variants on the shared endpoints of the 100 kb intervals (and next to them): a het SNP and an insertion on the other
    haplotype at the same position, so boundary sites carry several alleles from both intervals."""
    out = []
    for b in range(100_000, length, 100_000):
        out += [(b, "snp", "A" if b % 200_000 else "C", (0,)), (b, "ins", 3, (1,)), (b + 1, "snp", "G", (0, 1)), (b - 1, "del", 2, (1,))]
    return out


@pytest.fixture(scope="module")
def genome_files(tmp_path_factory):
    from pepper_b200 import synth, synth_files
    d = tmp_path_factory.mktemp("genome_dist")
    recs, fasta = {}, []
    for tid, (c, n, seed) in enumerate(CONTIGS):
        rec, genome = synth.simulate_contig_records(n, 20, synth.ONT, seed, truth=_planted(n))
        recs[tid] = rec
        fasta.append((c, genome))
    fasta.append(("chr3", synth.make_reference(5000, 44)))                 # in the FASTA only
    bam, fa = str(d / "g.bam"), str(d / "g.fa")
    synth_files.write_bam(bam, [(c, n) for c, n, _ in CONTIGS], recs)
    synth_files.write_fasta(fa, fasta)
    return dict(bam=bam, fa=fa, dir=d)


VCF_OPTS = dict(allowed_multiallelics=1, snp_q_cutoff=20, indel_q_cutoff=15, snp_q_cutoff_in_lc=20, indel_q_cutoff_in_lc=10)


def _files(d):
    from pepper_b200.vcf import VCF_FILES
    return [gzip.decompress(open(os.path.join(d, n + ".vcf.gz"), "rb").read()) for n in VCF_FILES]


def _play(dgc, src, shares, params, out_dir):
    """The per-rank work of each share in one process, with the collectives replaced by concatenation / sums."""
    from pepper_b200.dist import ListClaimer, group_table_rows, parse_rank_bytes
    from pepper_b200.vcf import write_vcfs_from_parts
    groups = src.groups(dgc.group_regions)
    parts = [dgc.run_groups(src, ListClaimer(ids), params, None, VCF_OPTS, world=len(shares)) for ids in shares]
    held = np.concatenate([p.held for p in parts])
    for p in parts:
        dgc.edge_pass(p, src, held, None, VCF_OPTS)
    table = sum(group_table_rows(p, len(groups)) for p in parts)
    totals = [dgc.compress(p, src, table) for p in parts]
    assert all(t == totals[0] for t in totals)
    got = {}
    for p in parts:
        got.update(parse_rank_bytes(np.concatenate([p.meta, p.comp.cpu().numpy()])))
    write_vcfs_from_parts(out_dir, "sample_b200", src.fasta_contigs(), src.names, [int(src.contig_of[g0]) for g0, _ in groups], got)
    return totals[0], parts, held


@pytest.mark.parametrize("gpu_inflate", [True, False])
def test_played_ranks_match_call_genome(genome_files, gpu_inflate):
    from oracle import nets
    from pepper_b200 import synth
    from pepper_b200.dist import DistributedGenomeCaller
    from pepper_b200.frontend import VariantFromFiles, VariantGenomeSource
    state = nets.make_variant_weights(0)
    params = synth.ont_params()
    d = genome_files["dir"]
    tag = "gpu" if gpu_inflate else "host"
    with VariantFromFiles(genome_files["bam"], genome_files["fa"], state, gpu_inflate=gpu_inflate) as vf:
        want = vf.call_genome(str(d / ("one_" + tag)), "sample_b200", params=params, vcf_options=VCF_OPTS, batch=1)
        want_files = _files(d / ("one_" + tag))
        dgc = DistributedGenomeCaller(None, 0, 1 << 26, "static", group_regions=1, distributed=False, caller=vf.caller)
        src = VariantGenomeSource(genome_files["bam"], genome_files["fa"], int(params["min_snp_baseq"]), gpu_inflate=gpu_inflate)
        try:
            groups = src.groups(1)
            assert [c for c in src.names] == ["chr1", "chr2", "chr10"] and len(groups) == 3 + 3 + 3
            n = len(groups)
            for k, shares in enumerate(([list(range(0, n, 2)), list(range(1, n, 2))], [list(range(n))], [list(range(n)), []])):
                out = str(d / ("play%d_%s" % (k, tag)))
                totals, parts, held = _play(dgc, src, shares, params, out)
                assert totals == want, (k, totals, want)
                got = _files(out)
                for a, b in zip(got, want_files):
                    assert a == b, k
                if k == 0:
                    # boundary sites with records from both sides, and edge lines written by the later group's owner
                    from pepper_b200.dist import GenomeRankPart  # noqa: F401
                    group_of = np.repeat(np.arange(n), [g1 - g0 for g0, g1 in groups])
                    both = 0
                    bnd = src.boundaries(groups)
                    for g in range(n):
                        b = bnd[g, 0]
                        if b >= 0:
                            m = held["position"] == b
                            both += bool(((group_of[held["region"]] == g - 1) & m).any() and ((group_of[held["region"]] == g) & m).any())
                    assert both >= 4, both
                    assert sum(len(p.edges) for p in parts) >= 4
        finally:
            src.close()
    assert want[0] > 100 and want[1] > 0 and want[2] > 0


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
    out = {}
    for schedule in ("static", "dynamic"):
        dgc = DistributedGenomeCaller(nets.make_variant_weights(0), rank, 1 << 26, schedule, group_regions=1)
        out[schedule] = dgc.call_genome(bam, fa, os.path.join(out_dir, schedule), "sample_b200", params=synth.ont_params(),
                                        vcf_options=VCF_OPTS)
        dgc.close()
    q.put((rank, out))
    dist.destroy_process_group()


def test_two_nccl_ranks_match_call_genome(genome_files):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    from oracle import nets
    from pepper_b200 import synth
    from pepper_b200.frontend import VariantFromFiles
    d = genome_files["dir"]
    with VariantFromFiles(genome_files["bam"], genome_files["fa"], nets.make_variant_weights(0)) as vf:
        want = vf.call_genome(str(d / "nccl_one"), "sample_b200", params=synth.ont_params(), vcf_options=VCF_OPTS, batch=1)
    want_files = _files(d / "nccl_one")
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + (os.getpid() % 2000) + 7
    procs = [ctx.Process(target=_rank_main, args=(r, world, port, q, genome_files["bam"], genome_files["fa"], str(d / "nccl")))
             for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=900) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
    for schedule in ("static", "dynamic"):
        assert res[0][schedule] == want and res[1][schedule] == want, schedule
        assert _files(d / "nccl" / schedule) == want_files, schedule
