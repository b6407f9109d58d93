"""GPU: k_bgzf_inflate on hand-built DEFLATE streams, and the device record path on files with every record shape, on both
symbol decoders (the warp-parallel speculative decode and the one-decoder-per-warp loop).

* The case table of tests/deflate_craft.py (pinned to zlib on the CPU by tests/test_deflate_craft_cpu.py): the kernel's verdict
  equals zlib's (accepted or rejected; on acceptance the exact bytes), with every payload starting at each address offset mod
  4; every valid stream is rejected when the expected size is one byte off or when the payload length is cut by 1-8 bytes
  while the stream's real bytes stay in memory right after it.
* pb_bam_fetch_device against the htslib iterator rule evaluated on the source arrays (not against the host reader): BGZF
  blocks of 1-2 kB written as stored, fixed and dynamic (long-code) DEFLATE blocks, records without SEQ between odd-length
  records, n_cigar = 0, all-insertion and soft-clip-only CIGARs, long CIGARs behind CG tags with aux tags of every type before
  or after CG, and records long enough to land in higher-level bins; host share 0 and 0.5."""
import gzip
import os
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest

from pepper_b200 import synth, synth_files
from tests import deflate_craft as dc
from tests.test_bamio_cpu import expected_fetch, subset

pytestmark = pytest.mark.gpu

CASES = dc.cases()
DECODERS = {"speculative": 1, "one_decoder": 0}


def _inflate(items, spec):
    """items: (stream bytes, payload length, out_len).  Each stream starts at the address offset mod 4 the list asks for:
    junk bytes after the previous payload fill the gap."""
    from pepper_b200.bamio import inflate_blocks
    return inflate_blocks([s for s, _, _ in items], [o for _, _, o in items], [n for _, n, _ in items], spec=spec)


def _aligned(entries):
    """entries: (stream, in_len, out_len, key) -> each at every start offset mod 4; a leading empty fixed block takes the
    first gap.  Returns (items, keys)."""
    rng = np.random.default_rng(4)
    items, keys = [[b"\x03\x00", 2, 0]], [None]
    cur = 2
    for s, n, o, key in entries:
        for k in range(4):
            pad = (k - cur) % 4
            items[-1][0] = items[-1][0] + bytes(rng.integers(0, 256, pad).astype(np.uint8))
            cur += pad
            items.append([s, n, o])
            keys.append((key, k))
            cur += len(s)
    return [tuple(i) for i in items], keys


@pytest.mark.parametrize("decoder", list(DECODERS))
def test_case_table_verdicts_equal_zlib(decoder):
    entries = [(c.stream, len(c.stream), c.out_len, c) for c in CASES]
    items, keys = _aligned(entries)
    outs, status = _inflate(items, DECODERS[decoder])
    assert status[0] == 0
    wrong = []
    for (c, k), o, s in zip(keys[1:], outs[1:], status[1:]):
        ok, z = dc.zlib_verdict(c.stream)
        assert ok == (c.expect is not None) and (not ok or z == c.expect), c.name         # the table still agrees with zlib
        if ok != (s == 0) or (ok and o != c.expect):
            wrong.append((c.name, int(s), "zlib accepts" if ok else z))
    assert not wrong, sorted(set(wrong))


@pytest.mark.parametrize("decoder", list(DECODERS))
def test_output_size_mismatch_is_rejected(decoder):
    valid = [c for c in CASES if c.expect is not None]
    entries = [(c.stream, len(c.stream), c.out_len + d, (c.name, d)) for c in valid for d in (-1, 1)]
    items, keys = _aligned(entries)
    _, status = _inflate(items, DECODERS[decoder])
    accepted = sorted({key for key, s in zip(keys[1:], status[1:]) if s == 0})
    assert not accepted, accepted


@pytest.mark.parametrize("decoder", list(DECODERS))
def test_payload_cut_short_is_rejected(decoder):
    """The whole stream stays in memory, the kernel is told a payload 1-8 bytes shorter: zlib, fed exactly that many bytes,
    does not reach the end of the stream, so the kernel must not either (a BGZF block whose BSIZE is a few bytes short)."""
    valid = [c for c in CASES if c.expect is not None]
    entries = []
    for c in valid:
        for cut in range(1, 9):
            if cut < len(c.stream):
                assert not dc.zlib_verdict(c.stream[:len(c.stream) - cut])[0]
                entries.append((c.stream, len(c.stream) - cut, c.out_len, (c.name, cut)))
    items, keys = _aligned(entries)
    _, status = _inflate(items, DECODERS[decoder])
    accepted = sorted({key[0] for key, s in zip(keys[1:], status[1:]) if s == 0})
    assert not accepted, accepted


@pytest.mark.parametrize("decoder", list(DECODERS))
def test_zlib_streams_on_both_decoders(decoder):
    rng = np.random.default_rng(8)
    data = [bytes(rng.integers(0, 4 + 60 * (i % 4), int(rng.integers(1, 65536))).astype(np.uint8)) for i in range(40)]
    streams = []
    for i, d in enumerate(data):
        co = zlib.compressobj(i % 10, zlib.DEFLATED, -15, 8, [zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY][i % 3])
        streams.append(co.compress(d) + co.flush())
    items, keys = _aligned([(s, len(s), len(d), i) for i, (s, d) in enumerate(zip(streams, data))])
    outs, status = _inflate(items, DECODERS[decoder])
    assert not status.any()
    assert all(o == data[i] for (i, _), o in zip(keys[1:], outs[1:]))


# ------------------------------------------------------------------------------------------------ device record path
ALL_TYPES = [(b"XA", b"A", b"Q"), (b"Xc", b"c", struct.pack("<b", -5)), (b"XC", b"C", struct.pack("<B", 200)),
             (b"Xs", b"s", struct.pack("<h", -300)), (b"XS", b"S", struct.pack("<H", 60000)),
             (b"Xi", b"i", struct.pack("<i", -70000)), (b"XI", b"I", struct.pack("<I", 4000000000)),
             (b"Xf", b"f", struct.pack("<f", 1.5))]
B_FMT = {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I", "f": "f"}


def aux_tags(r: int) -> bytes:
    """One tag of every type, Z / H / B sizes varying with the record index (B arrays of every subtype, one of them an
    I array that is not CG)."""
    out = b"".join(t + ty + v for t, ty, v in ALL_TYPES)
    out += b"XZZ" + b"z" * (r % 7) + b"\0" + b"XHH" + b"1AE3" * (r % 3) + b"\0"
    for st, fmt in B_FMT.items():
        n = (r + len(out)) % 5
        out += b"Y" + st.encode() + b"B" + st.encode() + struct.pack(f"<i{n}{fmt}", n, *range(n))
    return out


def parse_tags(a: bytes):
    """Pure-Python SAMv1 1.5 aux parse: list of (tag, type, raw value bytes)."""
    out, p = [], 0
    while p < len(a):
        tag, ty = a[p:p + 2], chr(a[p + 2])
        p += 3
        if ty in "AcC":
            n = 1
        elif ty in "sS":
            n = 2
        elif ty in "iIf":
            n = 4
        elif ty in "ZH":
            n = a.index(b"\0", p) - p + 1
        else:
            assert ty == "B"
            st, cnt = chr(a[p]), struct.unpack_from("<i", a, p + 1)[0]
            n = 5 + struct.calcsize("<" + B_FMT[st]) * cnt
        out.append((tag, ty, a[p:p + n]))
        p += n
    return out


def _codes(b):
    idx = np.arange(b.n_bases)
    byte = b.seq[idx >> 1]
    return np.where(idx & 1, byte & 15, byte >> 4).astype(np.uint8)


def _merge(*batches):
    """Records of several RecordBatches in one coordinate-sorted batch."""
    recs = []
    for b in batches:
        codes = _codes(b)
        for r in range(b.n_records):
            so, se, co, ce = int(b.seq_off[r]), int(b.seq_off[r + 1]), int(b.cigar_off[r]), int(b.cigar_off[r + 1])
            recs.append((int(b.pos[r]), codes[so:se], b.qual[so:se], b.cigar[co:ce], int(b.flag[r]), int(b.mapq[r])))
    recs.sort(key=lambda t: t[0])
    seq_off = np.concatenate([[0], np.cumsum([len(t[1]) for t in recs])]).astype(np.int64)
    cigar_off = np.concatenate([[0], np.cumsum([len(t[3]) for t in recs])]).astype(np.int64)
    cat = lambda k, dt: np.concatenate([np.asarray(t[k], dtype=dt) for t in recs]) if recs else np.zeros(0, dt)     # noqa: E731
    return synth.RecordBatch(np.array([t[0] for t in recs], np.int64), seq_off, cigar_off, np.array([t[4] for t in recs], np.uint16),
                             np.array([t[5] for t in recs], np.uint8), synth.pack_codes(cat(1, np.uint8)), cat(2, np.uint8),
                             cat(3, np.uint32))


def _shapes(contig_len: int, seed: int):
    """Hand-made record shapes, repeated along the contig."""
    rng = np.random.default_rng(seed)
    recs = []
    for p in range(300, contig_len - 200, 4099):
        recs += [dict(pos=p, seq="ACGTA", cigar=[(0, 5)]), dict(pos=p + 2, seq="", cigar=[(0, 30)], flag=256),
                 dict(pos=p + 4, seq="", cigar=[(0, 30)], flag=256), dict(pos=p + 5, seq="GGT", cigar=[(0, 3)]),
                 dict(pos=p + 9, seq="", cigar=[(0, 9)], flag=256), dict(pos=p + 20, seq="TTTTTTT", cigar=[(4, 2), (0, 5)]),
                 dict(pos=p + 21, seq="CAG", cigar=[]), dict(pos=p + 22, seq="", cigar=[]),
                 dict(pos=p + 23, seq="ACGTT", cigar=[(1, 5)]), dict(pos=p + 23, seq="GATTACA", cigar=[(4, 7)]),
                 dict(pos=p + 24, seq="TTACG", cigar=[(4, 2), (1, 3)]),
                 dict(pos=p + 30, seq="".join("ACGT"[i] for i in rng.integers(0, 4, 401)), cigar=[(0, 1), (1, 1)] * 200 + [(0, 1)])]
    for p in (1000, contig_len // 3, contig_len // 2):                               # bins above the 16 kb level
        recs += [dict(pos=p, seq="A" * 100, cigar=[(0, 50), (3, min(100_000, contig_len - p - 200)), (0, 50)]),
                 dict(pos=p + 1, seq="".join("ACGT"[i] for i in rng.integers(0, 4, 20_000)), cigar=[(0, 20_000)]),
                 dict(pos=p + 2, seq="C" * 61, cigar=[(0, 30), (2, 40_000), (0, 31)])]
    recs = [r for r in recs if r["pos"] + sum(l for op, l in r["cigar"] if op in (0, 2, 3)) < contig_len]
    recs.sort(key=lambda r: r["pos"])
    return synth.make_records(recs)


def crafted_deflate():
    """BGZF payloads as stored, fixed (literals only), dynamic with long codes on used literals (squared byte counts), and
    zlib blocks, in turn."""
    k = [0]

    def f(payload: bytes) -> bytes:
        i = k[0] % 4
        k[0] += 1
        if i == 0:
            return dc.Writer().stored(payload, final=True).bytes()
        if i == 1:
            return dc.Writer().fixed(list(payload), final=True).bytes()
        if i == 2:
            freq = np.bincount(np.frombuffer(payload, np.uint8), minlength=257).astype(np.int64) ** 2
            freq[256] = 1
            return dc.Writer().dynamic(list(payload), dc.huffman_lengths(freq.tolist(), 15), [1], final=True).bytes()
        co = zlib.compressobj(6, zlib.DEFLATED, -15)
        return co.compress(payload) + co.flush()
    return f


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("edges")
    LA, LB = 150_000, 50_000
    simA, _ = synth.simulate_contig_records(LA, 4, synth.ONT, 71)
    simB, _ = synth.simulate_contig_records(LB, 4, synth.HIFI, 72)
    batches = {0: _merge(simA, _shapes(LA, 1)), 1: _merge(simB, _shapes(LB, 2))}
    contigs = [("ctgA", LA), ("ctgB", LB)]
    out = {}
    path = str(d / "shapes.bam")
    synth_files.write_bam(path, contigs, batches, block_payload=1500, long_cigar_over=300, deflate=crafted_deflate())
    out["shapes"] = path
    for name, first in (("aux_before_cg", False), ("aux_after_cg", True)):
        path = str(d / f"{name}.bam")
        synth_files.write_bam(path, contigs, batches, block_payload=2000, long_cigar_over=40, aux=aux_tags, cg_first=first,
                              deflate=crafted_deflate())
        out[name] = path
    return out, batches, contigs


def _windows(length: int, seed: int):
    rng = np.random.default_rng(seed)
    w = [(0, length)]
    for _ in range(60):
        beg = int(rng.integers(0, length))
        w.append((beg, beg + int(rng.choice([1, 2, 10, 1201, 16384, 40_000, 150_000]))))
    for k in range(1, length // 16384 + 1):
        b = 16384 * k
        w += [(b - 1, b), (b, b + 1), (b - 100, b + 100), (b - 16384, b)]
    return w


@pytest.mark.parametrize("decoder", list(DECODERS))
def test_device_fetch_against_iterator_rule(files, decoder):
    """Every field of every window's records against the iterator rule on the source arrays, at host share 0 and 0.5.
    The decoder is chosen per process by PB_INFLATE_SPEC, so the one-decoder run repeats this test in a child process."""
    want_env = str(DECODERS[decoder])
    if os.environ.get("PB_INFLATE_SPEC", "1") != want_env:
        env = dict(os.environ, PB_INFLATE_SPEC=want_env)
        root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-x",
                            f"{os.path.abspath(__file__)}::test_device_fetch_against_iterator_rule[{decoder}]"],
                           cwd=root, env=env, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
        return
    from pepper_b200.bamio import BamReader
    paths, batches, contigs = files
    n_checked = 0
    for fname, path in paths.items():
        for share in (0.0, 0.5):
            rd = BamReader(path, 4)
            rd.set_host_share(share)
            for tid, (name, length) in enumerate(contigs):
                rec = batches[tid]
                for beg, end in _windows(length, 10 * tid + 1):
                    idx = expected_fetch(rec, beg, end)
                    want, wflag = subset(rec, idx)
                    got = rd.fetch_device(name, beg, end).to_batch()
                    key = (fname, share, name, beg, end)
                    assert got.n_records == want.n_reads, key
                    assert np.array_equal(got.pos, want.pos) and np.array_equal(got.flag, wflag), key
                    for f in ("seq_off", "cigar_off", "mapq", "seq", "qual", "cigar"):
                        assert np.array_equal(getattr(got, f), getattr(want, f)), key + (f,)
                    n_checked += got.n_records
            on_host, on_device = rd.inflate_split()
            assert on_device > 0 and (on_host > 0) == (share > 0)
            rd.close()
    assert n_checked > 10_000


def test_aux_files_against_python_parse(files):
    """The aux-tag files through gzip + struct: every record carries aux_tags(r) and, for long CIGARs, the CG array, in the
    order asked for; the core fields and CIGARs are the source's."""
    paths, batches, _ = files
    for fname, cg_first in (("aux_before_cg", False), ("aux_after_cg", True)):
        raw = gzip.open(paths[fname]).read()
        l_text, = struct.unpack_from("<i", raw, 4)
        p = 8 + l_text
        n_ref, = struct.unpack_from("<i", raw, p)
        p += 4
        for _ in range(n_ref):
            p += 8 + struct.unpack_from("<i", raw, p)[0]
        n_cg = 0
        for tid in range(n_ref):
            b = batches[tid]
            for r in range(b.n_records):
                bs, rtid, pos, l_name, _mapq, _bin, n_cig, flag, l_seq = struct.unpack_from("<iiiBBHHHi", raw, p)
                assert (rtid, pos, flag, l_seq) == (tid, int(b.pos[r]), int(b.flag[r]), int(b.seq_off[r + 1] - b.seq_off[r]))
                q = p + 36 + l_name + 4 * n_cig + (l_seq + 1) // 2 + l_seq
                tags = parse_tags(raw[q:p + 4 + bs])
                want_cig = b.cigar[b.cigar_off[r]:b.cigar_off[r + 1]]
                mine = [t for t in tags if t[0] != b"CG"]
                assert b"".join(t + ty.encode() + v for t, ty, v in mine) == aux_tags(r)
                cg = [i for i, t in enumerate(tags) if t[0] == b"CG"]
                if want_cig.shape[0] > 40:
                    assert cg == ([0] if cg_first else [len(tags) - 1])
                    assert np.array_equal(np.frombuffer(tags[cg[0]][2][5:], "<u4"), want_cig)
                    n_cg += 1
                else:
                    assert not cg and np.array_equal(np.frombuffer(raw, "<u4", n_cig, p + 36 + l_name), want_cig)
                p += 4 + bs
        assert n_cg > 50
