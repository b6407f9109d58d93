"""A DEFLATE (RFC 1951) stream writer for tests, and the table of hand-built streams the inflate tests share.

zlib's compressor never writes many legal streams (a distance of 32,768, codes near 15 bits, empty stored blocks between
Huffman blocks, code-length repeats that cross from the literal/length lengths into the distance lengths, ...) and no invalid
ones.  `Writer` writes any of them: bits go out LSB first and Huffman codes MSB first, blocks are stored, fixed or dynamic, a
dynamic block takes explicit code lengths and, optionally, an explicit code-length code and run-length encoding of them, and raw
bits can be appended anywhere.

Symbols are tokens:
  * an int 0..255: a literal;
  * a tuple (length, dist): a match, written with the canonical length and distance symbols;
  * Sym(sym, extra, dsym, dextra): an explicit literal/length symbol with its extra bits and, for a length, an explicit
    distance symbol with its extra bits (non-canonical 284 + 31, symbols 286/287, distance symbols 30/31).

`cases()` is the case table: tests/test_deflate_craft_cpu.py pins every case to zlib's verdict, and
tests/test_inflate_edges_gpu.py runs the same table through both decode paths of k_bgzf_inflate."""
from __future__ import annotations

import heapq
import zlib
from dataclasses import dataclass, field

import numpy as np

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
             8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CLEN_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32

# the inflate kernel's lookup tables (pepper_b200/csrc/bgzf_inflate.cuh): longer codes take the canonical slow path
LIT_TABLE_BITS, DIST_TABLE_BITS = 10, 8


@dataclass(frozen=True)
class Sym:
    sym: int
    extra: int = 0
    dsym: int | None = None
    dextra: int = 0


def canonical_codes(lens):
    """RFC 1951 3.2.2: the canonical code of every symbol (codes of an over-subscribed set are cut to their length)."""
    count = [0] * 17
    for l in lens:
        count[l] += 1
    count[0] = 0
    nxt, code = [0] * 17, 0
    for b in range(1, 16):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    out = []
    for l in lens:
        if l:
            out.append(nxt[l] & ((1 << l) - 1))
            nxt[l] += 1
        else:
            out.append(None)
    return out


def kraft(lens) -> int:
    """Sum of 2^(15 - len) over the used codes: 2^15 for a complete set, less when incomplete, more when over-subscribed."""
    return sum(1 << (15 - l) for l in lens if l)


def huffman_lengths(freqs, max_bits: int):
    """Complete Huffman code lengths limited to `max_bits` (frequencies are halved until the tree fits); a set with one used
    symbol gets a partner so that the code stays complete."""
    freqs = list(freqs)
    used = [s for s, f in enumerate(freqs) if f]
    if len(used) == 1:
        freqs[0 if used[0] else 1] = 1
        used = [s for s, f in enumerate(freqs) if f]
    lens = [0] * len(freqs)
    if not used:
        return lens
    while True:
        heap = [(freqs[s], i, [s]) for i, s in enumerate(used)]
        heapq.heapify(heap)
        depth = dict.fromkeys(used, 0)
        k = len(heap)
        while len(heap) > 1:
            fa, _, a = heapq.heappop(heap)
            fb, _, b = heapq.heappop(heap)
            for s in a + b:
                depth[s] += 1
            heapq.heappush(heap, (fa + fb, k, a + b))
            k += 1
        if max(depth.values()) <= max_bits:
            for s, d in depth.items():
                lens[s] = d
            return lens
        freqs = [(f + 1) // 2 if f else 0 for f in freqs]


def staircase(symbols, lens_total: int):
    """A complete code over `symbols` with lengths 1, 2, ..., n - 1, n - 1 (n = len(symbols) <= 16): the last symbols get the
    longest codes.  Returns a list of `lens_total` lengths."""
    n = len(symbols)
    assert 2 <= n <= 16
    out = [0] * lens_total
    for i, s in enumerate(symbols):
        out[s] = min(i + 1, n - 1)
    assert kraft(out) == 1 << 15
    return out


def rle_lengths(lens):
    """Code-length symbols for `lens` (one sequence: literal/length then distance lengths): 0..15, (16, rep), (17, rep),
    (18, rep).  Runs cross the literal/distance boundary when the lengths do."""
    out, i, n = [], 0, len(lens)
    while i < n:
        v, run = lens[i], 1
        while i + run < n and lens[i + run] == v:
            run += 1
        if v == 0 and run >= 3:
            r = min(run, 138)
            out.append((18, r) if r >= 11 else (17, r))
            i += r
        elif v and run >= 4:
            r = min(run - 1, 6)
            out += [v, (16, r)]
            i += 1 + r
        else:
            out.append(v)
            i += 1
    return out


def _length_sym(length: int):
    for li in range(28, -1, -1):
        if LEN_BASE[li] <= length:
            return 257 + li, length - LEN_BASE[li]
    raise ValueError(length)


def _dist_sym(dist: int):
    for di in range(29, -1, -1):
        if DIST_BASE[di] <= dist:
            return di, dist - DIST_BASE[di]
    raise ValueError(dist)


class Writer:
    """Builds one DEFLATE stream.  `out` is what a decoder must produce (None once a token makes the stream undecodable);
    `blocks` records per block its header bit, its first symbol bit, and every symbol's start bit with whether it needs the
    kernel's slow path (a literal/length code longer than its 10-bit table or a distance code longer than its 8-bit table)."""

    def __init__(self):
        self.acc = 0
        self.nbits = 0
        self.out: bytearray | None = bytearray()
        self.size = 0                     # bytes the tokens stand for, counted on after `out` becomes None
        self.blocks: list[dict] = []

    # ---- bits
    def bits(self, value: int, n: int) -> "Writer":
        """n raw bits, LSB first."""
        assert 0 <= value < (1 << n), (value, n)
        self.acc |= value << self.nbits
        self.nbits += n
        return self

    def code(self, code: int, n: int) -> "Writer":
        """A Huffman code of n bits, MSB first."""
        return self.bits(int(f"{code:0{n}b}"[::-1], 2) if n else 0, n)

    def align(self) -> "Writer":
        return self.bits(0, -self.nbits % 8)

    def bytes(self) -> bytes:
        n = (self.nbits + 7) // 8
        return self.acc.to_bytes(n, "little")

    # ---- blocks
    def stored(self, data: bytes, final: bool = False, nlen: int | None = None) -> "Writer":
        """A stored block.  `nlen` overrides NLEN (invalid streams)."""
        self.blocks.append(dict(type=0, start=self.nbits))
        self.bits(int(final), 1).bits(0, 2).align()
        self.bits(len(data), 16).bits((len(data) ^ 0xffff) if nlen is None else nlen, 16)
        self.acc |= int.from_bytes(data, "little") << self.nbits
        self.nbits += 8 * len(data)
        if self.out is not None:
            self.out += data
        self.size += len(data)
        return self

    def fixed(self, tokens, final: bool = False, eob: bool = True) -> "Writer":
        self.blocks.append(dict(type=1, start=self.nbits))
        self.bits(int(final), 1).bits(1, 2)
        return self._symbols(tokens, FIXED_LIT, FIXED_DIST, eob)

    def dynamic(self, tokens, lit_lens, dist_lens, final: bool = False, eob: bool = True, rle=None, clen_lens=None,
                hclen: int | None = None) -> "Writer":
        """A dynamic block: HLIT = len(lit_lens), HDIST = len(dist_lens).  `rle`: the code-length symbols (default
        rle_lengths of the concatenated lengths); `clen_lens`: the 19 lengths of the code-length code (default: a complete
        Huffman code of the symbols `rle` uses); `hclen`: how many of them are written (default: up to the last nonzero one
        in CLEN_ORDER, at least 4)."""
        lit_lens, dist_lens = list(lit_lens), list(dist_lens)
        assert 257 <= len(lit_lens) <= 288 and 1 <= len(dist_lens) <= 32
        rle = rle_lengths(lit_lens + dist_lens) if rle is None else rle
        if clen_lens is None:
            freq = [0] * 19
            for item in rle:
                freq[item[0] if isinstance(item, tuple) else item] += 1
            clen_lens = huffman_lengths(freq, 7)
        if hclen is None:
            hclen = max([4] + [i + 1 for i, s in enumerate(CLEN_ORDER) if clen_lens[s]])
        self.blocks.append(dict(type=2, start=self.nbits))
        self.bits(int(final), 1).bits(2, 2).bits(len(lit_lens) - 257, 5).bits(len(dist_lens) - 1, 5).bits(hclen - 4, 4)
        for i in range(hclen):
            self.bits(clen_lens[CLEN_ORDER[i]], 3)
        ccodes = canonical_codes(clen_lens)
        for item in rle:
            s, rep = item if isinstance(item, tuple) else (item, None)
            self.code(ccodes[s], clen_lens[s])
            if s == 16:
                self.bits(rep - 3, 2)
            elif s == 17:
                self.bits(rep - 3, 3)
            elif s == 18:
                self.bits(rep - 11, 7)
        return self._symbols(tokens, lit_lens, dist_lens, eob)

    def _symbols(self, tokens, lit_lens, dist_lens, eob: bool) -> "Writer":
        lcodes, dcodes = canonical_codes(lit_lens), canonical_codes(dist_lens)
        blk = self.blocks[-1]
        blk["sym_start"] = self.nbits
        syms = blk["syms"] = []

        def put(codes, lens, s):
            if s >= len(lens) or not lens[s]:
                raise ValueError(f"symbol {s} has no code in this block")
            self.code(codes[s], lens[s])
            return lens[s]
        for t in tokens:
            at = self.nbits
            if isinstance(t, tuple):
                ls, lx = _length_sym(t[0])
                ds, dx = _dist_sym(t[1])
                t = Sym(ls, lx, ds, dx)
            elif not isinstance(t, Sym):
                t = Sym(int(t))
            ll = put(lcodes, lit_lens, t.sym)
            dl = 0
            if t.sym < 256:
                self.size += 1
                if self.out is not None:
                    self.out.append(t.sym)
            elif t.sym == 256:
                pass
            else:
                lx = LEN_EXTRA[t.sym - 257] if t.sym <= 285 else 0
                self.bits(t.extra, lx)
                self.size += LEN_BASE[t.sym - 257] + t.extra if t.sym <= 285 else 0
                if t.dsym is not None:
                    dl = put(dcodes, dist_lens, t.dsym)
                    self.bits(t.dextra, DIST_EXTRA[t.dsym] if t.dsym < 30 else 0)
                if self.out is not None:
                    if t.sym > 285 or t.dsym is None or t.dsym > 29:
                        self.out = None
                    else:
                        length = LEN_BASE[t.sym - 257] + t.extra
                        dist = DIST_BASE[t.dsym] + t.dextra
                        if dist > len(self.out):
                            self.out = None
                        else:
                            for _ in range(length):
                                self.out.append(self.out[-dist])
            syms.append((at - blk["sym_start"], ll > LIT_TABLE_BITS or dl > DIST_TABLE_BITS))
        if eob:
            put(lcodes, lit_lens, 256)
        return self


def zlib_verdict(stream: bytes):
    """(True, output) when zlib inflates the raw stream to its end; (False, zlib's error text) otherwise."""
    d = zlib.decompressobj(-15)
    try:
        out = d.decompress(stream)
    except zlib.error as e:
        return False, str(e)
    if not d.eof:
        return False, "stream does not end"
    return True, out


@dataclass
class Case:
    """One stream.  `expect`: the bytes for a valid stream, None for an invalid one.  `zlib_error`: a substring of zlib's
    message for an invalid one.  `out_len`: what the decoder is told the output size is."""
    name: str
    stream: bytes
    expect: bytes | None
    zlib_error: str | None = None
    out_len: int = 0
    meta: dict = field(default_factory=dict)


def _valid(name, w: Writer, **meta) -> Case:
    assert w.out is not None, name
    return Case(name, w.bytes(), bytes(w.out), None, len(w.out), meta)


def _invalid(name, w: Writer, err: str, **meta) -> Case:
    """out_len: what a decoder that skipped the broken check would write, so that a size mismatch cannot hide the verdict."""
    return Case(name, w.bytes(), None, err, w.size, meta)


def round_offsets(sym_bits):
    """Offsets of each symbol inside the kernel's speculation rounds: a round covers the 32 bits after its first symbol, the
    next round starts at the first symbol at or after that.  sym_bits: start bits (relative to the block's first symbol)."""
    offs, base = [], 0
    for b in sym_bits:
        if b >= base + 32:
            base = b
        offs.append(b - base)
    return offs




# complete literal/length and distance sets close to the fixed code (the fixed code's own sets are complete only with the
# unusable symbols 286/287 and distances 30/31, which a dynamic block cannot declare)
LIT286 = [7, 7] + FIXED_LIT[2:286]                  # two 8-bit codes shortened to 7 bits fill the space of 286/287
LIT280 = [7] * 8 + FIXED_LIT[8:280] + [0] * 6       # length symbols 280..285 unused
DIST30 = [4, 4] + [5] * 28


def _random_bytes(rng, n: int) -> bytes:
    return bytes(rng.integers(0, 256, n).astype(np.uint8))


def _freq_lengths(data: bytes):
    """A complete literal code for `data` plus end-of-block."""
    freq = np.bincount(np.frombuffer(data, np.uint8), minlength=257)
    freq[256] = 1
    return huffman_lengths(freq.tolist(), 15)


def _long_code_block(rng, w: Writer, final: bool, n_tokens: int):
    """A dynamic block whose literal/length code reaches 15 bits on used literals and lengths, and whose distance code
    reaches 15 bits."""
    lit_syms = [65, 66, 256, 67, 265, 68, 260, 69, 270, 70, 257, 71, 280, 72, 284, 73]          # lengths 1..15, 15
    dsyms = list(range(16))
    lit, dist = staircase(lit_syms, 286), staircase(dsyms, 30)
    toks, hist = [], len(w.out)
    for _ in range(n_tokens):
        s = lit_syms[int(rng.integers(0, 16))]
        if s < 256:
            toks.append(s)
            hist += 1
        elif s > 256:
            li = s - 257
            extra = int(rng.integers(0, 1 << LEN_EXTRA[li]))
            ds = int(rng.integers(0, 16))
            while DIST_BASE[ds] > hist:
                ds -= 1
            dx = int(rng.integers(0, min(1 << DIST_EXTRA[ds], hist - DIST_BASE[ds] + 1)))
            toks.append(Sym(s, extra, ds, dx))
            hist += LEN_BASE[li] + extra
    w.dynamic(toks, lit, dist, final=final)


def _match_cases(rng, out):
    # every (dist, len) of the grid after a 32,768-byte history, with 0-2 literals between matches, so that matches sit at
    # many output offsets of a speculation round (the kernel copies lane-locally when len <= 8 and dist >= its offset + len,
    # cooperatively otherwise)
    dists = list(range(1, 10)) + [31, 32, 33, 32768]
    lens = list(range(3, 11)) + [31, 32, 33, 258]
    hist = _random_bytes(rng, 32768)
    grid = []
    for d in dists:
        for ln in lens:
            grid += [int(x) for x in rng.integers(0, 256, int(rng.integers(0, 3)))]
            grid.append((ln, d))
    out.append(_valid("match_grid_fixed", Writer().stored(hist).fixed(grid, final=True)))
    dfreq = [0] * 30
    for d in dists:
        dfreq[_dist_sym(d)[0]] = 1
    w = Writer().stored(hist).dynamic(grid, huffman_lengths([1] * 286, 15), huffman_lengths(dfreq, 15), final=True)
    out.append(_valid("match_grid_dynamic", w))
    # short codes: several short matches per round, each reading the bytes of the matches just before it
    freq = [0] * 265
    freq[65], freq[256], freq[257:265] = 50, 1, [40] * 8
    toks = [65] + [(ln, d) for d in range(1, 10) for ln in range(3, 11)] * 2
    w = Writer().stored(_random_bytes(rng, 40)).dynamic(toks, huffman_lengths(freq, 15), huffman_lengths([5] * 7, 15), final=True)
    out.append(_valid("match_grid_short_codes", w))
    # 258 written as symbol 285 and as 284 + 31 extra bits (zlib decides whether the second is legal)
    w = Writer().fixed([88, 89, 90]).fixed([Sym(285, 0, 2, 0), Sym(284, 31, 0, 0), (258, 3)], final=True)
    out.append(_valid("len258_as_285_and_as_284_plus_31", w))
    # the first match reaches back exactly to the first output byte; one byte further is too far
    out.append(_valid("match_dist_eq_pos", Writer().fixed([1, 2, 3, 4, 5, (10, 5)], final=True)))
    out.append(_invalid("match_dist_pos_plus_1", Writer().fixed([1, 2, 3, 4, 5, (10, 6)], final=True), "invalid distance too far back"))
    out.append(_invalid("match_at_start", Writer().fixed([(3, 1)], final=True), "invalid distance too far back"))
    out.append(_invalid("dist_32768_one_byte_short", Writer().stored(hist[:32767]).fixed([(3, 32768)], final=True),
                        "invalid distance too far back"))


def _long_code_cases(rng, out):
    # long-code symbols at every bit offset 0..31 of a speculation round (the kernel re-decodes them at true starts):
    # blocks are added until every offset is covered
    w = Writer().stored(_random_bytes(rng, 300))
    covered = set()
    while len(covered) < 32:
        _long_code_block(rng, w, False, 120)
        syms = w.blocks[-1]["syms"]
        covered |= {o for o, (_, slow) in zip(round_offsets([b for b, _ in syms]), syms) if slow}
    out.append(_valid("long_codes_at_every_round_offset", w.fixed([], final=True), blocks=len(w.blocks)))
    # only 13..15-bit literal codes in use (literals 76..79 of a staircase code)
    lit = staircase([256] + list(range(65, 80)), 286)
    w = Writer().dynamic([int(x) for x in rng.integers(76, 80, 200)], lit, [1], final=True)
    out.append(_valid("literal_codes_13_to_15_bits", w))
    # a round of 32 one-bit literals, then a block whose end-of-block code starts in lane 31
    lit = [0] * 257
    lit[65], lit[256], lit[66], lit[67] = 1, 2, 3, 3
    w = Writer().dynamic([65] * 32, lit, [1]).dynamic([65] * 31, lit, [1], final=True)
    out.append(_valid("one_bit_literals_eob_in_lane_31", w))


def _block_cases(rng, out):
    w = Writer().fixed([65, 66]).stored(b"").fixed([(5, 2)]).stored(b"", final=True)
    out.append(_valid("stored_empty_between_huffman", w))
    w = Writer().fixed([1, 2, 3]).stored(_random_bytes(rng, 65535)).fixed([(258, 32768), 7], final=True)
    out.append(_valid("stored_65535_between_huffman", w))
    # stored, fixed and dynamic blocks in one stream until the block after a Huffman block has started at every bit offset
    # mod 8 (the speculative path's resync, and the byte alignment of a stored block after it)
    w = Writer()

    def after_huffman():
        return {w.blocks[i + 1]["start"] % 8 for i in range(len(w.blocks) - 1) if w.blocks[i]["type"]}
    k = 0
    while k < 24 or len(after_huffman()) < 8:
        kind = k % 3 if k < 12 else int(rng.integers(0, 3))
        data = _random_bytes(rng, int(rng.integers(0, 40)))
        if kind == 0:
            w.stored(data)
        elif kind == 1:
            w.fixed(list(data) + ([(int(rng.integers(3, 20)), int(rng.integers(1, len(w.out) + 1)))] if w.out else []))
        else:
            w.dynamic(list(data), _freq_lengths(data), [1])
        k += 1
    w.fixed([9], final=True)
    out.append(_valid("mixed_blocks_at_every_bit_offset", w, offsets=sorted(after_huffman())))
    # literals only: HDIST = 1 and no distance code at all
    msg = b"literals only"
    out.append(_valid("no_distance_code", Writer().dynamic(list(msg), _freq_lengths(msg), [0], final=True)))
    # one distance code of length 1 (incomplete, legal)
    out.append(_valid("single_distance_code_of_length_1", Writer().dynamic([120, 121, (7, 2), (40, 2)], LIT286, [0, 1], final=True)))
    # code-length repeats crossing from the literal/length lengths into the distance lengths
    dist = [0] * 6 + [5] * 16 + [4] * 8                                    # distance symbols 0..5 unused
    toks = list(range(20)) + [(4, 9), (9, 17), (30, 25)]
    rl = rle_lengths(LIT280[:280]) + [(18, 12)] + rle_lengths(dist[6:])    # 280..285 and distances 0..5: one run of 12 zeros
    out.append(_valid("repeat_18_crosses_into_distance_lengths", Writer().dynamic(toks, LIT280, dist, rle=rl, final=True)))
    rl = rle_lengths(LIT280[:280]) + [(17, 4), (17, 8)] + rle_lengths(dist[6:])
    out.append(_valid("repeat_17_crosses_into_distance_lengths", Writer().dynamic(toks, LIT280, dist, rle=rl, final=True)))
    dist = [8, 8, 7, 6, 5, 4, 3, 2, 1]
    rl = rle_lengths(LIT286[:284]) + [8, (16, 3)] + rle_lengths(dist[2:])   # 16 repeats the 8 of symbol 284 into distances 0, 1
    toks = list(range(20)) + [(4, 1), (5, 2), (6, 3), (7, 4), (8, 7), (9, 20)]
    out.append(_valid("repeat_16_crosses_into_distance_lengths", Writer().dynamic(toks, LIT286, dist, rle=rl, final=True)))
    # HCLEN = 5 (16, 17, 18, 0 and 8): the fewest code-length codes that can describe a nonzero length
    lit = [8] * 255 + [0, 8]
    w = Writer().dynamic([int(x) for x in rng.integers(0, 255, 100)], lit, [0], final=True)
    out.append(_valid("hclen_5", w))
    cl = [5] * 6 + [4] * 13                                                 # all 19 code-length codes, complete
    out.append(_valid("hclen_19", Writer().dynamic(list(b"HCLEN 19"), LIT286, DIST30, clen_lens=cl, hclen=19, final=True)))


def _invalid_cases(rng, out):
    # HCLEN = 4 gives codes to 16, 17, 18 and 0 only, so every length is 0 and end-of-block has no code
    cl = [0] * 19
    cl[16], cl[17], cl[18], cl[0] = 2, 2, 2, 2
    w = Writer().dynamic([], [0] * 257, [0], rle=[(18, 138), (18, 119), 0], clen_lens=cl, hclen=4, final=True, eob=False)
    out.append(_invalid("hclen_4", w, "invalid code -- missing end-of-block"))
    lit = [0] * 257
    lit[65], lit[256] = 1, 2                                                # 'A' and end-of-block: 3/4 of the code space
    out.append(_invalid("incomplete_literal_set", Writer().dynamic([65] * 3, lit, [1], final=True), "invalid literal/lengths set"))
    out.append(_invalid("incomplete_distance_set", Writer().dynamic([65, (3, 1)], LIT286, [2, 2, 2], final=True), "invalid distances set"))
    out.append(_invalid("incomplete_distance_set_len2", Writer().dynamic([65, (3, 1)], LIT286, [2], final=True), "invalid distances set"))
    cl = [0] * 19
    for s, l in ((7, 2), (8, 2), (5, 2), (9, 3)):                            # 7/8 of the code space
        cl[s] = l
    out.append(_invalid("incomplete_code_length_set", Writer().dynamic([65], LIT286, DIST30, rle=[7, 8, 9, 5], clen_lens=cl, final=True),
                        "invalid code lengths set"))
    cl = [0] * 19
    cl[8] = 1                                                               # one code of length 1: legal for literals, not here
    out.append(_invalid("code_length_set_single_code", Writer().dynamic([65], LIT286, DIST30, rle=[8], clen_lens=cl, final=True),
                        "invalid code lengths set"))
    lit = [0] * 257
    lit[65], lit[66], lit[256] = 1, 1, 1
    out.append(_invalid("oversubscribed_literal_set", Writer().dynamic([], lit, [1], final=True), "invalid literal/lengths set"))
    out.append(_invalid("oversubscribed_distance_set", Writer().dynamic([65], LIT286, [1, 1, 1], final=True), "invalid distances set"))
    cl = [3] * 19
    out.append(_invalid("oversubscribed_code_length_set", Writer().dynamic([65], LIT286, DIST30, rle=[8], clen_lens=cl, final=True),
                        "invalid code lengths set"))
    out.append(_invalid("hlit_287", Writer().dynamic([65], LIT286 + [8], DIST30, final=True), "too many length or distance symbols"))
    out.append(_invalid("hdist_31", Writer().dynamic([65], LIT286, DIST30 + [5], final=True), "too many length or distance symbols"))
    rl = [(16, 3)] + rle_lengths(LIT286 + DIST30)
    out.append(_invalid("repeat_16_first", Writer().dynamic([65], LIT286, DIST30, rle=rl, final=True), "invalid bit length repeat"))
    rl = rle_lengths(LIT286 + DIST30[:27]) + [(18, 11)]
    out.append(_invalid("repeat_past_hlit_plus_hdist", Writer().dynamic([65], LIT286, DIST30, rle=rl, final=True),
                        "invalid bit length repeat"))
    lit = LIT286[:256] + [0] + LIT286[257:]
    out.append(_invalid("missing_end_of_block", Writer().dynamic([65], lit, DIST30, eob=False, final=True),
                        "invalid code -- missing end-of-block"))
    for s in (286, 287):
        out.append(_invalid(f"fixed_symbol_{s}", Writer().fixed([65, Sym(s)], final=True), "invalid literal/length code"))
    for d in (30, 31):
        out.append(_invalid(f"fixed_distance_{d}", Writer().fixed([65, 66, Sym(257, 0, d)], final=True), "invalid distance code"))
    out.append(_invalid("stored_bad_nlen", Writer().stored(b"abc", nlen=0x1234, final=True), "invalid stored block lengths"))
    out.append(_invalid("reserved_block_type", Writer().bits(1, 1).bits(3, 2).bits(0, 13), "invalid block type"))
    out.append(_invalid("no_final_block", Writer().fixed([65, 66]), "stream does not end"))


def cases() -> list[Case]:
    """The case table (deterministic)."""
    rng = np.random.default_rng(1951)
    out: list[Case] = []
    _match_cases(rng, out)
    _long_code_cases(rng, out)
    _block_cases(rng, out)
    _invalid_cases(rng, out)
    return out
