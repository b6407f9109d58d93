"""CPU: the DEFLATE writer of tests/deflate_craft.py against Python's zlib.  Every valid case of the shared case table inflates
to the bytes the writer intended and reaches the end of the stream; every invalid case is rejected with the recorded message;
every valid stream cut short by 1-8 bytes does not reach its end.  This pins the table that tests/test_inflate_edges_gpu.py
runs through the GPU inflate kernel."""
import zlib

import pytest

from tests import deflate_craft as dc

CASES = dc.cases()
VALID = [c for c in CASES if c.expect is not None]
INVALID = [c for c in CASES if c.expect is None]


def test_table_is_deterministic_and_names_are_unique():
    again = dc.cases()
    assert [c.stream for c in again] == [c.stream for c in CASES]
    assert len({c.name for c in CASES}) == len(CASES)
    assert len(VALID) >= 15 and len(INVALID) >= 20


@pytest.mark.parametrize("case", VALID, ids=lambda c: c.name)
def test_valid_case_round_trips_through_zlib(case):
    d = zlib.decompressobj(-15)
    assert d.decompress(case.stream) == case.expect
    assert d.eof and d.unused_data == b""
    assert case.out_len == len(case.expect)


@pytest.mark.parametrize("case", INVALID, ids=lambda c: c.name)
def test_invalid_case_is_rejected_by_zlib(case):
    ok, msg = dc.zlib_verdict(case.stream)
    assert not ok and case.zlib_error in msg, msg


@pytest.mark.parametrize("cut", range(1, 9))
def test_shortened_streams_do_not_end(cut):
    for c in VALID:
        ok, msg = dc.zlib_verdict(c.stream[:len(c.stream) - cut])
        assert not ok, (c.name, cut)


def test_writer_matches_zlib_fixed_and_stored_encoders():
    data = b"abcdefghij0123456789"
    co = zlib.compressobj(9, zlib.DEFLATED, -15, 8, zlib.Z_FIXED)
    assert dc.Writer().fixed(list(data), final=True).bytes() == co.compress(data) + co.flush()
    w = dc.Writer().stored(data, final=True)
    assert w.bytes() == bytes([1, len(data), 0, 0xff - len(data), 0xff]) + data
    assert zlib.decompress(dc.Writer().fixed([65, (258, 1), (3, 259)], final=True).bytes(), -15) == b"A" * 262


def test_code_sets_are_complete_where_the_table_relies_on_it():
    full = 1 << 15
    assert dc.kraft(dc.FIXED_LIT) == full and dc.kraft(dc.FIXED_DIST) == full
    assert dc.kraft(dc.LIT286) == full and dc.kraft(dc.LIT280) == full and dc.kraft(dc.DIST30) == full
    assert dc.kraft(dc.FIXED_LIT[:286]) < full              # why LIT286 exists
    for freqs in ([1] * 286, [5, 0, 0, 1], [1000, 1] + [1] * 30, [2 ** k for k in range(20)]):
        lens = dc.huffman_lengths(freqs, 7 if len(freqs) <= 19 else 15)
        assert dc.kraft(lens) == full and max(lens) <= 15


def test_table_covers_the_kernel_edges():
    by = {c.name: c for c in CASES}
    # long codes at every bit offset of a speculation round, block boundaries at every bit offset mod 8
    assert by["long_codes_at_every_round_offset"].meta["blocks"] > 2
    assert by["mixed_blocks_at_every_bit_offset"].meta["offsets"] == list(range(8))
    assert dc.round_offsets([0, 5, 31, 32, 40, 70, 80]) == [0, 5, 31, 0, 8, 0, 10]
    # a distance of exactly 32,768 and the 65,535-byte stored block
    assert len(by["stored_65535_between_huffman"].expect) > 65535
    assert by["match_grid_fixed"].out_len > 32768
