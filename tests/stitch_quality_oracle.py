"""TEST INFRASTRUCTURE ONLY.  The polish stitch with per-base qualities on in-memory prediction arrays: oracle/stitch.py's
restatement of Stitch.py:36-128 with the reference's commented-out quality plumbing put back (Stitch.py:39, 55, 73, 85, 88, 91).
The table keyed by (position, index) holds (base, phred), so a base and its QV always come from the same image column (the
last writer in string-sorted chunk-id order), and the quality string is built over the bases with a non-zero label.

One deliberate deviation: the reference wrote chr(phred + 33), which turns the network's phred 94-100 into bytes 127-133,
outside FASTQ's quality alphabet; here the phred is clamped to 93 ('~')."""
from __future__ import annotations

from collections import defaultdict

from oracle.stitch import BUFFER, LABEL_DECODER

MAX_QV = 93


def qv_char(phred: int) -> str:
    return chr(33 + min(int(phred), MAX_QV))


def stitch_with_qualities(bases, phred, position, index, image_region, chunk_id, region_starts, region_ends):
    """oracle.stitch.stitch's arguments plus phred uint8 [n,1000] -> (sequence, quality string)."""
    order = sorted(range(len(region_starts)), key=lambda r: (int(region_starts[r]), int(region_ends[r])))
    by_region = defaultdict(list)
    for i in range(len(image_region)):
        by_region[int(image_region[i])].append(i)
    table = {}
    for r in order:
        st = int(region_starts[r])
        imgs = sorted(by_region.get(r, []), key=lambda i: str(int(chunk_id[i])))
        for i in imgs:
            for pos, idx, b, q in zip(position[i].tolist(), index[i].tolist(), bases[i].tolist(), phred[i].tolist()):
                if st > 0 and pos <= st + BUFFER:
                    continue
                if idx < 0 or pos < 0:
                    continue
                table[(pos, idx)] = (b, q)                                            # Stitch.py:72-73
    values = [table[k] for k in sorted(table.keys())]
    seq = "".join(LABEL_DECODER[int(b)] for b, _ in values)
    qual = "".join(qv_char(q) for b, q in values if b != 0)                          # Stitch.py:91
    return seq, qual
