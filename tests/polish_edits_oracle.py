"""TEST INFRASTRUCTURE ONLY.  The polish edits VCF restated over in-memory predictions: the stitch's winners table
(tests/stitch_quality_oracle.py, Stitch.py:36-128 with label-0 winners kept) turned into records by the rules of DESIGN.md
section 4 ("Polish edits"), the text of their lines, and an applier that rebuilds the polished sequence from records."""
from __future__ import annotations

from collections import defaultdict

from oracle.stitch import BUFFER, LABEL_DECODER


def winners(bases, phred, position, index, image_region, chunk_id, region_starts, region_ends) -> dict:
    """{(position, index): (label, phred)} of the winning columns, label 0 included (the last writer in string-sorted
    chunk-id order, regions by start)."""
    order = sorted(range(len(region_starts)), key=lambda r: (int(region_starts[r]), int(region_ends[r])))
    by_region = defaultdict(list)
    for i in range(len(image_region)):
        by_region[int(image_region[i])].append(i)
    table = {}
    for r in order:
        st = int(region_starts[r])
        for i in sorted(by_region.get(r, []), key=lambda i: str(int(chunk_id[i]))):
            for pos, idx, b, q in zip(position[i].tolist(), index[i].tolist(), bases[i].tolist(), phred[i].tolist()):
                if (st > 0 and pos <= st + BUFFER) or idx < 0 or pos < 0:
                    continue
                table[(pos, idx)] = (b, q)
    return table


def stitched(table: dict) -> str:
    return "".join(LABEL_DECODER[int(table[k][0])] for k in sorted(table))


def records(table: dict, draft: str, span: tuple[int, int]) -> list[tuple]:
    """(0-based POS, REF, ALT, QUAL or None, UNCOVERED) of one contig polished over `span` (inclusive)."""
    s, e = span
    ins = defaultdict(list)
    for (p, k), (b, q) in sorted(table.items()):
        if k >= 1 and b != 0:
            ins[p].append((LABEL_DECODER[b], q))
    up = draft.upper()

    def state(p):
        w = table.get((p, 0))
        if w is None:
            return "U", None
        if w[0] == 0:
            return "D", w[1]
        return ("I", None) if LABEL_DECODER[w[0]] == up[p] else ("S", w[1])

    def alt(a, b):
        out, quals, unc = [], [], False
        for p in range(a, b + 1):
            st, q = state(p)
            if st == "S":
                out.append(LABEL_DECODER[table[(p, 0)][0]]); quals.append(q)
            elif st == "D":
                quals.append(q)
            elif st == "U":
                unc = True
            else:
                out.append(up[p])
            for base, q in ins[p]:
                out.append(base); quals.append(q)
        return "".join(out), (min(quals) if quals else None), unc

    edited = [p for p in range(s, e + 1) if state(p)[0] != "I" or ins[p]]
    runs = []
    for p in edited:
        if runs and runs[-1][1] == p - 1:
            runs[-1][1] = p
        else:
            runs.append([p, p])
    out, k = [], 0
    while k < len(runs):
        a, b = runs[k]
        alt_s, q, unc = alt(a, b)
        if not alt_s and a == s and k + 1 < len(runs) and runs[k + 1][0] == b + 2 and not alt(*runs[k + 1])[0]:
            b = runs[k + 1][1]
            alt_s, q, unc = alt(a, b)
            k += 1
        if alt_s:
            out.append((a, up[a:b + 1], alt_s, q, unc))
        elif a > s:
            out.append((a - 1, up[a - 1:b + 1], up[a - 1], q, unc))
        elif b < e:
            out.append((a, up[a:b + 2], up[b + 1], q, unc))
        else:
            out.append((a, up[a:b + 1], "", q, unc))
        k += 1
    return out


def line(contig: str, rec: tuple) -> str:
    pos, ref, alt, q, unc = rec
    return "%s\t%d\t.\t%s\t%s\t%s\t.\t%s\n" % (contig, pos + 1, ref, alt, "." if q is None else q, "UNCOVERED" if unc else ".")


def apply(recs: list[tuple], draft: str, span: tuple[int, int]) -> str:
    """Records applied to upper(draft[span]), POS in contig coordinates."""
    s, e = span
    up = draft.upper()
    out, cur = [], s
    for pos, ref, alt, _, _ in recs:
        assert pos >= cur and up[pos:pos + len(ref)] == ref, (pos, cur, ref)
        out.append(up[cur:pos]); out.append(alt)
        cur = pos + len(ref)
    out.append(up[cur:e + 1])
    return "".join(out)
