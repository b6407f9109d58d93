"""numpy statement of the gVCF rules (DESIGN.md section 4, "gVCF"): the binomial reference-confidence PL / GQ of each position,
the reference blocks over a track of (n_ref, n_alt) pairs, and the record-line rewrite.  Float64 numpy arithmetic with no fused
operations: the device computes each value with the same IEEE operations, so the two agree bit for bit."""
import math

import numpy as np

E = 0.001
A, B, H = math.log10(1.0 - E), math.log10(E), math.log10(0.5)


def pl_gq(n_ref, n_alt):
    """(PL [n, 3] int64, GQ [n] int64) of the counts."""
    r = np.asarray(n_ref, np.float64)
    x = np.asarray(n_alt, np.float64)
    l00 = r * A + x * B
    l01 = (r + x) * H
    l11 = r * B + x * A
    mx = np.maximum(np.maximum(l00, l01), l11)
    pl = np.stack([np.floor(10.0 * (mx - l) + 0.5) for l in (l00, l01, l11)], -1).astype(np.int64)
    gq = np.minimum(99, np.maximum(0, np.minimum(pl[..., 1], pl[..., 2]) - pl[..., 0]))
    return pl, gq


def counts_from_columns(ref_char: str, fwd, rev):
    """(n_ref, n_alt) of one position from the count matrix's columns 8-14 (fwd) and 19-25 (rev): A, C, G, T, I, D, other."""
    R = ref_char.upper()
    if R not in "ACGT":
        return 0, 0
    c = [abs(int(f)) + abs(int(r)) for f, r in zip(fwd, rev)]
    i, d, other = c[4], c[5], c[6]
    k = "ACGT".index(R)
    return max(0, c[k] - i - d), sum(c[b] for b in range(4) if b != k) + other + i + d


def blocks(track, segments, masks, ref: bytes, names, binsize: int = 5):
    """Block lines of a track: list of (contig id, 0-based pos, length, text)."""
    track = np.asarray(track, np.uint32)
    T = track.shape[0]
    nr, na = (track & 0xFFFF).astype(np.int64), (track >> 16).astype(np.int64)
    dp = nr + na
    pl, gq = pl_gq(nr, na)
    key = np.where(dp == 0, -1, gq // binsize)
    masked = np.zeros(T, bool)
    for a, b in np.asarray(masks, np.int64).reshape(-1, 2):
        masked[max(a, 0):min(b, T)] = True
    brk = np.zeros(T + 1, bool)
    toff = np.array([s["toff"] for s in segments], np.int64)
    for s in segments:
        if s["len"] > 0:
            brk[s["toff"]] = True
    keym = np.where(masked, -2, key)
    prev = np.concatenate([[-2], keym[:-1]])
    nxt = np.concatenate([keym[1:], [-2]])
    starts = np.flatnonzero((keym != -2) & (brk[:T] | (prev != keym)))
    ends = np.flatnonzero((keym != -2) & (brk[1:] | (nxt != keym)))
    out = []
    for a, b in zip(starts.tolist(), ends.tolist()):
        s = segments[int(np.searchsorted(toff, a, side="right")) - 1]
        pos = int(s["pos0"]) + a - int(s["toff"])
        last1 = int(s["pos0"]) + b - int(s["toff"]) + 1
        r = chr(ref[int(s["ref_off"]) + a - int(s["toff"])]).upper()
        r = r if r in "ACGT" else "N"
        k = a + int(np.argmin(gq[a:b + 1]))
        mdp = int(dp[a:b + 1].min())
        gt = "./." if mdp == 0 else "0/0"
        text = "%s\t%d\t.\t%s\t<*>\t.\t.\tEND=%d\tGT:GQ:MIN_DP:PL\t%s:%d:%d:%d,%d,%d\n" % (
            names[int(s["contig"])], pos + 1, r, last1, gt, int(gq[k]), mdp, *pl[k].tolist())
        out.append((int(s["contig"]), pos, b - a + 1, text))
    return out


def record_line(line: str) -> str:
    """A PEPPER_VARIANT_FULL line as the gVCF writes it: ",<*>" after ALT, ",." after AP, AD and VAF."""
    f = line.rstrip("\n").split("\t")
    f[4] += ",<*>"
    s = f[9].split(":")
    for i in (1, 4, 5):
        s[i] += ",."
    f[9] = ":".join(s)
    return "\t".join(f) + "\n"


def strip_record(line: str) -> str:
    """record_line's inverse."""
    f = line.rstrip("\n").split("\t")
    assert f[4].endswith(",<*>")
    f[4] = f[4][:-4]
    s = f[9].split(":")
    for i in (1, 4, 5):
        assert s[i].endswith(",.")
        s[i] = s[i][:-2]
    f[9] = ":".join(s)
    return "\t".join(f) + "\n"
