"""The contigs a whole-genome `call_variant` leaves out when no region is given: the decoy, alt, unplaced, HLA and viral
sequences of the human reference builds (hs37d5, GRCh38 analysis sets), where a call costs time and yields no usable variant.

The rule works on names alone.  A contig is excluded when its name
- ends in `_decoy`, `_alt` or `_random` (GRCh38 decoys, ALT haplotypes, unlocalized scaffolds: chr1_KI270706v1_random);
- starts with `chrUn_` (unplaced scaffolds) or `HLA-` (HLA allele sequences: HLA-A*01:01:01:01);
- is a versioned GenBank accession of a GRC scaffold: GL, JH, KB, KI, KN, KQ, KV, KZ, ML or MU, digits, a dot and a
  version (GL000207.1, KI270728.1: the unplaced contigs of b37 / hs37d5 and the unplaced, ALT and patch scaffolds of GRCh38
  in NCBI naming);
- is `chrEBV`, `hs37d5` (the hs37d5 decoy) or `NC_007605` (Epstein-Barr virus).
Names outside these shapes are kept: primary chromosomes in UCSC, Ensembl, GenBank or RefSeq naming (chr1, 1, chrX, MT,
chrM, CM000663.2, J01415.2, NC_000001.11), other organisms' chromosomes and assembly contigs (ctg1, tig00000001, contig_12)
and accessions outside the GRC scaffold prefixes (CP000001.1).  Give `-r` to call an excluded contig."""
from __future__ import annotations

import re

_EXCLUDED = re.compile(r".*_(decoy|alt|random)|chrUn_.*|HLA-.*|(GL|JH|KB|KI|KN|KQ|KV|KZ|ML|MU)\d{6}\.\d+|chrEBV|hs37d5|NC_007605")


def is_excluded_contig(name: str) -> bool:
    return _EXCLUDED.fullmatch(name) is not None


def excluded_contigs(names) -> list[str]:
    """The names of `names` the rule excludes, in their order."""
    return [c for c in names if is_excluded_contig(c)]
