"""Transcriptome ``--spliced_bam``: where every transcript lies on the genome (DESIGN §3 "Spliced mapped BAM"), as the flat
tables ``ns_set_splice`` takes.

The exons come from the GFF3 intron retention reads (``intron_retention.TranscriptStructures``, so seqid matching and its
``chr`` rule agree with intron retention).  A transcript's map is its exons sorted by coordinate and put in transcript
order: ascending on the plus strand, descending on the minus strand, whichever order the GFF3 lists them in (GENCODE
lists minus-strand exons descending).  Transcript base x is then one genome base, forward on the plus strand and
backward and complemented on the minus strand."""
import numpy as np

from .intron_retention import EXON


class SpliceMap:
    """Per transcript t its exons ``exon_off[t] .. exon_off[t+1]`` in transcript order (genome record, start, length; none:
    no map), its strand, the genome records' lengths, and the resident index of genome record 0 (None: the genome is not
    resident)."""

    def __init__(self, exon_off, exon_chrom, exon_start, exon_len, minus, genome_len, genome_first=None):
        self.exon_off, self.exon_chrom, self.exon_start, self.exon_len = exon_off, exon_chrom, exon_start, exon_len
        self.minus, self.genome_len, self.genome_first = minus, genome_len, genome_first

    def has_map(self):
        return np.diff(self.exon_off) > 0

    def exons(self, t):
        """Transcript t's exons in transcript order: [(genome record, start, end)]."""
        a, b = int(self.exon_off[t]), int(self.exon_off[t + 1])
        return [(int(c), int(s), int(s) + int(n)) for c, s, n in zip(self.exon_chrom[a:b], self.exon_start[a:b], self.exon_len[a:b])]


def build_splice_map(st, trx_lengths, genome_lengths, genome_first=None):
    """The SpliceMap of TranscriptStructures ``st`` (one per transcript record, of ``trx_lengths`` bases) on genome records
    of ``genome_lengths`` bases.  A transcript has no map when it has no exons, its exons lie on two records or two
    strands, overlap, an exon is empty or lies outside its record, their lengths do not add up to its length, or its
    chromosome is absent from the genome."""
    n = len(st.first) - 1
    trx_lengths = np.asarray(trx_lengths, dtype=np.int64)
    glen = np.asarray(genome_lengths, dtype=np.int64)
    owner = np.repeat(np.arange(n), np.diff(st.first))
    sel = st.ftype == EXON
    o, c, s, e, m = owner[sel], st.chrom[sel].astype(np.int64), st.start[sel], st.end[sel], st.minus[sel]
    order = np.lexsort((s, o))                                  # by transcript, then by coordinate
    o, c, s, e, m = o[order], c[order], s[order], e[order], m[order]
    bad = np.bincount(o, minlength=n) == 0
    known = (c >= 0) & (c < len(glen))
    rec_len = np.zeros(len(c), dtype=np.int64)
    rec_len[known] = glen[c[known]]
    outside = ~known | (s < 0) | (e <= s) | (e > rec_len)
    bad[o[outside]] = True
    same = o[1:] == o[:-1]
    clash = same & ((c[1:] != c[:-1]) | (m[1:] != m[:-1]) | (s[1:] < e[:-1]))
    bad[o[1:][clash]] = True
    total = np.zeros(n, dtype=np.int64)
    np.add.at(total, o, e - s)
    bad |= total != trx_lengths
    keep = ~bad[o]
    o, c, s, e, m = o[keep], c[keep], s[keep], e[keep], m[keep]
    cnt = np.bincount(o, minlength=n)
    exon_off = np.zeros(n + 1, dtype=np.uint64)
    exon_off[1:] = np.cumsum(cnt)
    first = exon_off[:-1].astype(np.int64)
    k = np.arange(len(o)) - first[o]                            # place by coordinate within the transcript
    dst = np.where(m, first[o] + cnt[o] - 1 - k, first[o] + k)
    exon_chrom, exon_start, exon_len = (np.zeros(len(o), dtype=np.uint32) for _ in range(3))
    exon_chrom[dst], exon_start[dst], exon_len[dst] = c, s, e - s
    minus = np.zeros(n, dtype=np.uint8)
    minus[o] = m
    return SpliceMap(exon_off, exon_chrom, exon_start, exon_len, minus, glen.astype(np.uint64), genome_first)
