"""``genome --vcf``: the haplotypes of a VCF's first sample as flat tables for ``ns_apply_variants``.

The VCF (4.x, plain or gzip/BGZF) is parsed with numpy over the whole file at once: tab, colon and comma positions are
found in one pass, and every column is sliced out of the byte buffer for all records together, so the cost per record
is a few array operations rather than a Python call.  Semantics (DESIGN §3, "Mode-specific design"):

* only records whose FILTER is ``PASS`` or ``.`` are applied; the others are skipped unchecked and counted;
* the first sample's ``GT``: ``|`` and ``/`` alike, the first allele goes to haplotype 1, the second to haplotype 2 (the
  order of ``bcftools consensus -H 1`` / ``-H 2``); ``0`` and ``.`` are the reference, ``k`` is ``ALT[k-1]``, ``*`` is
  the reference (a deletion on that haplotype already covers the position);
* REF must equal the reference bytes (case-insensitively); applied spans of one haplotype may touch but not overlap;
  all records of one chromosome have the same ploidy (1 or 2), a chromosome without records gets 2 copies;
* the symbolic structural variants ``<DEL>``, ``<INV>``, ``<DUP>`` and ``<DUP:TANDEM>`` are applied; every other
  symbolic or breakend ALT that a haplotype takes is an error, one that no haplotype takes is not checked.  A record
  whose allele a haplotype takes as one of those four has exactly one ALT and a one-base REF (the padding base at POS,
  which stays the FASTA's byte).  Its affected bases are POS+1 .. END (1-based, inclusive), END from INFO ``END=e``
  (END = e) or ``SVLEN=s`` (END = POS + |s|: VCF 4.3 writes deletions as negative, 4.4 as positive); with both they must
  agree, and POS < END <= the record's length.  With P = POS and E = END, ``ref[P:E]`` is what changes: ``<DEL>`` gives
  ``ref[:P] + ref[E:]``, ``<INV>`` ``ref[:P] + rc(ref[P:E]) + ref[E:]`` and ``<DUP>``/``<DUP:TANDEM>``
  ``ref[:E] + ref[P:E] + ref[E:]`` (one extra copy, in tandem).  ``rc`` reverses and complements A-T, C-G, R-Y, K-M,
  B-V and D-H in either case, keeping the case; every other byte stays.  For the overlap rule the record's span is
  ``[POS-1, END)``, the padding base included.  Only these few records are read one by one (their INFO).

Every error is a ``VcfError`` whose message names the line (1-based, header lines included).
"""
import gzip
import re

import numpy as np

_PASS = (b"PASS", b".")
_SYMBOLIC = {b"<DEL>": 1, b"<INV>": 2, b"<DUP>": 3, b"<DUP:TANDEM>": 3}     # the structural variants applied
_SV_DEL, _SV_INV, _SV_DUP = 1, 2, 3
_NUMBER = re.compile(rb"[+-]?[0-9]{1,18}")
_UPPER = np.arange(256, dtype=np.uint8)
_UPPER[ord("a"):ord("z") + 1] -= 32
_NOT_SEQUENCE = np.ones(256, dtype=bool)            # an applied ALT is IUPAC nucleotide codes in either case; this rejects
_NOT_SEQUENCE[np.frombuffer(b"ACGTUNRYSWKMBDHVacgtunryswkmbdhv", dtype=np.uint8)] = False    # <DEL>, N[chr2:5[, .A, G;X
_CHUNK = 1 << 18                                    # records per step of the fixed-width column gathers


class VcfError(ValueError):
    def __init__(self, line, msg):
        super().__init__(msg if line is None else "line %d: %s" % (line, msg))
        self.line = line


class HaplotypeTables:
    """What ``ns_apply_variants`` takes (``NsVariants``), plus the haplotype records' names and lengths.

    For haplotype record h (in order: reference records in file order, each with its copies in haplotype order):
    ``hap_chrom[h]`` is its source reference record, ``hap_number[h]`` 1 or 2, and its variants are
    ``var_off[h] .. var_off[h+1]``, in position order: reference span ``[var_pos, var_pos + var_ref_len)`` of that
    record, replaced by what ``alt_kind`` says: 0 ``alt[alt_off : alt_off + alt_len]``, 1 the source record's own bases
    ``[alt_off, alt_off + alt_len)``, 2 those bases reverse-complemented.  Symbolic alleles are encoded as
    ``<DEL>``: kind 0 with ``alt_len`` 0 (no other variant has an empty ALT); ``<INV>``: ``var_pos = alt_off = P``,
    ``var_ref_len = alt_len = E - P``, kind 2; ``<DUP>``: ``var_pos = E``, ``var_ref_len = 0``, ``alt_off = P``,
    ``alt_len = E - P``, kind 1."""

    def __init__(self, names, hap_chrom, hap_number, var_off, var_pos, var_ref_len, alt_off, alt_len, alt, lengths, skipped,
                 skipped_elsewhere=0, alt_kind=None):
        self.names = list(names)
        self.hap_chrom = np.ascontiguousarray(hap_chrom, dtype=np.uint32)
        self.hap_number = np.ascontiguousarray(hap_number, dtype=np.uint8)
        self.var_off = np.ascontiguousarray(var_off, dtype=np.uint64)
        self.var_pos = np.ascontiguousarray(var_pos, dtype=np.uint64)
        self.var_ref_len = np.ascontiguousarray(var_ref_len, dtype=np.uint32)
        self.alt_off = np.ascontiguousarray(alt_off, dtype=np.uint64)
        self.alt_len = np.ascontiguousarray(alt_len, dtype=np.uint32)
        self.alt = np.ascontiguousarray(alt, dtype=np.uint8)
        self.lengths = np.ascontiguousarray(lengths, dtype=np.int64)    # bases of every haplotype record
        self.skipped = np.ascontiguousarray(skipped, dtype=np.int64)    # records of its chromosome skipped by FILTER
        self.skipped_elsewhere = int(skipped_elsewhere)     # records skipped by FILTER on contigs the reference lacks
        self.alt_kind = np.ascontiguousarray(np.zeros(len(self.var_pos)) if alt_kind is None else alt_kind, dtype=np.uint8)
        self.ref_paired = None      # read_vcf: paired_ref_bytes over the reference the tables were read against

    @property
    def applied(self):
        return np.diff(self.var_off.astype(np.int64))

    @property
    def structural(self):
        """(n_hap, 3): per haplotype record, the deletions, inversions and duplications applied from symbolic alleles."""
        n = len(self.hap_chrom)
        h = np.repeat(np.arange(n), self.applied)
        kinds = ((self.alt_kind == 0) & (self.alt_len == 0), self.alt_kind == 2, self.alt_kind == 1)
        return np.stack([np.bincount(h[k], minlength=n) for k in kinds], axis=1)

    @property
    def offsets(self):
        return np.concatenate([[0], np.cumsum(self.lengths)]).astype(np.uint64)


def paired_ref_bytes(tables, ref):
    """The reference bytes [var_pos, var_pos + min(alt_len, var_ref_len)) of every kind-0 variant of ``tables``, back to
    back in table order: the REF bases a lifted alignment pairs an ALT's first bases with, which NM compares them to
    (``ns_set_aln_tags``).  ``ref``: the PackedReference the tables were read against."""
    n = np.where(tables.alt_kind == 0, np.minimum(tables.alt_len, tables.var_ref_len), 0).astype(np.int64)
    chrom = np.repeat(tables.hap_chrom.astype(np.int64), np.diff(tables.var_off.astype(np.int64)))
    pos, _ = _flat(np.asarray(ref.offsets, dtype=np.int64)[chrom] + tables.var_pos.astype(np.int64), n)
    return np.ascontiguousarray(np.asarray(ref.bases)[pos], dtype=np.uint8)


def _read_bytes(path):
    with open(path, "rb") as f:
        magic = f.read(2)
    if magic == b"\x1f\x8b":                        # gzip or BGZF (concatenated members)
        with gzip.open(path, "rb") as f:
            return f.read()
    with open(path, "rb") as f:
        return f.read()


def _gather(buf, s, e):
    """Bytes [s, e) of every row as a fixed-width (rows, W) uint8 matrix, zero-padded."""
    w = int((e - s).max()) if len(s) else 0
    w = max(w, 1)
    idx = s[:, None] + np.arange(w, dtype=np.int64)[None, :]
    keep = idx < e[:, None]
    m = buf[np.minimum(idx, len(buf) - 1)]
    m[~keep] = 0
    return m


def _codes(buf, s, e):
    """Dictionary encoding of the byte strings [s, e): (list of distinct strings, code per row)."""
    uniq, code = {}, np.empty(len(s), dtype=np.int64)
    for lo in range(0, len(s), _CHUNK):
        m = _gather(buf, s[lo:lo + _CHUNK], e[lo:lo + _CHUNK])
        u, inv = np.unique(np.ascontiguousarray(m).view("S%d" % m.shape[1]).ravel(), return_inverse=True)
        g = np.array([uniq.setdefault(bytes(x), len(uniq)) for x in u], dtype=np.int64)
        code[lo:lo + _CHUNK] = g[inv.ravel()]
    return list(uniq), code


def _integers(buf, s, e, line, what):
    """Decimal integers [s, e), or VcfError at the first row that is not one."""
    out = np.empty(len(s), dtype=np.int64)
    for lo in range(0, len(s), _CHUNK):
        ss, ee = s[lo:lo + _CHUNK], e[lo:lo + _CHUNK]
        m = _gather(buf, ss, ee).astype(np.int64) - 48
        n = ee - ss
        col = np.arange(m.shape[1])[None, :]
        inside = col < n[:, None]
        bad = (inside & ((m < 0) | (m > 9))).any(axis=1) | (n == 0) | (n > 18)
        if bad.any():
            raise VcfError(line[lo + int(np.argmax(bad))], "%s is not a number" % what)
        place = np.where(inside, n[:, None] - 1 - col, 0)
        out[lo:lo + _CHUNK] = (np.where(inside, m, 0) * 10 ** place).sum(axis=1)
    return out


def _first(mask, line, msg):
    if mask.any():
        raise VcfError(line[int(np.argmax(mask))], msg)


def _flat(s, n):
    """Positions s[i] .. s[i] + n[i] - 1 of every row, back to back, and each position's row."""
    total = int(n.sum())
    row = np.repeat(np.arange(len(s)), n)
    start = np.concatenate([[0], np.cumsum(n)[:-1]]) if len(n) else np.zeros(0, dtype=np.int64)
    return np.repeat(s - start, n) + np.arange(total, dtype=np.int64), row


def read_vcf(path, ref):
    """The haplotypes of ``path``'s first sample over ``ref`` (a PackedReference with host bases) -> HaplotypeTables.

    The checks run one kind at a time over all records, each finding its first offending line.  Every check looks at a
    record and the records before it only, so the file's first error is found by parsing again the records before the
    line reported, until no error is left there."""
    buf = np.frombuffer(_read_bytes(path), dtype=np.uint8)
    first_error, limit = None, None
    while True:
        try:
            tables = _read_records(buf, ref, path, limit)
        except VcfError as e:
            if e.line is None or (limit is not None and e.line >= limit):       # the header's own errors
                raise
            first_error, limit = e, e.line
            continue
        if first_error is not None:
            raise first_error
        tables.ref_paired = paired_ref_bytes(tables, ref)
        return tables


def _read_records(buf, ref, path, limit):
    """read_vcf over the records before line ``limit`` (None: all of them)."""
    nl = np.flatnonzero(buf == 10)
    starts = np.concatenate([[0], nl + 1]).astype(np.int64)
    ends = np.concatenate([nl, [len(buf)]]).astype(np.int64)
    if len(starts) and starts[-1] == len(buf):
        starts, ends = starts[:-1], ends[:-1]
    ends = ends - ((ends > starts) & (buf[np.maximum(ends - 1, 0)] == 13))        # CRLF
    lineno = np.arange(1, len(starts) + 1, dtype=np.int64)
    nonempty = ends > starts
    header = nonempty & (buf[np.minimum(starts, max(len(buf) - 1, 0))] == ord("#"))
    chrom_line = [i for i in np.flatnonzero(header) if bytes(buf[starts[i]:starts[i] + 6]) == b"#CHROM"]
    if not chrom_line:
        raise VcfError(None, "%s has no #CHROM header line" % path)
    cl = chrom_line[-1]
    if len(bytes(buf[starts[cl]:ends[cl]]).split(b"\t")) < 10:
        raise VcfError(lineno[cl], "the VCF has no sample column")
    body = np.flatnonzero(nonempty & ~header & ((lineno < limit) if limit is not None else True))
    s, e, line = starts[body], ends[body], lineno[body]

    tabs = np.flatnonzero(buf == 9)
    t0 = np.searchsorted(tabs, s)
    n_tabs = np.searchsorted(tabs, e) - t0
    _first(n_tabs < 9, line, "fewer than 10 columns (a sample column is needed)")
    tabs = np.concatenate([tabs, [len(buf)]])

    def field(k):
        fs = s if k == 0 else tabs[t0 + k - 1] + 1
        fe = np.where(n_tabs > k, tabs[np.minimum(t0 + k, len(tabs) - 1)], e)
        return fs, fe

    # FILTER first: records it skips are not checked
    filt, filt_code = _codes(buf, *field(6))
    passing = np.isin(filt_code, [i for i, f in enumerate(filt) if f in _PASS])
    chrom_names, chrom_code = _codes(buf, *field(0))
    raw_index = {n.encode(): i for i, n in enumerate(ref.raw_names)}
    chrom_of = np.array([raw_index.get(c, -1) for c in chrom_names], dtype=np.int64)
    rec_chrom_all = chrom_of[chrom_code] if len(chrom_code) else np.zeros(0, dtype=np.int64)
    n_ref = len(ref.names)
    skipped_chrom = np.bincount(rec_chrom_all[~passing & (rec_chrom_all >= 0)], minlength=n_ref)
    skipped_elsewhere = int((~passing & (rec_chrom_all < 0)).sum())

    keep = np.flatnonzero(passing)
    s, e, line, t0, n_tabs = s[keep], e[keep], line[keep], t0[keep], n_tabs[keep]
    rec_chrom = rec_chrom_all[keep]
    if (rec_chrom < 0).any():
        i = int(np.argmax(rec_chrom < 0))
        raise VcfError(line[i], "unknown contig %s (not a record of the reference)" % chrom_names[chrom_code[keep][i]].decode(errors="replace"))

    pos = _integers(buf, *field(1), line, "POS")
    ref_s, ref_e = field(3)
    alt_s, alt_e = field(4)

    # GT: its index in FORMAT, then that subfield of the first sample
    fmts, fmt_code = _codes(buf, *field(8))
    gt_index = np.array([f.split(b":").index(b"GT") if b"GT" in f.split(b":") else -1 for f in fmts], dtype=np.int64)
    rec_gt = gt_index[fmt_code] if len(fmt_code) else np.zeros(0, dtype=np.int64)
    _first(rec_gt < 0, line, "FORMAT has no GT")
    smp_s, smp_e = field(9)
    colons = np.flatnonzero(buf == ord(":"))
    c0 = np.searchsorted(colons, smp_s)
    n_sub = np.searchsorted(colons, smp_e) - c0 + 1
    _first(rec_gt >= n_sub, line, "the sample has no GT value")
    colons = np.concatenate([colons, [len(buf)]])
    gt_s = np.where(rec_gt == 0, smp_s, colons[np.minimum(c0 + rec_gt - 1, len(colons) - 1)] + 1)
    gt_e = np.where(rec_gt + 1 < n_sub, colons[np.minimum(c0 + rec_gt, len(colons) - 1)], smp_e)
    gts, gt_code = _codes(buf, gt_s, gt_e)
    parsed = []
    for g in gts:
        try:
            al = [0 if a == b"." else int(a) for a in g.replace(b"|", b"/").split(b"/")]
            ok = 1 <= len(al) <= 2 and min(al) >= 0
        except ValueError:
            al, ok = [], False
        parsed.append((len(al), al[0] if al else 0, al[1] if len(al) > 1 else 0, ok))
    table = np.array(parsed, dtype=np.int64).reshape(-1, 4)
    gt = table[gt_code] if len(gt_code) else np.zeros((0, 4), dtype=np.int64)
    _first(gt[:, 3] == 0, line, "GT is not one or two allele indices")
    ploidy, allele = gt[:, 0], gt[:, 1:3]

    # ploidy: every record of a chromosome agrees; a chromosome without records gets 2 copies
    chrom_ploidy = np.full(n_ref, 2, dtype=np.int64)
    if len(rec_chrom):
        u, first = np.unique(rec_chrom, return_index=True)
        chrom_ploidy[u] = ploidy[first]
        _first(ploidy != chrom_ploidy[rec_chrom], line, "GT ploidy differs from the chromosome's earlier records")

    # REF: inside the record, equal to the reference bytes
    ref_len = ref_e - ref_s
    _first(ref_len == 0, line, "empty REF")
    offs = ref.offsets.astype(np.int64)
    clen = offs[rec_chrom + 1] - offs[rec_chrom]
    _first((pos < 1) | (pos - 1 + ref_len > clen), line, "REF extends past the end of the reference record")
    vcf_idx, row = _flat(ref_s, ref_len)
    ref_idx, _ = _flat(offs[rec_chrom] + pos - 1, ref_len)
    bad = _UPPER[buf[vcf_idx]] != _UPPER[ref.bases[ref_idx]]
    if bad.any():
        raise VcfError(line[row[int(np.argmax(bad))]], "REF does not match the reference")

    # the ALT each haplotype takes: k -> ALT[k-1]
    commas = np.flatnonzero(buf == ord(","))
    a0 = np.searchsorted(commas, alt_s)
    n_alt = np.searchsorted(commas, alt_e) - a0 + 1
    commas = np.concatenate([commas, [len(buf)]])
    items = []          # (hap record key, record, alt start, alt len) per applied allele
    hap_base = np.concatenate([[0], np.cumsum(chrom_ploidy)])
    for h in range(2):
        k = allele[:, h]
        on = np.flatnonzero((ploidy > h) & (k > 0))
        _first((ploidy > h) & (k > n_alt), line, "a GT allele index is larger than the number of ALT alleles")
        kk = k[on]
        s_ = np.where(kk == 1, alt_s[on], commas[np.minimum(a0[on] + kk - 2, len(commas) - 1)] + 1)
        e_ = np.where(kk < n_alt[on], commas[np.minimum(a0[on] + kk - 1, len(commas) - 1)], alt_e[on])
        star = (e_ - s_ == 1) & (buf[np.minimum(s_, len(buf) - 1)] == ord("*"))
        on, s_, e_ = on[~star], s_[~star], e_[~star]
        items.append((hap_base[rec_chrom[on]] + h, on, s_, e_ - s_))
    key = np.concatenate([it[0] for it in items])
    rec = np.concatenate([it[1] for it in items])
    a_s = np.concatenate([it[2] for it in items])
    a_n = np.concatenate([it[3] for it in items])
    order = np.lexsort((rec, key))          # per haplotype record, in file order
    key, rec, a_s, a_n = key[order], rec[order], a_s[order], a_n[order]

    # the structural variants applied (a symbolic allele starts with '<'; few alleles do); they have no ALT bytes
    sv_type = np.zeros(len(rec), dtype=np.int64)
    for i in np.flatnonzero(buf[np.minimum(a_s, len(buf) - 1)] == ord("<")).tolist():
        sv_type[i] = _SYMBOLIC.get(bytes(buf[a_s[i]:a_s[i] + a_n[i]]), 0)
    sv = sv_type > 0
    a_n = np.where(sv, 0, a_n)

    bad_len = (a_n == 0) & ~sv
    alt_idx, arow = _flat(a_s, a_n)
    bad_byte = np.zeros(len(rec), dtype=bool)
    bad_byte[arow[_NOT_SEQUENCE[buf[alt_idx]]]] = True
    bad = bad_len | bad_byte
    if bad.any():
        raise VcfError(line[rec[bad]].min(), "a haplotype takes an ALT allele that is symbolic, a breakend, missing or not a "
                       "nucleotide sequence")

    # span end of every record (0-based, exclusive): END for a structural variant, checked record by record in file order
    rec_end = pos - 1 + ref_len
    if sv.any():
        info_s, info_e = field(7)
        for r in np.unique(rec[sv]).tolist():
            rec_end[r] = _sv_end(bytes(buf[info_s[r]:info_e[r]]), int(pos[r]), int(ref_len[r]), int(n_alt[r]), int(clen[r]), int(line[r]))

    # overlap: on one haplotype, a span that starts before the previous applied span ends
    v_pos = pos[rec] - 1
    v_end = rec_end[rec]
    same = key[1:] == key[:-1]
    over = same & (v_pos[1:] < v_end[:-1])
    if over.any():
        r = rec[1:][over][np.argmin(line[rec[1:][over]])]
        h = int(key[1:][over][np.argmin(line[rec[1:][over]])] - hap_base[rec_chrom[r]]) + 1
        raise VcfError(line[r], "overlaps an earlier variant on haplotype %d" % h)

    n_hap = int(hap_base[-1])
    hap_chrom = np.repeat(np.arange(n_ref), chrom_ploidy)
    hap_number = np.arange(n_hap) - hap_base[hap_chrom] + 1
    counts = np.bincount(key, minlength=n_hap)
    var_off = np.concatenate([[0], np.cumsum(counts)])
    # the table rows (HaplotypeTables), then the structural variants' own: P = POS and E = END
    t_pos, t_ref_len, t_alt_len, kind = v_pos, ref_len[rec], a_n, None
    t_alt_off = np.concatenate([[0], np.cumsum(a_n)[:-1]]) if len(a_n) else a_n
    if sv.any():
        P, E = pos[rec], rec_end[rec]
        t_pos = np.where(sv_type == _SV_DUP, E, np.where(sv, P, v_pos))
        t_ref_len = np.where(sv_type == _SV_DUP, 0, np.where(sv, E - P, t_ref_len))
        t_alt_off = np.where(sv_type >= _SV_INV, P, t_alt_off)
        t_alt_len = np.where(sv_type >= _SV_INV, E - P, a_n)
        kind = np.select([sv_type == _SV_INV, sv_type == _SV_DUP], [2, 1], 0)
    grow = np.concatenate([[0], np.cumsum(t_alt_len - t_ref_len)])
    delta = grow[var_off[1:]] - grow[var_off[:-1]]
    lengths = (offs[1:] - offs[:-1])[hap_chrom] + delta
    names = ["%s-hap%d" % (ref.names[c], h) for c, h in zip(hap_chrom, hap_number)]
    return HaplotypeTables(names, hap_chrom, hap_number, var_off, t_pos, t_ref_len, t_alt_off, t_alt_len, buf[alt_idx], lengths,
                           skipped_chrom[hap_chrom], skipped_elsewhere, kind)


def _sv_end(info, pos, ref_len, n_alt, clen, line):
    """END of a record whose allele a haplotype takes as a structural variant: its span's 0-based exclusive end."""
    if n_alt > 1:
        raise VcfError(line, "a symbolic structural variant must be the record's only ALT allele")
    if ref_len != 1:
        raise VcfError(line, "the REF of a symbolic structural variant must be one base (the padding base)")
    value = {}
    for item in info.split(b";"):
        k, _, v = item.partition(b"=")
        if k in (b"END", b"SVLEN") and k not in value:
            if not _NUMBER.fullmatch(v):
                raise VcfError(line, "INFO %s is not a number" % k.decode())
            value[k] = int(v)
    if not value:
        raise VcfError(line, "a symbolic structural variant needs END or SVLEN in INFO")
    end = value.get(b"END", pos + abs(value.get(b"SVLEN", 0)))
    if b"SVLEN" in value and end != pos + abs(value[b"SVLEN"]):
        raise VcfError(line, "END (%d) and SVLEN (%d) disagree" % (end, value[b"SVLEN"]))
    if end <= pos:
        raise VcfError(line, "END (%d) is not past POS (%d)" % (end, pos))
    if end > clen:
        raise VcfError(line, "END (%d) extends past the end of the reference record (%d bases)" % (end, clen))
    return end
