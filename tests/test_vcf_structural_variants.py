"""genome --vcf with the symbolic structural variants <DEL>, <INV>, <DUP> and <DUP:TANDEM> (nanosim_b200/variants.py,
alt_kind of ns_apply_variants, the reverse-complement path of hap_gather_kernel).

The reference implementation is ``build_haplotypes`` below, written from the semantics in DESIGN §3 ("Sample genome"):
it reads the VCF line by line and splices strings.  The parser's tables, spliced on the host with their kinds, must equal
it on the CPU; the device's haplotype bytes must equal it on the GPU, and ``genome -rg R --vcf V`` must write exactly what
``genome -rg H`` writes, H being the builder's FASTA of the haplotype records."""
import copy
import gzip
import os

import numpy as np
import pytest

import parity_checks as pc
import synth
from nanosim_b200.reference_fasta import PackedReference, normalise_name
from nanosim_b200.variants import VcfError, read_vcf

HEADER = ("##fileformat=VCFv4.3\n##contig=<ID=chr1>\n##ALT=<ID=DEL,Description=\"Deletion\">\n"
          "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tSAMPLE\n")
COMPLEMENT = bytes.maketrans(b"ATCGRYKMBVDHatcgrykmbvdh", b"TAGCYRMKVBHDtagcyrmkvbhd")     # every other byte stays


def rc(seq):
    return seq.translate(COMPLEMENT)[::-1]


def test_reverse_complement():
    assert rc(b"ACGTRYKMBVDHSWNU") == b"UNWSDHBVKMRYACGT"
    assert rc(b"acgtrykmbvdhswnu*-\x00\xff") == b"\xff\x00-*unwsdhbvkmryacgt"


def _sv_end(pos, info):
    kv = dict(x.split("=", 1) for x in info.split(";") if "=" in x)
    if "END" in kv:
        return int(kv["END"])
    return pos + abs(int(kv["SVLEN"]))


def build_haplotypes(records, vcf_text):
    """Reference implementation: [(fasta header, bytes)] + VCF text -> [(``{key}-hap{h}``, bytes)]."""
    index = {h.split()[0]: i for i, (h, _) in enumerate(records)}
    ploidy, edits = {}, {}
    for line in vcf_text.splitlines():
        if not line or line.startswith("#"):
            continue
        f = line.split("\t")
        if f[6] not in ("PASS", "."):
            continue
        c = index[f[0]]
        seq = records[c][1]
        gt = f[9].split(":")[f[8].split(":").index("GT")].replace("|", "/").split("/")
        ploidy[c] = len(gt)
        alts = f[4].split(",")
        pos = int(f[1])
        for h, a in enumerate(gt):
            if a in (".", "0") or alts[int(a) - 1] == "*":
                continue
            alt = alts[int(a) - 1]
            if alt.startswith("<"):
                p, e = pos, _sv_end(pos, f[7])             # the affected bases ref[p:e]; the padding base stays
                edit = {"<DEL>": (p, e, b""), "<INV>": (p, e, rc(seq[p:e])), "<DUP>": (e, e, seq[p:e]),
                        "<DUP:TANDEM>": (e, e, seq[p:e])}[alt]
            else:
                edit = (pos - 1, pos - 1 + len(f[3]), alt.encode())
            edits.setdefault((c, h), []).append(edit)
    out = []
    for c, (header, seq) in enumerate(records):
        for h in range(ploidy.get(c, 2)):
            parts, prev = [], 0
            for s, e, rep in edits.get((c, h), []):
                parts += [seq[prev:s], rep]
                prev = e
            parts.append(seq[prev:])
            out.append(("%s-hap%d" % (normalise_name(header), h + 1), b"".join(parts)))
    return out


def splice_tables(t, ref):
    """The haplotype bytes the tables describe, spliced on the host with each variant's kind."""
    out = []
    for h, c in enumerate(t.hap_chrom):
        seq = ref.bases[int(ref.offsets[c]):int(ref.offsets[c + 1])].tobytes()
        parts, prev = [], 0
        for j in range(int(t.var_off[h]), int(t.var_off[h + 1])):
            p, o, n = int(t.var_pos[j]), int(t.alt_off[j]), int(t.alt_len[j])
            alt = {0: t.alt[o:o + n].tobytes(), 1: seq[o:o + n], 2: rc(seq[o:o + n])}[int(t.alt_kind[j])]
            parts += [seq[prev:p], alt]
            prev = p + int(t.var_ref_len[j])
        parts.append(seq[prev:])
        out.append((t.names[h], b"".join(parts)))
    return out


def _write(path, text, gz=False):
    with (gzip.open(path, "wt") if gz else open(path, "w")) as f:
        f.write(text)
    return path


def _rows(*rows):
    return HEADER + "".join("\t".join(str(x) for x in r) + "\n" for r in rows)


def _row(chrom, pos, ref, alt, gt, info=".", filt="PASS"):
    return (chrom, pos, ".", ref, alt, 50, filt, info, "GT", gt)


SMALL = [("chr1 first", b"ACGTACGTACGTAAAACCCCGGGGTTTTacgtacgtNNNNACGTRYKMBDHVSWacgtrykmbdhvswUuACGTACGT"),
         ("chr2", b"GGGGCCCCAAAATTTTGGGGCCCCAAAATTTT"),
         ("chr3", b"TTGACCATGCAAGTCC")]
N1, N2, N3 = (len(s) for _, s in SMALL)


def _base(chrom, pos):
    return chr(dict((h.split()[0], s) for h, s in SMALL)[chrom][pos - 1])


def _sv(chrom, pos, alt, gt, info, filt="PASS"):
    return _row(chrom, pos, _base(chrom, pos), alt, gt, info, filt)


def _var(chrom, pos, n, alt, gt):
    """A small variant whose REF is the n reference bases at pos."""
    return _row(chrom, pos, "".join(_base(chrom, pos + i) for i in range(n)), alt, gt)


# every fixture the CPU checks the tables against and the GPU checks the device bytes against
CASES = {
    **{"%s_%s" % (alt.strip("<>").replace(":", "_"), name): [_sv("chr1", 10, alt, gt, "END=30")]
       for alt in ("<DEL>", "<INV>", "<DUP>", "<DUP:TANDEM>") for name, gt in (("het", "0|1"), ("hom", "1|1"))},
    "record_ends": [_sv("chr1", 1, "<INV>", "1|0", "END=%d" % N1), _sv("chr1", 1, "<DUP>", "0|1", "END=%d" % N1),
                    _sv("chr2", 1, "<DEL>", "1|1", "END=%d" % N2)],
    "one_base_spans": [_sv("chr1", 3, "<DEL>", "1|0", "END=4"), _sv("chr1", 5, "<INV>", "0|1", "SVLEN=1"),
                       _sv("chr1", 7, "<DUP>", "1|1", "END=8"), _sv("chr2", 4, "<INV>", "1|1", "END=5")],
    "adjacent": [_sv("chr1", 2, "<DEL>", "1|1", "END=5"), _sv("chr1", 6, "<INV>", "1|1", "END=9"),
                 _sv("chr1", 10, "<DUP>", "1|1", "END=14"), _var("chr1", 15, 3, "G", "1|1"),
                 _sv("chr1", 18, "<INV>", "1|0", "END=22"), _var("chr1", 23, 1, "GTT", "1|1"),
                 _var("chr1", 24, 1, "T", "0|1"), _sv("chr1", 25, "<DEL>", "0|1", "END=26")],
    "other_haplotype_small": [_sv("chr1", 4, "<DEL>", "1|0", "END=20"), _var("chr1", 6, 1, "T", "0|1"),
                              _var("chr1", 9, 4, "A", "0|1"), _var("chr1", 13, 1, "ATTT", "0|1"),
                              _sv("chr1", 21, "<INV>", "0|1", "END=40"), _var("chr1", 25, 1, "C", "1|0"),
                              _var("chr1", 30, 1, "CGA", "1|0")],
    "haploid": [_sv("chr3", 2, "<INV>", "1", "END=9"), _sv("chr3", 10, "<DUP>", "1", "END=14"), _sv("chr3", 15, "<DEL>", "0", "END=16")],
    "missing_ref_star": [_sv("chr1", 2, "<DEL>", "0|1", "END=10"), _var("chr1", 5, 1, "*,C", "2|1"),
                         _sv("chr1", 12, "<INV>", ".|1", "END=20"), _sv("chr1", 22, "<DUP>", "./.", "END=30"),
                         _sv("chr1", 32, "<DEL>", "0/0", "END=33")],
    "iupac_lower_case_inversion": [_sv("chr1", 28, "<INV>", "1|0", "END=%d" % (N1 - 3)), _sv("chr1", 40, "<DUP>", "0|1", "END=70")],
    "end_svlen_forms": [_sv("chr1", 2, "<DEL>", "1|1", "END=4"), _sv("chr1", 6, "<DEL>", "1|1", "SVLEN=-3"),
                        _sv("chr1", 12, "<DEL>", "1|1", "SVLEN=2"), _sv("chr1", 16, "<INV>", "1|1", "SVTYPE=INV;END=20;SVLEN=4"),
                        _sv("chr1", 22, "<DUP>", "1|1", "CIEND=-5,5;SVLEN=-3;SVLEN2=9"), _sv("chr1", 30, "<DUP>", "1|1", "SVLEN=+4")],
    "filtered_sv_skipped": [_sv("chr1", 2, "<INV>", "1|1", ".", filt="LowQual"), _sv("chr1", 3, "<DUP>", "0|1", "END=6"),
                            _row("chr1", 20, "G", "<INS>", "1|1", filt="q10"), _row("chr1", 30, "t", "<CNV>", "1|1", filt="q10")],
    "unchecked_other_alt": [_var("chr1", 10, 1, "G,<INS>", "1|0"), _var("chr1", 12, 1, "<DEL>,<CNV>", "0|0"),
                            _var("chr1", 14, 1, "T,<INV>", "0|1")],
}


def _small():
    return PackedReference.from_records(SMALL)


def _check(tmp_path, text, gz=False):
    path = _write(os.path.join(str(tmp_path), "v.vcf" + (".gz" if gz else "")), text, gz)
    ref = _small()
    t = read_vcf(path, ref)
    want = build_haplotypes(SMALL, text)
    assert splice_tables(t, ref) == want
    assert t.lengths.tolist() == [len(s) for _, s in want]
    return t, want


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", list(CASES))
def test_tables_equal_the_builder(name, tmp_path):
    t, want = _check(tmp_path, _rows(*CASES[name]))
    if name.startswith(("INV", "DUP", "DEL")):
        kind = {"DEL": 0, "INV": 2, "DUP": 1}[name[:3]]
        assert t.alt_kind.tolist() == [kind] * (2 if name.endswith("hom") else 1)
        assert t.structural.sum(axis=0).tolist() == [int(kind == k) * len(t.alt_kind) for k in (0, 2, 1)]


def test_gzip_vcf(tmp_path):
    _check(tmp_path, _rows(*CASES["adjacent"]), gz=True)


def test_kinds_and_lengths_of_each_encoding(tmp_path):
    t, want = _check(tmp_path, _rows(_sv("chr1", 5, "<DEL>", "1|0", "END=9"), _sv("chr1", 10, "<INV>", "1|0", "END=15"),
                                     _sv("chr1", 16, "<DUP:TANDEM>", "1|0", "SVLEN=-6")))
    assert t.var_pos[:3].tolist() == [5, 10, 22] and t.var_ref_len[:3].tolist() == [4, 5, 0]
    assert t.alt_off[1:3].tolist() == [10, 16] and t.alt_len[:3].tolist() == [0, 5, 6] and t.alt_kind.tolist() == [0, 2, 1]
    assert t.lengths.tolist() == [N1 - 4 + 6, N1, N2, N2, N3, N3]
    assert t.structural.tolist() == [[1, 1, 1], [0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0]]


def test_no_symbolic_alleles_gives_all_zero_kinds(tmp_path):
    t, _ = _check(tmp_path, _rows(_row("chr1", 2, "C", "G", "0|1"), _row("chr1", 5, "ACGT", "A", "1|1")))
    assert t.alt_kind.dtype == np.uint8 and t.alt_kind.tolist() == [0, 0, 0]


@pytest.mark.parametrize("rows, line, message", [
    ([_sv("chr1", 2, "<DEL>", "0|1", ".")], 5, "symbolic structural variant needs END or SVLEN"),
    ([_sv("chr1", 2, "<INV>", "0|1", "CIEND=-5,5;SVLEN2=3")], 5, "needs END or SVLEN"),
    ([_sv("chr1", 2, "<DUP>", "0|1", "END=1x")], 5, "INFO END is not a number"),
    ([_sv("chr1", 2, "<DUP>", "0|1", "SVLEN=3,4")], 5, "INFO SVLEN is not a number"),
    ([_sv("chr1", 2, "<DUP>", "0|1", "END")], 5, "INFO END is not a number"),
    ([_sv("chr1", 4, "<INV>", "1|0", "END=4")], 5, "is not past POS"),
    ([_sv("chr1", 4, "<DEL>", "1|0", "SVLEN=0")], 5, "is not past POS"),
    ([_sv("chr2", 4, "<DEL>", "1|0", "END=%d" % (N2 + 1))], 5, "past the end of the reference record"),
    ([_sv("chr2", 4, "<DUP>", "1|0", "SVLEN=%d" % (N2 - 3))], 5, "past the end of the reference record"),
    ([_sv("chr1", 4, "<DEL>", "1|0", "END=10;SVLEN=-5")], 5, "disagree"),
    ([_row("chr1", 4, "TA", "<DEL>", "1|0", "END=10")], 5, "must be one base"),
    ([_row("chr1", 4, "T", "<DEL>,C", "1|0", "END=10")], 5, "only ALT"),
    ([_row("chr1", 4, "T", "<DEL>,<INV>", "0|2", "END=10")], 5, "only ALT"),
    ([_row("chr1", 4, "A", "<DEL>", "1|0", "END=10")], 5, "REF does not match"),
    ([_sv("chr1", 4, "<DEL>", "1|0", "END=10"), _var("chr1", 8, 1, "G", "1|0")], 6, "overlaps an earlier variant on haplotype 1"),
    ([_sv("chr1", 4, "<INV>", "0|1", "END=10"), _sv("chr1", 10, "<DUP>", "1|1", "END=12")], 6, "overlaps an earlier variant on haplotype 2"),
    ([_row("chr1", 2, "CG", "C", "1|0"), _sv("chr1", 3, "<DEL>", "1|0", "END=10")], 6, "overlaps"),
])
def test_errors_name_the_line(rows, line, message, tmp_path):
    path = _write(os.path.join(str(tmp_path), "v.vcf"), _rows(*rows))
    with pytest.raises(VcfError) as e:
        read_vcf(path, _small())
    assert str(e.value).startswith("line %d:" % line) and message in str(e.value), str(e.value)


def test_sv_inside_a_deletion_on_the_other_haplotype_is_free(tmp_path):
    _check(tmp_path, _rows(_row("chr1", 2, "CGTACGTAC", "C", "1|0"), _sv("chr1", 4, "<INV>", "0|1", "END=8"),
                           _row("chr1", 9, "A", "T", "0|1")))


@pytest.mark.parametrize("alt", ["<INS>", "<CNV>", "<DEL:ME:ALU>", "G[chr2:5[", "<DUP:INT>", "<del>"])
def test_unsupported_symbolic_alts_keep_their_message(alt, tmp_path):
    path = _write(os.path.join(str(tmp_path), "v.vcf"), _rows(_row("chr1", 2, "C", "G", "0|1"), _sv("chr1", 3, alt, "0|1", "END=9")))
    with pytest.raises(VcfError, match="^line 6: a haplotype takes an ALT allele that is symbolic, a breakend, missing or not a "
                                       "nucleotide sequence$"):
        read_vcf(path, _small())


@pytest.mark.parametrize("late", [
    _sv("chr1", 30, "<DEL>", "1|0", "."),
    _sv("chr1", 30, "<DUP>", "1|0", "END=29"),
    _sv("chr1", 30, "<INV>", "1|0", "END=x"),
    _row("chr1", 30, "T", "<INS>", "1|0"),
    _row("chr1", 29, "TTa", "T", "1|0"),
])
@pytest.mark.parametrize("early", [
    _sv("chr1", 3, "<DEL>", "0|1", "SVLEN=4;END=9"),
    _sv("chr1", 3, "<INV>", "0|1", "END=%d" % (N1 + 1)),
    _row("chr1", 3, "GTA", "<DUP>", "0|1", "END=9"),
    _row("chr1", 3, "A", "<DUP>", "0|1", "END=9"),
])
def test_the_first_error_in_the_file_is_reported(early, late, tmp_path):
    rows = [_row("chr1", 2, "C", "G", "0|1"), early, _row("chr1", 21, "G", "A", "1|1"), late, _row("chr9", 40, "A", "C", "1|1")]
    path = _write(os.path.join(str(tmp_path), "v.vcf"), _rows(*rows))
    with pytest.raises(VcfError, match="^line 6: "):
        read_vcf(path, _small())
    path = _write(os.path.join(str(tmp_path), "v.vcf"), _rows(*(rows[:1] + rows[2:])))
    with pytest.raises(VcfError, match="^line 7: "):
        read_vcf(path, _small())


def synthetic_sv_genome(seed=11):
    """A multi-Mb reference (chrA and chrB diploid, chrC haploid) with lower case, N and IUPAC stretches, and a VCF of
    structural variants of 1 b to 200 kb (log-uniform) with SNVs and indels between them.  For each SV type, POS and
    END take every value mod 16; every record has an SV at POS 1 and one that ends at its last base.  Returns (records,
    vcf text)."""
    rng = np.random.default_rng(seed)
    lengths = {"chrA": 4_000_000, "chrB": 3_000_000, "chrC": 1_200_000}
    n_sv = {"chrA": 110, "chrB": 90, "chrC": 40}
    records = []
    for name, n in lengths.items():
        s = synth.synth_chrom(rng, n).copy()
        for _ in range(40):
            lo = int(rng.integers(0, n - 5000))
            s[lo:lo + int(rng.integers(100, 5000))] |= 32                        # lower case
        for _ in range(40):
            lo = int(rng.integers(0, n - 200))
            s[lo:lo + 200] = np.frombuffer(b"RYKMSWBDHVNUrykmswbdhvnu", dtype=np.uint8)[rng.integers(0, 24, 200)]
        records.append((name + " synthetic", s.tobytes()))
    seqs = {name: s for (name, _), s in zip(lengths.items(), (r[1] for r in records))}
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    rows, k = [], 0
    alts = ["<DEL>", "<INV>", "<DUP>", "<DUP:TANDEM>"]
    for chrom, n in lengths.items():
        gts = ["1"] if chrom == "chrC" else ["0|1", "1|0", "1|1", "1/0"]
        seq = seqs[chrom]
        cur = 1                                                                 # next free 1-based position
        for i in range(n_sv[chrom]):
            size = int(np.exp(rng.uniform(0, np.log(200_000))))
            pos = 1 if i == 0 else cur + int(rng.integers(1, 3000))
            if i:
                pos += ((k // 4) % 16 - pos) % 16                               # each type: every POS mod 16
            end = pos + size
            end += ((k // 4) * 7 % 16 - end) % 16                               # and every END mod 16
            last = i == n_sv[chrom] - 1 or end > n - 50
            assert pos < n - 50, (chrom, i)
            if last:
                end = n                                                          # the record's last base
            alt = alts[k % 4]
            info = ("END=%d" % end) if k % 3 == 0 else ("SVLEN=%d" % ((pos - end) if alt == "<DEL>" else (end - pos))) if k % 3 == 1 \
                else "END=%d;SVLEN=%d" % (end, end - pos)
            rows.append(_row(chrom, pos, chr(seq[pos - 1]), alt, gts[k % len(gts)], info))
            k += 1
            if last:
                break
            cur = end + 1
            # small variants behind it (the first one adjacent to the SV's span on the other haplotype or both)
            p = cur
            for _ in range(int(rng.integers(0, 6))):
                if p + 40 >= n:
                    break
                kind = int(rng.integers(0, 3))
                rl = 1 if kind != 1 else int(rng.integers(2, 12))
                alt_s = acgt[rng.integers(0, 4, 1 if kind != 2 else int(rng.integers(2, 20)))].tobytes().decode()
                rows.append(_row(chrom, p, seq[p - 1:p - 1 + rl].decode(), alt_s, gts[int(rng.integers(0, len(gts)))]))
                p += rl + int(rng.integers(0, 30))
            cur = p
    return records, HEADER + "".join("\t".join(str(x) for x in r) + "\n" for r in rows)


@pytest.fixture(scope="module")
def sv_genome(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("sv"))
    records, text = synthetic_sv_genome()
    ref = os.path.join(d, "ref.fa")
    synth.write_fasta(ref, [(h, np.frombuffer(s, dtype=np.uint8)) for h, s in records])
    vcf = _write(os.path.join(d, "sample.vcf.gz"), text, gz=True)
    haps = build_haplotypes(records, text)
    hap_fa = os.path.join(d, "hap.fa")
    synth.write_fasta(hap_fa, [(n, np.frombuffer(s, dtype=np.uint8)) for n, s in haps])
    return d, ref, vcf, hap_fa, records, text, haps


def test_synthetic_tables_equal_the_builder(sv_genome):
    d, ref, vcf, hap_fa, records, text, haps = sv_genome
    r = PackedReference.from_fasta(ref)
    t = read_vcf(vcf, r)
    assert splice_tables(t, r) == haps
    assert t.names == ["chrA-hap1", "chrA-hap2", "chrB-hap1", "chrB-hap2", "chrC-hap1"]
    sv = t.alt_kind > 0
    assert set(t.alt_kind.tolist()) == {0, 1, 2} and int(t.structural.sum()) >= 100
    assert set((t.alt_off[sv] % 16).tolist()) == set(range(16)) and set(((t.alt_off + t.alt_len)[sv] % 16).tolist()) == set(range(16))
    assert int(t.alt_len[sv].max()) > 50_000 and int(t.alt_len[sv].min()) <= 16


# ---------------------------------------------------------------------------------------------------------------- GPU
def _device_bytes(ref, t):
    from nanosim_b200.engine import Engine
    eng = Engine(device=0, seed=1)
    try:
        eng.set_reference(ref)
        eng.apply_variants(t)
        return eng.reference_bases(int(t.offsets[-1])).tobytes()
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_device_haplotypes_equal_the_builder(name, tmp_path):
    text = _rows(*CASES[name])
    ref = _small()
    t = read_vcf(_write(os.path.join(str(tmp_path), "v.vcf"), text), ref)
    assert _device_bytes(ref, t) == b"".join(s for _, s in build_haplotypes(SMALL, text))


@pytest.mark.gpu
def test_synthetic_device_haplotypes_equal_the_builder(sv_genome):
    d, ref, vcf, hap_fa, records, text, haps = sv_genome
    r = PackedReference.from_fasta(ref)
    t = read_vcf(vcf, r)
    assert _device_bytes(r, t) == b"".join(s for _, s in haps)


@pytest.mark.gpu
def test_null_kinds_equal_all_zero_kinds(tmp_path):
    text = _rows(_row("chr1", 2, "C", "G", "0|1"), _row("chr1", 5, "ACGT", "A", "1|1"), _row("chr2", 9, "A", "ATTTTTTTTTTTTTTTTTTTT", "1|0"))
    ref = _small()
    t = read_vcf(_write(os.path.join(str(tmp_path), "v.vcf"), text), ref)
    assert t.alt_kind.tolist() == [0] * 4
    zero = _device_bytes(ref, t)
    t.alt_kind = None                           # NsVariants.alt_kind = NULL
    assert _device_bytes(ref, t) == zero == b"".join(s for _, s in build_haplotypes(SMALL, text))


@pytest.mark.gpu
def test_bad_kinds_and_source_spans_are_rejected(tmp_path):
    from nanosim_b200.engine import Engine, NanoSimError
    ref = _small()
    t = read_vcf(_write(os.path.join(str(tmp_path), "v.vcf"), _rows(_sv("chr2", 4, "<INV>", "1|0", "END=10"),
                                                                       _sv("chr2", 12, "<DUP>", "1|0", "END=20"))), ref)
    assert t.alt_kind.tolist() == [2, 1]
    bad_kind = copy.deepcopy(t)
    bad_kind.alt_kind[1] = 3
    past_end = copy.deepcopy(t)                 # chr2's inversion reading past the end of its record
    past_end.alt_off[0] = N2 - 5
    past_end.alt_len[0] = 6
    dup_past_end = copy.deepcopy(t)
    dup_past_end.alt_off[1] = N2
    dup_past_end.alt_len[1] = 1
    for bad, message in ((bad_kind, "has ALT kind 3"), (past_end, "lies outside its source record"),
                         (dup_past_end, "lies outside its source record")):
        eng = Engine(device=0, seed=1)
        eng.set_reference(ref)
        with pytest.raises(NanoSimError, match=message + r".*\(rc=-1\)"):          # NS_EINVAL
            eng.apply_variants(bad)
        eng.apply_variants(t)                   # the failed call left the reference as it was
        assert eng.reference_bases(int(t.offsets[-1])).tobytes() == b"".join(s for _, s in splice_tables(t, ref))
        eng.close()


_E2E = {
    "guppy_fastq": ["-c", "guppy", "-n", "3000", "--fastq", "--seed", "51"],
    "gzip_gzip_error_profile": ["-c", "guppy", "-n", "3000", "--fastq", "--gzip", "--gzip_error_profile", "--seed", "52"],
    "dorado_hp6_chimeric_bam": ["-c", "dorado", "-n", "2000", "--fastq", "-hp", "-k", "6", "--chimeric", "--bam", "--seed", "53"],
}


def _argv(extra):
    extra = list(extra)
    extra[1] = os.path.join(pc.DATA, pc.MODELS[extra[1]])
    return extra + ["-t", "4"]


def _outputs(prefix):
    d, base = os.path.split(prefix)
    return sorted(f[len(base):] for f in os.listdir(d) if f.startswith(base + "_"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(_E2E))
def test_vcf_run_equals_a_run_on_the_haplotype_fasta(name, sv_genome):
    from nanosim_b200 import simulator
    d, ref, vcf, hap_fa, records, text, haps = sv_genome
    a, b = os.path.join(d, name + "_vcf"), os.path.join(d, name + "_hap")
    simulator.main(["genome", "-rg", ref, "--vcf", vcf, "-o", a] + _argv(_E2E[name]))
    simulator.main(["genome", "-rg", hap_fa, "-o", b] + _argv(_E2E[name]))
    files = _outputs(a)
    assert files == _outputs(b) and len(files) >= 3, files
    for f in files:
        x, y = open(a + f, "rb").read(), open(b + f, "rb").read()
        assert x == y and len(x) > 1000, f
