"""--aln_tags: NM and SA on the mapped records of --mapped_bam (plain and lifted) and --spliced_bam, computed on the GPU
(ns_set_aln_tags, DESIGN §3 "NM and SA tags").

The rules restated here: NM is what ``samtools calmd`` counts against the FASTA the header names (I and D lengths, and the
M positions whose 4-bit codes differ or either is N); a read with k > 1 records has on each an SA:Z with one
``rname,pos,strand,CIGAR,60,NM;`` entry per other record in record order; the aux order is HP/XS, NM:I, SA:Z, CG; and
removing NM and SA from a tagged file gives the untagged file's bytes.  GPU tests run with ``pytest -m gpu``; the CLI,
export and restatement tests need no GPU."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT

import synth
from test_bam_output import _CODE
from test_bgzf_output import check_bgzf_file
from test_mapped_bam import _ARGV, _circ, _config_args, _ecoli, _model
from test_vcf_haplotypes import genome  # noqa: F401  (module-scoped fixture: reference, VCF, haplotype FASTA)
from test_vcf_structural_variants import sv_genome  # noqa: F401

M, I, D, N, S, H = 0, 1, 2, 3, 4, 5
_OPS = "MIDNSHP=X"


# ------------------------------------------------------------------------------------------------------------ decoding
def _aux_fields(aux):
    """[(tag, type, value, start, end)] of a record's aux bytes."""
    out, p = [], 0
    sizes = {"A": 1, "c": 1, "C": 1, "s": 2, "S": 2, "i": 4, "I": 4, "f": 4}
    fmts = {"c": "<b", "C": "<B", "s": "<h", "S": "<H", "i": "<i", "I": "<I", "f": "<f"}
    while p < len(aux):
        tag, ty, q = aux[p:p + 2].decode(), chr(aux[p + 2]), p + 3
        if ty == "A":
            val, q = chr(aux[q]), q + 1
        elif ty in fmts:
            val, q = struct.unpack_from(fmts[ty], aux, q)[0], q + sizes[ty]
        elif ty == "Z":
            e = aux.index(b"\0", q)
            val, q = aux[q:e].decode(), e + 1
        else:
            assert ty == "B"
            sub, n = chr(aux[q]), struct.unpack_from("<I", aux, q + 1)[0]
            val = np.frombuffer(aux, dtype="<" + {"I": "u4", "i": "i4", "C": "u1", "c": "i1", "S": "u2", "s": "i2"}[sub], count=n,
                                offset=q + 5).copy()
            q += 5 + n * sizes[sub]
        out.append((tag, ty, val, p, q))
        p = q
    return out


def read_tagged_bam(data):
    """(header bytes, [SN names], records) of a decompressed BAM; a record: its fields, real CIGAR, 4-bit codes, aux
    fields, raw bytes and where its aux bytes start in them."""
    assert data[:4] == b"BAM\1"
    l_text = struct.unpack_from("<i", data, 4)[0]
    pos = 8 + l_text
    names = []
    for _ in range(struct.unpack_from("<i", data, pos)[0]):
        ln = struct.unpack_from("<i", data, pos + 4)[0]
        names.append(data[pos + 8:pos + 7 + ln].decode())
        pos += 8 + ln
    pos += 4
    head, recs = data[:pos], []
    while pos < len(data):
        block, ref_id, p, l_name, mapq, _, n_cig, flag, l_seq = struct.unpack_from("<iiiBBHHHI", data, pos)
        q = pos + 36
        name = data[q:q + l_name - 1]
        q += l_name
        cig = np.frombuffer(data, dtype="<u4", count=n_cig, offset=q).copy()
        q += 4 * n_cig
        packed = np.frombuffer(data, dtype=np.uint8, count=(l_seq + 1) // 2, offset=q)
        codes = np.empty(2 * len(packed), dtype=np.uint8)
        codes[0::2], codes[1::2] = packed >> 4, packed & 15
        q += (l_seq + 1) // 2 + l_seq
        raw = data[pos:pos + 4 + block]
        aux = _aux_fields(raw[q - pos:])
        cg = [v for t, _, v, _, _ in aux if t == "CG"]
        recs.append(dict(name=name, ref_id=ref_id, pos=p, mapq=mapq, flag=flag, l_seq=l_seq, codes=codes[:l_seq],
                         cigar=cg[0] if cg else cig, aux=aux, raw=raw, aux0=q - pos))
        pos += 4 + block
    assert pos == len(data)
    return head, names, recs


def strip_tags(rec):
    """The record's bytes without its NM and SA fields."""
    raw, a0 = rec["raw"], rec["aux0"]
    keep = b"".join(raw[a0 + s:a0 + e] for t, _, _, s, e in rec["aux"] if t not in ("NM", "SA"))
    body = raw[4:a0] + keep
    return struct.pack("<i", len(body)) + body


# --------------------------------------------------------------------------------------------------- the rules restated
def cigar_text(cig):
    return "".join("%d%s" % (int(w) >> 4, _OPS[int(w) & 15]) for w in cig)


def calmd_nm(cig, codes, ref, pos, ref_codes=None):
    """NM as samtools calmd counts it: I and D lengths, and the M positions whose codes differ or either is N (15).
    ref: the reference record's bytes (ref_codes: their codes, precomputed)."""
    rc = _CODE[np.frombuffer(ref, dtype=np.uint8)] if ref_codes is None else ref_codes
    nm, q, r = 0, 0, pos
    for w in cig:
        kind, n = int(w) & 15, int(w) >> 4
        if kind == M:
            a, b = codes[q:q + n], rc[r:r + n]
            nm += int(((a != b) | (a == 15) | (b == 15)).sum())
        elif kind in (I, D):
            nm += n
        q += n if kind in (M, I, S) else 0
        r += n if kind in (M, D, N) else 0
    return nm


def sa_entries(group, names, nms):
    """Every record's expected SA value (None for a read with one record)."""
    if len(group) < 2:
        return [None] * len(group)
    ent = ["%s,%d,%s,%s,60,%d;" % (names[r["ref_id"]], r["pos"] + 1, "-" if r["flag"] & 16 else "+", cigar_text(r["cigar"]), nm)
           for r, nm in zip(group, nms)]
    return ["".join(e for k, e in enumerate(ent) if k != j) for j in range(len(group))]


def groups(recs):
    """The records of each read (adjacent, one name)."""
    out = []
    for r in recs:
        if out and out[-1][0]["name"] == r["name"]:
            out[-1].append(r)
        else:
            out.append([r])
    return out


def check_tags(recs, names, refs, first_tag=None):
    """NM and SA of every record by the rules; refs: SN name -> (bytes, codes).  Returns the number of reads with SA."""
    n_sa = 0
    for g in groups(recs):
        if g[0]["flag"] & 4:
            assert len(g) == 1 and g[0]["aux"] == []
            continue
        nms = []
        for r in g:
            ref, rc = refs[names[r["ref_id"]]]
            nms.append(calmd_nm(r["cigar"], r["codes"], ref, r["pos"], rc))
        for r, nm, sa in zip(g, nms, sa_entries(g, names, nms)):
            tags = [t for t, *_ in r["aux"]]
            want = ([first_tag] if first_tag else []) + ["NM"] + (["SA"] if sa is not None else []) + (["CG"] if "CG" in tags else [])
            assert tags == want, (r["name"], tags)
            got = {t: (ty, v) for t, ty, v, _, _ in r["aux"]}
            assert got["NM"] == ("I", nm), (r["name"], got["NM"], nm)
            if sa is not None:
                assert got["SA"] == ("Z", sa), r["name"]
                n_sa += 1
    return n_sa


def fasta_refs(path):
    from nanosim_b200.reference_fasta import PackedReference
    r = PackedReference.from_fasta(path)
    out = {}
    for k, n in enumerate(r.raw_names):
        b = r.bases[int(r.offsets[k]):int(r.offsets[k + 1])].tobytes()
        out[n] = (b, _CODE[np.frombuffer(b, dtype=np.uint8)])
    return out


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_restatement_on_hand_built_records():
    def c(b):
        return _CODE[np.frombuffer(b, dtype=np.uint8)]
    assert calmd_nm([(4 << 4) | M], c(b"ACGA"), b"ACGT", 0) == 1
    # 1S 2M 1I 1D 2M: the clip is free, the I and the D count one each
    assert calmd_nm([(1 << 4) | S, (2 << 4) | M, (1 << 4) | I, (1 << 4) | D, (2 << 4) | M], c(b"TACTGT"), b"gACxGT", 1) == 2
    codes = c(b"ACG")
    assert calmd_nm([(3 << 4) | M], codes, b"ACN", 0) == 1                   # N in the reference always counts
    assert calmd_nm([(3 << 4) | M], _CODE[np.frombuffer(b"acu", dtype=np.uint8)], b"ACT", 0) == 0    # case and U as T
    assert calmd_nm([(2 << 4) | M, (5 << 4) | N, (1 << 4) | M], _CODE[np.frombuffer(b"ACG", dtype=np.uint8)], b"ACxxxxxG", 0) == 0
    recs = [dict(name=b"r", ref_id=1, pos=9, flag=0, cigar=np.array([(5 << 4) | M, (3 << 4) | H], dtype=np.uint32)),
            dict(name=b"r", ref_id=0, pos=0, flag=16 | 0x800, cigar=np.array([(5 << 4) | H, (2 << 4) | M, (1 << 4) | D, (1 << 4) | M], dtype=np.uint32))]
    assert sa_entries(recs, ["c0", "c1"], [2, 3]) == ["c0,1,-,5H2M1D1M,60,3;", "c1,10,+,5M3H,60,2;"]
    assert sa_entries(recs[:1], ["c0", "c1"], [2]) == [None]


def test_strip_and_aux_parsing():
    aux = b"HPC\x02" + b"NMI" + struct.pack("<I", 7) + b"SAZc,1,+,3M,60,0;\0" + b"CGBI" + struct.pack("<I", 1) + struct.pack("<I", 48)
    body = struct.pack("<iiBBHHHIiii", 0, 5, 2, 60, 4681, 1, 0, 0, -1, -1, 0) + b"r\0" + struct.pack("<I", 48)
    raw = struct.pack("<i", len(body) + len(aux)) + body + aux
    fields = _aux_fields(aux)
    assert [(t, ty) for t, ty, *_ in fields] == [("HP", "C"), ("NM", "I"), ("SA", "Z"), ("CG", "B")]
    rec = dict(raw=raw, aux0=4 + len(body), aux=fields)
    plain = body + b"HPC\x02" + b"CGBI" + struct.pack("<I", 1) + struct.pack("<I", 48)
    assert strip_tags(rec) == struct.pack("<i", len(plain)) + plain


@pytest.mark.parametrize("mode, extra, message", [
    ("genome", ["--bam", "--aln_tags"], "--aln_tags needs --mapped_bam"),
    ("metagenome", ["--bam", "--aln_tags"], "--aln_tags needs --mapped_bam"),
    ("transcriptome", ["--bam", "--aln_tags"], "--aln_tags needs --spliced_bam in transcriptome mode"),
    ("transcriptome", ["--bam", "--mapped_bam", "--aln_tags"], "--mapped_bam is not available in transcriptome mode"),
])
def test_usage_errors(mode, extra, message, tmp_path, capsys):
    from nanosim_b200 import simulator
    with pytest.raises(SystemExit) as e:
        simulator.main(_ARGV[mode] + ["-o", os.path.join(str(tmp_path), "sim")] + extra)
    assert e.value.code == 1
    assert message in capsys.readouterr().err
    assert os.listdir(str(tmp_path)) == []


def test_exports_name_the_new_entry_point():
    from nanosim_b200 import _lib
    header = open(os.path.join(ROOT, "include", "nanosim_b200.h")).read()
    assert "ns_set_aln_tags" in _lib.EXPORTS and "ns_set_aln_tags(" in header


def test_paired_ref_bytes_are_the_ref_spans_of_sequence_alts():
    import types
    from nanosim_b200.variants import HaplotypeTables, paired_ref_bytes
    ref = types.SimpleNamespace(bases=np.frombuffer(b"ACGTACGTAA" + b"ttggccaaNN", dtype=np.uint8), offsets=np.array([0, 10, 20]))
    # haplotype 0 on record 1: SNV at 2, deletion 4..7 -> A, <INV> kind 2; haplotype 1 on record 0: insertion at 5, <DUP>
    t = HaplotypeTables(["a", "b"], [1, 0], [1, 1], [0, 3, 5], [2, 4, 8, 5, 9], [1, 3, 2, 1, 0], [0, 1, 8, 2, 3], [1, 1, 2, 3, 4],
                        np.frombuffer(b"CAGTT", dtype=np.uint8), [10, 10], [0, 0], alt_kind=[0, 0, 2, 0, 1])
    assert paired_ref_bytes(t, ref).tobytes() == b"g" + b"c" + b"C"


# ------------------------------------------------------------------------------------------------------------------ GPU
def _iupac_fa(tmp):
    """A reference with lower case stretches, N runs and IUPAC codes."""
    path = os.path.join(tmp, "iupac.fa")
    if not os.path.exists(path):
        rng = np.random.default_rng(17)
        s = synth.synth_chrom(rng, 400000).copy()
        for start in rng.integers(0, len(s) - 3000, 60):
            s[start:start + 2000] = np.char.lower(s[start:start + 2000].view("S1")).view(np.uint8)
        for start in rng.integers(0, len(s) - 200, 40):
            s[start:start + rng.integers(1, 150)] = ord("N")
        codes = np.frombuffer(b"RYSWKMBDHVNryswkmbdhvn", dtype=np.uint8)
        s[rng.integers(0, len(s), 600)] = codes[rng.integers(0, len(codes), 600)]
        t = synth.synth_chrom(rng, 150000)
        synth.write_fasta(path, [("chrI iupac", s), ("chrP plain", t)])
    return path


def _genome_configs(tmp):
    iu = _iupac_fa(tmp)
    return {
        "iupac_guppy_fastq": (["genome", "-rg", iu, "-c", _model("guppy"), "-n", "2000", "--fastq", "--seed", "71"], iu),
        "dorado_hp6_chimeric": (_config_args("dorado_hp6_chimeric", tmp)[0], _ecoli(tmp)),
        "perfect_iupac": (["genome", "-rg", iu, "-c", _model("guppy"), "-n", "1500", "--fastq", "--perfect", "--seed", "72"], iu),
        "genome_circular": (_config_args("genome_circular", tmp)[0], _circ(tmp)),
        "metagenome_chimeric": (_config_args("metagenome_chimeric", tmp)[0], None),
    }


_RUNS = {}


def _pair(key, args, d):
    """args run with --bam plus ``extra`` mapped flags, without and with --aln_tags (same seed): the two prefixes."""
    from nanosim_b200 import simulator
    if key not in _RUNS:
        plain, tagged = os.path.join(d, key + "_untagged"), os.path.join(d, key + "_tagged")
        simulator.main(args + ["-o", plain, "-t", "4"])
        simulator.main(args + ["-o", tagged, "-t", "4", "--aln_tags"])
        _RUNS[key] = (plain, tagged)
    return _RUNS[key]


def _same_but_tags(plain, tagged, suffixes=("",), extra_files=()):
    """The tagged file less its NM and SA is the untagged file; every other file is byte-identical.  Returns the tagged
    files' decoded (names, records) per suffix."""
    out = []
    for p in suffixes:
        a = check_bgzf_file(plain + p + "_aligned_reads.bam")
        b = check_bgzf_file(tagged + p + "_aligned_reads.bam")
        head, names, recs = read_tagged_bam(b)
        assert a == head + b"".join(strip_tags(r) for r in recs)
        assert len(b) > len(a)
        for f in ("_unaligned_reads.bam",) + tuple(extra_files):
            if os.path.exists(plain + p + f):
                assert open(plain + p + f, "rb").read() == open(tagged + p + f, "rb").read(), f
        out.append((names, recs))
    return out


@pytest.fixture(scope="module")
def workdir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("aln_tags"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["iupac_guppy_fastq", "dorado_hp6_chimeric", "perfect_iupac", "genome_circular", "metagenome_chimeric"])
def test_genome_and_metagenome_tags(name, workdir):
    from nanosim_b200.reference_fasta import MetaReference
    from conftest import GOLDEN
    args, fa = _genome_configs(workdir)[name]
    plain, tagged = _pair(name, args + ["--bam", "--mapped_bam"], workdir)
    suffixes = ["_sample0", "_sample1"] if name == "metagenome_chimeric" else [""]
    if fa is None:
        m = MetaReference.from_genome_list(os.path.join(GOLDEN, "meta", "genome_list_local.tsv"),
                                           os.path.join(GOLDEN, "meta", "dna_type.tsv"))
        refs = {}
        for k, n in enumerate(m.raw_names):
            b = m.bases[int(m.offsets[k]):int(m.offsets[k + 1])].tobytes()
            refs[n] = (b, _CODE[np.frombuffer(b, dtype=np.uint8)])
    else:
        refs = fasta_refs(fa)
    n_sa = 0
    for names, recs in _same_but_tags(plain, tagged, suffixes, ("_aligned_error_profile",)):
        n_sa += check_tags(recs, names, refs)
        mapped = [r for r in recs if not r["flag"] & 4]
        nm = [dict((t, v) for t, _, v, _, _ in r["aux"])["NM"] for r in mapped]
        assert len(mapped) > 100
        if name == "perfect_iupac":
            # no simulated error: NM is the bytes under M that are not a/c/g/t
            assert sum(nm) > 0 and all(r["cigar"].tolist() == [(r["l_seq"] << 4) | M] for r in mapped)
        else:
            assert np.mean(nm) > 0
    if name in ("dorado_hp6_chimeric", "genome_circular", "metagenome_chimeric"):
        assert n_sa > 0


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["genome", "sv"])
def test_lifted_tags(which, genome, sv_genome):  # noqa: F811
    """NM against the haploid -rg FASTA; a simulated MIS on an SNV that gives back the REF base counts as a match.  sv:
    <DEL>, <INV> and <DUP> with small variants between them, on a reference with lower case, N, IUPAC and U bytes (an
    inversion's haplotype keeps U, the haploid base there is a U whose complement is A)."""
    from nanosim_b200.reference_fasta import PackedReference
    from nanosim_b200.variants import read_vcf
    d, ref, vcf = (genome if which == "genome" else sv_genome)[:3]
    args = ["genome", "-rg", ref, "--vcf", vcf, "-c", _model("guppy"), "-n", "4000", "--fastq", "--seed", "73", "--bam", "--mapped_bam",
            "--lift_mapped_bam"] + (["--chimeric"] if which != "genome" else [])
    plain, tagged = _pair("lift_" + which, args, d)
    [(names, recs)] = _same_but_tags(plain, tagged, extra_files=("_aligned_error_profile",))
    refs = fasta_refs(ref)
    n_sa = check_tags(recs, names, refs, first_tag="HP")
    if which != "genome":
        assert n_sa > 0
        # records inside an <INV>: on the other strand from the read (its name's F or R)
        assert any(("_F_" in r["name"].decode()) == bool(r["flag"] & 16) for r in recs if not r["flag"] & 4)
    # SNVs per haplotype: haploid position -> (REF code, ALT code)
    r = PackedReference.from_fasta(ref)
    t = read_vcf(vcf, r)
    snv = {}
    for h in range(len(t.hap_chrom)):
        for j in range(int(t.var_off[h]), int(t.var_off[h + 1])):
            if t.alt_kind[j] == 0 and t.var_ref_len[j] == 1 and t.alt_len[j] == 1:
                c = int(t.hap_chrom[h])
                rb = r.bases[int(r.offsets[c]) + int(t.var_pos[j])]
                snv.setdefault((c, int(t.hap_number[h])), {})[int(t.var_pos[j])] = (_CODE[rb], _CODE[t.alt[int(t.alt_off[j])]])
    back = 0
    for rec in recs:
        if rec["flag"] & 4:
            continue
        hp = dict((tg, v) for tg, _, v, _, _ in rec["aux"])["HP"]
        s = snv.get((rec["ref_id"], hp), {})
        q, p = 0, rec["pos"]
        for w in rec["cigar"]:
            kind, n = int(w) & 15, int(w) >> 4
            if kind == M:
                for k in range(n):
                    v = s.get(p + k)
                    if v is not None and v[0] != v[1] and rec["codes"][q + k] == v[0]:
                        back += 1
            q += n if kind in (M, I, S) else 0
            p += n if kind in (M, D, N) else 0
    if which == "genome":
        assert back > 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["ir_fastq", "no_ir"])
def test_spliced_tags(name, tmp_path_factory, monkeypatch):
    """NM against the -rg genome the fixture's transcripts are spliced from, on plus- and minus-strand transcripts; with
    intron retention also on reads laid out on the genome (chains), forward and reverse-complemented."""
    from nanosim_b200 import _lib as L
    from nanosim_b200.engine import Engine
    from test_ir_homopolymer import _hp_model, _write_fixture
    chains, orig = set(), Engine.compress_bam_mapped

    def compress(self, names):
        for k in self.fetch(want_ops=True).pieces["kind"].astype(np.int64):
            if k & L.NS_PIECE_GENOME and k & L.NS_PIECE_KIND_MASK == L.NS_PIECE_SEGMENT:
                chains.add(bool(k & L.NS_PIECE_REF_REV))
        return orig(self, names)
    monkeypatch.setattr(Engine, "compress_bam_mapped", compress)
    d = str(tmp_path_factory.mktemp("tags_" + name))
    _write_fixture(d)
    model, _ = _hp_model(d)
    args = ["transcriptome", "-rt", os.path.join(d, "transcripts.fa"), "-rg", os.path.join(d, "genome.fa"), "-e",
            os.path.join(d, "expression.tsv"), "-c", model, "-n", "1500", "--ir_markov_model", os.path.join(d, "IR_markov_model"),
            "--ir_gff3", os.path.join(d, "annotation.gff3"), "--fastq", "--seed", "74", "--bam", "--spliced_bam"]
    if name == "no_ir":
        args.append("--no_model_ir")
    plain, tagged = _pair("splice_" + name, args, d)
    [(names, recs)] = _same_but_tags(plain, tagged, extra_files=("_aligned_error_profile",))
    check_tags(recs, names, fasta_refs(os.path.join(d, "genome.fa")), first_tag="XS")
    xs = {dict((t, v) for t, _, v, _, _ in r["aux"])["XS"] for r in recs if not r["flag"] & 4}
    assert xs == {"+", "-"}
    assert chains == ({False, True} if name == "ir_fastq" else set())


@pytest.mark.gpu
def test_sa_with_a_cigar_of_more_than_65535_ops(tmp_path):
    """Reads of about 1 Mb on a 4 Mb circular record: those across the origin have two records, one beyond 65 535 ops,
    whose SA entry carries the real CIGAR from CG."""
    ref = os.path.join(str(tmp_path), "long.fa")
    synth.write_fasta(ref, [("big", synth.synth_chrom(np.random.default_rng(9), 4_000_000))])
    args = ["genome", "-rg", ref, "-c", _model("guppy"), "-n", "24", "--fastq", "-med", "1000000", "-sd", "0.05", "-dna_type",
            "circular", "--seed", "75", "--bam", "--mapped_bam", "--no_error_profile"]
    plain, tagged = _pair("cg", args, str(tmp_path))
    [(names, recs)] = _same_but_tags(plain, tagged)
    assert check_tags(recs, names, fasta_refs(ref)) > 0
    assert any(len(g) > 1 and any(len(r["cigar"]) > 65535 for r in g) for g in groups(recs))


@pytest.mark.gpu
def test_independent_of_batching(tmp_path):
    from nanosim_b200 import simulator
    ref = _ecoli(str(tmp_path))
    outs = []
    for batch in (["--batch_reads", "700"], []):
        out = os.path.join(str(tmp_path), "b%d" % len(batch))
        simulator.main(["genome", "-rg", ref, "-c", _model("guppy"), "-n", "3000", "--fastq", "--chimeric", "--seed", "76", "-t", "3",
                        "--bam", "--mapped_bam", "--aln_tags", "-o", out] + batch)
        outs.append(out)
    a, b = (check_bgzf_file(o + "_aligned_reads.bam") for o in outs)
    assert a == b and len(read_tagged_bam(a)[2]) > 100


@pytest.mark.gpu
def test_set_aln_tags_rejects_other_tables_and_clones(genome):  # noqa: F811
    from nanosim_b200 import simulator
    from nanosim_b200.engine import NanoSimError
    d, ref, vcf = genome[:3]
    prof = simulator.read_profile(ref, [10], _model("guppy"), False, "genome", None, dna_type="linear", vcf=vcf, lift=True)
    t = prof.haplotypes
    names = list(prof.haploid.raw_names)
    with pytest.raises(NanoSimError, match="REF bytes table is for"):
        prof.engine.set_aln_tags(names, t.ref_paired, len(t.var_pos) + 1)
    with pytest.raises(NanoSimError, match="REF bytes table has"):
        prof.engine.set_aln_tags(names, t.ref_paired[:-1], len(t.var_pos))
    assert prof.engine.set_aln_tags(names, t.ref_paired, len(t.var_pos)) > 0
    clone = prof.engine.clone()
    with pytest.raises(NanoSimError, match=r"cloned context.*\(rc=-3\)"):
        clone.set_aln_tags(names, t.ref_paired, len(t.var_pos))
    clone.close()
    prof.engine.close()


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_ranks_equal_one_rank(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs (this box has %d)" % torch.cuda.device_count())
    ref = _ecoli(str(tmp_path))
    args = ["genome", "-rg", ref, "-c", _model("guppy"), "-n", "4000", "--fastq", "--chimeric", "--seed", "77", "--batch_reads",
            "700", "-t", "4", "--bam", "--mapped_bam", "--aln_tags"]
    one, two = os.path.join(str(tmp_path), "one"), os.path.join(str(tmp_path), "two")
    env = dict(os.environ, PYTHONPATH=ROOT)
    subprocess.run([sys.executable, "-m", "nanosim_b200.simulator"] + args + ["-o", one], check=True, env=env, cwd=ROOT)
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                    "--master-port", "29757", "-m", "nanosim_b200.simulator"] + args + ["-o", two], check=True, env=env, cwd=ROOT)
    for f in ("_aligned_reads.bam", "_unaligned_reads.bam"):
        assert check_bgzf_file(two + f) == check_bgzf_file(one + f), f
