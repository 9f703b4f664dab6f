"""--lift_mapped_bam: the true alignments of a --vcf run lifted onto the -rg records (ns_set_lift, ns_compress_bam_mapped).

The Python lift below restates DESIGN §3 "Lifted mapped BAM": a read's alignment to its haplotype record (the ops
test_mapped_bam.script_ops yields) is composed with the haplotype's segments, cut where the reference stops advancing
forward, and trimmed, merged and laid out by the rules of "Mapped BAM".  The CPU tests check it on hand-built cases; the
GPU tests compare the decompressed file with it byte for byte, and check the records without it against the haploid FASTA
and the VCF.  GPU tests run with ``pytest -m gpu``."""
import copy
import gzip
import os
import struct
import subprocess
import sys
import types

import numpy as np
import pytest

from conftest import ROOT

from test_bam_output import _CODE, bam_record
from test_bgzf_output import check_bgzf_file
from test_mapped_bam import (COMP_TABLE, D, H, I, M, N, S, _CUT, _header_of, _model, capture, read_mapped_bam,  # noqa: F401
                             reg2bin, script_ops)
from test_vcf_haplotypes import genome  # noqa: F401  (module-scoped fixtures: reference, VCF, haplotype FASTA)
from test_vcf_structural_variants import sv_genome  # noqa: F401

SEQ, DUP, INV = 0, 1, 2


# --------------------------------------------------------------------------------------------------------- Python lift
def lift_segments(t, haploid_lengths):
    """Per haplotype of a variants.HaplotypeTables: its segments in haplotype order, (hap0, hap_len, ref0, ref_len, kind):
    the stretch before each variant, the variant (a <DUP> copy onto its source span), the stretch behind the last one."""
    out = []
    for h in range(len(t.hap_chrom)):
        clen = int(haploid_lengths[int(t.hap_chrom[h])])
        segs, hp, end = [], 0, 0
        for j in range(int(t.var_off[h]), int(t.var_off[h + 1])):
            p, r, a, k = int(t.var_pos[j]), int(t.var_ref_len[j]), int(t.alt_len[j]), int(t.alt_kind[j])
            segs.append((hp, p - end, end, p - end, SEQ))
            hp += p - end
            segs.append((hp, a, int(t.alt_off[j]), a, DUP) if k == DUP else (hp, a, p, r, k))
            hp += a
            end = p + r
        segs.append((hp, clen - end, end, clen - end, SEQ))
        out.append(segs)
    return out


def compose(segs, pos, ops):
    """A script's ops (M I D over the haplotype from base pos) composed with the segments: (kind, n, at, inv) and
    (_CUT, 0, None, None).  at: the reference coordinate of an M or D's first base, or for inv (inside an <INV>) one past
    it in reference order.  M over an inserted ALT base is I, D over one vanishes; the reference-only bases of a sequence
    ALT are a D when the walk reaches them; a cut goes where a <DUP> copy begins and at both ends of an <INV>."""
    s = max(k for k, g in enumerate(segs) if g[0] <= pos)
    t, d_done, out = pos - segs[s][0], False, []

    def advance():
        nonlocal s, t, d_done
        while t >= segs[s][1]:
            hap0, a, ref0, r, kind = segs[s]
            if kind == SEQ and r > a and not d_done:
                out.append((D, r - a, ref0 + a, False))
                d_done = True
            if s == len(segs) - 1:
                return
            s, t, d_done = s + 1, 0, False
            if kind == INV or segs[s][4] != SEQ:
                out.append((_CUT, 0, None, None))

    for kind, n in ops:
        if kind == I:
            out.append((I, n, None, None))
            continue
        while n:
            hap0, a, ref0, r, k = segs[s]
            one = a if k != SEQ else min(a, r)
            assert t < a, "past the record's end"
            if k == INV:
                m = min(n, a - t)
                out.append((kind, m, ref0 + r - t, True))
            elif t < one:
                m = min(n, one - t)
                out.append((kind, m, ref0 + t, False))
            else:
                m = min(n, a - t)
                if kind == M:
                    out.append((I, m, None, None))
            t, n = t + m, n - m
            advance()
    return out


def lift_alignments(segs, pos, ops, q_start=0):
    """The lifted alignments of one segment: (pos, span, q0, q1, body, inv) per part with an M, read offsets forward."""
    parts, cur = [], []
    for o in compose(segs, pos, ops):
        if o[0] == _CUT:
            parts.append(cur)
            cur = []
        else:
            cur.append(o)
    parts.append(cur)
    alns, q = [], q_start
    for part in parts:
        ms = [j for j, o in enumerate(part) if o[0] == M]
        body, span = [], 0
        for j, (kind, n, at, inv) in enumerate(part):
            if ms and ms[0] <= j <= ms[-1]:
                if j == ms[0]:
                    q0, at0, inv0 = q, at, inv
                if body and body[-1][0] == kind:
                    body[-1] = (kind, body[-1][1] + n)
                else:
                    body.append((kind, n))
                span += n if kind != I else 0
                if j == ms[-1]:
                    q1 = q + n
            q += n if kind != D else 0
        if ms:
            alns.append((at0 - span if inv0 else at0, span, q0, q1, body, inv0))
    return alns


def lifted_layout(alns, L, rev):
    """The records of a read's lifted alignments [(ref_id, hp, pos, span, q0, q1, body, inv)]: dicts of ref_id, pos,
    span, flag, cigar (clips included, in the record's orientation), the stored range [lo, hi) of the read in that
    orientation, and hp."""
    prim = max(range(len(alns)), key=lambda k: (alns[k][3], -k))
    out = []
    for k, (ref_id, hp, pos, span, q0, q1, body, inv) in enumerate(alns):
        clip = S if k == prim else H
        cig = ([(clip, q0)] if q0 else []) + body + ([(clip, L - q1)] if q1 < L else [])
        lo, hi = (0, L) if k == prim else (q0, q1)
        if inv:
            cig, lo, hi = cig[::-1], L - hi, L - lo
        out.append(dict(ref_id=ref_id, pos=pos, span=span, flag=(16 if rev != inv else 0) | (0 if k == prim else 0x800), cigar=cig,
                        lo=lo, hi=hi, hp=hp))
    return out


def encode_record(name, rec, codes, q):
    """One lifted record's bytes; codes / q: the read's 4-bit codes and qualities in the record's orientation."""
    lo, hi = rec["lo"], rec["hi"]
    c = codes[lo:hi]
    if len(c) % 2:
        c = np.append(c, np.uint8(0))
    packed = ((c[0::2] << 4) | c[1::2]).astype(np.uint8).tobytes()
    words = np.array([(n << 4) | kind for kind, n in rec["cigar"]], dtype="<u4")
    aux = b"HPC" + bytes([rec["hp"]])
    if len(words) > 65535:
        field = struct.pack("<II", ((hi - lo) << 4) | S, (rec["span"] << 4) | N)
        aux += b"CGBI" + struct.pack("<I", len(words)) + words.tobytes()
    else:
        field = words.tobytes()
    pos, span = rec["pos"], rec["span"]
    body = struct.pack("<iiBBHHHIiii", rec["ref_id"], pos, len(name) + 1, 60, reg2bin(pos, pos + span), len(field) // 4, rec["flag"],
                       hi - lo, -1, -1, 0) + name + b"\0" + field + packed + q[lo:hi].astype(np.uint8).tobytes() + aux
    return struct.pack("<i", len(body)) + body


def lifted_records(b, i, name, lifts, hap_chrom, hap_number, fastq):
    """Read i's lifted records (or the unmapped record), as the rules lay them out."""
    r = b.reads[i]
    o, L, rev = int(r["seq_off"]), int(r["seq_len"]), bool(r["reversed"])
    seq = b.seq[o:o + L].tobytes()
    qual = b.qual[o:o + L].tobytes() if fastq else None
    alns = []
    for k in range(int(r["n_pieces"])):
        p = b.pieces[int(r["piece_first"]) + k]
        if int(p["kind"]) & 0xffff != 0:
            continue
        h = int(p["chrom"])
        ops = script_ops(b.ops[int(p["op_off"]):int(p["op_off"]) + int(p["n_ops"])], None)
        alns += [(int(hap_chrom[h]), int(hap_number[h])) + a for a in lift_alignments(lifts[h], int(p["pos"]), ops, int(p["out_rel"]))]
    if not alns:
        return bam_record(name, seq, qual)
    codes = _CODE[np.frombuffer(seq, dtype=np.uint8)]
    q = np.frombuffer(qual, dtype=np.uint8) - 33 if fastq else np.full(L, 0xff, dtype=np.uint8)
    if rev:
        codes, q = COMP_TABLE[codes[::-1]], q[::-1]
    rc_codes, rc_q = COMP_TABLE[codes[::-1]], q[::-1]
    out = b""
    for rec in lifted_layout(alns, L, rev):
        inv = bool(rec["flag"] & 16) != rev
        out += encode_record(name, rec, rc_codes if inv else codes, rc_q if inv else q)
    return out


def cigar_str(cig):
    return "".join("%d%s" % (n, "MIDNSH"[k]) for k, n in cig)


# ---------------------------------------------------------------------------------------------------------------- CPU
def _segs(clen, *variants):
    """One haplotype of a record of clen bases with variants (pos, ref_len, alt_len, kind[, alt_off])."""
    t = types.SimpleNamespace(hap_chrom=[0], var_off=[0, len(variants)], var_pos=[v[0] for v in variants],
                              var_ref_len=[v[1] for v in variants], alt_len=[v[2] for v in variants], alt_kind=[v[3] for v in variants],
                              alt_off=[v[4] if len(v) > 4 else v[0] for v in variants])
    return lift_segments(t, [clen])[0]


def _records(segs, pos, ops, L, rev=False, q_start=0, hp=1):
    alns = [(0, hp) + a for a in lift_alignments(segs, pos, ops, q_start)]
    if not alns:
        return []
    return [(r["pos"], r["flag"], cigar_str(r["cigar"]), r["lo"], r["hi"]) for r in lifted_layout(alns, L, rev)]


def test_snv_and_mnp_are_m():
    segs = _segs(100, (10, 1, 1, SEQ), (20, 3, 3, SEQ))
    assert _records(segs, 5, [(M, 30)], 30) == [(5, 0, "30M", 0, 30)]
    # a read D over the MNP's middle base and a read I behind it stay as they are
    assert _records(segs, 15, [(M, 6), (D, 1), (M, 4), (I, 2), (M, 5)], 17, rev=True) == [(15, 16, "6M1D4M2I5M", 0, 17)]


def test_padded_insertion_deletion_and_complex_alt():
    # REF A / ALT ATTT at 10 (insertion of 3), REF ATT / ALT A at 30 (1M2D), REF ACG / ALT TTTTT at 50 (3M then 2I)
    segs = _segs(100, (10, 1, 4, SEQ), (30, 3, 1, SEQ), (50, 3, 5, SEQ))
    # haplotype bases: [0,10) 1:1, 10 the ALT's first base, 11-13 inserted, 14.. = ref 11..; the deletion's ALT base is
    # haplotype 33 = ref 30, ref 31-32 deleted; the complex ALT is haplotype 51-55 = ref 50-52 and two inserted bases
    assert _records(segs, 0, [(M, 60)], 60) == [(0, 0, "11M3I20M2D20M2I4M", 0, 60)]
    # the 3 inserted bases sit at haplotype 11-13: a read starting inside them begins with I, which is clip
    assert _records(segs, 12, [(M, 10)], 10) == [(11, 0, "2S8M", 0, 10)]
    # ending inside them: the I after the last M is clip too
    assert _records(segs, 5, [(M, 8)], 8) == [(5, 0, "6M2S", 0, 8)]


def test_symbolic_deletion_is_d():
    segs = _segs(1000, (100, 400, 0, SEQ))                     # <DEL> of ref [100, 500)
    assert _records(segs, 90, [(M, 20)], 20) == [(90, 0, "10M400D10M", 0, 20)]
    # a read I at the deleted position comes after the D
    assert _records(segs, 90, [(M, 10), (I, 3), (M, 10)], 23) == [(90, 0, "10M400D3I10M", 0, 23)]
    # starting exactly behind the deletion: POS is the first base behind it
    assert _records(segs, 100, [(M, 10)], 10) == [(500, 0, "10M", 0, 10)]


def test_read_d_over_inserted_bases_vanishes():
    segs = _segs(100, (10, 1, 6, SEQ))                         # 5 inserted bases at haplotype 11-15
    assert _records(segs, 5, [(M, 6), (D, 5), (M, 6)], 12) == [(5, 0, "12M", 0, 12)]
    assert _records(segs, 5, [(M, 6), (D, 3), (M, 8)], 14) == [(5, 0, "6M2I6M", 0, 14)]


def test_read_wholly_inside_an_insertion_is_unmapped():
    segs = _segs(100, (10, 1, 50, SEQ))
    assert _records(segs, 15, [(M, 20)], 20) == []


def test_dup_copy_is_cut_into_two_records_over_the_source():
    segs = _segs(1000, (300, 0, 100, DUP, 200))                # <DUP> of ref [200, 300): a copy behind 300
    recs = _records(segs, 250, [(M, 100)], 100)
    assert recs == [(250, 0, "50M50S", 0, 100), (200, 0x800, "50H50M", 50, 100)]
    # the longer part is primary; both lie on [200, 300)
    recs = _records(segs, 290, [(M, 80)], 80)
    assert recs == [(290, 0x800, "10M70H", 0, 10), (200, 0, "10S70M", 0, 80)]


def test_inversion_containing_the_alignment_flips_the_strand():
    segs = _segs(1000, (100, 200, 200, INV))                   # <INV> of ref [100, 300)
    # haplotype 150..170 is ref 249..230 backwards: one record on the other strand, CIGAR reversed, clips mirrored
    recs = _records(segs, 150, [(M, 5), (D, 2), (M, 8), (I, 1), (M, 5)], 22, q_start=3)
    assert recs == [(230, 16, "5M1I8M2D5M3S", 0, 22)]
    assert _records(segs, 150, [(M, 20)], 20, rev=True) == [(230, 0, "20M", 0, 20)]


def test_inversion_crossing_one_or_both_ends():
    segs = _segs(1000, (100, 200, 200, INV))
    # 90..110 crosses the left end: 10 forward bases, then haplotype 100-109 = ref 299..290 on the other strand, where the
    # read's first 10 bases come last
    recs = _records(segs, 90, [(M, 20)], 20)
    assert recs == [(90, 0, "10M10S", 0, 20), (290, 0x800 | 16, "10M10H", 0, 10)]
    # a supplementary inverted part in the middle of a read: its stored range is mirrored
    recs = _records(segs, 280, [(M, 40)], 40)
    assert recs == [(100, 16, "20S20M", 0, 40), (300, 0x800, "20H20M", 20, 40)]
    # crossing both ends: forward, inverted (primary), forward
    recs = _records(segs, 95, [(M, 210)], 210)
    assert recs == [(95, 0x800, "5M205H", 0, 5), (100, 16, "5S200M5S", 0, 210), (300, 0x800, "205H5M", 205, 210)]


def test_hp_comes_before_cg():
    segs = _segs(400000, (10, 1, 1, SEQ))
    ops = [(M, 2), (I, 1)] * 40000 + [(M, 2)]
    alns = [(3, 2) + a for a in lift_alignments(segs, 0, ops)]
    rec = lifted_layout(alns, 120002, False)[0]
    assert len(rec["cigar"]) > 65535
    L = 120002
    data = encode_record(b"r", rec, np.ones(L, dtype=np.uint8), np.full(L, 30, dtype=np.uint8))
    l_seq = struct.unpack_from("<I", data, 20)[0]
    aux = data[4 + 32 + 2 + 8 + (l_seq + 1) // 2 + l_seq:]
    assert aux[:4] == b"HPC\x02" and aux[4:8] == b"CGBI"
    _, _, recs = read_mapped_bam_with_hp(b"BAM\1" + struct.pack("<i", 0) + struct.pack("<i", 0) + data)
    assert recs[0]["hp"] == 2 and recs[0]["cg"] and recs[0]["ref_id"] == 3


def read_mapped_bam_with_hp(data):
    """read_mapped_bam of a lifted file: each mapped record's leading HP:C field is taken off (its value in "hp") first."""
    head_end = len(_header_of(data))
    out = bytearray(data[:head_end])
    pos, hps = head_end, []
    while pos < len(data):
        block, flag, l_seq = struct.unpack_from("<i", data, pos)[0], struct.unpack_from("<H", data, pos + 18)[0], \
            struct.unpack_from("<I", data, pos + 20)[0]
        rec = bytearray(data[pos:pos + 4 + block])
        if flag & 4:
            hps.append(None)
        else:
            l_name, n_cig = rec[12], struct.unpack_from("<H", rec, 16)[0]
            a = 36 + l_name + 4 * n_cig + (l_seq + 1) // 2 + l_seq
            assert rec[a:a + 3] == b"HPC" and rec[a + 3] in (1, 2)
            hps.append(rec[a + 3])
            del rec[a:a + 4]
            struct.pack_into("<i", rec, 0, block - 4)
        out += rec
        pos += 4 + block
    text, refs, recs = read_mapped_bam(bytes(out))
    for r, hp in zip(recs, hps):
        r["hp"] = hp
    return text, refs, recs


_ARGV = ["genome", "-rg", "x.fa"]


@pytest.mark.parametrize("extra, message", [
    (["--bam", "--mapped_bam", "--lift_mapped_bam"], "--lift_mapped_bam needs --vcf"),
    (["--bam", "--vcf", "v.vcf", "--lift_mapped_bam"], "--lift_mapped_bam needs --mapped_bam"),
])
def test_usage_errors(extra, message, tmp_path, capsys):
    from nanosim_b200 import simulator
    with pytest.raises(SystemExit) as e:
        simulator.main(_ARGV + ["-o", os.path.join(str(tmp_path), "sim")] + extra)
    assert e.value.code == 1
    assert message + "!" in capsys.readouterr().err
    assert os.listdir(str(tmp_path)) == []


def test_header_names_the_haploid_records(tmp_path, monkeypatch):
    from nanosim_b200 import simulator
    from nanosim_b200.simulator import BGZF_EOF
    from test_bgzf_output import _EmptyPipeline, _empty_profile

    def profile(*a, **kw):
        prof = _empty_profile()
        prof.ref = types.SimpleNamespace(names=["chrA-hap1", "chrA-hap2"], raw_names=["chrA-hap1", "chrA-hap2"], lengths=np.array([990, 1004]),
                                         max_chrom=1004)
        prof.haploid = simulator._RemoteReference(["chrA"], [0, 1000], ["chrA"])
        return prof
    monkeypatch.setattr(simulator, "read_profile", profile)
    monkeypatch.setattr(simulator, "BatchPipeline", _EmptyPipeline)
    out = os.path.join(str(tmp_path), "sim")
    simulator.main(_ARGV + ["-o", out, "--bam", "--mapped_bam", "--vcf", "v.vcf", "--lift_mapped_bam"])
    data = open(out + "_aligned_reads.bam", "rb").read()
    assert data == simulator.bam_header([("chrA", 1000, False)]) + BGZF_EOF
    text, refs, recs = read_mapped_bam(gzip.decompress(data))
    assert refs == [(b"chrA", 1000)] and b"@SQ\tSN:chrA\tLN:1000\n" in text and recs == []


def test_haploid_header_of_a_vcf(genome):  # noqa: F811
    """The haploid reference's bam_refs: raw names (the FASTA header up to the first blank) and lengths."""
    from nanosim_b200.reference_fasta import PackedReference
    from nanosim_b200.simulator import bam_header, bam_refs
    d, ref = genome[:2]
    r = PackedReference.from_fasta(ref)
    refs = bam_refs(r)
    assert [n for n, _, _ in refs] == list(r.raw_names) and [ln for _, ln, _ in refs] == [int(x) for x in r.lengths]
    _, got, _ = read_mapped_bam(gzip.decompress(bam_header(refs)))
    assert got == [(n.encode(), ln) for n, ln, _ in refs]


def test_exports_name_the_new_entry_point():
    from nanosim_b200 import _lib
    header = open(os.path.join(ROOT, "include", "nanosim_b200.h")).read()
    assert "ns_set_lift" in _lib.EXPORTS and "ns_set_lift(" in header


# ---------------------------------------------------------------------------------------------------------------- GPU
_RUNS = {}


def _tables(ref_fa, vcf):
    from nanosim_b200.reference_fasta import PackedReference
    from nanosim_b200.variants import read_vcf
    r = PackedReference.from_fasta(ref_fa)
    t = read_vcf(vcf, r)
    return r, t, lift_segments(t, r.lengths)


_CONFIGS = {
    "genome_guppy_fastq": ("genome", ["-c", "guppy", "-n", "2500", "--fastq", "--seed", "61"]),
    "genome_fasta": ("genome", ["-c", "guppy", "-n", "2000", "--seed", "62"]),
    "sv_guppy_fastq": ("sv", ["-c", "guppy", "-n", "2500", "--fastq", "--seed", "63"]),
    "sv_dorado_hp6_chimeric": ("sv", ["-c", "dorado", "-n", "2000", "--fastq", "-hp", "-k", "6", "--chimeric", "--seed", "64"]),
}


def _argv(extra):
    extra = list(extra)
    extra[1] = _model(extra[1])
    return extra + ["-t", "4", "--bam", "--mapped_bam"]


def _run(name, fixture):
    """The configuration with --vcf --bam --mapped_bam, without and with --lift_mapped_bam (same seed)."""
    from nanosim_b200 import simulator
    if name not in _RUNS:
        d, ref, vcf = fixture[:3]
        plain, lifted = os.path.join(d, name + "_mapped"), os.path.join(d, name + "_lifted")
        args = ["genome", "-rg", ref, "--vcf", vcf] + _argv(_CONFIGS[name][1])
        simulator.main(args + ["-o", plain])
        simulator.main(args + ["-o", lifted, "--lift_mapped_bam"])
        _RUNS[name] = (plain, lifted, "--fastq" in _CONFIGS[name][1])
    return _RUNS[name]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(_CONFIGS))
def test_lifted_bam_equals_the_python_lift(name, genome, sv_genome, capture):  # noqa: F811
    from nanosim_b200 import simulator
    fixture = genome if _CONFIGS[name][0] == "genome" else sv_genome
    plain, lifted, fastq = _run(name, fixture)
    r, t, lifts = _tables(fixture[1], fixture[2])
    data = check_bgzf_file(lifted + "_aligned_reads.bam")
    head = _header_of(data)
    assert head == gzip.decompress(simulator.bam_header(simulator.bam_refs(r)))
    batches = sorted(capture[lifted], key=lambda bn: int(bn[0].first_id))
    twin = b"".join(lifted_records(b, i, names[i], lifts, t.hap_chrom, t.hap_number, fastq) for b, names in batches for i in range(len(names)))
    assert data[len(head):] == twin
    _, refs, recs = read_mapped_bam_with_hp(data)
    assert [n for n, _ in refs] == [n.encode() for n in r.raw_names]
    mapped = [x for x in recs if not x["flag"] & 4]
    assert len(mapped) > 100 and {x["hp"] for x in mapped} == {1, 2}
    assert any(x["cigar"][(x["cigar"] & 15) == D].size for x in mapped) and any(x["cigar"][(x["cigar"] & 15) == I].size for x in mapped)
    if _CONFIGS[name][0] == "sv":
        assert any(x["flag"] & 0x800 for x in mapped)


def _hap_variants(t, r, h):
    """Haplotype h's source record as 4-bit codes, whether each base is A, C, G or T (a read resolves other codes at
    random, and an inversion keeps U as it is), and the variants in reference coordinates: mismatching 1:1 positions, deletions and insertions (pos, n),
    inversion spans."""
    c = int(t.hap_chrom[h])
    raw = r.bases[int(r.offsets[c]):int(r.offsets[c + 1])]
    ref, acgt = _CODE[raw], np.isin(raw, np.frombuffer(b"ACGTacgt", dtype=np.uint8))
    mis, dels, ins, invs = set(), set(), set(), []
    for j in range(int(t.var_off[h]), int(t.var_off[h + 1])):
        p, rl, a, k = int(t.var_pos[j]), int(t.var_ref_len[j]), int(t.alt_len[j]), int(t.alt_kind[j])
        if k == INV:
            invs.append((p, p + rl))
        if k != SEQ:
            continue
        alt = _CODE[t.alt[int(t.alt_off[j]):int(t.alt_off[j]) + a]]
        mis |= {p + x for x in range(min(a, rl)) if alt[x] != ref[p + x]}
        if rl > a:
            dels.add((p + a, rl - a))
        if a > rl:
            ins.add((p + rl, a - rl))
    return ref, acgt, {p for p in mis if acgt[p]}, dels, ins, invs


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["genome", "sv"])
def test_perfect_records_are_the_haplotypes_variants(which, genome, sv_genome):  # noqa: F811
    """Without the Python lift, --perfect: every record's CIGAR walked over the haploid FASTA mismatches exactly at the
    SNV/MNP positions of its HP haplotype inside its span (at A/C/G/T reference bases); its D runs are that haplotype's deletions and its I runs its
    insertions; records inside an <INV> are on the other strand from the read's other records."""
    from nanosim_b200 import simulator
    fixture = genome if which == "genome" else sv_genome
    d, ref_fa, vcf = fixture[:3]
    out = os.path.join(d, which + "_perfect_lifted")
    simulator.main(["genome", "-rg", ref_fa, "--vcf", vcf, "-o", out, "--perfect", "--lift_mapped_bam"] +
                   _argv(["-c", "guppy", "-n", "1500", "--fastq", "--seed", "65"]))
    r, t, _ = _tables(ref_fa, vcf)
    _, refs, recs = read_mapped_bam_with_hp(check_bgzf_file(out + "_aligned_reads.bam"))
    hap_of = {(int(t.hap_chrom[h]), int(t.hap_number[h])): h for h in range(len(t.hap_chrom))}
    cache = {}
    n_mis = n_del = n_ins = n_inv = 0
    by_read = {}
    for x in recs:
        if x["flag"] & 4:
            continue
        h = hap_of[(x["ref_id"], x["hp"])]
        if h not in cache:
            cache[h] = _hap_variants(t, r, h)
        ref, acgt, mis, dels, ins, invs = cache[h]
        kinds, lens = x["cigar"] & 15, (x["cigar"] >> 4).astype(np.int64)
        rp, qp = x["pos"], int(lens[0]) if kinds[0] == S else 0
        got_mis, got_d, got_i = [], set(), set()
        for kind, n in zip(kinds, lens):
            n = int(n)
            if kind == M:
                got_mis += (rp + np.nonzero((ref[rp:rp + n] != x["codes"][qp:qp + n]) & acgt[rp:rp + n])[0]).tolist()
            if kind == D:
                got_d.add((rp, n))
            if kind == I:
                got_i.add((rp, n))
            rp += n if kind in (M, D) else 0
            qp += n if kind in (M, I) else 0
        lo, hi = x["pos"], rp
        assert sorted(got_mis) == sorted(p for p in mis if lo <= p < hi), x["name"]
        assert got_d == {(p, n) for p, n in dels if lo < p and p + n < hi}, x["name"]
        assert got_i == {(p, n) for p, n in ins if lo < p < hi}, x["name"]
        inside = any(a <= lo and hi <= b for a, b in invs)
        by_read.setdefault(x["name"], []).append((inside, x["flag"] & 16))
        n_mis, n_del, n_ins, n_inv = n_mis + len(got_mis), n_del + len(got_d), n_ins + len(got_i), n_inv + inside
    assert n_mis > 100 and n_del > 20 and n_ins > 20
    n_mixed = 0
    for parts in by_read.values():
        fwd = {s for inside, s in parts if not inside}
        rev = {s for inside, s in parts if inside}
        if fwd and rev:
            assert len(fwd) == len(rev) == 1 and fwd != rev
            n_mixed += 1
    if which == "sv":
        assert n_inv > 10 and n_mixed > 0


@pytest.mark.gpu
def test_all_reference_genotypes_give_the_mapped_records(genome, tmp_path):  # noqa: F811
    """A VCF whose sample is 0|0 everywhere: the lifted records are the --mapped_bam ones with HP taken off and the
    haplotype refIDs mapped to their source records."""
    from nanosim_b200 import simulator
    d, ref_fa, vcf = genome[:3]
    text = gzip.open(vcf, "rt").read().splitlines(True)
    rows = [ln if ln.startswith("#") else "\t".join(ln.rstrip("\n").split("\t")[:9] + ["0|0"]) + "\n" for ln in text]
    ref_vcf = os.path.join(str(tmp_path), "ref.vcf")
    open(ref_vcf, "w").write("".join(rows))
    args = ["genome", "-rg", ref_fa, "--vcf", ref_vcf] + _argv(["-c", "guppy", "-n", "2000", "--fastq", "--chimeric", "--seed", "66"])
    a, b = os.path.join(str(tmp_path), "mapped"), os.path.join(str(tmp_path), "lifted")
    simulator.main(args + ["-o", a])
    simulator.main(args + ["-o", b, "--lift_mapped_bam"])
    _, t, _ = _tables(ref_fa, ref_vcf)
    assert int(t.applied.sum()) == 0
    _, _, want = read_mapped_bam(check_bgzf_file(a + "_aligned_reads.bam"))
    _, _, got = read_mapped_bam_with_hp(check_bgzf_file(b + "_aligned_reads.bam"))
    assert len(got) == len(want) > 100
    for x, y in zip(got, want):
        if not y["flag"] & 4:
            assert x["hp"] == int(t.hap_number[y["ref_id"]])
            y["ref_id"] = int(t.hap_chrom[y["ref_id"]])
        x = dict(x)
        x.pop("hp")
        assert {k: (v.tolist() if isinstance(v, np.ndarray) else v) for k, v in x.items()} == \
            {k: (v.tolist() if isinstance(v, np.ndarray) else v) for k, v in y.items()}


@pytest.mark.gpu
def test_independent_of_batching(sv_genome):  # noqa: F811
    from nanosim_b200 import simulator
    d, ref_fa, vcf = sv_genome[:3]
    outs = []
    for batch in (["--batch_reads", "700"], []):
        out = os.path.join(d, "lift_batch%d" % len(batch))
        simulator.main(["genome", "-rg", ref_fa, "--vcf", vcf, "-o", out, "--lift_mapped_bam"] + batch +
                       _argv(["-c", "guppy", "-n", "3000", "--fastq", "--chimeric", "--seed", "67"]))
        outs.append(out)
    a, b = (check_bgzf_file(o + "_aligned_reads.bam") for o in outs)
    assert a == b and len(read_mapped_bam_with_hp(a)[2]) > 100


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_ranks_equal_one_rank(sv_genome, tmp_path):  # noqa: F811
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs (this box has %d)" % torch.cuda.device_count())
    d, ref_fa, vcf = sv_genome[:3]
    args = ["genome", "-rg", ref_fa, "--vcf", vcf, "--lift_mapped_bam", "--batch_reads", "700"] + \
        _argv(["-c", "guppy", "-n", "4000", "--fastq", "--chimeric", "--seed", "68"])
    one, two = os.path.join(str(tmp_path), "one"), os.path.join(str(tmp_path), "two")
    env = dict(os.environ, PYTHONPATH=ROOT)
    subprocess.run([sys.executable, "-m", "nanosim_b200.simulator"] + args + ["-o", one], check=True, env=env, cwd=ROOT)
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                    "--master-port", "29751", "-m", "nanosim_b200.simulator"] + args + ["-o", two], check=True, env=env, cwd=ROOT)
    for f in ("_aligned_reads.bam", "_unaligned_reads.bam"):
        assert check_bgzf_file(two + f) == check_bgzf_file(one + f), f


@pytest.mark.gpu
def test_set_lift_rejects_other_tables_and_clones(sv_genome):  # noqa: F811
    from nanosim_b200.engine import Engine, NanoSimError
    d, ref_fa, vcf = sv_genome[:3]
    r, t, _ = _tables(ref_fa, vcf)
    eng = Engine(device=0, seed=1)
    eng.set_reference(r)
    with pytest.raises(NanoSimError, match=r"not the haplotypes of ns_apply_variants.*\(rc=-3\)"):
        eng.set_lift(t)
    eng.apply_variants(t)
    longer = copy.deepcopy(t)                                   # haplotype 1 one base longer than its resident record
    j = int(np.nonzero((t.alt_kind == 0) & (np.arange(len(t.alt_len)) >= int(t.var_off[1])))[0][0])
    longer.alt_len[j] += 1
    with pytest.raises(NanoSimError, match=r"ns_set_lift: haplotype 1 has .*\(rc=-1\)"):
        eng.set_lift(longer)
    bad_kind = copy.deepcopy(t)
    bad_kind.alt_kind[0] = 3
    with pytest.raises(NanoSimError, match=r"ns_set_lift: variant 0 of haplotype 0 has ALT kind 3.*\(rc=-1\)"):
        eng.set_lift(bad_kind)
    assert eng.set_lift(t) >= 17 * (2 * len(t.var_pos) + len(t.hap_chrom))
    clone = eng.clone()
    with pytest.raises(NanoSimError, match=r"cloned context.*\(rc=-3\)"):
        clone.set_lift(t)
    clone.close()
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["genome_guppy_fastq", "sv_dorado_hp6_chimeric"])
def test_the_rest_of_the_output_is_unchanged(name, genome, sv_genome):  # noqa: F811
    """The unaligned file, the read names and the error profile are those of the same seed without the flag, and every
    record's SEQ/QUAL is the read in that record's orientation."""
    fixture = genome if _CONFIGS[name][0] == "genome" else sv_genome
    plain, lifted, fastq = _run(name, fixture)
    assert open(lifted + "_unaligned_reads.bam", "rb").read() == open(plain + "_unaligned_reads.bam", "rb").read()
    assert open(lifted + "_aligned_error_profile", "rb").read() == open(plain + "_aligned_error_profile", "rb").read()
    _, _, before = read_mapped_bam(check_bgzf_file(plain + "_aligned_reads.bam"))
    _, _, after = read_mapped_bam_with_hp(check_bgzf_file(lifted + "_aligned_reads.bam"))
    reads = {}
    for x in before:
        if not x["flag"] & 0x800:
            codes, qual = x["codes"], np.frombuffer(x["qual"], dtype=np.uint8)
            if x["flag"] & 16:
                codes, qual = COMP_TABLE[codes[::-1]], qual[::-1]
            reads[x["name"]] = (codes, qual)             # the read as sequenced
    assert [x["name"] for x in after if not x["flag"] & 0x800] == [x["name"] for x in before if not x["flag"] & 0x800]
    for x in after:
        codes, qual = reads[x["name"]]
        if x["flag"] & 16:
            codes, qual = COMP_TABLE[codes[::-1]], qual[::-1]
        kinds, lens = x["cigar"] & 15, (x["cigar"] >> 4).astype(np.int64)
        lo = int(lens[0]) if not x["flag"] & 4 and kinds[0] == H else 0
        assert (x["codes"] == codes[lo:lo + x["l_seq"]]).all()
        assert np.frombuffer(x["qual"], dtype=np.uint8).tolist() == qual[lo:lo + x["l_seq"]].tolist()
