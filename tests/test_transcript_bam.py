"""--transcript_bam: the true alignment of every transcriptome read to the -rt transcript it was simulated from, as mapped
BAM records built on the GPU (ns_compress_bam_transcript).

The Python encoder below restates DESIGN §3 "Transcript-coordinate mapped BAM" from a fetched batch (reads, pieces, emitted
ops, bases, qualities, names) and the splice map: a read on a transcript piece gets the records of "Mapped BAM", a read
that retains an intron walks its chain of genome pieces, each exon piece placed on the transcript through the map and
each retained intron's bases an insertion.  The decompressed ``<out>_aligned_reads.bam`` must be the transcript header
followed by its records.  Other tests check the records without the encoder: ``--perfect`` records against
transcripts.fa and the chains' retained pieces, NM against transcripts.fa, and that the rest of the output is what
``--bam`` and ``--spliced_bam`` write.  The fixture is test_spliced_bam's.  GPU tests run with ``pytest -m gpu``; the
rules, header and CLI tests need no GPU."""
import gzip
import os
import struct
import subprocess
import sys
import types

import numpy as np
import pytest

from conftest import ROOT

from test_aln_tags import check_tags, fasta_refs, read_tagged_bam, strip_tags
from test_bam_output import _CODE, bam_record, read_bam
from test_bgzf_output import _EmptyPipeline, _empty_profile, check_bgzf_file
from test_lifted_bam import cigar_str
from test_mapped_bam import COMP_TABLE, D, H, I, M, N, S, _CUT, _header_of, _names, mapped_records, read_mapped_bam, reg2bin, script_ops
from test_spliced_bam import _args, fixture_dir, fx  # noqa: F401  (module-scoped fixtures: the spliced transcripts)

NS_PIECE_RETAINED, NS_PIECE_GENOME = 0x20000000, 0x10000000


# ------------------------------------------------------------------------------------------------------ Python encoder
def trx_compose(chain, ops):
    """Ops (kind, n) over a chain's pieces back to back [(transcript offset of the piece's first base in chain order, or
    None for a retained intron, bases)], composed with the transcript: (kind, n, at) with at the transcript offset of an M
    or D's first base, and (_CUT, 0, None).  M and D over an exon piece stay; over a retained intron an M is I and a D
    vanishes; an exon piece that does not start where the last exon piece ended is a cut."""
    out, k, t = [], 0, 0
    off, ln = chain[0]
    end = None if off is None else off + ln
    for kind, n in ops:
        if kind == I:
            out.append((I, n, None))
            continue
        while n:
            while t >= ln and k + 1 < len(chain):
                k, t = k + 1, 0
                off, ln = chain[k]
                if off is not None:
                    if end is not None and off != end:
                        out.append((_CUT, 0, None))
                    end = off + ln
            m = min(n, ln - t) if t < ln else n
            if off is not None:
                out.append((kind, m, off + t))
            elif kind == M:
                out.append((I, m, None))
            t, n = t + m, n - m
    return out


def trx_alignments(chain, ops, q_start=0):
    """The alignments of one chain (or one transcript piece: a chain of one piece): (pos, span, q0, q1, body) per part
    with an M, read offsets forward; what lies before the first M and after the last one leaves the alignment."""
    parts, cur = [], []
    for o in trx_compose(chain, ops):
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
        for j, (kind, n, at) in enumerate(part):
            if ms and ms[0] <= j <= ms[-1]:
                if j == ms[0]:
                    q0, at0 = q, at
                if body and body[-1][0] == kind:
                    body[-1] = (kind, body[-1][1] + n)
                else:
                    body.append((kind, n))
                span += n if kind != I else 0
                if j == ms[-1]:
                    q1 = q + n
            q += n if kind != D else 0
        if ms:
            alns.append((at0, span, q0, q1, body))
    return alns


def exon_offset(smap, trx, chrom, start, end):
    """The transcript offset of the first base in transcript order of genome bases [start, end) of genome record chrom,
    when one exon of the transcript's map holds them (a linear scan), else None."""
    cum = 0
    for c, s, e in smap.exons(trx):
        if c == chrom and s <= start and end <= e:
            return cum + (e - end if smap.minus[trx] else start - s)
        cum += e - s
    return None


def read_alignments(b, i, smap, genome_first):
    """Read i's alignments [(refID, pos, span, q0, q1, body)] in record order: each transcript piece's, or its chain's (none
    when the chain's transcript has no map or an exon piece lies in none of its exons)."""
    r = b.reads[i]
    pf, n_pc = int(r["piece_first"]), int(r["n_pieces"])
    p0 = b.pieces[pf]
    if int(p0["kind"]) & NS_PIECE_GENOME:
        trx = int(p0["ref_req"])
        if smap is None or trx >= len(smap.minus) or not smap.exons(trx):
            return []
        segs = [b.pieces[pf + 2 * j] for j in range((n_pc + 1) // 2)]
        chain = []
        for p in segs:
            s, ln = int(p["pos"]), int(p["ref_len"])
            off = None if int(p["kind"]) & NS_PIECE_RETAINED else exon_offset(smap, trx, int(p["chrom"]) - genome_first, s, s + ln)
            if off is None and not int(p["kind"]) & NS_PIECE_RETAINED:
                return []
            chain.append((off, ln))
        ops = np.concatenate([b.ops[int(p["op_off"]):int(p["op_off"]) + int(p["n_ops"])] for p in segs])
        return [(trx,) + a for a in trx_alignments(chain, script_ops(ops, None), int(p0["out_rel"]))]
    alns = []
    for k in range(n_pc):
        p = b.pieces[pf + k]
        if int(p["kind"]) & 0xffff != 0:
            continue
        ops = script_ops(b.ops[int(p["op_off"]):int(p["op_off"]) + int(p["n_ops"])], None)
        alns += [(int(p["chrom"]),) + a for a in trx_alignments([(int(p["pos"]), int(p["ref_len"]))], ops, int(p["out_rel"]))]
    return alns


def layout(alns, L, rev):
    """The records of a read's alignments as "Mapped BAM" lays them out: refID, pos, span, flag, CIGAR with the clips,
    the stored range [lo, hi) of the read in forward orientation."""
    prim = max(range(len(alns)), key=lambda k: (alns[k][2], -k))
    out = []
    for k, (ref_id, pos, span, q0, q1, body) in enumerate(alns):
        clip = S if k == prim else H
        cig = ([(clip, q0)] if q0 else []) + body + ([(clip, L - q1)] if q1 < L else [])
        lo, hi = (0, L) if k == prim else (q0, q1)
        out.append(dict(ref_id=ref_id, pos=pos, span=span, flag=(16 if rev else 0) | (0 if k == prim else 0x800), cigar=cig, lo=lo, hi=hi))
    return out



def encode(name, rec, codes, q):
    """One record's bytes: no aux field but CG beyond 65 535 ops; codes / q the read's in the record's orientation."""
    lo, hi = rec["lo"], rec["hi"]
    c = codes[lo:hi]
    if len(c) % 2:
        c = np.append(c, np.uint8(0))
    packed = ((c[0::2] << 4) | c[1::2]).astype(np.uint8).tobytes()
    words = np.array([(n << 4) | kind for kind, n in rec["cigar"]], dtype="<u4")
    aux = b""
    if len(words) > 65535:
        field = struct.pack("<II", ((hi - lo) << 4) | S, (rec["span"] << 4) | N)
        aux = b"CGBI" + struct.pack("<I", len(words)) + words.tobytes()
    else:
        field = words.tobytes()
    pos, span = rec["pos"], rec["span"]
    body = struct.pack("<iiBBHHHIiii", rec["ref_id"], pos, len(name) + 1, 60, reg2bin(pos, pos + span), len(field) // 4, rec["flag"],
                       hi - lo, -1, -1, 0) + name + b"\0" + field + packed + q[lo:hi].astype(np.uint8).tobytes() + aux
    return struct.pack("<i", len(body)) + body


def transcript_records(b, i, name, smap, genome_first, fastq):
    """Read i's records against the transcripts (or the unmapped record), as the rules lay them out."""
    r = b.reads[i]
    o, L, rev = int(r["seq_off"]), int(r["seq_len"]), bool(r["reversed"])
    seq = b.seq[o:o + L].tobytes()
    qual = b.qual[o:o + L].tobytes() if fastq else None
    alns = read_alignments(b, i, smap, genome_first)
    if not alns:
        return bam_record(name, seq, qual)
    codes = _CODE[np.frombuffer(seq, dtype=np.uint8)]
    q = np.frombuffer(qual, dtype=np.uint8) - 33 if fastq else np.full(L, 0xff, dtype=np.uint8)
    if rev:
        codes, q = COMP_TABLE[codes[::-1]], q[::-1]
    return b"".join(encode(name, rec, codes, q) for rec in layout(alns, L, rev))


# ---------------------------------------------------------------------------------------------------------------- CPU
def _recs(chain, ops, L, rev=False, q_start=0, ref_id=0):
    alns = [(ref_id,) + a for a in trx_alignments(chain, ops, q_start)]
    return [(r["ref_id"], r["pos"], r["flag"], cigar_str(r["cigar"]), r["lo"], r["hi"]) for r in layout(alns, L, rev)] if alns else []


def _op(t, n, base=0):
    return (t << 28) | (base << 26) | n if t == 5 else (t << 28) | n


# a transcript of three exons in transcript order (cum 0, 100, 200), on either strand
_PLUS = [(0, 100, 200), (0, 300, 400), (0, 700, 800)]
_MINUS = [(1, 700, 800), (1, 300, 400), (1, 100, 200)]


def _smap(*transcripts):
    """A SpliceMap of transcripts [(exons in transcript order, minus)]."""
    from nanosim_b200.splice import SpliceMap
    ex = [e for t, _ in transcripts for e in t]
    off = np.concatenate([[0], np.cumsum([len(t) for t, _ in transcripts])]).astype(np.uint64)
    return SpliceMap(off, np.array([c for c, _, _ in ex], np.uint32), np.array([s for _, s, _ in ex], np.uint32),
                     np.array([e - s for _, s, e in ex], np.uint32), np.array([int(m) for _, m in transcripts], np.uint8),
                     np.array([1000, 1000], np.uint64), 2)


def test_exon_pieces_are_placed_through_the_map():
    m = _smap((_PLUS, False), (_MINUS, True))
    assert exon_offset(m, 0, 0, 150, 200) == 50 and exon_offset(m, 0, 0, 300, 340) == 100
    # minus strand: the piece's first base in transcript order is its highest genome base
    assert exon_offset(m, 1, 1, 700, 760) == 40 and exon_offset(m, 1, 1, 350, 400) == 100 and exon_offset(m, 1, 1, 100, 110) == 290
    # across an exon's end, on another record, in an intron: no exon holds it
    assert exon_offset(m, 0, 0, 190, 210) is None and exon_offset(m, 0, 1, 150, 200) is None and exon_offset(m, 0, 0, 250, 260) is None


def test_retained_intron_is_an_insertion():
    # plus: exon bases 50..99, the intron behind exon 0, exon 1 from its start
    assert _recs([(50, 50), (None, 100), (100, 40)], [(M, 190)], 190) == [(0, 50, 0, "50M100I40M", 0, 190)]
    # minus: genome 700..760 of exon 0 (transcript 40..99), the intron 400..700, genome 350..400 of exon 1 (transcript 100..149)
    m = _smap((_PLUS, False), (_MINUS, True))
    chain = [(exon_offset(m, 1, 1, 700, 760), 60), (None, 300), (exon_offset(m, 1, 1, 350, 400), 50)]
    assert _recs(chain, [(M, 410)], 410, ref_id=1) == [(1, 40, 0, "60M300I50M", 0, 410)]
    assert _recs(chain, [(M, 410)], 410, rev=True, ref_id=1) == [(1, 40, 16, "60M300I50M", 0, 410)]


def test_read_starting_in_a_retained_intron_is_clipped():
    assert _recs([(None, 50), (100, 100)], [(M, 150)], 150) == [(0, 100, 0, "50S100M", 0, 150)]
    # and one ending in it
    assert _recs([(60, 40), (None, 70)], [(M, 110)], 110) == [(0, 60, 0, "40M70S", 0, 110)]


def test_deletion_in_a_retained_intron_vanishes():
    assert _recs([(50, 50), (None, 100), (100, 100)], [(M, 80), (D, 10), (M, 160)], 240) == [(0, 50, 0, "50M90I100M", 0, 240)]
    # a D over exon bases stays
    assert _recs([(50, 50), (None, 100), (100, 100)], [(M, 40), (D, 10), (M, 200)], 240) == [(0, 50, 0, "40M10D100I100M", 0, 240)]


def test_lit_group_across_an_exon_intron_boundary():
    # the first piece's script ends in a LIT run, the retained piece's begins with the DEL that closes the group:
    # LIT 3 + DEL 6 -> 3 D (the exon's last bases) then 3 M (LIT) over the intron, as I
    ops = script_ops([_op(0, 47), _op(5, 3), _op(3, 6), _op(0, 94), _op(0, 100)], None)
    assert ops == [(M, 47), (D, 3), (M, 3), (M, 94), (M, 100)]
    assert _recs([(50, 50), (None, 100), (100, 100)], ops, 244) == [(0, 50, 0, "47M3D100I97M", 0, 244)]
    # LIT 8 + DEL 2 -> 6 I, then 2 M (LIT) across the boundary: one base on the exon, one in the intron
    ops = script_ops([_op(0, 49), _op(5, 8), _op(3, 2), _op(0, 99), _op(0, 10)], None)
    assert _recs([(50, 50), (None, 100), (100, 100)], ops, 166) == [(0, 50, 0, "49M6I1M100I10M", 0, 166)]


def test_non_contiguous_exon_pieces_are_split():
    # exon 1 first, then exon 0: the second piece does not continue the first in transcript offsets
    assert _recs([(100, 50), (50, 50)], [(M, 100)], 100) == [(0, 100, 0, "50M50S", 0, 100), (0, 50, 0x800, "50H50M", 50, 100)]
    # a retained intron between two contiguous exon pieces does not matter; between two others it goes with the first part
    assert _recs([(100, 50), (None, 30), (150, 20)], [(M, 100)], 100) == [(0, 100, 0, "50M30I20M", 0, 100)]
    assert _recs([(100, 50), (None, 30), (10, 60)], [(M, 140)], 140) == \
        [(0, 100, 0x800, "50M90H", 0, 50), (0, 10, 0, "80S60M", 0, 140)]


def test_polya_and_head_tail_are_s():
    ops = script_ops([_op(4, 4), _op(0, 30), _op(5, 10)], None)   # HT, COPY, a polyA LIT run
    assert ops == [(I, 4), (M, 30), (I, 10)]
    assert _recs([(20, 30)], ops, 44) == [(0, 20, 0, "4S30M10S", 0, 44)]
    assert _recs([(20, 10), (None, 5), (30, 15)], ops, 44) == [(0, 20, 0, "4S10M5I15M10S", 0, 44)]


def _batch(pieces, ops, seq=b"ACGTACGTAC", rev=0):
    from nanosim_b200 import _lib as L
    reads = np.zeros(1, dtype=L.READ_DTYPE)
    reads[0]["seq_len"], reads[0]["n_pieces"], reads[0]["reversed"] = len(seq), len(pieces), rev
    pc = np.zeros(len(pieces), dtype=L.PIECE_DTYPE)
    for k, p in enumerate(pieces):
        for key, v in p.items():
            pc[k][key] = v
    return types.SimpleNamespace(reads=reads, pieces=pc, ops=np.asarray(ops, dtype=np.uint32), seq=np.frombuffer(seq, dtype=np.uint8),
                                 qual=np.full(len(seq), 40, dtype=np.uint8))


def test_chains_outside_the_map_are_unmapped():
    m = _smap((_PLUS, False), ([], False))
    g = NS_PIECE_GENOME
    ok = [dict(kind=g, chrom=2, pos=190, ref_len=10, ref_req=0, n_ops=1, op_off=0)]
    b = _batch(ok, [10])
    _, _, recs = read_mapped_bam(b"BAM\1" + struct.pack("<i", 0) + struct.pack("<i", 0) + transcript_records(b, 0, b"r0", m, 2, True))
    assert [(r["ref_id"], r["pos"], r["flag"], r["cigar"].tolist()) for r in recs] == [(0, 90, 0, [(10 << 4) | M])]
    unmapped = bam_record(b"r0", b"ACGTACGTAC", bytes([40] * 10))
    # an exon piece across an exon's end, and a transcript without a map
    for piece in (dict(ok[0], pos=195), dict(ok[0], ref_req=1)):
        assert transcript_records(_batch([piece], [10]), 0, b"r0", m, 2, True) == unmapped
    # a transcript piece needs no map
    b = _batch([dict(kind=0, chrom=1, pos=7, ref_len=10, n_ops=1, op_off=0)], [10])
    assert transcript_records(b, 0, b"r0", None, 2, True) == mapped_records(b, 0, b"r0", [100, 100], True)


def test_transcript_pieces_agree_with_the_plain_encoder():
    """A transcript piece's records are the plain walk's: test_mapped_bam's encoder gives the same bytes."""
    ops = [_op(4, 3), _op(0, 20), _op(2, 2), _op(1, 1), _op(3, 4), _op(0, 30), _op(5, 2), _op(3, 1), _op(5, 9)]
    seq = bytes(np.random.default_rng(3).choice(list(b"ACGT"), 67).astype(np.uint8))
    b = _batch([dict(kind=0, chrom=1, pos=40, ref_len=56, n_ops=len(ops), op_off=0)], ops, seq=seq, rev=1)
    for fastq in (False, True):
        assert transcript_records(b, 0, b"r", None, 0, fastq) == mapped_records(b, 0, b"r", [100, 500], fastq)


_ARGV = ["transcriptome", "-rt", "t.fa", "-e", "e.tsv"]


@pytest.mark.parametrize("extra, message", [
    (["--no_model_ir", "--transcript_bam"], "--transcript_bam needs --bam"),
    (["--no_model_ir", "--bam", "--transcript_bam", "--spliced_bam", "-rg", "g.fa"], "both write <out>_aligned_reads.bam"),
    (["--bam", "--transcript_bam"], "Please provide a reference genome to simulate intron retention events"),
    (["--bam", "--transcript_bam", "-rg", "g.fa", "--ir_gff3", "/nonexistent/ann.gff3"],
     "--transcript_bam: the GFF3 annotation /nonexistent/ann.gff3 does not exist"),
    # the messages of the other truth BAMs keep their text
    (["--no_model_ir", "--bam", "--mapped_bam"], "--mapped_bam is not available in transcriptome mode"),
    (["--no_model_ir", "--bam", "--mapped_bam", "--transcript_bam"], "--mapped_bam is not available in transcriptome mode"),
    (["--no_model_ir", "--bam", "--aln_tags"], "--aln_tags needs --spliced_bam in transcriptome mode"),
])
def test_usage_errors(extra, message, tmp_path, capsys):
    from nanosim_b200 import simulator
    with pytest.raises(SystemExit) as e:
        simulator.main(_ARGV + ["-o", os.path.join(str(tmp_path), "sim")] + extra)
    assert e.value.code == 1
    assert message in capsys.readouterr().err
    assert os.listdir(str(tmp_path)) == []


class _SpliceEngine:
    """The engine calls of a --transcript_bam run's set-up, without a GPU."""

    def __init__(self):
        self.calls = []

    def configure(self, **kw):
        self.calls.append(("configure", kw.get("trx_records")))

    def set_splice(self, m):
        self.calls.append(("set_splice", m))

    def set_aln_tags(self, names, *a):
        self.calls.append(("set_aln_tags", list(names)))


def _profile(ir, raw=("ENST1.1", "ENST2.1")):
    """An empty run's profile over transcripts of 1000 and 900 bases, with intron retention the genome behind them."""
    from nanosim_b200.simulator import _RemoteReference

    def profile(*a, **kw):
        prof = _empty_profile()
        names, lens = ["t1", "t2"] + (["chr1", "chr2"] if ir else []), [1000, 900] + ([50000, 40000] if ir else [])
        prof.ref = _RemoteReference(names, np.concatenate([[0], np.cumsum(lens)]), list(raw) + (["chr1", "chr2"] if ir else []))
        prof.engine = _SpliceEngine()
        if ir:
            prof.ir, prof.n_trx, prof.splice = object(), 2, "the map"
        return prof
    return profile


@pytest.mark.parametrize("ir", [False, True])
@pytest.mark.parametrize("tags", [False, True])
def test_flag_writes_the_transcript_header(ir, tags, tmp_path, monkeypatch):
    from nanosim_b200 import simulator
    from nanosim_b200.simulator import BGZF_EOF
    profile = _profile(ir)
    seen = []
    monkeypatch.setattr(simulator, "read_profile", lambda *a, **kw: seen.append(profile()) or seen[-1])
    monkeypatch.setattr(simulator, "BatchPipeline", _EmptyPipeline)
    gff = os.path.join(str(tmp_path), "ann.gff3")
    open(gff, "w").close()
    out = os.path.join(str(tmp_path), "sim")
    extra = (["-rg", "g.fa", "--ir_gff3", gff] if ir else ["--no_model_ir"]) + (["--aln_tags"] if tags else [])
    simulator.main(_ARGV + ["-o", out, "--bam", "--transcript_bam"] + extra)
    refs = [("ENST1.1", 1000, False), ("ENST2.1", 900, False)]
    head = simulator.bam_header(refs)
    assert open(out + "_aligned_reads.bam", "rb").read() == head + BGZF_EOF
    assert open(out + "_unaligned_reads.bam", "rb").read() == simulator.bam_header() + BGZF_EOF
    assert b"chr1" not in gzip.decompress(head)
    calls = seen[0].engine.calls
    assert (("set_splice", "the map") in calls) == ir
    assert (("set_aln_tags", ["ENST1.1", "ENST2.1"]) in calls) == tags


@pytest.mark.parametrize("ir", [False, True])
@pytest.mark.parametrize("bad", ["duplicate", "oversized"])
def test_bad_transcript_records_are_usage_errors(ir, bad, tmp_path, monkeypatch, capsys):
    from nanosim_b200 import simulator
    profile = _profile(ir, raw=("ENST1.1", "ENST1.1"))
    if bad == "oversized":
        def profile(*a, **kw):                  # noqa: F811
            prof = _profile(ir)()
            prof.ref.offsets = prof.ref.offsets.copy()
            prof.ref.offsets[2:] += 1 << 31
            return prof
    monkeypatch.setattr(simulator, "read_profile", profile)
    monkeypatch.setattr(simulator, "BatchPipeline", _EmptyPipeline)
    gff = os.path.join(str(tmp_path), "ann.gff3")
    open(gff, "w").close()
    out = os.path.join(str(tmp_path), "out")
    os.mkdir(out)
    with pytest.raises(SystemExit) as e:
        simulator.main(_ARGV + ["-o", os.path.join(out, "sim"), "--bam", "--transcript_bam"] +
                       (["-rg", "g.fa", "--ir_gff3", gff] if ir else ["--no_model_ir"]))
    assert e.value.code == 1
    err = capsys.readouterr().err
    assert "--transcript_bam: " in err
    assert ("have the same name ENST1.1" if bad == "duplicate" else "record 1 (t2) has 2147484548 bases") in err
    assert os.listdir(out) == []


def test_merge_rank_files_writes_the_transcript_header_once(tmp_path):
    from nanosim_b200.simulator import BGZF_EOF, bam_header, merge_rank_files
    from test_bgzf_output import _zlib_member
    out = os.path.join(str(tmp_path), "sim")
    refs = [("ENST1.1", 1000, False), ("ENST2.1", 900, False)]
    parts = []
    for r in range(2):
        parts.append(_zlib_member(bam_record(b"aligned_%d" % r, b"ACGTA", None)))
        with open(out + "_aligned_reads%d.bam" % r, "wb") as f:
            f.write(parts[-1])
        with open(out + "_unaligned_reads%d.bam" % r, "wb") as f:
            f.write(parts[-1])
        open(out + "_error_profile%d" % r, "w").close()
    merge_rank_files(out, False, False, 2, bam=True, mapped_refs=refs)
    assert open(out + "_aligned_reads.bam", "rb").read() == bam_header(refs) + parts[0] + parts[1] + BGZF_EOF


def test_exports_name_the_new_entry_point():
    from nanosim_b200 import _lib
    header = open(os.path.join(ROOT, "include", "nanosim_b200.h")).read()
    assert "ns_compress_bam_transcript" in _lib.EXPORTS and "ns_compress_bam_transcript(" in header


# ------------------------------------------------------------------------------------------------------------- GPU runs
_CAPTURE = {}


@pytest.fixture
def capture(monkeypatch):
    """Every batch ns_compress_bam_transcript is called on, fetched (with its ops) as it stands, and its names, by output
    prefix; and the run's splice map."""
    from nanosim_b200 import simulator
    from nanosim_b200.engine import Engine
    orig, orig_sim = Engine.compress_bam_transcript, simulator.simulation
    cur = {}

    def compress(self, names):
        cur["list"].append((self.fetch(want_ops=True), _names(names)))
        return orig(self, names)

    def simulation(prof, mode, out, *a, **kw):
        cur["list"] = _CAPTURE.setdefault(out, [])
        _CAPTURE[out + ":splice"] = getattr(prof, "splice", None)
        return orig_sim(prof, mode, out, *a, **kw)

    monkeypatch.setattr(Engine, "compress_bam_transcript", compress)
    monkeypatch.setattr(simulator, "simulation", simulation)
    return _CAPTURE


_CONFIGS = ["ir_fastq", "ir_hp_polya", "no_ir", "perfect"]
_RUNS = {}


def _run(fx, name, *flags):
    """The configuration run with --bam and ``flags`` (same seed): the output prefix."""
    from nanosim_b200 import simulator
    key = (name,) + flags
    if key not in _RUNS:
        args, _ = _args(fx, name)
        out = os.path.join(fx["d"], "trx_" + name + "".join(flags).replace("-", "_"))
        simulator.main(args + ["-o", out, "--bam"] + list(flags))
        _RUNS[key] = out
    return _RUNS[key]


def _transcripts(fx):
    from nanosim_b200.reference_fasta import PackedReference
    return PackedReference.from_fasta(os.path.join(fx["d"], "transcripts.fa"))


def _batches(out):
    return sorted(_CAPTURE[out], key=lambda bn: int(bn[0].first_id))


def _is_chain(b, i):
    return bool(int(b.pieces[int(b.reads[i]["piece_first"])]["kind"]) & NS_PIECE_GENOME)


def _inner_retained(b, i):
    """The bases of chain read i's retained pieces between its first and last exon piece."""
    r = b.reads[i]
    pf = int(r["piece_first"])
    segs = [b.pieces[pf + 2 * j] for j in range((int(r["n_pieces"]) + 1) // 2)]
    ex = [j for j, p in enumerate(segs) if not int(p["kind"]) & NS_PIECE_RETAINED]
    return sum(int(p["ref_len"]) for j, p in enumerate(segs) if ex and ex[0] < j < ex[-1] and int(p["kind"]) & NS_PIECE_RETAINED)


@pytest.mark.gpu
@pytest.mark.parametrize("name", _CONFIGS)
def test_transcript_bam_equals_the_python_encoder(name, fx, capture):
    from nanosim_b200 import simulator
    out = _run(fx, name, "--transcript_bam")
    _, fastq = _args(fx, name)
    data = check_bgzf_file(out + "_aligned_reads.bam")
    head = _header_of(data)
    assert head == gzip.decompress(simulator.bam_header(simulator.bam_refs(_transcripts(fx))))
    smap = _CAPTURE[out + ":splice"]
    assert (smap is not None) == (name != "no_ir")
    g0 = smap.genome_first if smap is not None else 0
    batches = _batches(out)
    twin = b"".join(transcript_records(b, i, names[i], smap, g0, fastq) for b, names in batches for i in range(len(names)))
    assert data[len(head):] == twin
    _, refs, recs = read_mapped_bam(data)
    mapped = [r for r in recs if not r["flag"] & 4]
    assert len(mapped) > 500 and len({r["ref_id"] for r in mapped}) > 5 and not any(r["cg"] for r in mapped)
    if name.startswith("ir"):
        # chain reads on both strands, some with an insertion from a retained intron
        chains = [(b, i) for b, names in batches for i in range(len(names)) if _is_chain(b, i)]
        assert {bool(smap.minus[int(b.pieces[int(b.reads[i]["piece_first"])]["ref_req"])]) for b, i in chains} == {False, True}
        with_ir = 0
        for b, i in chains:
            inner = _inner_retained(b, i)
            ins = sum(n for a in read_alignments(b, i, smap, g0) for k, n in a[5] if k == I)
            with_ir += inner > 0 and ins >= inner // 2
        assert with_ir > 10


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["ir_fastq", "no_ir"])
def test_transcript_pieces_agree_with_the_mapped_encoder(name, fx, capture):
    """Reads that do not retain an intron: their records are what test_mapped_bam's plain restatement writes with the
    transcripts as the reference."""
    out = _run(fx, name, "--transcript_bam")
    _, fastq = _args(fx, name)
    lengths = _transcripts(fx).lengths
    data = check_bgzf_file(out + "_aligned_reads.bam")
    got = {}
    _, _, recs = read_mapped_bam(data)
    for r in recs:
        got.setdefault(r["name"], []).append(r)
    n = 0
    for b, names in _batches(out):
        for i in range(len(names)):
            if _is_chain(b, i):
                continue
            want = mapped_records(b, i, names[i], lengths, fastq)
            _, _, wr = read_mapped_bam(b"BAM\1" + struct.pack("<i", 0) + struct.pack("<i", 0) + want)
            assert [(r["ref_id"], r["pos"], r["flag"], r["cigar"].tolist()) for r in got[names[i]]] == \
                [(r["ref_id"], r["pos"], r["flag"], r["cigar"].tolist()) for r in wr]
            n += 1
    assert n > 50


def _check_perfect(recs, trx):
    """Every M base of SEQ is the transcript base (case-folded; an IUPAC code matches any base it allows), and POS + span
    lies within the transcript.  Returns the M bases."""
    n_m = 0
    for r in recs:
        if r["flag"] & 4:
            continue
        ref = _CODE[trx.bases[int(trx.offsets[r["ref_id"]]):int(trx.offsets[r["ref_id"] + 1])]]
        kinds, lens = r["cigar"] & 15, (r["cigar"] >> 4).astype(np.int64)
        rp, qp = r["pos"], 0
        for kind, n in zip(kinds, lens):
            if kind == M:
                assert ((ref[rp:rp + n] & r["codes"][qp:qp + n]) != 0).all(), r["name"]
                n_m += int(n)
            rp += int(n) if kind in (M, D) else 0
            qp += int(n) if kind in (M, I, S) else 0
        assert rp <= len(ref), r["name"]
    return n_m


@pytest.mark.gpu
def test_perfect_records_are_the_transcripts(fx):
    """Without the encoder, on --perfect reads: the CLI's (which retain no intron) against transcripts.fa, and a batch of
    the engine with intron retention applied as the CLI applies it (plan_batch, ns_reemit).  A read that retains an
    intron has, in its one record, I bases adding up to its retained pieces between its first and last exon piece (those
    at either end are clip)."""
    from nanosim_b200 import _lib as L
    from nanosim_b200 import intron_retention as ir
    from nanosim_b200.reference_fasta import PackedReference, read_expression
    from nanosim_b200.splice import build_splice_map
    import parity_checks as pc
    trx = _transcripts(fx)
    _, _, recs = read_mapped_bam(check_bgzf_file(_run(fx, "perfect", "--transcript_bam") + "_aligned_reads.bam"))
    assert _check_perfect(recs, trx) > 100000
    d = fx["d"]
    genome = PackedReference.from_fasta(os.path.join(d, "genome.fa"))
    n_trx = len(trx.names)
    chrom, w = read_expression(os.path.join(d, "expression.tsv"), trx)
    st = ir.TranscriptStructures.from_gff3(os.path.join(d, "annotation.gff3"), trx.names, genome.raw_names)
    eng, _, _ = pc.make_trx_engine(PackedReference.concat(trx, genome), chrom, w, perfect=True, seed=72, trx_records=n_trx,
                                   max_len=trx.max_chrom)
    try:
        eng.set_splice(build_splice_map(st, trx.lengths, genome.lengths, n_trx))
        info = eng.simulate(L.NS_KIND_ALIGNED, 0, 1500)
        irm = ir.IntronRetention(ir.read_ir_markov_model(os.path.join(d, "IR_markov_model")), st, trx.lengths, n_trx)
        reads, pieces, ops = eng.fetch_meta()
        eng.reemit(*irm.plan_batch(reads, pieces, ops, 0, 72, info.n_pieces, info.n_ops, info.raw_ev_off))
        b = eng.fetch(want_ops=True)
        names = ["r%d" % i for i in range(len(b.reads))]
        eng.compress_bam_transcript(names)
        data = gzip.decompress(eng.fetch_compressed().tobytes())
    finally:
        eng.close()
    _, _, recs = read_mapped_bam(b"BAM\1" + struct.pack("<i", 0) + struct.pack("<i", 0) + data)
    assert _check_perfect(recs, trx) > 100000
    by_name = {}
    for r in recs:
        by_name.setdefault(r["name"].decode(), []).append(r)
    n_chain = 0
    for i, name in enumerate(names):
        if not _is_chain(b, i):
            continue
        got = by_name[name]
        assert len(got) == 1 and not got[0]["flag"] & 4, name
        inner = _inner_retained(b, i)
        assert sum(int(x) >> 4 for x in got[0]["cigar"] if int(x) & 15 == I) == inner, name
        n_chain += inner > 0
    assert n_chain > 50


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["ir_fastq", "no_ir"])
def test_the_rest_of_the_output_is_what_bam_writes(name, fx, capture):
    out, bam, spliced = (_run(fx, name, *f) for f in (["--transcript_bam"], [], ["--spliced_bam"]))
    for f in ("_unaligned_reads.bam", "_aligned_error_profile"):
        ref = open(bam + f, "rb").read()
        assert open(out + f, "rb").read() == ref == open(spliced + f, "rb").read(), f
    _, unmapped = read_bam(check_bgzf_file(bam + "_aligned_reads.bam"))
    _, _, recs = read_mapped_bam(check_bgzf_file(out + "_aligned_reads.bam"))
    prim = [r for r in recs if not r["flag"] & 0x800]
    assert [r["name"] for r in prim] == [u["name"] for u in unmapped]
    for r, u in zip(prim, unmapped):
        codes, qual = r["codes"], r["qual"]
        if r["flag"] & 16:
            codes, qual = COMP_TABLE[codes[::-1]], qual[::-1]
        assert (codes == u["codes"]).all() and qual == u["qual"]


@pytest.mark.gpu
def test_independent_of_batching(fx):
    from nanosim_b200 import simulator
    args, _ = _args(fx, "ir_hp_polya")
    outs = []
    for batch in ("64", "1000"):
        out = os.path.join(fx["d"], "trx_batch" + batch)
        simulator.main(args + ["-o", out, "--bam", "--transcript_bam", "--batch_reads", batch])
        outs.append(out)
    a, b = (check_bgzf_file(o + "_aligned_reads.bam") for o in outs)
    assert a == b and len(read_mapped_bam(a)[2]) > 500


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["ir_fastq", "no_ir"])
def test_tags_are_calmd_against_the_transcripts(name, fx, capture):
    """NM against transcripts.fa, on transcript pieces and on chains (compared base by base: the read was copied from the
    genome); removing NM and SA gives the untagged file."""
    plain = _run(fx, name, "--transcript_bam")
    tagged = _run(fx, name, "--transcript_bam", "--aln_tags")
    a = check_bgzf_file(plain + "_aligned_reads.bam")
    head, names, recs = read_tagged_bam(check_bgzf_file(tagged + "_aligned_reads.bam"))
    assert a == head + b"".join(strip_tags(r) for r in recs)
    for f in ("_unaligned_reads.bam", "_aligned_error_profile"):
        assert open(plain + f, "rb").read() == open(tagged + f, "rb").read(), f
    check_tags(recs, names, fasta_refs(os.path.join(fx["d"], "transcripts.fa")))
    nm = [dict((t, v) for t, _, v, _, _ in r["aux"])["NM"] for r in recs if not r["flag"] & 4]
    assert len(nm) > 500 and np.mean(nm) > 0
    if name == "ir_fastq":
        assert any(_is_chain(b, i) for b, ns in _batches(tagged) for i in range(len(ns)))


@pytest.mark.gpu
def test_engine_needs_a_matching_splice_map_with_intron_retention(fx):
    from nanosim_b200 import _lib as L
    from nanosim_b200 import intron_retention as ir
    from nanosim_b200.engine import Engine, NanoSimError
    from nanosim_b200.model import DeviceTables, build_alias, load_model
    from nanosim_b200.reference_fasta import PackedReference, read_expression
    from nanosim_b200.splice import build_splice_map
    d = fx["d"]
    trx = _transcripts(fx)
    genome = PackedReference.from_fasta(os.path.join(d, "genome.fa"))
    chrom, w = read_expression(os.path.join(d, "expression.tsv"), trx)
    names = ["r%d" % i for i in range(20)]
    tables = DeviceTables(load_model(fx["model"]), fastq=True)
    pr, al = build_alias(w)
    engines = []

    def engine(ref, **kw):
        eng = Engine(device=0, seed=71)
        engines.append(eng)
        eng.set_reference(ref)
        eng.set_model(tables)
        if kw.get("transcriptome"):
            eng.set_expression(pr, al, chrom, None)
        eng.configure(fastq=True, min_len=50, max_len=trx.max_chrom, **kw)
        return eng
    try:
        # intron retention: the genome behind the transcripts, and a map that is the run's
        eng = engine(PackedReference.concat(trx, genome), transcriptome=True, trx_records=len(trx.names))
        eng.simulate(L.NS_KIND_ALIGNED, 0, 20)
        with pytest.raises(NanoSimError, match="splice map.*rc=-1"):
            eng.compress_bam_transcript(names)
        st = ir.TranscriptStructures.from_gff3(os.path.join(d, "annotation.gff3"), trx.names, genome.raw_names)
        eng.set_splice(build_splice_map(st, trx.lengths, genome.lengths))
        with pytest.raises(NanoSimError, match="not the run's.*rc=-1"):
            eng.compress_bam_transcript(names)
        eng.set_splice(build_splice_map(st, trx.lengths, genome.lengths, len(trx.names)))
        assert eng.compress_bam_transcript(names) > 0
        eng.simulate(L.NS_KIND_UNALIGNED, 0, 20)
        with pytest.raises(NanoSimError, match="unaligned.*rc=-1"):
            eng.compress_bam_transcript(names)
        # without intron retention no map is needed, and compress_bam_mapped still wants one
        eng = engine(trx, transcriptome=True)
        eng.simulate(L.NS_KIND_ALIGNED, 0, 20)
        assert eng.compress_bam_transcript(names) > 0
        with pytest.raises(NanoSimError, match="splice map.*rc=-1"):
            eng.compress_bam_mapped(names)
        # a genome context
        eng = engine(genome)
        eng.simulate(L.NS_KIND_ALIGNED, 0, 20)
        with pytest.raises(NanoSimError, match="transcriptome context.*rc=-1"):
            eng.compress_bam_transcript(names)
    finally:
        for e in engines:
            e.close()


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_ranks_equal_one_rank(fx):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs (this box has %d)" % torch.cuda.device_count())
    args, _ = _args(fx, "ir_hp_polya")
    args = args + ["--bam", "--transcript_bam", "--aln_tags", "--batch_reads", "300"]
    one, two = os.path.join(fx["d"], "trx_rank_one"), os.path.join(fx["d"], "trx_rank_two")
    env = dict(os.environ, PYTHONPATH=ROOT)
    subprocess.run([sys.executable, "-m", "nanosim_b200.simulator"] + args + ["-o", one], check=True, env=env, cwd=ROOT)
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                    "--master-port", "29763", "-m", "nanosim_b200.simulator"] + args + ["-o", two], check=True, env=env, cwd=ROOT)
    for f in ("_aligned_reads.bam", "_unaligned_reads.bam"):
        assert check_bgzf_file(two + f) == check_bgzf_file(one + f), f
