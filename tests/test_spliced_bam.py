"""--spliced_bam: the true spliced alignment of every transcriptome read to the genome, as mapped BAM records built on the
GPU (ns_set_splice + ns_compress_bam_mapped).

The Python encoder below restates the rules of DESIGN §3 "Spliced mapped BAM" from a fetched batch (reads, pieces, emitted
ops, bases, qualities, names) and the splice map; the decompressed ``<out>_aligned_reads.bam`` must be the genome header
followed by its records.  Other tests check the records without the encoder: ``--perfect`` records against genome.fa and
the annotation, every N against the read's transcript's introns, and that the rest of the output is what ``--bam``
writes.  The fixture is test_ir_homopolymer's seeded genome with plus- and minus-strand transcripts spliced from it.  GPU
tests run with ``pytest -m gpu``; the rules, map builder and CLI tests need no GPU."""
import gzip
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT

from test_bam_output import _CODE, bam_record
from test_bgzf_output import check_bgzf_file
from test_ir_homopolymer import _hp_model, _write_fixture
from test_lifted_bam import cigar_str, lifted_layout
from test_mapped_bam import COMP_TABLE, D, I, M, N, S, _CUT, _header_of, _names, read_mapped_bam, reg2bin, script_ops

NS_PIECE_REF_REV, NS_PIECE_GENOME = 0x80000000, 0x10000000


# ------------------------------------------------------------------------------------------------------ Python encoder
def splice_compose(ivs, k, t, inv, ops):
    """Ops (kind, n) over the walk's intervals ivs [(genome record, start, end)] in walk order, from offset t of interval k,
    composed with them: (kind, n, at, record), at the genome coordinate of an M or D's first base (inv: one past it), and
    (_CUT, 0, None, None).  An M or D that reaches the next interval's first base first emits the distance to it in the
    walk's direction as N (nothing when it is 0), or a cut when that interval is on another record or not further on."""
    out = []
    c, s, e = ivs[k]
    for kind, n in ops:
        if kind == I:
            out.append((I, n, None, None))
            continue
        while n:
            if t >= e - s and k + 1 < len(ivs):
                c2, s2, e2 = ivs[k + 1]
                gap = s - e2 if inv else s2 - e
                if c2 != c or gap < 0:
                    out.append((_CUT, 0, None, None))
                elif gap:
                    out.append((N, gap, None, c))
                k, t, (c, s, e) = k + 1, 0, ivs[k + 1]
            m = min(n, e - s - t) if t < e - s else n
            out.append((kind, m, e - t if inv else s + t, c))
            t, n = t + m, n - m
    return out


def splice_alignments(ivs, k, t, inv, ops, q_start=0):
    """The spliced alignments of one read: (record, pos, span, q0, q1, body) per part with an M, read offsets forward;
    everything before the first M and after the last one leaves the alignment (an N or D before it moves POS)."""
    parts, cur = [], []
    for o in splice_compose(ivs, k, t, inv, ops):
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
        for j, (kind, n, at, c) in enumerate(part):
            if ms and ms[0] <= j <= ms[-1]:
                if j == ms[0]:
                    q0, at0, c0 = q, at, c
                if body and body[-1][0] == kind:
                    body[-1] = (kind, body[-1][1] + n)
                else:
                    body.append((kind, n))
                span += n if kind != I else 0
                if j == ms[-1]:
                    q1 = q + n
            q += n if kind in (M, I) else 0
        if ms:
            alns.append((c0, at0 - span if inv else at0, span, q0, q1, body))
    return alns


def read_walk(b, i, smap, genome_first):
    """Read i's walk: (intervals, k, t, minus, ops, q_start), or None (no map: the unmapped record)."""
    r = b.reads[i]
    pf, n_pc = int(r["piece_first"]), int(r["n_pieces"])
    p0 = b.pieces[pf]
    if int(p0["kind"]) & 0xffff != 0:
        return None
    if int(p0["kind"]) & NS_PIECE_GENOME:                       # it retains an intron: its chain of genome pieces
        chain = [b.pieces[pf + 2 * j] for j in range((n_pc + 1) // 2)]
        ivs = [(int(p["chrom"]) - genome_first, int(p["pos"]), int(p["pos"]) + int(p["ref_len"])) for p in chain]
        ops = np.concatenate([b.ops[int(p["op_off"]):int(p["op_off"]) + int(p["n_ops"])] for p in chain])
        return ivs, 0, 0, bool(int(p0["kind"]) & NS_PIECE_REF_REV), ops, int(p0["out_rel"])
    trx = int(p0["chrom"])
    ivs = smap.exons(trx)
    if not ivs:
        return None
    cum = np.cumsum([0] + [e - s for _, s, e in ivs])
    pos = int(p0["pos"])
    k = int(np.searchsorted(cum[:-1], pos, side="right")) - 1
    return ivs, k, pos - int(cum[k]), bool(smap.minus[trx]), b.ops[int(p0["op_off"]):int(p0["op_off"]) + int(p0["n_ops"])], \
        int(p0["out_rel"])


def spliced_layout(alns, L, rev, minus):
    """The records of a read's spliced alignments, as lifted_layout lays out lifted ones: a minus-strand transcript's part
    is a record on the other strand (CIGAR reversed, stored range mirrored); hp carries the strand."""
    return lifted_layout([(c, int(minus), pos, span, q0, q1, body, minus) for c, pos, span, q0, q1, body in alns], L, rev)


def encode_spliced(name, rec, codes, q):
    """One spliced record's bytes (XS:A first, then CG when the CIGAR has more than 65 535 ops); codes / q: the read's
    4-bit codes and qualities in the record's orientation."""
    lo, hi = rec["lo"], rec["hi"]
    c = codes[lo:hi]
    if len(c) % 2:
        c = np.append(c, np.uint8(0))
    packed = ((c[0::2] << 4) | c[1::2]).astype(np.uint8).tobytes()
    words = np.array([(n << 4) | kind for kind, n in rec["cigar"]], dtype="<u4")
    aux = b"XSA" + (b"-" if rec["hp"] else b"+")
    if len(words) > 65535:
        field = struct.pack("<II", ((hi - lo) << 4) | S, (rec["span"] << 4) | N)
        aux += b"CGBI" + struct.pack("<I", len(words)) + words.tobytes()
    else:
        field = words.tobytes()
    pos, span = rec["pos"], rec["span"]
    body = struct.pack("<iiBBHHHIiii", rec["ref_id"], pos, len(name) + 1, 60, reg2bin(pos, pos + span), len(field) // 4, rec["flag"],
                       hi - lo, -1, -1, 0) + name + b"\0" + field + packed + q[lo:hi].astype(np.uint8).tobytes() + aux
    return struct.pack("<i", len(body)) + body


def spliced_records(b, i, name, smap, genome_first, fastq):
    """Read i's spliced records (or the unmapped record), as the rules lay them out."""
    r = b.reads[i]
    o, L, rev = int(r["seq_off"]), int(r["seq_len"]), bool(r["reversed"])
    seq = b.seq[o:o + L].tobytes()
    qual = b.qual[o:o + L].tobytes() if fastq else None
    walk = read_walk(b, i, smap, genome_first)
    alns = []
    if walk is not None:
        ivs, k, t, minus, ops, q_start = walk
        alns = splice_alignments(ivs, k, t, minus, script_ops(ops, None), q_start)
    if not alns:
        return bam_record(name, seq, qual)
    codes = _CODE[np.frombuffer(seq, dtype=np.uint8)]
    q = np.frombuffer(qual, dtype=np.uint8) - 33 if fastq else np.full(L, 0xff, dtype=np.uint8)
    if rev:
        codes, q = COMP_TABLE[codes[::-1]], q[::-1]
    if minus:
        codes, q = COMP_TABLE[codes[::-1]], q[::-1]
    return b"".join(encode_spliced(name, rec, codes, q) for rec in spliced_layout(alns, L, rev, minus))


def read_spliced_bam(data):
    """read_mapped_bam of a spliced file: each mapped record's leading XS:A field is taken off (its value in "xs") first."""
    head_end = len(_header_of(data))
    out = bytearray(data[:head_end])
    pos, xs = head_end, []
    while pos < len(data):
        block, flag, l_seq = struct.unpack_from("<i", data, pos)[0], struct.unpack_from("<H", data, pos + 18)[0], \
            struct.unpack_from("<I", data, pos + 20)[0]
        rec = bytearray(data[pos:pos + 4 + block])
        if flag & 4:
            xs.append(None)
        else:
            l_name, n_cig = rec[12], struct.unpack_from("<H", rec, 16)[0]
            a = 36 + l_name + 4 * n_cig + (l_seq + 1) // 2 + l_seq
            assert rec[a:a + 3] == b"XSA" and rec[a + 3:a + 4] in (b"+", b"-")
            xs.append(rec[a + 3:a + 4].decode())
            del rec[a:a + 4]
            struct.pack_into("<i", rec, 0, block - 4)
        out += rec
        pos += 4 + block
    text, refs, recs = read_mapped_bam(bytes(out))
    for r, x in zip(recs, xs):
        r["xs"] = x
    return text, refs, recs


# ---------------------------------------------------------------------------------------------------------------- CPU
def _recs(ivs, k, t, minus, ops, L, rev=False, q_start=0):
    alns = splice_alignments(ivs, k, t, minus, ops, q_start)
    return [(r["ref_id"], r["pos"], r["flag"], cigar_str(r["cigar"]), r["lo"], r["hi"]) for r in spliced_layout(alns, L, rev, minus)] \
        if alns else []


_PLUS = [(0, 100, 200), (0, 300, 400), (0, 700, 800)]           # transcript order, plus strand: introns of 100 and 300
_MINUS = [(1, 700, 800), (1, 300, 400), (1, 100, 200)]          # transcript order, minus strand


def test_inside_one_exon_is_m():
    assert _recs(_PLUS, 0, 10, False, [(M, 50)], 50) == [(0, 110, 0, "50M", 0, 50)]
    assert _recs(_PLUS, 2, 0, False, [(M, 100)], 100) == [(0, 700, 0, "100M", 0, 100)]


def test_across_a_junction_is_n():
    assert _recs(_PLUS, 0, 80, False, [(M, 50)], 50) == [(0, 180, 0, "20M100N30M", 0, 50)]
    assert _recs(_PLUS, 0, 80, False, [(M, 150)], 150) == [(0, 180, 0, "20M100N100M300N30M", 0, 150)]


def test_insertion_at_a_junction_stays_before_the_n():
    assert _recs(_PLUS, 0, 80, False, [(M, 20), (I, 3), (M, 30)], 53) == [(0, 180, 0, "20M3I100N30M", 0, 53)]


def test_deletion_across_a_junction_is_d_n_d():
    assert _recs(_PLUS, 0, 80, False, [(M, 18), (D, 4), (M, 30)], 48) == [(0, 180, 0, "18M2D100N2D30M", 0, 48)]
    # a D ending exactly at the exon's end: the N waits for the next M
    assert _recs(_PLUS, 0, 80, False, [(M, 18), (D, 2), (M, 30)], 48) == [(0, 180, 0, "18M2D100N30M", 0, 48)]


def test_leading_d_and_n_move_pos():
    assert _recs(_PLUS, 0, 90, False, [(D, 20), (M, 30)], 30) == [(0, 310, 0, "30M", 0, 30)]
    # a leading insertion is clip, the D behind it moves POS
    assert _recs(_PLUS, 0, 90, False, [(I, 4), (D, 10), (M, 30)], 34) == [(0, 300, 0, "4S30M", 0, 34)]


def test_minus_strand_is_the_other_strand():
    # transcript base t of the first exon is genome base 799 - t: the walk runs down the genome
    assert _recs(_MINUS, 0, 80, True, [(M, 50)], 50) == [(1, 370, 16, "30M300N20M", 0, 50)]
    assert _recs(_MINUS, 0, 80, True, [(M, 50)], 50, rev=True) == [(1, 370, 0, "30M300N20M", 0, 50)]
    # walk order 5S 20M 3I 300N 30M 2D 10M: reversed onto the genome, clips mirrored
    assert _recs(_MINUS, 0, 80, True, [(I, 5), (M, 20), (I, 3), (M, 30), (D, 2), (M, 10)], 68, q_start=0) == \
        [(1, 358, 16, "10M2D30M300N3I20M5S", 0, 68)]


def test_polya_and_head_tail_are_s():
    def op(t, n):
        return (t << 28) | n
    ops = script_ops([op(4, 4), op(0, 30), op(5, 10)], None)   # HT, COPY, a polyA LIT run
    assert ops == [(I, 4), (M, 30), (I, 10)]
    assert _recs(_PLUS, 1, 20, False, ops, 44) == [(0, 320, 0, "4S30M10S", 0, 44)]


def test_exon_and_adjacent_retained_intron_merge():
    chain = [(0, 100, 200), (0, 200, 300), (0, 400, 500)]      # exon, the retained intron behind it, the next exon
    assert _recs(chain, 0, 50, False, [(M, 250)], 250) == [(0, 150, 0, "150M100N100M", 0, 250)]
    minus = [(0, 400, 500), (0, 300, 400), (0, 100, 200)]
    assert _recs(minus, 0, 0, True, [(M, 250)], 250) == [(0, 150, 16, "50M100N200M", 0, 250)]


def test_non_monotone_chain_is_split():
    chain = [(0, 400, 500), (0, 100, 200)]
    assert _recs(chain, 0, 0, False, [(M, 150)], 150) == [(0, 400, 0, "100M50S", 0, 150), (0, 100, 0x800, "100H50M", 100, 150)]
    # on another record too
    chain = [(0, 100, 200), (1, 300, 400)]
    assert _recs(chain, 0, 40, False, [(M, 30), (M, 70)], 100) == [(0, 140, 0, "60M40S", 0, 100), (1, 300, 0x800, "60H40M", 60, 100)]


def _batch(pieces, ops, seq=b"ACGTACGTAC", rev=0):
    import types
    from nanosim_b200 import _lib as L
    reads = np.zeros(1, dtype=L.READ_DTYPE)
    reads[0]["seq_len"], reads[0]["n_pieces"], reads[0]["reversed"] = len(seq), len(pieces), rev
    pc = np.zeros(len(pieces), dtype=L.PIECE_DTYPE)
    for k, p in enumerate(pieces):
        for key, v in p.items():
            pc[k][key] = v
    return types.SimpleNamespace(reads=reads, pieces=pc, ops=np.asarray(ops, dtype=np.uint32), seq=np.frombuffer(seq, dtype=np.uint8),
                                 qual=np.full(len(seq), 40, dtype=np.uint8))


def test_transcript_without_a_map_is_unmapped():
    from nanosim_b200.splice import SpliceMap
    smap = SpliceMap(np.array([0, 0, 1], dtype=np.uint64), np.array([0], np.uint32), np.array([5], np.uint32), np.array([10], np.uint32),
                     np.array([0, 0], np.uint8), np.array([100], np.uint64))
    b = _batch([dict(chrom=0, pos=0, ref_len=10, n_ops=1, op_off=0)], [10])
    assert spliced_records(b, 0, b"r0", smap, 0, True) == bam_record(b"r0", b"ACGTACGTAC", bytes([40] * 10))
    b = _batch([dict(chrom=1, pos=0, ref_len=10, n_ops=1, op_off=0)], [10])
    text = spliced_records(b, 0, b"r0", smap, 0, True)
    _, _, recs = read_spliced_bam(b"BAM\1" + struct.pack("<i", 0) + struct.pack("<i", 0) + text)
    assert [(r["ref_id"], r["pos"], r["flag"], r["xs"]) for r in recs] == [(0, 5, 0, "+")]


def test_xs_comes_before_cg():
    ops = [(M, 2), (I, 1)] * 40000 + [(M, 2)]
    L = 120002
    alns = splice_alignments([(3, 0, 400000)], 0, 0, True, ops)
    rec = spliced_layout(alns, L, False, True)[0]
    assert len(rec["cigar"]) > 65535
    data = encode_spliced(b"r", rec, np.ones(L, dtype=np.uint8), np.full(L, 30, dtype=np.uint8))
    l_seq = struct.unpack_from("<I", data, 20)[0]
    aux = data[4 + 32 + 2 + 8 + (l_seq + 1) // 2 + l_seq:]
    assert aux[:4] == b"XSA-" and aux[4:8] == b"CGBI"
    _, _, recs = read_spliced_bam(b"BAM\1" + struct.pack("<i", 0) + struct.pack("<i", 0) + data)
    assert recs[0]["xs"] == "-" and recs[0]["cg"] and recs[0]["ref_id"] == 3 and recs[0]["flag"] == 16


def _gff(path, rows):
    with open(path, "w") as f:
        f.write("##gff-version 3\n")
        for chrom, tid, a, b, strand in rows:
            f.write("%s\tT\texon\t%d\t%d\t.\t%s\t.\tParent=transcript:%s;transcript_id=%s\n" % (chrom, a + 1, b, strand, tid, tid))


def _map(tmp_path, name, rows, trx, lengths, genome=(("chr1", 10000), ("chr2", 5000))):
    from nanosim_b200.intron_retention import TranscriptStructures
    from nanosim_b200.splice import build_splice_map
    path = os.path.join(str(tmp_path), name)
    _gff(path, rows)
    st = TranscriptStructures.from_gff3(path, trx, [g for g, _ in genome])
    return build_splice_map(st, lengths, [n for _, n in genome])


def test_map_is_the_same_from_ascending_and_descending_exons(tmp_path):
    exons = {"T1": ("chr1", "+", [(100, 200), (300, 350), (900, 1000)]), "T2": ("chr2", "-", [(50, 80), (200, 400), (1000, 1010)])}
    trx, lengths = ["T1", "T2"], [250, 240]
    up = [(c, t, a, b, s) for t, (c, s, ex) in exons.items() for a, b in ex]
    down = [(c, t, a, b, s) for t, (c, s, ex) in exons.items() for a, b in ex[::-1]]
    m1, m2 = _map(tmp_path, "up.gff3", up, trx, lengths), _map(tmp_path, "down.gff3", down, trx, lengths)
    for m in (m1, m2):
        assert m.exons(0) == [(0, 100, 200), (0, 300, 350), (0, 900, 1000)]
        assert m.exons(1) == [(1, 1000, 1010), (1, 200, 400), (1, 50, 80)]
        assert m.minus.tolist() == [0, 1] and m.genome_len.tolist() == [10000, 5000] and m.genome_first is None


@pytest.mark.parametrize("rows, length", [
    ([], 100),                                                                          # no exons
    ([("chr1", "T", 0, 50, "+"), ("chr2", "T", 100, 150, "+")], 100),                   # two records
    ([("chr1", "T", 0, 50, "+"), ("chr1", "T", 100, 150, "-")], 100),                   # two strands
    ([("chr1", "T", 0, 60, "+"), ("chr1", "T", 50, 90, "+")], 100),                     # overlapping exons
    ([("chr1", "T", 9990, 10040, "+"), ("chr1", "T", 0, 50, "+")], 100),                # an exon outside its record
    ([("chr1", "T", 0, 50, "+"), ("chr1", "T", 100, 149, "+")], 100),                   # lengths that do not add up
    ([("chr9", "T", 0, 50, "+"), ("chr9", "T", 100, 150, "+")], 100),                   # a chromosome -rg lacks
])
def test_invalid_structures_get_no_map(rows, length, tmp_path):
    rows = rows + [("chr1", "OK", 2000, 2100, "+")]
    m = _map(tmp_path, "bad.gff3", rows, ["T", "OK"], [length, 100])
    assert m.exons(0) == [] and m.has_map().tolist() == [False, True]


@pytest.fixture(scope="module")
def fixture_dir(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("spliced"))
    _write_fixture(d)
    return d


def _trx_args(d, out, extra=()):
    return ["transcriptome", "-rt", os.path.join(d, "transcripts.fa"), "-e", os.path.join(d, "expression.tsv"), "-o", out] + list(extra)


@pytest.mark.parametrize("extra, message", [
    (["-rg", "G", "--no_model_ir", "--spliced_bam"], "--spliced_bam needs --bam"),
    (["--no_model_ir", "--bam", "--spliced_bam"], "--spliced_bam needs -rg"),
    (["-rg", "G", "--no_model_ir", "--bam", "--spliced_bam", "--ir_gff3", "/nonexistent/ann.gff3"],
     "the GFF3 annotation /nonexistent/ann.gff3 does not exist"),
    (["-rg", "G", "--bam", "--mapped_bam", "--spliced_bam"], "--mapped_bam is not available in transcriptome mode"),
])
def test_usage_errors(extra, message, fixture_dir, tmp_path, capsys):
    from nanosim_b200 import simulator
    extra = [os.path.join(fixture_dir, "genome.fa") if x == "G" else x for x in extra]
    with pytest.raises(SystemExit) as e:
        simulator.main(_trx_args(fixture_dir, os.path.join(str(tmp_path), "sim"), extra))
    assert e.value.code == 1
    assert message in capsys.readouterr().err
    assert os.listdir(str(tmp_path)) == []


@pytest.mark.parametrize("ir", [False, True])
@pytest.mark.parametrize("bad", ["duplicate", "oversized"])
def test_bad_genome_records_are_usage_errors(ir, bad, fixture_dir, tmp_path, monkeypatch, capsys):
    """The genome's records as bam_refs sees them: two with one name (a FASTA reader merges records with one key, so the
    names are made equal on the way), or one longer than BAM's l_ref holds."""
    from nanosim_b200 import simulator
    orig = simulator.bam_refs

    def spoiled(ref, circular=False):
        if bad == "duplicate":
            ref.raw_names = [ref.raw_names[0]] * len(ref.raw_names)
        else:
            ref.offsets = ref.offsets.copy()
            ref.offsets[-1] = ref.offsets[-2] + (1 << 31)
        return orig(ref, circular)
    monkeypatch.setattr(simulator, "bam_refs", spoiled)
    out = os.path.join(str(tmp_path), "out")
    os.mkdir(out)
    extra = ["-rg", os.path.join(fixture_dir, "genome.fa"), "--bam", "--spliced_bam", "--ir_gff3", os.path.join(fixture_dir, "annotation.gff3"),
             "--ir_markov_model", os.path.join(fixture_dir, "IR_markov_model"), "-c", os.path.join(fixture_dir, "none")]
    with pytest.raises(SystemExit) as e:
        simulator.main(_trx_args(fixture_dir, os.path.join(out, "sim"), extra + ([] if ir else ["--no_model_ir"])))
    assert e.value.code == 1
    err = capsys.readouterr().err
    assert ("have the same name chr1" if bad == "duplicate" else "more than the 2147483647") in err
    assert os.listdir(out) == []


def test_exports_name_the_new_entry_point():
    from nanosim_b200 import _lib
    header = open(os.path.join(ROOT, "include", "nanosim_b200.h")).read()
    assert "ns_set_splice" in _lib.EXPORTS and "ns_set_splice(" in header


# ------------------------------------------------------------------------------------------------------------- GPU runs
_CAPTURE = {}


@pytest.fixture
def capture(monkeypatch):
    """Every batch ns_compress_bam_mapped is called on, fetched (with its ops) as it stands, and its names, by output
    prefix; and the run's splice map."""
    from nanosim_b200 import simulator
    from nanosim_b200.engine import Engine
    orig, orig_sim = Engine.compress_bam_mapped, simulator.simulation
    cur = {}

    def compress(self, names):
        cur["list"].append((self.fetch(want_ops=True), _names(names)))
        return orig(self, names)

    def simulation(prof, mode, out, *a, **kw):
        cur["list"] = _CAPTURE.setdefault(out, [])
        _CAPTURE[out + ":splice"] = getattr(prof, "splice", None)
        return orig_sim(prof, mode, out, *a, **kw)

    monkeypatch.setattr(Engine, "compress_bam_mapped", compress)
    monkeypatch.setattr(simulator, "simulation", simulation)
    return _CAPTURE


@pytest.fixture(scope="module")
def fx(fixture_dir):
    model, _ = _hp_model(fixture_dir)
    return dict(d=fixture_dir, model=model)


def _args(fx, name):
    d = fx["d"]
    base = ["transcriptome", "-rt", os.path.join(d, "transcripts.fa"), "-rg", os.path.join(d, "genome.fa"), "-e",
            os.path.join(d, "expression.tsv"), "-c", fx["model"], "-n", "1500", "-t", "4", "--ir_markov_model",
            os.path.join(d, "IR_markov_model"), "--ir_gff3", os.path.join(d, "annotation.gff3")]
    if name == "ir_fastq":
        return base + ["--fastq", "--seed", "61"], True
    if name == "ir_hp_polya":
        return base + ["--fastq", "-hp", "-k", "6", "--polya", os.path.join(d, "polya.txt"), "-b", "guppy", "--seed", "62"], True
    if name == "no_ir":
        return base + ["--no_model_ir", "--fastq", "--seed", "63"], True
    assert name == "perfect"
    return base + ["--perfect", "--fastq", "--seed", "64"], True


_CONFIGS = ["ir_fastq", "ir_hp_polya", "no_ir", "perfect"]
_RUNS = {}


def _run(fx, name):
    """The configuration run with --bam and with --bam --spliced_bam (same seed)."""
    from nanosim_b200 import simulator
    if name not in _RUNS:
        args, fastq = _args(fx, name)
        bam, spliced = (os.path.join(fx["d"], name + s) for s in ("_bam", "_spliced"))
        simulator.main(args + ["-o", bam, "--bam"])
        simulator.main(args + ["-o", spliced, "--bam", "--spliced_bam"])
        _RUNS[name] = (bam, spliced, fastq)
    return _RUNS[name]


def _genome(fx):
    from nanosim_b200.reference_fasta import PackedReference
    return PackedReference.from_fasta(os.path.join(fx["d"], "genome.fa"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", _CONFIGS)
def test_spliced_bam_equals_the_python_encoder(name, fx, capture):
    from nanosim_b200 import simulator
    bam, spliced, fastq = _run(fx, name)
    data = check_bgzf_file(spliced + "_aligned_reads.bam")
    head = _header_of(data)
    assert head == gzip.decompress(simulator.bam_header(simulator.bam_refs(_genome(fx))))
    smap = _CAPTURE[spliced + ":splice"]
    g0 = smap.genome_first if smap.genome_first is not None else 0
    batches = sorted(_CAPTURE[spliced], key=lambda bn: int(bn[0].first_id))
    twin = b"".join(spliced_records(b, i, names[i], smap, g0, fastq) for b, names in batches for i in range(len(names)))
    assert data[len(head):] == twin
    _, refs, recs = read_spliced_bam(data)
    mapped = [r for r in recs if not r["flag"] & 4]
    assert len(mapped) > 500 and {r["xs"] for r in mapped} == {"+", "-"} and {r["ref_id"] for r in mapped} == {0, 1}
    assert any(N in (r["cigar"] & 15).tolist() for r in mapped)
    if name.startswith("ir"):
        assert any(int(b.pieces[int(b.reads[i]["piece_first"])]["kind"]) & NS_PIECE_GENOME for b, names in batches
                   for i in range(len(names)))


def _annotation(fx):
    """Per transcript name: its introns on the genome, as (record index, start, end)."""
    from nanosim_b200.intron_retention import INTRON, TranscriptStructures
    from nanosim_b200.reference_fasta import PackedReference
    trx = PackedReference.from_fasta(os.path.join(fx["d"], "transcripts.fa"))
    st = TranscriptStructures.from_gff3(os.path.join(fx["d"], "annotation.gff3"), trx.names, _genome(fx).raw_names)
    out = {}
    for t, name in enumerate(trx.names):
        a, b = int(st.first[t]), int(st.first[t + 1])
        out[name] = {(int(st.chrom[j]), int(st.start[j]), int(st.end[j])) for j in range(a, b) if st.ftype[j] == INTRON}
    return out


def _walk_n(r):
    """The record's N operations as genome intervals, and its span."""
    kinds, lens = r["cigar"] & 15, (r["cigar"] >> 4).astype(np.int64)
    rp, ns = r["pos"], []
    for kind, n in zip(kinds, lens):
        if kind == N:
            ns.append((r["ref_id"], rp, rp + int(n)))
        if kind in (M, D, N):
            rp += int(n)
    return ns, rp - r["pos"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["perfect", "ir_fastq", "ir_hp_polya"])
def test_records_agree_with_the_genome_and_the_annotation(name, fx, capture):
    """Without the encoder: every N is exactly one annotated intron of the read's transcript and none lies over an intron
    the read retains (its name lists them); POS + span lies within the record; with --perfect every M base of SEQ is the
    genome base (case-folded; an IUPAC code matches any base it allows)."""
    bam, spliced, fastq = _run(fx, name)
    _, refs, recs = read_spliced_bam(check_bgzf_file(spliced + "_aligned_reads.bam"))
    introns = _annotation(fx)
    g = _genome(fx)
    n_n = n_m = 0
    for r in recs:
        if r["flag"] & 4:
            continue
        qname = r["name"].decode()
        trx = qname.split("_")[0]
        ns, span = _walk_n(r)
        assert r["pos"] + span <= refs[r["ref_id"]][1]
        assert all(x in introns[trx] for x in ns), (qname, ns)
        if "_RetainedIntron_" in qname:
            kept = [tuple(int(v) for v in iv.split("-")) for iv in qname.split("_RetainedIntron_")[1].split("_")[0].split(";") if iv]
            assert not any(c == r["ref_id"] and s < b and a < e for c, a, b in ns for s, e in kept), qname
        n_n += len(ns)
        if name == "perfect":
            chrom = _CODE[g.bases[int(g.offsets[r["ref_id"]]):int(g.offsets[r["ref_id"] + 1])]]
            kinds, lens = r["cigar"] & 15, (r["cigar"] >> 4).astype(np.int64)
            rp, qp = r["pos"], int(lens[0]) if kinds[0] == S else 0
            for kind, n in zip(kinds, lens):
                if kind == M:
                    assert ((chrom[rp:rp + n] & r["codes"][qp:qp + n]) != 0).all(), qname
                    n_m += int(n)
                if kind in (M, D, N):
                    rp += int(n)
                if kind in (M, I):
                    qp += int(n)
    assert n_n > 100
    if name == "perfect":
        assert n_m > 100000


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["ir_fastq", "no_ir"])
def test_the_rest_of_the_output_is_what_bam_writes(name, fx, capture):
    from test_bam_output import read_bam
    bam, spliced, fastq = _run(fx, name)
    assert open(spliced + "_unaligned_reads.bam", "rb").read() == open(bam + "_unaligned_reads.bam", "rb").read()
    assert open(spliced + "_aligned_error_profile", "rb").read() == open(bam + "_aligned_error_profile", "rb").read()
    _, unmapped = read_bam(check_bgzf_file(bam + "_aligned_reads.bam"))
    _, _, recs = read_spliced_bam(check_bgzf_file(spliced + "_aligned_reads.bam"))
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
        out = os.path.join(fx["d"], "batch" + batch)
        simulator.main(args + ["-o", out, "--bam", "--spliced_bam", "--batch_reads", batch])
        outs.append(out)
    a, b = (check_bgzf_file(o + "_aligned_reads.bam") for o in outs)
    assert a == b and len(read_spliced_bam(a)[2]) > 500


@pytest.mark.gpu
def test_engine_needs_a_matching_splice_map(fx):
    import copy
    from nanosim_b200 import _lib as L
    from nanosim_b200 import intron_retention as ir
    from nanosim_b200.engine import Engine, NanoSimError
    from nanosim_b200.model import DeviceTables, build_alias, load_model
    from nanosim_b200.reference_fasta import PackedReference, read_expression
    from nanosim_b200.splice import build_splice_map
    d = fx["d"]
    trx = PackedReference.from_fasta(os.path.join(d, "transcripts.fa"))
    genome = _genome(fx)
    chrom, w = read_expression(os.path.join(d, "expression.tsv"), trx)
    eng = Engine(device=0, seed=70)
    eng.set_reference(trx)
    eng.set_model(DeviceTables(load_model(fx["model"]), fastq=True))
    pr, al = build_alias(w)
    eng.set_expression(pr, al, chrom, None)
    eng.configure(fastq=True, min_len=50, max_len=trx.max_chrom, transcriptome=True)
    eng.simulate(L.NS_KIND_ALIGNED, 0, 20)
    names = ["r%d" % i for i in range(20)]
    with pytest.raises(NanoSimError, match="splice map.*rc=-1"):
        eng.compress_bam_mapped(names)
    st = ir.TranscriptStructures.from_gff3(os.path.join(d, "annotation.gff3"), trx.names, genome.raw_names)
    smap = build_splice_map(st, trx.lengths, genome.lengths)
    bad = copy.copy(smap)
    bad.exon_len = smap.exon_len.copy()
    bad.exon_len[0] -= 1
    with pytest.raises(NanoSimError, match="transcript 0 add up to .*rc=-1"):
        eng.set_splice(bad)
    assert eng.set_splice(smap) > 0
    assert eng.compress_bam_mapped(names) > 0
    clone = eng.clone()
    with pytest.raises(NanoSimError, match="rc=-3"):
        clone.set_splice(smap)
    clone.close()
    eng.close()


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_ranks_equal_one_rank(fx):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs (this box has %d)" % torch.cuda.device_count())
    args, _ = _args(fx, "ir_hp_polya")
    args = args + ["--bam", "--spliced_bam", "--batch_reads", "300"]
    one, two = os.path.join(fx["d"], "rank_one"), os.path.join(fx["d"], "rank_two")
    env = dict(os.environ, PYTHONPATH=ROOT)
    subprocess.run([sys.executable, "-m", "nanosim_b200.simulator"] + args + ["-o", one], check=True, env=env, cwd=ROOT)
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                    "--master-port", "29751", "-m", "nanosim_b200.simulator"] + args + ["-o", two], check=True, env=env, cwd=ROOT)
    for f in ("_aligned_reads.bam", "_unaligned_reads.bam"):
        assert check_bgzf_file(two + f) == check_bgzf_file(one + f), f
