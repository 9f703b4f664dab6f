"""--mapped_bam: the true alignment of every aligned read as mapped BAM records, built on the GPU (ns_compress_bam_mapped).

The Python encoder below restates the rules of DESIGN §3 "Mapped BAM" from a fetched batch (reads, pieces, emitted ops,
bases, qualities, names); the decompressed ``<out>_aligned_reads.bam`` must be the header followed by its records.  Other
tests check the alignments without the encoder: every record's SEQ against the plain FASTQ, the CIGAR against the
reference, and that the rest of the output is what ``--bam`` writes.  GPU tests run with ``pytest -m gpu``; the header,
CLI, rank-merge and encoder tests at the end need no GPU."""
import gzip
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

import parity_checks as pc
import synth
from test_bam_output import _CODE, SAM_CODES, bam_record, parse_records
from test_bgzf_output import _EmptyPipeline, _empty_profile, bgzf_members, check_bgzf_file

M, I, D, N, S, H = 0, 1, 2, 3, 4, 5
_CUT = -1
# complement of every 4-bit code, from the specification's letters
_COMP_LETTER = dict(zip("=ACMGRSVTWYHKDBN", "=TGKCYSBAWRDMHVN"))
COMP_TABLE = np.array([SAM_CODES.index(_COMP_LETTER[c]) for c in SAM_CODES], dtype=np.uint8)


# ------------------------------------------------------------------------------------------------------ Python encoder
def script_ops(ops, cut, period=None):
    """A segment's emitted script as CIGAR kinds (M I D, HT as I), LIT groups resolved, zero lengths dropped, and a _CUT
    before the reference base at offset ``cut`` and every ``period`` bases behind it (None: the segment does not cross its
    record's origin)."""
    out, rf, lit = [], 0, 0

    def put(kind, n):
        nonlocal rf, cut
        if n == 0:
            return
        while kind != I and cut is not None and rf <= cut < rf + n:
            a = cut - rf
            if a:
                out.append((kind, a))
            out.append((_CUT, 0))
            rf, n, cut = rf + a, n - a, cut + period
        out.append((kind, n))
        if kind != I:
            rf += n

    for op in ops:
        ty = int(op) >> 28
        n = int(op) & (0x00ffffff if ty == 5 else 0x0fffffff)
        if ty == 5:
            lit += n
            continue
        if lit and ty == 3:
            put(I if lit > n else D, abs(lit - n))
            put(M, min(lit, n))
            lit = 0
            continue
        put(I, lit)
        lit = 0
        put(D if ty == 3 else M if ty in (0, 1) else I, n)
    put(I, lit)
    return out


def read_alignments(b, i, lengths):
    """Read i's alignments in read order: (chrom, pos, span, q0, q1, merged body ops)."""
    r = b.reads[i]
    alns = []
    for k in range(int(r["n_pieces"])):
        p = b.pieces[int(r["piece_first"]) + k]
        if int(p["kind"]) & 0xffff != 0:
            continue
        clen, pos, ref_len = int(lengths[int(p["chrom"])]), int(p["pos"]), int(p["ref_len"])
        ops = script_ops(b.ops[int(p["op_off"]):int(p["op_off"]) + int(p["n_ops"])],
                         max(clen - pos, 0) if pos + ref_len > clen else None, clen)
        parts, cur = [], []
        for o in ops:
            if o[0] == _CUT:
                parts.append(cur)
                cur = []
            else:
                cur.append(o)
        parts.append(cur)
        q, rf = int(p["out_rel"]), 0
        for part in parts:
            ms = [j for j, o in enumerate(part) if o[0] == M]
            body, q0 = [], None
            for j, (kind, n) in enumerate(part):
                if ms and ms[0] <= j <= ms[-1]:
                    if j == ms[0]:
                        q0, rf0 = q, rf
                    if body and body[-1][0] == kind:
                        body[-1] = (kind, body[-1][1] + n)
                    else:
                        body.append((kind, n))
                    if j == ms[-1]:
                        q1, rf1 = q + n, rf + n
                q += n if kind != D else 0
                rf += n if kind != I else 0
            if ms:
                alns.append((int(p["chrom"]), (pos + rf0) % clen, rf1 - rf0, q0, q1, body))
    return alns


def reg2bin(beg, end):
    if end > 1 << 29:
        return 4680
    end -= 1
    for shift, off in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        if beg >> shift == end >> shift:
            return off + (beg >> shift)
    return 0


def mapped_records(b, i, name, lengths, fastq):
    """Read i's mapped records (or the unmapped record) as the rules lay them out."""
    r = b.reads[i]
    o, L, rev = int(r["seq_off"]), int(r["seq_len"]), bool(r["reversed"])
    seq = b.seq[o:o + L].tobytes()
    qual = b.qual[o:o + L].tobytes() if fastq else None
    alns = read_alignments(b, i, lengths)
    if not alns:
        return bam_record(name, seq, qual)
    codes = _CODE[np.frombuffer(seq, dtype=np.uint8)]
    q = np.frombuffer(qual, dtype=np.uint8) - 33 if fastq else np.full(L, 0xff, dtype=np.uint8)
    if rev:
        codes, q = COMP_TABLE[codes[::-1]], q[::-1]
    prim = max(range(len(alns)), key=lambda k: (alns[k][2], -k))
    out = b""
    for k, (chrom, pos, span, q0, q1, body) in enumerate(alns):
        clip = S if k == prim else H
        cig = ([(clip, q0)] if q0 else []) + body + ([(clip, L - q1)] if q1 < L else [])
        words = np.array([(n << 4) | kind for kind, n in cig], dtype="<u4")
        lo, hi = (0, L) if k == prim else (q0, q1)
        c = codes[lo:hi]
        if len(c) % 2:
            c = np.append(c, np.uint8(0))
        packed = ((c[0::2] << 4) | c[1::2]).astype(np.uint8).tobytes()
        if len(words) > 65535:
            field, aux = struct.pack("<II", ((hi - lo) << 4) | S, (span << 4) | N), b"CGBI" + struct.pack("<I", len(words)) + words.tobytes()
        else:
            field, aux = words.tobytes(), b""
        flag = (16 if rev else 0) | (0 if k == prim else 0x800)
        body_ = struct.pack("<iiBBHHHIiii", chrom, pos, len(name) + 1, 60, reg2bin(pos, pos + span), len(field) // 4, flag, hi - lo,
                            -1, -1, 0) + name + b"\0" + field + packed + q[lo:hi].astype(np.uint8).tobytes() + aux
        out += struct.pack("<i", len(body_)) + body_
    return out


def _names(names):
    from nanosim_b200.records import _name_blob
    blob, offs = _name_blob(names)
    blob = bytes(blob)
    return [blob[int(o):blob.index(b"\0", int(o))] for o in offs]


def read_mapped_bam(data):
    """(header text, [(name, ref_id, pos, span)], records) of a decompressed BAM: every record's fields and CIGAR."""
    assert data[:4] == b"BAM\1"
    l_text = struct.unpack_from("<i", data, 4)[0]
    text = data[8:8 + l_text]
    pos = 8 + l_text
    n_ref = struct.unpack_from("<i", data, pos)[0]
    pos += 4
    refs = []
    for _ in range(n_ref):
        ln = struct.unpack_from("<i", data, pos)[0]
        refs.append((data[pos + 4:pos + 3 + ln], struct.unpack_from("<i", data, pos + 4 + ln)[0]))
        pos += 8 + ln
    recs = []
    while pos < len(data):
        block, ref_id, p, l_name, mapq, bin_, n_cig, flag, l_seq, nref, npos, tlen = struct.unpack_from("<iiiBBHHHIiii", data, pos)
        q = pos + 36
        name = data[q:q + l_name - 1]
        q += l_name
        cig = np.frombuffer(data, dtype="<u4", count=n_cig, offset=q).copy()
        q += 4 * n_cig
        packed = np.frombuffer(data, dtype=np.uint8, count=(l_seq + 1) // 2, offset=q)
        codes = np.empty(2 * len(packed), dtype=np.uint8)
        codes[0::2], codes[1::2] = packed >> 4, packed & 15
        q += (l_seq + 1) // 2
        qual = data[q:q + l_seq]
        q += l_seq
        aux = data[q:pos + 4 + block]
        if aux:
            assert aux[:4] == b"CGBI"
            n = struct.unpack_from("<I", aux, 4)[0]
            real = np.frombuffer(aux, dtype="<u4", count=n, offset=8).copy()
            assert len(aux) == 8 + 4 * n and n > 65535
            assert cig.tolist() == [(l_seq << 4) | S, (int((real[(real & 15) == M] >> 4).sum() + (real[(real & 15) == D] >> 4).sum()) << 4) | N]
            cig = real
        recs.append(dict(name=name, ref_id=ref_id, pos=p, mapq=mapq, bin=bin_, flag=flag, l_seq=l_seq, cigar=cig,
                         codes=codes[:l_seq], qual=qual, next=(nref, npos, tlen), cg=bool(aux)))
        pos += 4 + block
    assert pos == len(data)
    return text, refs, recs


# ------------------------------------------------------------------------------------------------------------- GPU runs
_CAPTURE = {}


@pytest.fixture
def capture(monkeypatch):
    """Every batch ns_compress_bam_mapped is called on, fetched (with its ops) as it stands, and its names, by output
    prefix of the simulation() call."""
    from nanosim_b200 import simulator
    from nanosim_b200.engine import Engine
    orig, orig_sim = Engine.compress_bam_mapped, simulator.simulation
    cur = {}

    def compress(self, names):
        cur["list"].append((self.fetch(want_ops=True), _names(names)))
        return orig(self, names)

    def simulation(prof, mode, out, *a, **kw):
        cur["list"] = _CAPTURE.setdefault(out, [])
        cur["lengths"] = np.asarray(prof.ref.lengths)
        _CAPTURE[out + ":lengths"] = cur["lengths"]
        return orig_sim(prof, mode, out, *a, **kw)

    monkeypatch.setattr(Engine, "compress_bam_mapped", compress)
    monkeypatch.setattr(simulator, "simulation", simulation)
    return _CAPTURE


def _ecoli(tmp):
    ref = os.path.join(tmp, "ecoli5m.fa")
    if not os.path.exists(ref):
        synth.ecoli5m(ref)
    return ref


def _circ(tmp):
    ref = os.path.join(tmp, "circ60k.fa")
    if not os.path.exists(ref):
        synth.write_fasta(ref, [("plasmid_1 circular test record", synth.synth_chrom(np.random.default_rng(7), 60000))])
    return ref


def _model(m):
    return os.path.join(pc.DATA, pc.MODELS[m])


def _config_args(name, tmp):
    if name == "guppy_fastq":
        return ["genome", "-rg", _ecoli(tmp), "-c", _model("guppy"), "-n", "2500", "--fastq", "--seed", "41"], True
    if name == "dorado_hp6_chimeric":
        return ["genome", "-rg", _ecoli(tmp), "-c", _model("dorado"), "-n", "2000", "--fastq", "-hp", "-k", "6", "--chimeric",
                "--seed", "42"], True
    if name == "metagenome_chimeric":
        from conftest import meta_fixture
        meta_fixture()
        Mg = os.path.join(GOLDEN, "meta")
        return ["metagenome", "-gl", os.path.join(Mg, "genome_list_local.tsv"), "-a", os.path.join(Mg, "abundance.tsv"), "-dl",
                os.path.join(Mg, "dna_type.tsv"), "-c", _model("even"), "--fastq", "--chimeric", "--seed", "43"], True
    if name == "genome_circular":
        return ["genome", "-rg", _circ(tmp), "-c", _model("guppy"), "-n", "1500", "--fastq", "-dna_type", "circular",
                "--seed", "44"], True
    if name == "perfect":
        return ["genome", "-rg", _ecoli(tmp), "-c", _model("guppy"), "-n", "1500", "--fastq", "--perfect", "--seed", "45"], True
    return ["genome", "-rg", _ecoli(tmp), "-c", _model("guppy"), "-n", "2000", "--seed", "46"], False


_CONFIGS = ["guppy_fastq", "dorado_hp6_chimeric", "metagenome_chimeric", "genome_circular", "perfect", "fasta"]
_RUNS = {}


def _run_config(name, tmp, capture):
    """The configuration run plain, with --bam and with --bam --mapped_bam (same seed): prefixes, fastq, sample suffixes."""
    from nanosim_b200 import simulator
    if name not in _RUNS:
        args, fastq = _config_args(name, tmp)
        plain, bam, mapped = (os.path.join(tmp, name + s) for s in ("_plain", "_bam", "_mapped"))
        simulator.main(args + ["-o", plain, "-t", "4"])
        simulator.main(args + ["-o", bam, "-t", "4", "--bam"])
        simulator.main(args + ["-o", mapped, "-t", "4", "--bam", "--mapped_bam"])
        _RUNS[name] = (plain, bam, mapped, fastq, ["_sample0", "_sample1"] if name == "metagenome_chimeric" else [""])
    return _RUNS[name]


@pytest.fixture(scope="module")
def workdir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("mapped_bam"))


def _twin(out, fastq):
    batches = sorted(_CAPTURE[out], key=lambda bn: int(bn[0].first_id))
    lengths = _CAPTURE[out + ":lengths"]
    return b"".join(mapped_records(b, i, names[i], lengths, fastq) for b, names in batches for i in range(len(names)))


def _header_of(data):
    l_text = struct.unpack_from("<i", data, 4)[0]
    pos = 12 + l_text
    for _ in range(struct.unpack_from("<i", data, 8 + l_text)[0]):
        pos += 8 + struct.unpack_from("<i", data, pos)[0]
    return data[:pos]


@pytest.mark.gpu
@pytest.mark.parametrize("name", _CONFIGS)
def test_mapped_bam_equals_the_python_encoder(name, workdir, capture):
    from nanosim_b200 import simulator
    from nanosim_b200.reference_fasta import MetaReference, PackedReference
    plain, bam, mapped, fastq, samples = _run_config(name, workdir, capture)
    for p in samples:
        data = check_bgzf_file(mapped + p + "_aligned_reads.bam")
        head = _header_of(data)
        if name == "metagenome_chimeric":
            ref = MetaReference.from_genome_list(os.path.join(GOLDEN, "meta", "genome_list_local.tsv"),
                                                 os.path.join(GOLDEN, "meta", "dna_type.tsv"))
        else:
            ref = PackedReference.from_fasta(_config_args(name, workdir)[0][2])
        assert head == gzip.decompress(simulator.bam_header(simulator.bam_refs(ref, name == "genome_circular")))
        twin = _twin(mapped + p, fastq)
        assert data[len(head):] == twin
        _, refs, recs = read_mapped_bam(data)
        assert len(recs) > 100 and any(r["flag"] & 16 for r in recs)
        if name != "metagenome_chimeric":                       # the metagenome model's reads are all reversed
            assert any(not r["flag"] & 16 for r in recs)
        if "chimeric" in name:
            assert any(r["flag"] & 0x800 for r in recs)
        if name == "genome_circular":
            assert b"TP:circular" in head and sum(r["flag"] & 0x800 != 0 for r in recs) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", _CONFIGS)
def test_alignments_agree_with_the_reads_and_the_reference(name, workdir, capture):
    """Without the encoder, every configuration: CIGAR query length = l_seq, POS + span <= LN, SEQ/QUAL with the clips
    restored (and oriented back) are the read of the plain run, and the CIGAR walked over the reference leaves fewer than
    10 % of the M bases mismatched (none with --perfect).  test_alignments_are_the_error_profile checks the mismatches and
    indels exactly, read by read."""
    from nanosim_b200.reference_fasta import MetaReference, PackedReference
    plain, bam, mapped, fastq, samples = _run_config(name, workdir, capture)
    ext = ".fastq" if fastq else ".fasta"
    if name == "metagenome_chimeric":
        ref = MetaReference.from_genome_list(os.path.join(GOLDEN, "meta", "genome_list_local.tsv"),
                                             os.path.join(GOLDEN, "meta", "dna_type.tsv"))
    else:
        ref = PackedReference.from_fasta(_config_args(name, workdir)[0][2])
    for p in samples:
        _, refs, recs = read_mapped_bam(check_bgzf_file(mapped + p + "_aligned_reads.bam"))
        reads = {n: (s, q) for n, s, q in parse_records(open(plain + p + "_aligned_reads" + ext, "rb").read(), fastq)}
        n_mis = n_m = 0
        for r in recs:
            s, q = reads[r["name"]]
            if r["flag"] & 4:
                continue
            cig = r["cigar"]
            kinds, lens = cig & 15, (cig >> 4).astype(np.int64)
            assert lens[np.isin(kinds, [M, I, S])].sum() == r["l_seq"]
            span = int(lens[np.isin(kinds, [M, D])].sum())
            assert r["pos"] + span <= refs[r["ref_id"]][1]
            assert r["mapq"] == 60 and r["next"] == (-1, -1, 0) and r["bin"] == reg2bin(r["pos"], r["pos"] + span)
            lo = int(lens[0]) if kinds[0] == H else 0
            want = _CODE[np.frombuffer(s, dtype=np.uint8)]
            qual = np.frombuffer(q, dtype=np.uint8) - 33 if fastq else None
            if r["flag"] & 16:
                want = COMP_TABLE[want[::-1]]
                qual = qual[::-1] if fastq else None
            assert (r["codes"] == want[lo:lo + r["l_seq"]]).all()
            if fastq:
                assert r["qual"] == qual[lo:lo + r["l_seq"]].astype(np.uint8).tobytes()
            else:
                assert r["qual"] == b"\xff" * r["l_seq"]
            # the CIGAR over the reference: M positions compared base by base
            a, b = int(ref.offsets[r["ref_id"]]), int(ref.offsets[r["ref_id"] + 1])
            chrom = _CODE[ref.bases[a:b]]
            rp, qp = r["pos"], (lens[0] if kinds[0] == S else 0)
            for kind, n in zip(kinds, lens):
                if kind == M:
                    n_mis += int((chrom[rp:rp + n] != r["codes"][qp:qp + n]).sum())
                    n_m += int(n)
                if kind in (M, D):
                    rp += n
                if kind in (M, I):
                    qp += n
        if name == "perfect":
            assert n_mis == 0
        else:
            assert 0 < n_mis < 0.1 * n_m


def _profile_rows(path):
    """The rows of a plain error profile by read name: (type, Seq_pos, length)."""
    rows = {}
    with open(path, "rb") as f:
        next(f)
        for line in f:
            n, p, ty, ln = line.split(b"\t", 4)[:4]
            rows.setdefault(n, []).append((ty, int(p), int(ln)))
    return rows


def _overlap(a0, a1, b0, b1):
    return max(0, min(a1, b1) - max(a0, b0))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["guppy_fastq", "genome_circular", "fasta"])
def test_alignments_are_the_error_profile(name, workdir, capture):
    """Read by read, without the encoder, on plain-ACGT references without -hp (one segment per read, so every row of the
    error profile belongs to it; on the circular record segments that wrap give two records): each record's CIGAR walked
    over the reference mismatches the stored bases exactly at the `mis` rows' positions; its D total is the `del` rows'
    bases inside the records' reference intervals (a D outside them was trimmed); its I total is the `ins` rows strictly
    inside an interval (the others are at an alignment's edge, so in the clip); and the M and I bases plus those clipped
    insertions are the read less its head and tail (from the read name)."""
    from nanosim_b200.reference_fasta import PackedReference
    plain, bam, mapped, fastq, samples = _run_config(name, workdir, capture)
    ref = PackedReference.from_fasta(_config_args(name, workdir)[0][2])
    _, refs, recs = read_mapped_bam(check_bgzf_file(mapped + "_aligned_reads.bam"))
    rows = _profile_rows(mapped + "_aligned_error_profile")
    assert rows == _profile_rows(plain + "_aligned_error_profile")
    by_read = {}
    for r in recs:
        by_read.setdefault(r["name"], []).append(r)
    assert set(rows) <= set(by_read) and len(by_read) > 500
    n_split = n_mis = n_del = n_ins = n_clipped = 0
    for qname, rr in by_read.items():
        chrom, pos, _, _, _, head, _, tail = qname.rsplit(b"_", 7)
        pos, head, tail = int(pos), int(head), int(tail)
        ev = rows.get(qname, [])
        prim = [r for r in rr if not r["flag"] & 0x800]
        assert len(prim) == 1
        L = prim[0]["l_seq"]
        if prim[0]["flag"] & 4:                                 # no M in the read: nothing to check but that
            assert not [e for e in ev if e[0] == b"mis"]
            continue
        cid = rr[0]["ref_id"]
        assert ref.names[cid] == chrom.decode() and all(r["ref_id"] == cid for r in rr)
        a, clen = int(ref.offsets[cid]), refs[cid][1]
        bases = _CODE[ref.bases[a:a + clen]]
        mis, d_tot, i_tot, q_tot, spans = [], 0, 0, 0, []
        for r in rr:
            kinds, lens = r["cigar"] & 15, (r["cigar"] >> 4).astype(np.int64)
            rp, qp = r["pos"], int(lens[0]) if kinds[0] == S else 0
            for kind, n in zip(kinds, lens):
                if kind == M:
                    bad = np.nonzero(bases[rp:rp + n] != r["codes"][qp:qp + n])[0]
                    mis += (rp + bad).tolist()
                d_tot += int(n) if kind == D else 0
                i_tot += int(n) if kind == I else 0
                q_tot += int(n) if kind in (M, I) else 0
                rp += int(n) if kind in (M, D) else 0
                qp += int(n) if kind in (M, I) else 0
            rs = (r["pos"] - pos) % clen                        # the record's reference interval in segment offsets
            while spans and rs < spans[-1][1]:
                rs += clen
            spans.append((rs, rs + rp - r["pos"]))
        want_mis = sorted((pos + s + t) % clen for ty, s, n in ev if ty == b"mis" for t in range(n))
        assert sorted(mis) == want_mis, qname
        want_d = sum(_overlap(s, s + n, r0, r1) for ty, s, n in ev if ty == b"del" for r0, r1 in spans)
        inside = sum(n for ty, s, n in ev if ty == b"ins" and any(r0 < s < r1 for r0, r1 in spans))
        clipped = sum(n for ty, s, n in ev if ty == b"ins") - inside
        assert (d_tot, i_tot) == (want_d, inside), qname
        assert q_tot + clipped == L - head - tail, qname
        n_split += len(rr) > 1
        n_mis, n_del, n_ins, n_clipped = n_mis + len(want_mis), n_del + want_d, n_ins + inside, n_clipped + clipped
    assert n_mis > 1000 and n_del > 1000 and n_ins > 1000
    if name == "genome_circular":
        assert n_split > 10


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["guppy_fastq", "metagenome_chimeric"])
def test_the_rest_of_the_output_is_what_bam_writes(name, workdir, capture):
    """The unaligned .bam is byte for byte the --bam one; every aligned read's primary SEQ and QUAL, oriented back, are its
    --bam record's; the members stay near-optimal (check_bgzf_file)."""
    from test_bam_output import read_bam
    plain, bam, mapped, fastq, samples = _run_config(name, workdir, capture)
    for p in samples:
        assert open(mapped + p + "_unaligned_reads.bam", "rb").read() == open(bam + p + "_unaligned_reads.bam", "rb").read()
        _, unmapped = read_bam(check_bgzf_file(bam + p + "_aligned_reads.bam"))
        _, _, recs = read_mapped_bam(check_bgzf_file(mapped + p + "_aligned_reads.bam"))
        prim = [r for r in recs if not r["flag"] & 0x800]
        assert [r["name"] for r in prim] == [u["name"] for u in unmapped]
        for r, u in zip(prim, unmapped):
            codes, qual = r["codes"], r["qual"]
            if r["flag"] & 16:
                codes, qual = COMP_TABLE[codes[::-1]], qual[::-1]
            assert (codes == u["codes"]).all() and qual == u["qual"]
        assert open(mapped + p + "_aligned_error_profile", "rb").read() == open(plain + p + "_aligned_error_profile", "rb").read()


@pytest.mark.gpu
def test_independent_of_batching(tmp_path):
    from nanosim_b200 import simulator
    ref = _ecoli(str(tmp_path))
    outs = []
    for batch in (["--batch_reads", "700"], []):
        out = os.path.join(str(tmp_path), "b%d" % len(batch))
        simulator.main(["genome", "-rg", ref, "-c", _model("guppy"), "-n", "3000", "--fastq", "--chimeric", "--seed", "47", "-t", "3",
                        "--bam", "--mapped_bam", "-o", out] + batch)
        outs.append(out)
    a, b = (check_bgzf_file(o + "_aligned_reads.bam") for o in outs)
    assert a == b and len(read_mapped_bam(a)[2]) > 100


@pytest.mark.gpu
def test_cigar_of_more_than_65535_ops_goes_into_cg(tmp_path, capture):
    """Reads of a few hundred kb carry more than 65 535 CIGAR ops: CIGAR kSmN and the real one in CG:B,I."""
    from nanosim_b200 import simulator
    ref = os.path.join(str(tmp_path), "long.fa")
    synth.write_fasta(ref, [("big", synth.synth_chrom(np.random.default_rng(9), 4_000_000))])
    out = os.path.join(str(tmp_path), "cg")
    simulator.main(["genome", "-rg", ref, "-c", _model("guppy"), "-n", "12", "--fastq", "-med", "1000000", "-sd", "0.05",
                    "--seed", "48", "--bam", "--mapped_bam", "--no_error_profile", "-o", out])
    data = check_bgzf_file(out + "_aligned_reads.bam")
    head = _header_of(data)
    assert data[len(head):] == _twin(out, True)
    recs = read_mapped_bam(data)[2]
    assert any(r["cg"] for r in recs)


from test_vcf_haplotypes import genome  # noqa: E402,F401  (the module-scoped fixture: reference, VCF, haplotype FASTA)


@pytest.mark.gpu
def test_vcf_run_equals_a_run_on_the_haplotype_fasta(genome):  # noqa: F811
    """-rg R --vcf V --mapped_bam writes what -rg H --mapped_bam writes: the records are named after the haplotypes."""
    from nanosim_b200 import simulator
    d, ref, vcf, hap_fa = genome[:4]
    args = ["-c", _model("dorado"), "-n", "2000", "--fastq", "-hp", "-k", "6", "--chimeric", "--seed", "51", "-t", "4", "--bam",
            "--mapped_bam", "--gzip_error_profile"]
    a, b = os.path.join(d, "mapped_vcf"), os.path.join(d, "mapped_hap")
    simulator.main(["genome", "-rg", ref, "--vcf", vcf, "-o", a] + args)
    simulator.main(["genome", "-rg", hap_fa, "-o", b] + args)
    for f in ("_aligned_reads.bam", "_unaligned_reads.bam", "_aligned_error_profile.gz"):
        assert open(a + f, "rb").read() == open(b + f, "rb").read(), f
    text, refs, recs = read_mapped_bam(check_bgzf_file(a + "_aligned_reads.bam"))
    assert [n for n, _ in refs] == [b"chrA-hap1", b"chrA-hap2", b"chrB-hap1", b"chrB-hap2", b"chrC-hap1"]
    assert len(recs) > 100 and len({r["ref_id"] for r in recs}) >= 3


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_ranks_equal_one_rank(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs (this box has %d)" % torch.cuda.device_count())
    ref = _ecoli(str(tmp_path))
    args = ["genome", "-rg", ref, "-c", _model("guppy"), "-n", "4000", "--fastq", "--chimeric", "--seed", "49", "--batch_reads",
            "700", "-t", "4", "--bam", "--mapped_bam"]
    one, two = os.path.join(str(tmp_path), "one"), os.path.join(str(tmp_path), "two")
    env = dict(os.environ, PYTHONPATH=ROOT)
    subprocess.run([sys.executable, "-m", "nanosim_b200.simulator"] + args + ["-o", one], check=True, env=env, cwd=ROOT)
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                    "--master-port", "29747", "-m", "nanosim_b200.simulator"] + args + ["-o", two], check=True, env=env, cwd=ROOT)
    for f in ("_aligned_reads.bam", "_unaligned_reads.bam"):
        assert check_bgzf_file(two + f) == check_bgzf_file(one + f), f


@pytest.mark.gpu
def test_engine_rejects_unaligned_batches():
    from nanosim_b200 import _lib as L
    from nanosim_b200.engine import NanoSimError
    from nanosim_b200.reference_fasta import PackedReference
    ref = PackedReference.from_records(synth.ecoli5m())
    eng, _, _ = pc.make_engine("guppy", ref, fastq=True, seed=50)
    eng.simulate(L.NS_KIND_UNALIGNED, 0, 10)
    with pytest.raises(NanoSimError, match="unaligned.*rc=-1"):
        eng.compress_bam_mapped(["r%d" % i for i in range(10)])
    eng.close()


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_header_with_references_parses_back():
    from nanosim_b200.simulator import VERSION, bam_header
    refs = [("chr%d" % i, 1000 + i, i == 3) for i in range(5000)]
    m = bam_header(refs)
    assert len(bgzf_members(m)) > 1
    data = gzip.decompress(m)
    text, got, recs = read_mapped_bam(data)
    lines = text.decode().splitlines()
    assert lines[0] == "@HD\tVN:1.6\tSO:unknown" and lines[-1] == "@PG\tID:NanoSim\tPN:NanoSim\tVN:%s" % VERSION
    assert lines[1:-1] == ["@SQ\tSN:%s\tLN:%d%s" % (n, ln, "\tTP:circular" if c else "") for n, ln, c in refs]
    assert got == [(n.encode(), ln) for n, ln, _ in refs] and recs == []
    assert bam_header([]) == bam_header()


def test_bam_refs_names_and_duplicates():
    import types
    from nanosim_b200.simulator import bam_refs
    ref = types.SimpleNamespace(raw_names=["a", "b"], names=["a", "b"], lengths=np.array([5, 7]))
    assert bam_refs(ref, True) == [("a", 5, True), ("b", 7, True)]
    meta = types.SimpleNamespace(raw_names=["x", "x"], names=["s1-x", "s2-x"], lengths=np.array([5, 7]), chrom_circular=np.array([1, 0]))
    with pytest.raises(ValueError, match=r"records 0 \(s1-x\) and 1 \(s2-x\) have the same name x"):
        bam_refs(meta)
    big = types.SimpleNamespace(raw_names=["a", "b"], names=["a", "b"], lengths=np.array([5, 1 << 31]))
    with pytest.raises(ValueError, match=r"record 1 \(b\) has 2147483648 bases, more than the 2147483647"):
        bam_refs(big)
    assert bam_refs(types.SimpleNamespace(raw_names=["a"], names=["a"], lengths=np.array([(1 << 31) - 1])))[0][1] == (1 << 31) - 1


def test_metagenome_records_keep_their_fasta_names(tmp_path):
    from nanosim_b200.reference_fasta import MetaReference
    d = str(tmp_path)
    synth.write_fasta(os.path.join(d, "a.fa"), [("NC_1.1 first one", synth.synth_chrom(np.random.default_rng(1), 100))])
    synth.write_fasta(os.path.join(d, "b.fa"), [("NC_2 second", synth.synth_chrom(np.random.default_rng(2), 100))])
    with open(os.path.join(d, "gl.tsv"), "w") as f:
        f.write("sp A\t%s\nspB\t%s\n" % (os.path.join(d, "a.fa"), os.path.join(d, "b.fa")))
    m = MetaReference.from_genome_list(os.path.join(d, "gl.tsv"))
    assert m.raw_names == ["NC_1.1", "NC_2"] and m.names == ["sp_A-NC-1", "spB-NC-2"]


_ARGV = {"genome": ["genome", "-rg", "x.fa"], "metagenome": ["metagenome", "-gl", "gl.tsv", "-a", "ab.tsv"],
         "transcriptome": ["transcriptome", "-rt", "t.fa", "-e", "e.tsv", "--no_model_ir"]}


@pytest.mark.parametrize("mode, extra, message", [
    ("genome", ["--mapped_bam"], "--mapped_bam needs --bam"),
    ("metagenome", ["--mapped_bam", "--gzip"], "--mapped_bam needs --bam"),
    ("transcriptome", ["--bam", "--mapped_bam"], "--mapped_bam is not available in transcriptome mode"),
])
def test_usage_errors(mode, extra, message, tmp_path, capsys):
    from nanosim_b200 import simulator
    with pytest.raises(SystemExit) as e:
        simulator.main(_ARGV[mode] + ["-o", os.path.join(str(tmp_path), "sim")] + extra)
    assert e.value.code == 1
    assert message in capsys.readouterr().err
    assert os.listdir(str(tmp_path)) == []


def test_duplicate_reference_names_are_a_usage_error(tmp_path, monkeypatch, capsys):
    import types
    from nanosim_b200 import simulator

    def profile(*a, **kw):
        prof = _empty_profile()
        prof.ref = types.SimpleNamespace(names=["c", "c2"], raw_names=["c", "c"], lengths=np.array([1000, 900]), max_chrom=1000)
        return prof
    monkeypatch.setattr(simulator, "read_profile", profile)
    monkeypatch.setattr(simulator, "BatchPipeline", _EmptyPipeline)
    with pytest.raises(SystemExit) as e:
        simulator.main(_ARGV["genome"] + ["-o", os.path.join(str(tmp_path), "sim"), "--bam", "--mapped_bam"])
    assert e.value.code == 1 and "have the same name c" in capsys.readouterr().err


def test_flag_writes_the_reference_header(tmp_path, monkeypatch):
    import types
    from nanosim_b200 import simulator
    from nanosim_b200.simulator import BGZF_EOF

    def profile(*a, **kw):
        prof = _empty_profile()
        prof.ref = types.SimpleNamespace(names=["c"], raw_names=["chrA"], lengths=np.array([1000]), max_chrom=1000)
        return prof
    monkeypatch.setattr(simulator, "read_profile", profile)
    monkeypatch.setattr(simulator, "BatchPipeline", _EmptyPipeline)
    out = os.path.join(str(tmp_path), "sim")
    simulator.main(_ARGV["genome"] + ["-o", out, "--bam", "--mapped_bam", "-dna_type", "circular"])
    assert open(out + "_aligned_reads.bam", "rb").read() == simulator.bam_header([("chrA", 1000, True)]) + BGZF_EOF
    assert open(out + "_unaligned_reads.bam", "rb").read() == simulator.bam_header() + BGZF_EOF


def test_merge_rank_files_writes_the_header_once(tmp_path):
    from nanosim_b200.simulator import BGZF_EOF, bam_header, merge_rank_files
    from test_bgzf_output import _zlib_member
    out = os.path.join(str(tmp_path), "sim")
    refs = [("chr1", 100, False)]
    parts = {}
    for kind in ("aligned", "unaligned"):
        for r in range(2):
            parts[kind, r] = _zlib_member(bam_record(b"%s_%d" % (kind.encode(), r), b"ACGTA", None))
            with open(out + "_%s_reads%d.bam" % (kind, r), "wb") as f:
                f.write(parts[kind, r])
    for r in range(2):
        open(out + "_error_profile%d" % r, "w").close()
    merge_rank_files(out, False, False, 2, bam=True, mapped_refs=refs)
    assert open(out + "_aligned_reads.bam", "rb").read() == bam_header(refs) + parts["aligned", 0] + parts["aligned", 1] + BGZF_EOF
    assert open(out + "_unaligned_reads.bam", "rb").read() == bam_header() + parts["unaligned", 0] + parts["unaligned", 1] + BGZF_EOF


def test_nibble_complement_is_the_bit_reversal():
    assert [int("{:04b}".format(c)[::-1], 2) for c in range(16)] == COMP_TABLE.tolist()


def test_encoder_rules():
    """LIT groups, merging, trimming and the cut, on hand-made scripts."""
    def op(t, n, base=0):
        return (t << 28) | (base << 26) | n if t == 5 else (t << 28) | n
    # LIT 3 + DEL 5 -> 2 D then 3 M; LIT 4 + DEL 2 -> 2 I then 2 M; a lone LIT -> I; zero-length ops vanish
    assert script_ops([op(0, 4), op(5, 1), op(5, 2), op(3, 5), op(0, 0), op(5, 4), op(3, 2), op(5, 1)], None) == \
        [(M, 4), (D, 2), (M, 3), (I, 2), (M, 2), (I, 1)]
    # an M across the cut is split, an insertion at the cut stays before it, a D across it is split too
    assert script_ops([op(0, 5), op(2, 2), op(0, 3)], 5, 100) == [(M, 5), (I, 2), (_CUT, 0), (M, 3)]
    assert script_ops([op(0, 4), op(3, 3), op(0, 2)], 5, 100) == [(M, 4), (D, 1), (_CUT, 0), (D, 2), (M, 2)]
    # a segment longer than its record passes the origin more than once: a cut every record length
    assert script_ops([op(0, 12), op(2, 1), op(0, 9)], 2, 8) == [(M, 2), (_CUT, 0), (M, 8), (_CUT, 0), (M, 2), (I, 1), (M, 6),
                                                                (_CUT, 0), (M, 3)]
    assert reg2bin(0, 1) == 4681 and reg2bin(0, 1 << 14) == 4681 and reg2bin(0, (1 << 14) + 1) == 585 and reg2bin(0, 1 << 30) == 4680


def test_exports_name_the_new_entry_point():
    from nanosim_b200 import _lib
    header = open(os.path.join(ROOT, "include", "nanosim_b200.h")).read()
    assert "ns_compress_bam_mapped" in _lib.EXPORTS and "ns_compress_bam_mapped(" in header
