"""-hp/-k on transcriptome reads that retain introns (simulator.py:1156-1183, then mutate_read with the -k filter and
mutate_homo on the GENOMIC read).

The parity target is the oracle's simulation_aligned_transcriptome(..., kmer_bias=K, model_ir=True).  Its intron-retention
loop is pinned against the unmodified reference without -hp (test_oracle_ir_golden.py), and mutate_read / mutate_homo are
pinned on their own (test_oracle_golden.py): the combination is the oracle composing pinned parts.

The fixture is generated here from a seed: a genome rich in homopolymer runs, some planted across exon / intron boundaries,
with a lower-case stretch and N / IUPAC bytes inside introns; plus- and minus-strand transcripts spliced from it; an IR
model that retains often.  The model is the shipped dRNA model with the dorado model's homopolymer table added."""
import os
import random

import numpy as np
import pytest

import parity_checks as pc
import run_stats as rs

COMP = str.maketrans("ACGTacgt", "TGCAtgca")


def _write_fixture(d, seed=5):
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    genome = {}
    for chrom, n in (("chr1", 40000), ("chr2", 30000)):
        s = acgt[rng.integers(0, 4, n)].copy()
        for _ in range(n // 60):
            p = int(rng.integers(0, n - 20))
            s[p:p + int(rng.integers(4, 15))] = acgt[int(rng.integers(0, 4))]
        genome[chrom] = s
    gff, trx = ["##gff-version 3"], []
    cursor = {"chr1": 400, "chr2": 300}
    for i in range(14):
        chrom = "chr1" if i % 3 else "chr2"
        strand = "+" if i % 2 == 0 else "-"
        s = genome[chrom]
        start = cursor[chrom] + int(rng.integers(50, 300))
        feats, pos, exons = [], start, []
        n_exon = int(rng.integers(3, 7))
        for e in range(n_exon):
            el = int(rng.integers(90, 600))
            feats.append(("exon", pos, pos + el - 1))
            exons.append((pos - 1, pos - 1 + el))
            pos += el
            if e + 1 < n_exon:
                il = int(rng.integers(80, 400))
                feats.append(("intron", pos, pos + il - 1))
                a, b = pos - 1, pos - 1 + il                   # 0-based intron
                lo = a + int(rng.integers(10, il // 2))
                if rng.random() < 0.5:
                    s[lo:lo + 25] |= 0x20                       # lower case
                for _ in range(3):
                    s[a + int(rng.integers(0, il))] = ord("NRYN"[int(rng.integers(0, 4))])
                pos += il
        # runs planted across the exon / intron boundaries (after the IUPAC bytes: exons stay plain)
        for (ty, a, b) in feats[:-1]:
            if rng.random() < 0.7:
                L = int(rng.integers(4, 15))
                c = b - int(rng.integers(1, L))                 # 0-based start: the run covers base b-1 / b
                s[c:c + L] = acgt[int(rng.integers(0, 4))]
        cursor[chrom] = pos
        tid = "ENST%011d.1" % (3000 + i)
        gff.append("%s\tTEST\ttranscript\t%d\t%d\t.\t%s\t.\tID=transcript%d;transcript_id=%s" % (chrom, start, pos - 1, strand, i, tid))
        for ty, a, b in feats:
            gff.append("%s\tTEST\t%s\t%d\t%d\t.\t%s\t.\tParent=transcript%d;transcript_id=%s" % (chrom, ty, a, b, strand, i, tid))
        trx.append((tid, chrom, strand, exons))
    for k in genome:
        assert cursor[k] < len(genome[k]) - 100
    with open(os.path.join(d, "genome.fa"), "w") as f:
        for k, s in genome.items():
            f.write(">%s\n%s\n" % (k, s.tobytes().decode()))
    with open(os.path.join(d, "annotation.gff3"), "w") as f:
        f.write("\n".join(gff) + "\n")
    with open(os.path.join(d, "transcripts.fa"), "w") as f, open(os.path.join(d, "expression.tsv"), "w") as e, \
            open(os.path.join(d, "polya.txt"), "w") as pa:
        e.write("target_id\test_counts\ttpm\n")
        for i, (tid, chrom, strand, exons) in enumerate(trx):
            sp = "".join(genome[chrom][a:b].tobytes().decode() for a, b in exons)
            if strand == "-":
                sp = sp.translate(COMP)[::-1]
            f.write(">%s\n%s\n" % (tid, sp))
            e.write("%s\t10.0\t%.3f\n" % (tid, 5.0 + i))
            if i % 2 == 0:
                pa.write(tid + "\n")
    with open(os.path.join(d, "IR_markov_model"), "w") as f:
        f.write("succedent\tno_IR\tIR\nstart\t0.4\t0.6\nno_IR\t0.5\t0.5\nIR\t0.4\t0.6\n")


def _hp_model(d):
    """The shipped dRNA model plus the dorado model's homopolymer table, as one .npz."""
    from nanosim_b200.model import CompiledModel
    cm = CompiledModel.load(os.path.join(pc.DATA, pc.MODELS["drna"]))
    cm.text["hp_lengths_model_parameters.tsv"] = CompiledModel.load(os.path.join(pc.DATA, pc.MODELS["dorado"])).text["hp_lengths_model_parameters.tsv"]
    path = os.path.join(d, "drna_hp.npz")
    cm.save(path)
    return path, cm


@pytest.fixture(scope="module")
def fx(tmp_path_factory):
    from nanosim_b200 import intron_retention as ir
    from nanosim_b200.reference_fasta import PackedReference, read_expression, read_polya_list
    d = str(tmp_path_factory.mktemp("ir_hp"))
    _write_fixture(d)
    model, cm = _hp_model(d)
    trx = PackedReference.from_fasta(os.path.join(d, "transcripts.fa"))
    genome = PackedReference.from_fasta(os.path.join(d, "genome.fa"))
    ref = PackedReference.concat(trx, genome)
    chrom, w = read_expression(os.path.join(d, "expression.tsv"), trx)
    polya = np.concatenate([read_polya_list(os.path.join(d, "polya.txt"), trx), np.zeros(len(genome.names), dtype=np.uint8)])
    st = ir.TranscriptStructures.from_gff3(os.path.join(d, "annotation.gff3"), trx.names, genome.raw_names)
    irm = ir.IntronRetention(ir.read_ir_markov_model(os.path.join(d, "IR_markov_model")), st, trx.lengths, len(trx.names))
    return dict(d=d, model=model, cm=cm, trx=trx, genome=genome, ref=ref, chrom=chrom, w=w, polya=polya, irm=irm)


def _engine(fx, K, seed, polya=True, kde2d_sample=400):
    from nanosim_b200.engine import Engine
    from nanosim_b200.model import DeviceTables, build_alias
    from nanosim_b200.reference_fasta import POLYA_SCALE
    t = DeviceTables(fx["cm"], fastq=True, homopolymer=bool(K))
    eng = Engine(device=0, seed=seed)
    eng.set_reference(fx["ref"])
    eng.set_model(t)
    pr, al = build_alias(fx["w"])
    eng.set_expression(pr, al, fx["chrom"], fx["polya"] if polya else None)
    eng.configure(fastq=True, min_len=50, max_len=fx["trx"].max_chrom, transcriptome=True, kmer_bias=K,
                  polya_scale=POLYA_SCALE["guppy"] if polya else 0.0, kde2d_sample=kde2d_sample, trx_records=len(fx["trx"].names))
    return eng


def _simulate_and_retain(eng, irm, first, n, seed):
    info = eng.simulate(0, first, n)
    b0 = eng.fetch(want_ops=True)
    patch = irm.plan_batch(b0.reads, b0.pieces, b0.ops, first, seed, info.n_pieces, info.n_ops, info.raw_ev_off)
    eng.reemit(*patch)
    return info, b0, patch, eng.fetch(want_ops=True)


def _in_hp_mask(seq, k):
    """Bases of seq inside a run of >= k equal A/C/G/T (any other byte breaks runs and is never inside one)."""
    if len(seq) == 0:
        return np.zeros(0, dtype=bool)
    bounds = np.concatenate([[0], np.flatnonzero(seq[1:] != seq[:-1]) + 1, [len(seq)]])
    runs = np.diff(bounds)
    ok = np.isin(seq[bounds[:-1]], np.frombuffer(b"ACGT", dtype=np.uint8))
    return np.repeat((runs >= k) & ok, runs)


def _events(b, pcs, events=True):
    """[(type, chain offset, length)] of the error events of a chain's pieces."""
    out, base = [], 0
    for q in pcs:
        ty, ln, _, _, _, ref_start = pc._piece_layout(b, q, events=events)
        for j in np.flatnonzero((ty >= 1) & (ty <= 3) & (ln > 0)):
            out.append((int(ty[j]), base + int(ref_start[j]), int(ln[j])))
        base += int(q["ref_len"])
    return out


# reference bytes read on the minus strand: A C G T and the IUPAC codes complemented (R <-> Y, K <-> M, B <-> V, D <-> H)
_COMP_CODE = np.arange(256, dtype=np.uint8)
for _a, _b in (("A", "T"), ("C", "G"), ("R", "Y"), ("K", "M"), ("B", "V"), ("D", "H")):
    _COMP_CODE[ord(_a)], _COMP_CODE[ord(_b)] = ord(_b), ord(_a)


def _check_genome_reads(b, ref, slots):
    """The re-application of parity_checks.check_edit_scripts for reads laid out on the genome, whose minus-strand pieces
    may hold IUPAC codes (the generated fixture puts some in introns): there a copied base must be a member of the
    COMPLEMENTED code.  Rewritten scripts hold COPY / DEL / LIT / HT only.  Returns the number of bases verified."""
    off = ref.offsets.astype(np.int64)
    verified = 0
    for i in slots.tolist():
        r = b.reads[i]
        n, so = int(r["seq_len"]), int(r["seq_off"])
        assert so % 16 == 0
        raw = b.seq[so:so + n]
        fwd = pc._COMP[raw[::-1]] if r["reversed"] else raw
        assert pc._IS_ACGT[fwd].all(), "non-ACGT base in read %d" % i
        q = b.qual[so:so + n]
        assert q.min() >= 33 + 1 and q.max() <= 33 + 93, "quality out of [1,93] in read %d" % i
        p0, npc = int(r["piece_first"]), int(r["n_pieces"])
        cursor = 0
        for k in range(npc):
            pcs = b.pieces[p0 + k]
            assert int(pcs["read_slot"]) == i and int(pcs["out_rel"]) == cursor
            ty, ln, out_adv, ref_adv, out_start, ref_start = pc._piece_layout(b, pcs)
            assert int(out_adv.sum()) == int(pcs["out_len"]) and int(ref_adv.sum()) == int(pcs["ref_len"])
            assert (ln > 0).all() and not (ty == 1).any() and not (ty == 2).any()
            if k == 0 and int(r["head"]) > 0:
                assert ty[0] == 4 and ln[0] == int(r["head"])
            if k == npc - 1 and int(r["tail"]) > 0:
                assert ty[-1] == 4 and ln[-1] == int(r["tail"])
            seg = fwd[cursor:cursor + int(pcs["out_len"])]

            def spread(sel):
                return np.repeat(out_start[sel], ln[sel]) + (np.arange(int(ln[sel].sum())) - np.repeat(np.cumsum(ln[sel]) - ln[sel], ln[sel]))
            lit = ty == 5
            if lit.any():
                o_ops = b.ops[int(pcs["op_off"]): int(pcs["op_off"]) + int(pcs["n_ops"])]
                want = np.frombuffer(b"ACTG", dtype=np.uint8)[((o_ops[lit] >> 26) & 3).astype(np.int64)]
                assert (seg[spread(lit)] == np.repeat(want, ln[lit])).all(), "literal base mismatch (read %d piece %d)" % (i, k)
            cp = ty == 0
            if cp.any():
                ridx = np.repeat(ref_start[cp], ln[cp]) + (np.arange(int(ln[cp].sum())) - np.repeat(np.cumsum(ln[cp]) - ln[cp], ln[cp]))
                c0, rl, pos = int(off[pcs["chrom"]]), int(pcs["ref_len"]), int(pcs["pos"])
                if int(pcs["kind"]) & 0x80000000:           # NS_PIECE_REF_REV: the genome read backwards, complemented
                    rb = _COMP_CODE[pc._UPPER[ref.bases[c0 + pos + rl - 1 - ridx]]]
                else:
                    rb = pc._UPPER[ref.bases[c0 + pos + ridx]]
                assert pc._MEMBER[rb, seg[spread(cp)]].all(), "copied base differs from the genome (read %d piece %d)" % (i, k)
                verified += len(ridx)
            cursor += int(pcs["out_len"])
        assert cursor == n
    return verified


@pytest.mark.gpu
@pytest.mark.parametrize("K", [6, 3])
def test_ir_hp_reemit_bit_exact(fx, K, monkeypatch):
    """simulate -> fetch -> plan_batch -> reemit -> fetch: reads that keep their transcript layout are untouched byte for
    byte; replaced reads re-apply bit-exactly to the genome (minus strand and IUPAC bytes included), no surviving event
    touches a run >= K of the unmutated genomic read, the filter demonstrably ran on the genome, rewritten runs straddle
    piece boundaries, intervals and names are those of the same run without -hp / of the oracle's extract_read_pos, and
    the error-profile formatters agree."""
    import nanosim_oracle as no
    from nanosim_b200 import _lib as L
    from nanosim_b200 import intron_retention as ir
    from nanosim_b200.records import error_profile_rows, format_error_profile, name_table, read_names
    ref, irm, trx, d = fx["ref"], fx["irm"], fx["trx"], fx["d"]
    seed, first, n = 71 + K, 500, 4000
    eng = _engine(fx, K, seed)
    info0, b0, patch, b1 = _simulate_and_retain(eng, irm, first, n, seed)
    assert info0.raw_ev_off > 0 and b1.info.seq_bytes >= (1 << 20)      # large enough for the 2-bit transfer
    slots = patch[0]
    assert 0.2 * n < len(slots) < 0.95 * n
    touched = np.zeros(n, dtype=bool)
    touched[slots] = True
    for i in np.flatnonzero(~touched):
        a, m = int(b0.reads["seq_off"][i]), int(b0.reads["seq_len"][i])
        assert int(b1.reads["seq_off"][i]) == a and int(b1.reads["seq_len"][i]) == m
        assert np.array_equal(b0.seq[a:a + m], b1.seq[a:a + m]) and np.array_equal(b0.qual[a:a + m], b1.qual[a:a + m])
    assert (b1.reads["seq_off"][slots] >= b0.info.seq_bytes).all() and (b1.reads["seq_off"] % 16 == 0).all()
    assert int(b1.reads["seq_len"].astype(np.int64).sum()) == b1.info.total_bases
    assert int(b1.info.n_pieces) == len(b1.pieces) and b1.info.n_ops == len(b1.ops)
    assert pc.check_edit_scripts(b0, ref, True) > 0                     # transcript layout (plain A C G T)
    assert _check_genome_reads(b1, ref, slots) > 0
    assert not np.array_equal(b0.reads["seq_len"][slots], b1.reads["seq_len"][slots])

    # the same batch without -hp: the same reads retain introns, on the same intervals, under the same names
    eng0 = _engine(fx, 0, seed)
    _, _, patch0, c1 = _simulate_and_retain(eng0, irm, first, n, seed)
    eng0.close()
    assert np.array_equal(patch0[0], slots)
    keep = ["kind", "chrom", "pos", "ref_len", "read_slot"]
    assert all(np.array_equal(c1.pieces[k][len(c1.pieces) - len(patch0[2]):], b1.pieces[k][len(b1.pieces) - len(patch[2]):]) for k in keep)
    names = read_names(b1, ref.names, first, transcriptome=True)
    assert names == read_names(c1, ref.names, first, transcriptome=True)
    assert name_table(b1, ref.names, first, transcriptome=True).tolist() == names

    # the -k filter ran on the genomic read
    gbytes = ref.bases
    off = ref.offsets.astype(np.int64)
    comp = np.arange(256, dtype=np.uint8)
    for x, y in (("A", "T"), ("C", "G")):
        comp[ord(x)], comp[ord(y)] = ord(y), ord(x)
    n_ev = g_only = t_only = straddle = 0
    for i in slots.tolist():
        p0, npc = int(b1.reads["piece_first"][i]), int(b1.reads["n_pieces"][i])
        segs = b1.pieces[p0:p0 + npc:2]
        chain = []
        for q in segs:
            s = gbytes[off[q["chrom"]] + q["pos"]: off[q["chrom"]] + q["pos"] + q["ref_len"]].copy()
            s[(s >= 97) & (s <= 122)] -= 32
            chain.append(comp[s[::-1]] if int(q["kind"]) & L.NS_PIECE_REF_REV else s)
        mask = _in_hp_mask(np.concatenate(chain), K)
        got = _events(b1, segs)
        for t, rp, ln in got:
            lo, hi = rp - (1 if t == 2 else 0), rp + ln - 1
            assert not mask[max(lo, 0):min(hi, len(mask) - 1) + 1].any(), "event inside a homopolymer of the genomic read survived"
        n_ev += len(got)
        q0 = b0.pieces[int(b0.reads["piece_first"][i])]
        raw = b0.ops[int(info0.raw_ev_off) + int(q0["ev_off"]): int(info0.raw_ev_off) + int(q0["ev_off"]) + int(q0["ev_n_ops"])]
        t_kept = {(t, rp) for t, rp, _ in _events(b0, [q0])}
        g_kept = {(t, rp) for t, rp, _ in got}
        ty = (raw >> 28).astype(np.int64)
        ln = np.where(ty == 5, raw & 0xffffff, raw & 0xfffffff).astype(np.int64)
        rs0 = np.concatenate([[0], np.cumsum(np.where((ty == 2) | (ty >= 4), 0, ln))[:-1]])
        for j in np.flatnonzero((ty >= 1) & (ty <= 3) & (ln > 0)):
            e = (int(ty[j]), int(rs0[j]))
            g_only += e in g_kept and e not in t_kept
            t_only += e in t_kept and e not in g_kept
        # a rewritten run carried across a boundary: the next piece's script opens with its share of the run's reference
        # skip although that piece's event script does not open with a deletion
        for q in segs[1:]:
            o = b1.ops[int(q["op_off"]): int(q["op_off"]) + int(q["n_ops"])]
            e = b1.ops[int(q["ev_off"]): int(q["ev_off"]) + int(q["ev_n_ops"])]
            e = e[(e & 0xfffffff) > 0]
            straddle += len(o) > 0 and (o[0] >> 28) == 3 and (len(e) == 0 or (e[0] >> 28) != 3)
    print("K=%d: %d replaced reads, %d events; kept only on the genome %d, only on the transcript %d; straddling runs %d"
          % (K, len(slots), n_ev, g_only, t_only, straddle))
    assert n_ev > 1000 and g_only > 0 and t_only > 0 and straddle > 20

    # intervals: the oracle's extract_read_pos from the same uniforms (first 300 replaced reads)
    oref = no.OracleTrxReference.from_files(os.path.join(d, "transcripts.fa"), os.path.join(d, "expression.tsv"), os.path.join(d, "polya.txt"))
    oref.load_ir(os.path.join(d, "genome.fa"), os.path.join(d, "annotation.gff3"), os.path.join(d, "IR_markov_model"))
    for i in slots[:300].tolist():
        p1 = b1.pieces[int(b1.reads["piece_first"][i]):int(b1.reads["piece_first"][i]) + int(b1.reads["n_pieces"][i])][::2]
        t0 = int(b0.pieces["chrom"][int(b0.reads["piece_first"][i])])
        key, n_int = trx.names[t0], int(irm.st.n_introns[t0])
        u = ir.ir_uniforms(seed, [first + i], n_int + 1)[0]
        feed = iter(u[:n_int].tolist())
        monkeypatch.setattr(random, "random", lambda: next(feed))
        monkeypatch.setattr(random, "randint", lambda lo, hi: min(int(u[n_int] * (hi + 1)), hi) if hi > 0 else 0)
        flag, st_new = no.update_structure(oref.structure[key], oref.ir_model)
        assert flag
        ivs, _, _ = no.extract_read_pos(int(p1["ref_len"].sum()), oref.seq_len[key], st_new, False)
        assert sorted((int(x["pos"]), int(x["pos"]) + int(x["ref_len"])) for x in p1) == [(s, e) for _, s, e, _ in ivs]
    monkeypatch.undo()
    want = "".join(error_profile_rows(b1, names, ref, seed=seed)).encode()
    assert format_error_profile(b1, name_table(b1, ref.names, first, transcriptome=True), ref, seed=seed, n_threads=4) == want
    eng.close()


@pytest.mark.gpu
def test_ir_hp_statistics_vs_oracle(fx, tmp_path):
    """Device against the oracle's simulation_aligned_transcriptome(..., kmer_bias=6, model_ir=True) on the fixture (no
    polyA tails: the device keeps a retaining read's first-pass polyA decision, a documented deviation): homopolymer run
    lengths, middle qualities, read lengths, middle bases per reference base, share of reads that retain an intron."""
    import nanosim_oracle as no
    from conftest import oracle_model
    from nanosim_b200 import _lib as L
    K, N, d = 6, 700, fx["d"]
    eng = _engine(fx, K, 23, polya=False, kde2d_sample=N)
    s_dev = rs.empty()
    n_ir_dev = 0
    for j in range(2):
        _, _, patch, b1 = _simulate_and_retain(eng, fx["irm"], j * 6000, 6000, 23)
        pc.batch_stats(b1, fx["ref"], True, s_dev)
        # reads whose intervals cover a retained intron (the oracle names only those)
        n_ir_dev += len(np.unique(b1.pieces["read_slot"][(b1.pieces["kind"] & L.NS_PIECE_RETAINED) != 0]))
    eng.close()
    oref = no.OracleTrxReference.from_files(os.path.join(d, "transcripts.fa"), os.path.join(d, "expression.tsv"), None)
    oref.load_ir(os.path.join(d, "genome.fa"), os.path.join(d, "annotation.gff3"), os.path.join(d, "IR_markov_model"))
    m = oracle_model(fx["cm"], tmp_path, fastq=True, homopolymer=True)
    s_or = rs.empty()
    n_ir_or = 0
    for rep in range(3):                                    # three independent workers of N reads each
        random.seed(900 + rep)
        np.random.seed(900 + rep)
        sink = no.ReadSink()
        no.simulation_aligned_transcriptome(oref, m, sink, K, "guppy", N, False, True, model_ir=True)
        prefix = os.path.join(str(tmp_path), "o%d" % rep)
        with open(prefix + "_aligned_reads.fastq", "w") as f:
            f.write(no.format_records(sink.records, True))
        with open(prefix + "_aligned_error_profile", "w") as f:
            f.write("Seq_name\tSeq_pos\terror_type\terror_length\tref_base\tseq_base\n")
            f.writelines(r + "\n" for r in sink.error_rows)
        rs.merge(s_or, rs.stats_from_prefix(prefix, True))
        n_ir_or += sum("_RetainedIntron_" in name for name, _, _ in sink.records)
    fails = []
    for k in ("hp_runs", "qual_middle", "len_aligned"):
        st, dof, p = pc.chi2_two_sample(s_dev[k], s_or[k])
        print(k, "chi2 %.1f dof %d p %.3g" % (st, dof, p))
        if p < 1e-5:
            fails.append("%s chi2 %.1f dof %d p %.3g" % (k, st, dof, p))
    rd = (s_dev["aligned_bases"] - s_dev["head_bases"] - s_dev["tail_bases"]) / s_dev["ref_bases"]
    ro = (s_or["aligned_bases"] - s_or["head_bases"] - s_or["tail_bases"]) / s_or["ref_bases"]
    print("middle bases per reference base: device %.5f oracle %.5f" % (rd, ro))
    if abs(rd / ro - 1) >= 3e-3:
        fails.append("middle bases per reference base %.5f vs %.5f" % (rd, ro))
    f_d, f_o = n_ir_dev / s_dev["n_aligned"], n_ir_or / s_or["n_aligned"]
    print("share of reads that retain an intron: device %.4f oracle %.4f" % (f_d, f_o))
    if abs(f_d - f_o) > 5 * np.sqrt(f_o * (1 - f_o) * (1 / s_dev["n_aligned"] + 1 / s_or["n_aligned"])):
        fails.append("share of IR reads %.4f vs %.4f" % (f_d, f_o))
    assert not fails, "\n".join(fails)


def _cli_args(fx, out, extra=()):
    d = fx["d"]
    return ["transcriptome", "-rt", os.path.join(d, "transcripts.fa"), "-rg", os.path.join(d, "genome.fa"),
            "-e", os.path.join(d, "expression.tsv"), "-c", fx["model"], "-n", "1500", "-o", out, "--fastq",
            "--polya", os.path.join(d, "polya.txt"), "-b", "guppy", "--seed", "9", "-hp", "-k", "6",
            "--ir_markov_model", os.path.join(d, "IR_markov_model"), "--ir_gff3", os.path.join(d, "annotation.gff3")] + list(extra)


@pytest.mark.gpu
def test_cli_transcriptome_hp_with_intron_retention(fx, tmp_path):
    """`transcriptome ... -hp -k 6` with intron retention on: output independent of the batch split, retaining reads
    present, read counts right."""
    from nanosim_b200 import simulator
    outs = []
    for tag, batch in (("a", "100000"), ("b", "211")):
        out = os.path.join(str(tmp_path), tag)
        simulator.main(_cli_args(fx, out, ["--batch_reads", batch]))
        outs.append(out)
    for suffix in ("_aligned_reads.fastq", "_unaligned_reads.fastq", "_aligned_error_profile"):
        a, b = open(outs[0] + suffix, "rb").read(), open(outs[1] + suffix, "rb").read()
        assert a == b and len(a) > 1000, suffix
    heads = [line for line in open(outs[0] + "_aligned_reads.fastq") if line.startswith("@ENST")]
    assert sum("_RetainedIntron_" in h for h in heads) > 100
    s = rs.stats_from_prefix(outs[0], True)
    assert s["n_aligned"] + s["n_unaligned"] == 1500 and s["n_aligned"] == len(heads)


# ---------------------------------------------------------------------------------------------------- CPU
def _merged(ops):
    """The op sequence with adjacent ops of one reference-consuming type joined (undoes split_script's cuts)."""
    out = []
    for o in ops.tolist():
        t, n = o >> 28, o & 0x0fffffff
        if out and t in (0, 1, 3) and out[-1][0] == t:
            out[-1][1] += n
        else:
            out.append([t, n if t != 5 else o & 0xffffff])
    return out


def test_plan_batch_cuts_raw_scripts_when_given():
    """plan_batch on a hand-built batch whose emitted scripts differ from the unfiltered copy at raw_ev_off: with
    raw_ev_off it cuts the copy, without it the emitted script; the decisions and intervals are the same."""
    from conftest import GOLDEN
    from nanosim_b200 import _lib as L
    from nanosim_b200 import intron_retention as ir
    from nanosim_b200.reference_fasta import PackedReference
    D = os.path.join(GOLDEN, "ir")
    trx = PackedReference.from_fasta(os.path.join(D, "transcripts.fa"))
    genome = PackedReference.from_fasta(os.path.join(D, "genome.fa"))
    st = ir.TranscriptStructures.from_gff3(os.path.join(D, "annotation.gff3"), trx.names, genome.raw_names)
    irm = ir.IntronRetention(ir.read_ir_markov_model(os.path.join(D, "IR_markov_model")), st, trx.lengths, len(trx.names))
    rng = np.random.default_rng(3)
    n = 300
    reads = np.zeros(n, dtype=L.READ_DTYPE)
    pieces = np.zeros(n, dtype=L.PIECE_DTYPE)
    emitted, raw = [], []
    for i in range(n):
        t = int(rng.integers(0, len(trx.names)))
        want = int(rng.integers(20, int(trx.lengths[t]) - 5))
        script, rf = [(L.NS_OP_HT << 28) | 4], 0
        while rf < want:
            ty = int(rng.choice([L.NS_OP_COPY, L.NS_OP_MIS, L.NS_OP_INS, L.NS_OP_DEL]))
            ln = int(rng.integers(1, 20 if ty == L.NS_OP_COPY else 4))
            if ty != L.NS_OP_INS:
                ln = min(ln, want - rf)
                rf += ln
            script.append((ty << 28) | ln)
        script.append((L.NS_OP_HT << 28) | 3)
        # the emitted script as the homopolymer pass leaves it: substitutions dropped (copies), insertions gone
        em = [((L.NS_OP_COPY << 28) | (o & 0xfffffff)) if (o >> 28) == L.NS_OP_MIS else o for o in script if (o >> 28) != L.NS_OP_INS]
        reads[i]["piece_first"], reads[i]["n_pieces"], reads[i]["head"], reads[i]["tail"] = i, 1, 4, 3
        pieces[i]["chrom"], pieces[i]["ref_len"], pieces[i]["read_slot"] = t, rf, i
        pieces[i]["op_off"], pieces[i]["n_ops"] = len(emitted), len(em)
        pieces[i]["ev_off"], pieces[i]["ev_n_ops"] = len(raw), len(script)
        emitted += em
        raw += script
    raw_off = len(emitted)
    ops = np.asarray(emitted + raw, dtype=np.uint32)
    with_raw = irm.plan_batch(reads, pieces, ops, 1000, 5, n, len(ops), raw_ev_off=raw_off)
    without = irm.plan_batch(reads, pieces, ops, 1000, 5, n, len(ops))
    assert np.array_equal(with_raw[0], without[0]) and len(with_raw[0]) > 0.15 * n
    for k in ("kind", "chrom", "pos", "ref_len", "read_slot"):
        assert np.array_equal(with_raw[2][k], without[2][k])
    for patch, src in ((with_raw, "raw"), (without, "emitted")):
        slots, nr, npc, nops = patch
        for k, i in enumerate(slots.tolist()):
            r = nr[k]
            own = npc[int(r["piece_first"]) - n: int(r["piece_first"]) - n + int(r["n_pieces"])][::2]
            parts = np.concatenate([nops[int(q["op_off"]) - len(ops): int(q["op_off"]) - len(ops) + int(q["n_ops"])] for q in own])
            p = pieces[i]
            script = ops[raw_off + int(p["ev_off"]): raw_off + int(p["ev_off"]) + int(p["ev_n_ops"])] if src == "raw" else \
                ops[int(p["op_off"]): int(p["op_off"]) + int(p["n_ops"])]
            assert _merged(parts) == _merged(script), (src, i)


def test_cli_accepts_hp_with_intron_retention(fx, monkeypatch):
    """-hp -k 6 with intron retention passes the CLI's checks and the model set-up up to the GPU context; a model without
    homopolymer parameters fails with the model error, as in genome mode."""
    from nanosim_b200 import simulator

    class Reached(Exception):
        pass

    def no_gpu(*a, **k):
        raise Reached()

    monkeypatch.setattr(simulator, "Engine", no_gpu)
    out = os.path.join(fx["d"], "cli_cpu")
    with pytest.raises(Reached):
        simulator.main(_cli_args(fx, out))
    args = _cli_args(fx, out)
    args[args.index("-c") + 1] = os.path.join(pc.DATA, pc.MODELS["drna"])
    with pytest.raises(FileNotFoundError, match="hp_lengths"):
        simulator.main(args)
