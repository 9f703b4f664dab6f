"""Intron retention in transcriptome mode: the host half.

Mirrors ``read_profile``'s model_ir block (/root/reference/src/simulator.py:404-453), ``update_structure`` (:114-146),
``extract_read_pos`` (:149-191) and the IR part of ``simulation_aligned_transcriptome`` (:1156-1192).

Division of labour.  The device simulates every aligned read against its transcript as usual.  Per batch the host then
draws, from the read metadata alone, the IR / no_IR state of every intron of every read's transcript (two-state Markov
chain, vectorised over the batch, uniforms a pure function of seed and read id), and for the few reads that retain an intron (~2 % with the
shipped models) it lays the read out on the GENOME instead: the exon / retained-intron intervals the read covers become
the read's pieces (one per interval, walked backwards for transcripts on the minus strand) and the read's edit script is
cut at the interval boundaries.  ``ns_reemit`` uploads those pieces and runs the emit kernel on them again; as all emit
randomness is indexed by the position in the read, inserted / head / tail bases and every quality value stay what they
were -- only the bases copied or substituted from the reference change, exactly as when ``mutate_read`` is handed the
genomic sequence instead of the spliced one (:1163-1181).  With -hp/-k the reference filters and rewrites the genomic
read: the device then keeps the unfiltered event scripts (``raw_ev_off``), those are cut, and ``ns_reemit`` runs the
homopolymer pass again over the read's genome pieces; the read changes length and its qualities are drawn anew.

Kept from the device's first pass (documented deviation): whether the read carries a polyA tail (the reference re-decides
it from the genomic end of the last feature, :186-189, which would change the read length).
"""
import numpy as np

from . import _lib as L

ST_IR = 9                      # stream tag of the IR draws (the device's Philox streams use purposes 1..8)
EXON, INTRON = 0, 1


def read_ir_markov_model(path):
    """``_IR_markov_model`` (:413-422) -> P(no_IR | previous state) for start / no_IR / IR; the IR interval is the rest."""
    thr = {}
    with open(path) as f:
        f.readline()
        for line in f:
            info = line.strip().split()
            if info:
                thr[info[0]] = float(info[1])
    return np.asarray([thr["start"], thr["no_IR"], thr["IR"]], dtype=np.float64)


class TranscriptStructures:
    """``dict_ref_structure`` (:424-453) as flat arrays: for transcript record t the features
    ``first[t] .. first[t+1]`` in GFF3 file order, each (type, genome record or -1, start, end, strand)."""

    def __init__(self, first, ftype, chrom, start, end, minus):
        self.first, self.ftype, self.chrom, self.start, self.end, self.minus = first, ftype, chrom, start, end, minus
        n = len(first) - 1
        self.n_introns = np.add.reduceat(np.concatenate([ftype == INTRON, [False]]).astype(np.int64), first[:-1])[:n] if n else np.zeros(0, np.int64)
        self.n_introns[np.diff(first) == 0] = 0

    @staticmethod
    def from_gff3(path, trx_names, genome_raw_names):
        """trx_names: transcript record names (IDs cut at '.'), genome_raw_names: FASTA record names of the genome."""
        index = {k: i for i, k in enumerate(trx_names)}
        flag_chrom = any("chr" in g for g in genome_raw_names)                         # :1066-1069
        gidx = {g: i for i, g in enumerate(genome_raw_names)}
        per = {}
        with open(path) as f:
            for line in f:
                if line[:1] == "#":
                    continue
                c = line.rstrip("\n").split("\t", 8)
                if len(c) < 9 or c[2] not in ("exon", "intron"):
                    continue
                attr = c[8]
                k = attr.find("transcript_id=")
                if k >= 0:
                    e = attr.find(";", k)
                    fid = attr[k + 14:e if e >= 0 else None]
                elif "Parent=" in attr:                                               # :432-441
                    first = attr.split(";", 1)[0].split("=", 1)[-1].strip().strip('"')
                    info = first.split(":")
                    if len(info) == 1:
                        fid = info[0]
                    elif info[0] == "transcript":
                        fid = info[1]
                    else:
                        continue
                else:
                    continue
                t = index.get(fid.strip().strip('"').split(".")[0])
                if t is None:
                    continue
                chrom = c[0].strip("chr") if "chr" in c[0] else c[0]                   # :448-450
                g = gidx.get(("chr" + chrom) if flag_chrom else chrom, -1)             # :1165-1167
                per.setdefault(t, []).append((EXON if c[2] == "exon" else INTRON, g, int(c[3]) - 1, int(c[4]), c[6] == "-"))
        n = len(trx_names)
        first = np.zeros(n + 1, dtype=np.int64)
        for t, feats in per.items():
            first[t + 1] = len(feats)
        first = np.cumsum(first)
        tot = int(first[-1])
        ftype, chrom = np.zeros(tot, dtype=np.int8), np.zeros(tot, dtype=np.int64)
        start, end, minus = np.zeros(tot, dtype=np.int64), np.zeros(tot, dtype=np.int64), np.zeros(tot, dtype=bool)
        for t, feats in per.items():
            a = int(first[t])
            for j, (ty, g, s, e, m) in enumerate(feats):
                ftype[a + j], chrom[a + j], start[a + j], end[a + j], minus[a + j] = ty, g, s, e, m
        return TranscriptStructures(first, ftype, chrom, start, end, minus)


def expressed_with_structure(expr_chrom, expr_weights, st, trx_lengths):
    """With intron retention on, the reference only accepts a drawn transcript that has features in the GFF3 and whose
    exon lengths add up to its length in the transcriptome FASTA (simulator.py:1094-1099, ref_len_from_structure :100-105);
    anything else is drawn again.  Redrawing from fixed weights == dropping those transcripts from the expressed set."""
    expr_chrom = np.asarray(expr_chrom)
    n = len(st.first) - 1
    is_exon = st.ftype == EXON
    exon_len = np.zeros(n, dtype=np.int64)
    owner = np.repeat(np.arange(n), np.diff(st.first))
    np.add.at(exon_len, owner[is_exon], (st.end - st.start)[is_exon])
    has = np.diff(st.first) > 0
    t = expr_chrom.astype(np.int64)
    keep = has[t] & (exon_len[t] == np.asarray(trx_lengths, dtype=np.int64)[t])
    return expr_chrom[keep], np.asarray(expr_weights)[keep], int((~keep).sum())


def ir_uniforms(seed, rids, n, counts=None):
    """n uniforms in [0, 1) per read id, a pure function of (seed, read id, column): SplitMix64's finaliser over a counter
    built from the three (host-side draws: a handful per read, no need for the device's Philox streams).  counts[i]
    (optional): only the first counts[i] uniforms of read i are needed -- most transcripts have few introns, a few hundreds."""
    rids = np.asarray(rids, dtype=np.uint64)
    counts = np.full(len(rids), n, dtype=np.int64) if counts is None else np.minimum(np.asarray(counts, dtype=np.int64), n)
    rows = np.repeat(np.arange(len(rids)), counts)
    cols = np.arange(int(counts.sum())) - np.repeat(np.cumsum(counts) - counts, counts)
    with np.errstate(over="ignore"):
        z = (rids[rows] * np.uint64(0x9E3779B97F4A7C15) + (cols.astype(np.uint64) + np.uint64(1)) * np.uint64(0xD1B54A32D192ED03)
             + np.uint64(seed & 0xFFFFFFFFFFFFFFFF) * np.uint64(0x8CB92BA72F3D8DD7) + np.uint64(ST_IR))
        z ^= z >> np.uint64(30)
        z *= np.uint64(0xBF58476D1CE4E5B9)
        z ^= z >> np.uint64(27)
        z *= np.uint64(0x94D049BB133111EB)
        z ^= z >> np.uint64(31)
    out = np.zeros((len(rids), n), dtype=np.float64)
    out[rows, cols] = (z >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)
    return out


def draw_ir_states(p_no_ir, n_introns, u):
    """update_structure's chain (:121-133) for many reads at once.  u[i, j] is the uniform of read i's j-th intron.
    Returns a bool matrix: intron j of read i is retained."""
    n, m = u.shape
    state = np.zeros(n, dtype=np.int64)                     # 0 start, 1 no_IR, 2 IR
    retained = np.zeros((n, m), dtype=bool)
    for j in range(m):
        active = j < n_introns
        is_ir = u[:, j] >= p_no_ir[state]
        retained[:, j] = is_ir & active
        state = np.where(active, np.where(is_ir, 2, 1), state)
    return retained


def extract_read_pos(length, ref_len, feats, retained, u_start):
    """extract_read_pos (:149-183) on one transcript: feats = [(type, genome record, start, end, minus)], retained[j] for its
    j-th intron, u_start the uniform behind ``random.randint(0, min(ref_len - length, len_before))``.
    Returns [(genome record, start, end, minus, is_retained_intron)] in genomic (file) order."""
    len_before, j = 0, 0
    kinds = []
    for ty, g, s, e, m in feats:
        if ty == EXON:
            kinds.append(1)
        else:
            kinds.append(2 if retained[j] else 0)
            j += 1
    for k, (ty, g, s, e, m) in zip(kinds, feats):
        if k == 1:
            len_before += e - s
        elif k == 2:
            break
    hi = min(ref_len - length, len_before)
    start_pos = min(int(u_start * (hi + 1)), hi) if hi > 0 else 0
    ivs = []
    for k, (ty, g, s, e, m) in zip(kinds, feats):
        if length == 0:
            break
        if k == 0:
            continue
        if start_pos < e - s:
            a = start_pos + s
            b = a + length if a + length <= e else e
            length -= b - a
            start_pos = 0
            ivs.append((g, a, b, m, k == 2))
        else:
            start_pos -= e - s
    return ivs


def split_script(ops, cuts):
    """Cuts one edit script at cumulative reference offsets ``cuts`` (ascending, the last one = total reference length).
    Ops that consume no reference (INS, HT, LIT) stay with the piece that is open when they occur; the leading HT goes to
    the first piece, everything after the last reference base to the last.  Returns a list of uint32 arrays."""
    out, cur, consumed, k = [], [], 0, 0
    for op in ops.tolist():
        ty = op >> 28
        ln = (op & 0x00ffffff) if ty == L.NS_OP_LIT else (op & 0x0fffffff)
        if ty in (L.NS_OP_COPY, L.NS_OP_MIS, L.NS_OP_DEL):
            while ln > 0:
                while k < len(cuts) - 1 and consumed >= cuts[k]:
                    out.append(cur)
                    cur = []
                    k += 1
                take = min(ln, cuts[k] - consumed) if k < len(cuts) - 1 else ln
                cur.append((ty << 28) | take)
                consumed += take
                ln -= take
        else:
            cur.append(op)
    out.append(cur)
    while len(out) < len(cuts):
        out.append([])
    return [np.asarray(x, dtype=np.uint32) for x in out]


def _out_len(ops):
    ty = ops >> 28
    ln = np.where(ty == L.NS_OP_LIT, ops & 0x00ffffff, ops & 0x0fffffff)
    return int(ln[ty != L.NS_OP_DEL].sum())


class IntronRetention:
    """Everything the aligned-read sink needs: p(no_IR), the structures, and where the genome records sit in the reference."""

    def __init__(self, p_no_ir, structures, trx_lengths, genome_first_record):
        self.p_no_ir, self.st, self.trx_len, self.g0 = p_no_ir, structures, np.asarray(trx_lengths, dtype=np.int64), int(genome_first_record)

    def plan_batch(self, reads, pieces, ops, first_id, seed, n_pieces_total, n_ops_total, raw_ev_off=0):
        """reads / pieces / ops: the fetched metadata of an aligned batch.  Returns None when no read of the batch retains an
        intron, else (slots, new_reads, new_pieces, new_ops): the patch ``Engine.reemit`` takes.  Offsets in the new
        pieces are absolute (they land behind the batch's n_pieces_total pieces / n_ops_total ops).
        raw_ev_off (NsBatchInfo.raw_ev_off, -hp/-k): where the unfiltered event scripts start; the read's script is cut from
        there (the -k filter and mutate_homo run again on the genomic read), else from the emitted script."""
        st = self.st
        p0 = reads["piece_first"].astype(np.int64)
        trx = pieces["chrom"][p0].astype(np.int64)
        n_int = st.n_introns[trx]
        if len(n_int) == 0 or int(n_int.max()) == 0:
            return None
        rids = first_id + np.arange(len(reads), dtype=np.uint64)
        # most transcripts have a handful of introns, a few have hundreds: two groups keep the uniform matrices small
        decided = {}
        for sel in (np.flatnonzero((n_int > 0) & (n_int <= 31)), np.flatnonzero(n_int > 31)):
            if len(sel) == 0:
                continue
            m = int(n_int[sel].max())
            u = ir_uniforms(seed, rids[sel], m + 1, counts=n_int[sel] + 1)
            ret = draw_ir_states(self.p_no_ir, n_int[sel], u[:, :m])
            for k in np.flatnonzero(ret.any(axis=1)).tolist():
                i = int(sel[k])
                decided[i] = (ret[k, :int(n_int[i])].tolist(), float(u[k, int(n_int[i])]))
        hit = sorted(decided)
        slots, new_reads, new_pieces, new_ops = [], [], [], []
        piece_cursor, op_cursor = int(n_pieces_total), int(n_ops_total)
        for i in hit:
            retained_i, u_start = decided[i]
            t = int(trx[i])
            a, b = int(st.first[t]), int(st.first[t + 1])
            feats = list(zip(st.ftype[a:b].tolist(), st.chrom[a:b].tolist(), st.start[a:b].tolist(), st.end[a:b].tolist(),
                             st.minus[a:b].tolist()))
            pc = pieces[int(p0[i])]
            length = int(pc["ref_len"])
            # u_start: the uniform after the read's own intron draws (not after the batch's longest chain: results must not
            # depend on which reads share a batch)
            ivs = extract_read_pos(length, int(self.trx_len[t]), feats, retained_i, u_start)
            if not ivs or any(g < 0 for g, *_ in ivs) or sum(e - s for _, s, e, _, _ in ivs) != length:
                continue                                     # a chromosome the genome file lacks (:1168-1170) / inconsistent annotation
            minus = bool(ivs[-1][3])                         # `interval.strand` after the loop (:1177)
            order = ivs[::-1] if minus else ivs              # pieces in the direction of the transcript
            if raw_ev_off:
                script = ops[int(raw_ev_off) + int(pc["ev_off"]):int(raw_ev_off) + int(pc["ev_off"]) + int(pc["ev_n_ops"])]
            else:
                script = ops[int(pc["op_off"]):int(pc["op_off"]) + int(pc["n_ops"])]
            parts = split_script(script, np.cumsum([e - s for _, s, e, _, _ in order]).tolist())
            rd = reads[i].copy()
            rd["piece_first"] = piece_cursor
            rd["n_pieces"] = 2 * len(order) - 1
            out_rel = 0
            for k, ((g, s, e, mi, is_ir), part) in enumerate(zip(order, parts)):
                if k:
                    gap = np.zeros((), dtype=L.PIECE_DTYPE)
                    gap["kind"] = L.NS_PIECE_GAP
                    gap["read_slot"] = i
                    gap["out_rel"] = out_rel
                    gap["op_off"] = gap["ev_off"] = op_cursor
                    new_pieces.append(gap)
                q = pc.copy()
                q["kind"] = (L.NS_PIECE_SEGMENT | L.NS_PIECE_GENOME | (L.NS_PIECE_REF_REV if minus else 0) |
                             (L.NS_PIECE_CONT if k else 0) | (L.NS_PIECE_RETAINED if is_ir else 0))
                q["chrom"] = self.g0 + g
                q["pos"] = s
                q["ref_len"] = e - s
                q["ref_req"] = t                             # the transcript the read belongs to (names)
                q["op_off"] = q["ev_off"] = op_cursor
                q["n_ops"] = q["ev_n_ops"] = len(part)
                q["out_len"] = _out_len(part) if len(part) else 0
                q["out_rel"] = out_rel
                q["polya_len"] = pc["polya_len"] if k == 0 else 0
                out_rel += int(q["out_len"])
                op_cursor += len(part)
                new_pieces.append(q)
                new_ops.append(part)
            piece_cursor += 2 * len(order) - 1
            slots.append(i)
            new_reads.append(rd)
        if not slots:
            return None
        return (np.asarray(slots, dtype=np.uint32), np.asarray(new_reads, dtype=L.READ_DTYPE),
                np.asarray(new_pieces, dtype=L.PIECE_DTYPE), np.concatenate(new_ops) if new_ops else np.zeros(0, dtype=np.uint32))
