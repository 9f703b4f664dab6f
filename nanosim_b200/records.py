"""Host-side text formatting of a fetched batch: read names, FASTA/FASTQ records, error-profile rows.

Formats follow the reference exactly:
  aligned   {chrom}_{pos}[;{chrom}_{pos}...]_aligned_{idx}[_chimeric]_{F|R}_{head}_{seg[;seg...]}_{tail}
            (/root/reference/src/simulator.py:1390-1402)
  perfect   {chrom}_{pos}_perfect_{idx}_{F|R}_0_{len}_0                                   (:1332-1343)
  unaligned {chrom}_{pos}_unaligned_{idx}_{F|R}_0_{middle_ref}_0                          (:1511, :1529-1534)
  records   '@'|'>' name, sequence, ['+', chr(q+33)...]                                   (:1437-1443)
  errors    Seq_name Seq_pos error_type error_length ref_base seq_base, right to left      (:1634, :2006-2008)
"""
import ctypes as C

import numpy as np

from . import _lib as L

_COMP = np.arange(256, dtype=np.uint8)
for _a, _b in (("A", "T"), ("C", "G")):
    _COMP[ord(_a)], _COMP[ord(_b)] = ord(_b), ord(_a)


def read_names(batch, ref_names, index_base, perfect=False, metagenome=False, transcriptome=False):
    """index_base: value of the reference's shared ``total_simulated`` counter for the batch's first read."""
    reads, pieces = batch.reads, batch.pieces
    names = []
    unaligned = batch.kind == L.NS_KIND_UNALIGNED
    for i in range(len(reads)):
        r = reads[i]
        p0, npc = int(r["piece_first"]), int(r["n_pieces"])
        strand = "R" if r["reversed"] else "F"
        idx = index_base + i
        if unaligned:
            pc = pieces[p0]
            names.append("%s_%d_unaligned_%d_%s_0_%d_0" % (ref_names[pc["chrom"]], pc["pos"], idx, strand, pc["ref_len"]))
            continue
        segs = [pieces[p0 + k] for k in range(0, npc, 2)]
        if transcriptome and int(segs[0]["kind"]) & L.NS_PIECE_GENOME:
            # intron-retention layout (:1188-1192): genomic start of the first interval, retained introns in genomic order
            loc = sorted(segs, key=lambda x: int(x["pos"]))
            ir = "".join("%d-%d;" % (x["pos"], int(x["pos"]) + int(x["ref_len"])) for x in loc if int(x["kind"]) & L.NS_PIECE_RETAINED)
            names.append("%s_%d_aligned_%d%s_%s_%d_%d_%d" % (ref_names[segs[0]["ref_req"]], loc[0]["pos"], idx, "_RetainedIntron_" + ir if ir else "",
                                                             strand, r["head"], sum(int(x["ref_len"]) for x in segs),
                                                             int(r["tail"]) + int(segs[0]["polya_len"])))
            continue
        if transcriptome:       # {trx}_{pos}_aligned|perfect_{idx}_{F|R}_{head}_{middle_ref}_{tail+polyA} (:1188-1219)
            pc = segs[0]
            names.append("%s_%d_%s_%d_%s_%d_%d_%d" % (ref_names[pc["chrom"]], pc["pos"], "perfect" if perfect else "aligned", idx,
                                                      strand, r["head"], pc["ref_len"], int(r["tail"]) + int(pc["polya_len"])))
            continue
        if perfect:
            loc = "".join("%s_%d" % (ref_names[s["chrom"]], s["pos"]) for s in segs)
            names.append("%s_perfect_%d_%s_0_%d_0" % (loc, idx, strand, sum(int(s["ref_len"]) for s in segs)))
            continue
        if metagenome:          # gap lengths are part of the name in metagenome mode (:965-969)
            comps = []
            for k in range(npc):
                pc = pieces[p0 + k]
                comps.append("gap_%d" % pc["out_len"] if k & 1 else "%s_%d" % (ref_names[pc["chrom"]], pc["pos"]))
            loc = ";".join(comps)
        else:
            loc = ";".join("%s_%d" % (ref_names[s["chrom"]], s["pos"]) for s in segs)
        nm = "%s_aligned_%d" % (loc, idx)
        if len(segs) > 1:
            nm += "_chimeric"
        nm += "_%s_%d_%s_%d" % (strand, r["head"], ";".join(str(int(s["ref_len"])) for s in segs), r["tail"])
        names.append(nm)
    return names


def format_records(batch, names, fastq, n_threads=8, as_array=False):
    """FASTA/FASTQ text of the batch via the library's multi-threaded formatter -> bytes (or the uint8 array itself)."""
    lib = L.lib()
    blob, offs = _name_blob(names)
    reads = np.ascontiguousarray(batch.reads)
    qual_ptr = batch.qual.ctypes.data_as(C.c_void_p) if fastq else None
    need = lib.ns_format_records(batch.seq.ctypes.data_as(C.c_void_p), qual_ptr, reads.ctypes.data_as(C.c_void_p),
                                 len(names), blob, offs.ctypes.data_as(C.c_void_p), int(fastq), None, 0, n_threads)
    if need < 0:
        raise RuntimeError("ns_format_records failed: %d" % need)
    out = np.empty(int(need), dtype=np.uint8)
    got = lib.ns_format_records(batch.seq.ctypes.data_as(C.c_void_p), qual_ptr, reads.ctypes.data_as(C.c_void_p),
                                len(names), blob, offs.ctypes.data_as(C.c_void_p), int(fastq),
                                out.ctypes.data_as(C.c_void_p), int(need), n_threads)
    if got != need:
        raise RuntimeError("ns_format_records failed: %d" % got)
    return out if as_array else out.tobytes()


def write_records(fd, file_off, batch, names, fastq, n_threads=8):
    """format_records() straight into file descriptor ``fd`` at byte ``file_off`` (ns_write_records: every formatter thread
    pwrite()s its own stretch).  Returns the number of bytes written."""
    lib = L.lib()
    blob, offs = _name_blob(names)
    reads = np.ascontiguousarray(batch.reads)
    qual_ptr = batch.qual.ctypes.data_as(C.c_void_p) if fastq else None
    got = lib.ns_write_records(int(fd), C.c_uint64(int(file_off)), batch.seq.ctypes.data_as(C.c_void_p), qual_ptr,
                               reads.ctypes.data_as(C.c_void_p), len(names), blob, offs.ctypes.data_as(C.c_void_p), int(fastq), n_threads)
    if got < 0:
        raise OSError("ns_write_records failed: %d" % got)
    return int(got)


def write_error_profile(fd, file_off, batch, names, ref, seed=0, n_threads=8):
    """format_error_profile() straight into file descriptor ``fd`` at byte ``file_off`` (ns_write_error_profile)."""
    lib = L.lib()
    blob, offs = _name_blob(names)
    reads = np.ascontiguousarray(batch.reads)
    pieces = np.ascontiguousarray(batch.pieces)
    ops = np.ascontiguousarray(batch.ops, dtype=np.uint32)
    bases = np.ascontiguousarray(ref.bases)
    coff = np.ascontiguousarray(ref.offsets, dtype=np.uint64)
    got = lib.ns_write_error_profile(int(fd), C.c_uint64(int(file_off)), batch.seq.ctypes.data_as(C.c_void_p),
                                     reads.ctypes.data_as(C.c_void_p), pieces.ctypes.data_as(C.c_void_p), ops.ctypes.data_as(C.c_void_p),
                                     len(names), bases.ctypes.data_as(C.c_void_p), coff.ctypes.data_as(C.c_void_p), blob,
                                     offs.ctypes.data_as(C.c_void_p), C.c_uint64(int(seed)), C.c_uint64(int(batch.first_id)), n_threads)
    if got < 0:
        raise OSError("ns_write_error_profile failed: %d" % got)
    return int(got)


class NameTable:
    """Read names as the formatters take them: NUL-terminated strings back to back + the offset of each."""

    def __init__(self, blob, offs):
        self.blob, self.offs = blob, offs

    def __len__(self):
        return len(self.offs)

    def __getitem__(self, i):
        a = int(self.offs[i])
        return bytes(self.blob[a:self.blob.index(b"\0", a)]).decode()

    def tolist(self):
        return [x.decode() for x in bytes(self.blob).split(b"\0")[:-1]]


_CHROM_CACHE = {}


def name_table(batch, ref_names, index_base, perfect=False, metagenome=False, transcriptome=False):
    """read_names() through the library (ns_format_names): same strings, no per-read Python."""
    lib = L.lib()
    key = id(ref_names)
    entry = _CHROM_CACHE.get(key)          # one lookup: pipeline workers call this concurrently
    if entry is None or entry[0] is not ref_names:
        entry = (ref_names,) + _name_blob(ref_names)
        _CHROM_CACHE.clear()
        _CHROM_CACHE[key] = entry
    _, cblob, coffs = entry
    reads = np.ascontiguousarray(batch.reads)
    pieces = np.ascontiguousarray(batch.pieces)
    flags = (1 if perfect else 0) | (2 if metagenome else 0) | (4 if transcriptome else 0)
    n = len(reads)

    def call(out_ptr, cap, off_ptr):
        return lib.ns_format_names(reads.ctypes.data_as(C.c_void_p), pieces.ctypes.data_as(C.c_void_p), n, int(batch.kind), flags,
                                   C.c_uint64(int(index_base)), cblob, coffs.ctypes.data_as(C.c_void_p), out_ptr, cap, off_ptr)

    offs = np.zeros(n, dtype=np.uint64)
    # one call with a buffer that almost always suffices (names are ~60 characters); sized exactly when it does not
    out = np.empty(max(n, 1) * 160, dtype=np.uint8)
    got = call(out.ctypes.data_as(C.c_void_p), len(out), offs.ctypes.data_as(C.c_void_p))
    if got == -4:                                    # NS_ENOMEM
        need = call(None, 0, None)
        if need < 0:
            raise RuntimeError("ns_format_names failed: %d" % need)
        out = np.empty(int(need), dtype=np.uint8)
        got = call(out.ctypes.data_as(C.c_void_p), int(need), offs.ctypes.data_as(C.c_void_p))
    if got < 0:
        raise RuntimeError("ns_format_names failed: %d" % got)
    return NameTable(out[:int(got)].tobytes(), offs)


def _name_blob(names):
    if isinstance(names, NameTable):
        return names.blob, names.offs
    blob = ("\0".join(names) + "\0").encode()
    offs = np.zeros(len(names), dtype=np.uint64)
    pos = 0
    for i, nm in enumerate(names):
        offs[i] = pos
        pos += len(nm.encode()) + 1
    return blob, offs


def format_error_profile(batch, names, ref, seed=0, n_threads=8, as_array=False):
    """The rows of ``<out>_aligned_error_profile`` for a fetched batch (needs batch.ops) via the library's multi-threaded
    formatter -> bytes.  Same text as ``"".join(error_profile_rows(...))``, which stays as the readable reference
    implementation the tests compare against."""
    lib = L.lib()
    blob, offs = _name_blob(names)
    reads = np.ascontiguousarray(batch.reads)
    pieces = np.ascontiguousarray(batch.pieces)
    ops = np.ascontiguousarray(batch.ops, dtype=np.uint32)
    bases = np.ascontiguousarray(ref.bases)
    coff = np.ascontiguousarray(ref.offsets, dtype=np.uint64)

    def call(out_ptr, cap):
        return lib.ns_format_error_profile(batch.seq.ctypes.data_as(C.c_void_p), reads.ctypes.data_as(C.c_void_p),
                                           pieces.ctypes.data_as(C.c_void_p), ops.ctypes.data_as(C.c_void_p), len(names),
                                           bases.ctypes.data_as(C.c_void_p), coff.ctypes.data_as(C.c_void_p), blob,
                                           offs.ctypes.data_as(C.c_void_p), C.c_uint64(int(seed)), C.c_uint64(int(batch.first_id)),
                                           out_ptr, cap, n_threads)

    need = call(None, 0)
    if need < 0:
        raise RuntimeError("ns_format_error_profile failed: %d" % need)
    out = np.empty(int(need), dtype=np.uint8)
    got = call(out.ctypes.data_as(C.c_void_p), int(need))
    if got != need:
        raise RuntimeError("ns_format_error_profile failed: %d" % got)
    return out if as_array else out.tobytes()


_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85


def _philox4x32(ctr, key, rounds):
    """numpy Philox4x32 (vectorised over the first axis of ctr [n,4] uint64-held uint32 words); mirrors
    csrc/device_common.cuh:philox4x32."""
    c = [ctr[:, i].astype(np.uint64) for i in range(4)]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    mask = np.uint64(0xFFFFFFFF)
    for _ in range(rounds):
        p0 = np.uint64(_M0) * c[0]
        p1 = np.uint64(_M1) * c[2]
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ k0) & mask, p1 & mask, ((p0 >> np.uint64(32)) ^ c[3] ^ k1) & mask, p0 & mask]
        k0 = (k0 + np.uint64(_W0)) & mask
        k1 = (k1 + np.uint64(_W1)) & mask
    return np.stack(c, axis=1)


def event_bases_hp(seed, rid, piece_in_read, k, n, is_mis, orig_idx=None):
    """Bases the homopolymer pass assigned to error event k of a segment (csrc/hp_kernel.cuh): 16 bits h of Philox-7
    block (k<<9)+(t>>3) per base (csrc/device_common.cuh:event_base).  Returns ACGT index array in the device's order
    A C T G = 0 1 2 3."""
    t = np.arange(n, dtype=np.uint64)
    stream = (6 << 28) | (piece_in_read & 0x07ffffff)            # ST_EMIT_B, kind 0
    ctr = np.stack([np.full(n, rid & 0xFFFFFFFF, dtype=np.uint64), np.full(n, (rid >> 32) & 0xFFFFFFFF, dtype=np.uint64),
                    np.full(n, stream, dtype=np.uint64), (np.uint64(k) << np.uint64(9)) + (t >> np.uint64(3))], axis=1)
    blk = _philox4x32(ctr, (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF), 7)
    word = blk[np.arange(n), ((t >> np.uint64(1)) & np.uint64(3)).astype(np.int64)]
    h = ((word >> (np.uint64(16) * (t & np.uint64(1)))) & np.uint64(0xFFFF)).astype(np.int64)
    if not is_mis:
        return h & 3
    return (orig_idx + 1 + ((h * 3) >> 16)) & 3


_IDX_BASE = np.frombuffer(b"ACTG", dtype=np.uint8)
_BASE_IDX = np.zeros(256, dtype=np.int64)
for _i, _c in enumerate(b"ACTG"):
    _BASE_IDX[_c] = _i


def error_profile_rows(batch, names, ref, seed=0):
    """The rows mutate_read logs for every aligned segment (needs batch.ops).  ``ref`` is the PackedReference.
    Reference bases are shown upper-cased as stored (an IUPAC code is shown as the code itself)."""
    rows = []
    reads, pieces, ops_all = batch.reads, batch.pieces, batch.ops
    ref_off = ref.offsets.astype(np.int64)
    for i in range(len(reads)):
        r = reads[i]
        L_read = int(r["seq_len"])
        so = int(r["seq_off"])
        fwd = batch.seq[so:so + L_read]
        if r["reversed"]:
            fwd = _COMP[fwd[::-1]]
        p0, npc = int(r["piece_first"]), int(r["n_pieces"])
        group, ref_base = [], 0                 # rows of one mutate_read call: a segment and the pieces continuing it
        for k in range(0, npc, 2):
            pc = pieces[p0 + k]
            kind = int(pc["kind"])
            if kind & L.NS_PIECE_KIND_MASK != L.NS_PIECE_SEGMENT:
                continue
            if not kind & L.NS_PIECE_CONT:
                rows.extend(reversed(group))
                group, ref_base = [], 0
            back = bool(kind & L.NS_PIECE_REF_REV)
            ops = ops_all[int(pc["ev_off"]): int(pc["ev_off"]) + int(pc["ev_n_ops"])]    # the error-event script
            rewritten = int(pc["ev_off"]) != int(pc["op_off"])                        # -hp: bases fixed by the hp pass
            ty = (ops >> 28).astype(np.int64)
            ln = np.where(ty == L.NS_OP_LIT, ops & 0x00ffffff, ops & 0x0fffffff).astype(np.int64)
            out_adv = np.where(ty == L.NS_OP_DEL, 0, ln)
            ref_adv = np.where((ty == L.NS_OP_COPY) | (ty == L.NS_OP_MIS) | (ty == L.NS_OP_DEL), ln, 0)
            out_start = int(pc["out_rel"]) + np.concatenate([[0], np.cumsum(out_adv)[:-1]])
            ref_start = np.concatenate([[0], np.cumsum(ref_adv)[:-1]])
            cstart, clen = int(ref_off[pc["chrom"]]), int(ref_off[pc["chrom"] + 1] - ref_off[pc["chrom"]])
            base, plen = int(pc["pos"]), int(pc["ref_len"])
            for j in np.nonzero((ty >= 1) & (ty <= 3) & (ln > 0))[0]:
                t, n, rs, os_ = int(ty[j]), int(ln[j]), int(ref_start[j]), int(out_start[j])
                if t == L.NS_OP_INS:
                    refb = "-" * n
                else:
                    f = rs + np.arange(n)                      # offsets in the piece, in the direction of the read
                    idx = (base + (plen - 1 - f if back else f)) % clen
                    rb = ref.bases[cstart + idx]
                    rb = np.where((rb >= 97) & (rb <= 122), rb - 32, rb).astype(np.uint8)
                    refb = (_COMP[rb] if back else rb).tobytes().decode()
                if t == L.NS_OP_DEL:
                    seqb = "-" * n
                elif rewritten:
                    orig = _BASE_IDX[np.frombuffer(refb.encode(), dtype=np.uint8)] if t == L.NS_OP_MIS else None
                    bi = event_bases_hp(seed, batch.first_id + i, k, int(j), n, t == L.NS_OP_MIS, orig)
                    seqb = _IDX_BASE[bi].tobytes().decode()
                else:
                    seqb = fwd[os_:os_ + n].tobytes().decode()
                group.append("%s\t%d\t%s\t%d\t%s\t%s\n" % (names[i], ref_base + rs, ("mis", "ins", "del")[t - 1], n, refb, seqb))
            ref_base += plen
        rows.extend(reversed(group))
    return rows
