"""Thin object wrapper over the C ABI (one context == one GPU)."""
import ctypes as C

import numpy as np

from . import _lib as L
from .model import DeviceTables


class NanoSimError(RuntimeError):
    pass


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _variants(t, out):
    """NsVariants over the arrays of a variants.HaplotypeTables; out (c_uint64) receives peak_bytes."""
    return L.NsVariants(len(t.hap_chrom), _ptr(t.hap_chrom), _ptr(t.var_off), len(t.var_pos), _ptr(t.var_pos), _ptr(t.var_ref_len),
                        _ptr(t.alt_off), _ptr(t.alt_len), _ptr(t.alt), len(t.alt), C.pointer(out), _ptr(t.alt_kind))


class Batch:
    """Host copy of one simulated batch."""

    def __init__(self, info, seq, qual, reads, pieces, ops, kind, first_id):
        self.info, self.seq, self.qual, self.reads, self.pieces, self.ops = info, seq, qual, reads, pieces, ops
        self.kind, self.first_id = kind, first_id

    def read_seq(self, i):
        r = self.reads[i]
        o = int(r["seq_off"])
        return self.seq[o:o + int(r["seq_len"])].tobytes().decode()

    def read_qual(self, i):
        r = self.reads[i]
        o = int(r["seq_off"])
        return self.qual[o:o + int(r["seq_len"])]


class Engine:
    def __init__(self, device=0, seed=0):
        self._lib = L.lib()
        self._ctx = C.c_void_p()
        rc = self._lib.ns_create(int(device), C.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), C.byref(self._ctx))
        if rc != 0:
            raise NanoSimError("ns_create failed (rc=%d): no usable CUDA device %d?" % (rc, device))
        self.device = device
        self._keep = {}
        self.fastq = False
        self.info = None
        self._z_bytes = self._ep_bytes = 0

    def clone(self):
        """A context that shares this engine's reference + model in HBM (own stream and batch buffers)."""
        other = Engine.__new__(Engine)
        other._lib = self._lib
        other._ctx = C.c_void_p()
        self._check(self._lib.ns_clone(self._ctx, C.byref(other._ctx)))
        other.device, other._keep, other.fastq, other.info = self.device, {}, self.fastq, None
        other._z_bytes = other._ep_bytes = 0
        other._parent = self            # keep the parent alive
        for k in ("ref", "tables"):
            if hasattr(self, k):
                setattr(other, k, getattr(self, k))
        return other

    def close(self):
        if self._ctx:
            self._lib.ns_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise NanoSimError(self._lib.ns_last_error(self._ctx).decode() + " (rc=%d)" % rc)

    # ---- read_profile()
    def set_reference(self, ref):
        """ref: PackedReference (host) -- or pass device pointers via set_reference_ptr."""
        self.ref = ref
        sp = getattr(ref, "chrom_species", None)
        if sp is not None:
            sp = np.ascontiguousarray(sp, dtype=np.uint32)
            circ = np.ascontiguousarray(ref.chrom_circular, dtype=np.uint8)
            r = L.NsReference(_ptr(ref.bases), ref.genome_len, _ptr(ref.offsets), len(ref.names), len(ref.species),
                              _ptr(sp), _ptr(circ))
        else:
            r = L.NsReference(_ptr(ref.bases), ref.genome_len, _ptr(ref.offsets), len(ref.names), 0, None, None)
        self._check(self._lib.ns_set_reference(self._ctx, C.byref(r)))

    def apply_variants(self, tables):
        """genome --vcf: replaces the resident reference with the haplotype records of ``tables`` (a
        variants.HaplotypeTables over it), built in HBM (ns_apply_variants).  Returns the device memory the reference and
        the build held at the build's peak, in bytes."""
        peak = C.c_uint64()
        self._check(self._lib.ns_apply_variants(self._ctx, C.byref(_variants(tables, peak))))
        return int(peak.value)

    def set_lift(self, tables):
        """genome --vcf --lift_mapped_bam: after apply_variants(tables), keeps the lift of the haplotype records onto the
        haploid reference (ns_set_lift), so that compress_bam_mapped() writes the reads' alignments to the haploid
        records.  Call before clone().  Returns the device bytes the lift keeps."""
        n = C.c_uint64()
        self._check(self._lib.ns_set_lift(self._ctx, C.byref(_variants(tables, n))))
        return int(n.value)

    def set_splice(self, m):
        """transcriptome --spliced_bam: keeps the transcripts' exons on the genome records (a splice.SpliceMap; ns_set_splice),
        so that compress_bam_mapped() writes the reads' spliced alignments to the genome (and compress_bam_transcript()
        places the reads that retain an intron on their transcripts).  Call before clone().  Returns the
        device bytes the map keeps."""
        n = C.c_uint64()
        arrs = [np.ascontiguousarray(x, dtype=d) for x, d in ((m.exon_off, np.uint64), (m.exon_chrom, np.uint32), (m.exon_start, np.uint32),
                                                               (m.exon_len, np.uint32), (m.minus, np.uint8), (m.genome_len, np.uint64))]
        first = L.NS_SPLICE_NO_GENOME if m.genome_first is None else int(m.genome_first)
        s = L.NsSplice(len(arrs[0]) - 1, _ptr(arrs[0]), _ptr(arrs[1]), _ptr(arrs[2]), _ptr(arrs[3]), _ptr(arrs[4]), len(arrs[5]), _ptr(arrs[5]),
                       first, C.pointer(n))
        self._check(self._lib.ns_set_splice(self._ctx, C.byref(s)))
        return int(n.value)

    def set_aln_tags(self, ref_names, ref_paired=None, n_var=0):
        """--aln_tags: compress_bam_mapped() adds NM and SA to every mapped record (ns_set_aln_tags).  ref_names: the mapped
        header's @SQ names in refID order; with set_lift(tables), ref_paired = tables.ref_paired (the REF bytes the ALTs'
        first bases pair with) and n_var = its variant count.  Call after set_lift() / set_splice() and before clone().
        Returns the device bytes the tables keep."""
        enc = [n.encode() for n in ref_names]
        blob = np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8)
        off = np.concatenate([[0], np.cumsum([len(e) for e in enc])]).astype(np.uint64)
        paired = np.ascontiguousarray(ref_paired if ref_paired is not None else np.zeros(0), dtype=np.uint8)
        n = C.c_uint64()
        t = L.NsAlnTags(len(enc), _ptr(blob), _ptr(off), int(n_var), _ptr(paired) if len(paired) else None, len(paired), C.pointer(n))
        self._check(self._lib.ns_set_aln_tags(self._ctx, C.byref(t)))
        return int(n.value)

    def set_abundance(self, abun, inflated=None):
        """dict_abun / dict_abun_inflated of one sample, per species in genome-list order (metagenome mode)."""
        a = np.ascontiguousarray(abun, dtype=np.float64)
        i = np.ascontiguousarray(inflated, dtype=np.float64) if inflated is not None else None
        self._check(self._lib.ns_set_abundance(self._ctx, _ptr(a), _ptr(i), len(a)))

    def set_reference_ptr(self, bases_ptr, n_bases, offsets, chrom_species=None, chrom_circular=None, n_species=0):
        """Reference whose bases already sit in device (or pinned host) memory, e.g. after an NCCL broadcast."""
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        sp = np.ascontiguousarray(chrom_species, dtype=np.uint32) if n_species else None
        circ = np.ascontiguousarray(chrom_circular, dtype=np.uint8) if n_species else None
        r = L.NsReference(C.c_void_p(int(bases_ptr)), int(n_bases), _ptr(offsets), len(offsets) - 1, int(n_species), _ptr(sp), _ptr(circ))
        self._check(self._lib.ns_set_reference(self._ctx, C.byref(r)))

    # ---- multi-GPU init: one NCCL broadcast of the reference (ns_bcast_nccl)
    def nccl_unique_id(self):
        buf = (C.c_uint8 * 128)()
        rc = self._lib.ns_nccl_unique_id(buf)
        if rc != 0:
            raise NanoSimError("ns_nccl_unique_id failed (rc=%d): libnccl.so.2 not loadable?" % rc)
        return bytes(buf)

    def bcast_reference(self, nccl_id, rank, world, root=0):
        """Collective over the ranks of a job: rank `root` (which has set its reference) sends it to the others' HBM."""
        buf = (C.c_uint8 * 128).from_buffer_copy(nccl_id)
        self._check(self._lib.ns_bcast_nccl(self._ctx, buf, int(rank), int(world), int(root)))

    def reference_bases(self, n_bases):
        out = np.empty(int(n_bases), dtype=np.uint8)
        self._check(self._lib.ns_get_reference(self._ctx, _ptr(out), C.c_uint64(len(out))))
        return out

    def fetch_packs_bases(self):
        """True when ns_fetch sends the bases over PCIe as 2 bits each (ns_transfer_info)."""
        packed, threads = C.c_uint32(), C.c_uint32()
        self._check(self._lib.ns_transfer_info(self._ctx, C.byref(packed), C.byref(threads)))
        return bool(packed.value)

    def set_model(self, t: DeviceTables, perfect=False):
        m = L.NsModel()
        keep = []

        def kde(name):
            if name not in t.kde:
                return L.NsKde(None, 0, 0.0)
            data, bw = t.kde[name]
            d = np.ascontiguousarray(data.reshape(-1), dtype=np.float32)
            keep.append(d)
            return L.NsKde(_ptr(d), len(d), float(bw))

        m.kde_aligned = kde("aligned_reads" if perfect else "aligned_region")
        m.kde_ht = kde("ht_length")
        m.kde_ht_ratio = kde("ht_ratio")
        m.kde_unaligned = kde("unaligned_length")
        m.kde_gap = kde("gap_length")
        if getattr(t, "kde2d", None) is not None:
            keep.append(t.kde2d)
            m.kde2d_x, m.kde2d_y = _ptr(t.kde2d[0]), _ptr(t.kde2d[1])
            m.n_kde2d, m.kde2d_bandwidth = len(t.kde2d[0]), float(t.kde2d[2])
        arrays = dict(prob=np.ascontiguousarray(t.alias_prob, dtype=np.uint32),
                      idx=np.ascontiguousarray(t.alias_idx, dtype=np.uint32),
                      desc=np.ascontiguousarray(t.alias_desc.reshape(-1), dtype=np.uint32),
                      lo=np.ascontiguousarray(t.match_bin_lo, dtype=np.uint32),
                      hi=np.ascontiguousarray(t.match_bin_hi, dtype=np.uint32))
        keep.append(arrays)
        m.alias_prob, m.alias_idx, m.alias_desc = _ptr(arrays["prob"]), _ptr(arrays["idx"]), _ptr(arrays["desc"])
        m.n_tables, m.alias_len = len(t.alias_desc), len(arrays["prob"])
        m.match_bin_lo, m.match_bin_hi, m.n_match_bins = _ptr(arrays["lo"]), _ptr(arrays["hi"]), len(arrays["lo"])
        m.has_qual = 1 if t.has_qual else 0
        for i in range(L.NS_N_ERR_STATES):
            for j in range(3):
                m.trans[i][j] = int(t.trans[i, j])
        for i in range(L.NS_N_QUAL_STATES):
            for j in range(L.NS_QUAL_SLOTS):
                m.qual_cdf[i][j] = int(t.qual_cdf[i, j])
        for i in range(2):
            for j in range(6):
                m.hp[i][j] = float(t.hp[i, j])
        m.hp_mis_rate = float(t.hp_mis_rate)
        m.has_hp = 1 if t.has_hp else 0
        m.strandness_rate = float(t.strandness)
        m.segment_mean = float(t.segment_mean)
        m.mean_ref_per_event = float(t.mean_ref_per_event)
        m.ref_per_event_cv = float(getattr(t, "ref_per_event_cv", 1.0))
        self._check(self._lib.ns_set_model(self._ctx, C.byref(m)))
        self.tables = t

    def set_expression(self, alias_prob, alias_idx, expr_chrom, chrom_has_polya=None):
        """Transcriptome mode: alias table over the expressed transcripts, their reference record indices, polyA flags."""
        a = np.ascontiguousarray(alias_prob, dtype=np.uint32)
        b = np.ascontiguousarray(alias_idx, dtype=np.uint32)
        c = np.ascontiguousarray(expr_chrom, dtype=np.uint32)
        d = np.ascontiguousarray(chrom_has_polya, dtype=np.uint8) if chrom_has_polya is not None else None
        ex = L.NsExpression(_ptr(a), _ptr(b), _ptr(c), len(a), _ptr(d))
        self._check(self._lib.ns_set_expression(self._ctx, C.byref(ex)))

    def configure(self, circular=False, perfect=False, fastq=False, chimeric=False, kmer_bias=0, min_len=50,
                  max_len=None, median_len=0.0, sd_len=0.0, unaligned_scripts=False, metagenome=False,
                  transcriptome=False, uracil=False, polya_scale=0.0, kde2d_sample=0, trx_records=0, emit_exact=False, emit_whole=False):
        if max_len is None or max_len == float("inf"):
            max_len = 0x0fffffff
        flags = (L.NS_FLAG_UNALIGNED_SCRIPTS if unaligned_scripts else 0) | (L.NS_FLAG_URACIL if uracil else 0) | \
            (L.NS_FLAG_EMIT_EXACT if emit_exact else 0) | (L.NS_FLAG_EMIT_WHOLE if emit_whole else 0)
        cfg = L.NsRunConfig(2 if transcriptome else (1 if metagenome else 0), int(circular), int(perfect), int(fastq),
                            int(chimeric), int(kmer_bias or 0), int(min_len), int(min(max_len, 0x0fffffff)),
                            float(median_len or 0.0), float(sd_len or 0.0), flags, int(kde2d_sample), float(polya_scale or 0.0),
                            int(trx_records), 0)
        self._check(self._lib.ns_configure(self._ctx, C.byref(cfg)))
        self.fastq = bool(fastq)

    # ---- simulation workers
    def simulate(self, kind, first_id, n_reads):
        info = L.NsBatchInfo()
        self._check(self._lib.ns_simulate(self._ctx, int(kind), C.c_uint64(int(first_id)), int(n_reads), C.byref(info)))
        self.info = info
        self._kind, self._first = kind, first_id
        return info

    def reemit(self, slots, new_reads, new_pieces, new_ops):
        """Intron retention (intron_retention.py): replaces the piece lists of reads `slots` of the last aligned batch and
        emits those reads again (ns_reemit; with -hp/-k they change length and move to new slots)."""
        slots = np.ascontiguousarray(slots, dtype=np.uint32)
        new_reads = np.ascontiguousarray(new_reads, dtype=L.READ_DTYPE)
        new_pieces = np.ascontiguousarray(new_pieces, dtype=L.PIECE_DTYPE)
        new_ops = np.ascontiguousarray(new_ops, dtype=np.uint32)
        self._check(self._lib.ns_reemit(self._ctx, _ptr(slots), _ptr(new_reads), len(slots), _ptr(new_pieces), len(new_pieces),
                                        _ptr(new_ops), C.c_uint64(len(new_ops))))
        info = L.NsBatchInfo()
        self._check(self._lib.ns_batch_info(self._ctx, C.byref(info)))
        self.info = info

    def fetch_meta(self, want_ops=True):
        """reads / pieces / (ops) of the last batch without the sequence bytes."""
        info = self.info
        reads = np.empty(int(info.n_reads), dtype=L.READ_DTYPE)
        pieces = np.empty(int(info.n_pieces), dtype=L.PIECE_DTYPE)
        ops = np.empty(int(info.n_ops), dtype=np.uint32) if want_ops else None
        self._check(self._lib.ns_fetch(self._ctx, None, None, _ptr(reads), _ptr(pieces), _ptr(ops)))
        return reads, pieces, ops

    def fetch(self, want_ops=False, want_pieces=True):
        info = self.info
        seq = np.empty(int(info.seq_bytes), dtype=np.uint8)
        qual = np.empty(int(info.seq_bytes), dtype=np.uint8) if self.fastq else None
        reads = np.empty(int(info.n_reads), dtype=L.READ_DTYPE)
        pieces = np.empty(int(info.n_pieces), dtype=L.PIECE_DTYPE) if want_pieces else None
        ops = np.empty(int(info.n_ops), dtype=np.uint32) if want_ops else None
        self._check(self._lib.ns_fetch(self._ctx, _ptr(seq), _ptr(qual), _ptr(reads), _ptr(pieces), _ptr(ops)))
        return Batch(info, seq, qual, reads, pieces, ops, self._kind, self._first)

    def fetch_into(self, seq_ptr, qual_ptr, reads_ptr, pieces_ptr=None, ops_ptr=None):
        """Raw-pointer variant for pinned buffers owned by the caller."""
        def vp(x):
            return C.c_void_p(int(x)) if x else None
        self._check(self._lib.ns_fetch(self._ctx, vp(seq_ptr), vp(qual_ptr), vp(reads_ptr), vp(pieces_ptr), vp(ops_ptr)))

    def _compress(self, name, names):
        """ns_<name> over the last batch with its read ``names`` (a records.NameTable or a list of str) -> the size of the
        members it keeps on the device."""
        from .records import _name_blob
        blob, offs = _name_blob(names)
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        if len(offs) != int(self.info.n_reads):
            raise ValueError("%s: %d names for %d reads" % (name, len(offs), int(self.info.n_reads)))
        n = C.c_uint64()
        self._check(getattr(self._lib, "ns_" + name)(self._ctx, blob, _ptr(offs), C.byref(n)))
        return int(n.value)

    def compress_records(self, names):
        """The last batch's FASTA/FASTQ records (read ``names``: a records.NameTable or a list of str) as BGZF members,
        built on the device and kept there (ns_compress_records).  Returns their size in bytes; no end-of-file block."""
        self._z_bytes = self._compress("compress_records", names)
        return self._z_bytes

    def compress_bam(self, names):
        """The last batch's reads as unaligned BAM records (``names`` as for compress_records; at most 254 bytes each)
        as BGZF members, built on the device and kept there (ns_compress_bam); they replace those of the last
        compress_records().  Returns their size in bytes; neither the BAM header nor the end-of-file block."""
        self._z_bytes = self._compress("compress_bam", names)
        return self._z_bytes

    def compress_bam_mapped(self, names):
        """The last aligned batch as mapped BAM records, the true alignment of every read (``names`` as for compress_bam),
        as BGZF members built on the device and kept there (ns_compress_bam_mapped); they replace those of the last
        compress_records() / compress_bam().  After set_lift() the records are lifted onto the haploid reference; in
        transcriptome mode set_splice() must come first, and the records are spliced onto the genome.  Returns
        their size in bytes; neither the BAM header nor the end-of-file block."""
        self._z_bytes = self._compress("compress_bam_mapped", names)
        return self._z_bytes

    def compress_bam_transcript(self, names):
        """The last aligned batch of a transcriptome run as mapped BAM records against the transcripts, the true alignment of
        every read (``names`` as for compress_bam), as BGZF members built on the device and kept there
        (ns_compress_bam_transcript); they replace those of the last compress_records() / compress_bam().  With intron
        retention set_splice() must come first: the reads that retain an intron are composed with it.  Returns their size
        in bytes; neither the BAM header nor the end-of-file block."""
        self._z_bytes = self._compress("compress_bam_transcript", names)
        return self._z_bytes

    def fetch_compressed(self, out=None):
        """The members of the last compress_records(), compress_bam(), compress_bam_mapped() or compress_bam_transcript() -> uint8 array (into ``out`` when given: a
        uint8 array, pinned memory recommended, at least that large)."""
        if out is None:
            out = np.empty(self._z_bytes, dtype=np.uint8)
        self._check(self._lib.ns_fetch_compressed(self._ctx, _ptr(out), C.c_uint64(len(out))))
        return out[:self._z_bytes]

    def compress_error_profile(self, names):
        """The last aligned batch's error-profile rows (records.format_error_profile's bytes, no header line) as BGZF
        members, formatted and compressed on the device and kept there (ns_compress_error_profile).  ``names`` as for
        compress_records.  Returns their size in bytes (0: no error events); no end-of-file block."""
        self._ep_bytes = self._compress("compress_error_profile", names)
        return self._ep_bytes

    def fetch_compressed_error_profile(self, out=None):
        """The members of the last compress_error_profile() -> uint8 array (into ``out`` when given, as for
        fetch_compressed)."""
        if out is None:
            out = np.empty(self._ep_bytes, dtype=np.uint8)
        self._check(self._lib.ns_fetch_compressed_error_profile(self._ctx, _ptr(out), C.c_uint64(len(out))))
        return out[:self._ep_bytes]

    def device_buffers(self):
        ps = [C.c_void_p() for _ in range(5)]
        self._check(self._lib.ns_device_buffers(self._ctx, *[C.byref(p) for p in ps]))
        return dict(zip(("seq", "qual", "reads", "pieces", "ops"), (p.value for p in ps)))

    def op_stats(self):
        out = np.zeros(L.NS_STATS_WORDS, dtype=np.uint64)
        self._check(self._lib.ns_op_stats(self._ctx, _ptr(out)))
        ev, run = L.NS_STATS_EV_CAP + 1, L.NS_STATS_RUN_CAP + 1
        o = out.astype(np.int64)
        d = {"n_segments": int(o[0]), "ref_bases": int(o[1]), "segment_out_bases": int(o[2]), "ht_bases": int(o[3]),
             "n_gaps": int(o[4]), "gap_bases": int(o[5]), "n_events": int(o[6]),
             "events": {"mis": int(o[8]), "ins": int(o[9]), "del": int(o[10])},
             "event_bases": {"mis": int(o[11]), "ins": int(o[12]), "del": int(o[13])},
             "ev_len": {k: o[16 + i * ev: 16 + (i + 1) * ev].copy() for i, k in enumerate(("mis", "ins", "del"))},
             "match_run": o[16 + 3 * ev: 16 + 3 * ev + run].copy(),
             "first_match": o[16 + 3 * ev + run: 16 + 3 * ev + 2 * run].copy(),
             # error events per aligned segment (exact counts; the last slot collects >= NS_STATS_EPR_CAP)
             "events_per_segment": o[L.NS_STATS_EPR_OFF: L.NS_STATS_EPR_OFF + L.NS_STATS_EPR_CAP + 1].copy(),
             # 1-base mismatches: reference base x read base, inserted bases, read composition (A C G T order)
             "mis_sub": o[L.NS_STATS_SUB_OFF: L.NS_STATS_SUB_OFF + 16].reshape(4, 4).copy(),
             "ins_base": o[L.NS_STATS_INS_OFF: L.NS_STATS_INS_OFF + 4].copy(),
             "base_comp": o[L.NS_STATS_COMP_OFF: L.NS_STATS_COMP_OFF + 4].copy()}
        return d
