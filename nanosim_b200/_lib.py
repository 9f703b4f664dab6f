"""ctypes binding of libnanosim_b200.so (include/nanosim_b200.h).  No CPU fallback: if the shared library is
missing, importing this module's ``lib()`` raises."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NANOSIM_B200_LIB") or os.path.join(_HERE, "libnanosim_b200.so")     # env: A/B builds of the kernels

NS_MAX_SEGMENTS = 16
NS_N_ERR_STATES = 7
NS_N_QUAL_STATES = 5
NS_QUAL_SLOTS = 94
NS_KIND_ALIGNED, NS_KIND_UNALIGNED = 0, 1
NS_PIECE_SEGMENT, NS_PIECE_GAP, NS_PIECE_UNALIGNED = 0, 1, 2
NS_PIECE_REF_REV, NS_PIECE_CONT, NS_PIECE_RETAINED, NS_PIECE_GENOME, NS_PIECE_KIND_MASK = 0x80000000, 0x40000000, 0x20000000, 0x10000000, 0xffff
NS_OP_COPY, NS_OP_MIS, NS_OP_INS, NS_OP_DEL, NS_OP_HT, NS_OP_LIT = 0, 1, 2, 3, 4, 5
NS_STATS_EV_CAP, NS_STATS_RUN_CAP = 64, 512
NS_STATS_EPR_CAP = 131072
NS_STATS_EPR_OFF = 8 + 8 + 3 * (NS_STATS_EV_CAP + 1) + 2 * (NS_STATS_RUN_CAP + 1)
NS_STATS_SUB_OFF = NS_STATS_EPR_OFF + NS_STATS_EPR_CAP + 1
NS_STATS_INS_OFF = NS_STATS_SUB_OFF + 16
NS_STATS_COMP_OFF = NS_STATS_INS_OFF + 4
NS_STATS_WORDS = NS_STATS_COMP_OFF + 4

EXPORTS = ["ns_create", "ns_destroy", "ns_last_error", "ns_clone", "ns_set_abundance", "ns_set_expression", "ns_set_reference", "ns_set_model", "ns_configure",
           "ns_simulate", "ns_fetch", "ns_reemit", "ns_batch_info", "ns_device_buffers", "ns_op_stats", "ns_format_records", "ns_format_error_profile", "ns_format_names", "ns_transfer_info", "ns_write_records", "ns_write_error_profile", "ns_read_fasta", "ns_nccl_unique_id", "ns_bcast_nccl", "ns_get_reference", "ns_unpack_bases",
           "ns_compress_records", "ns_fetch_compressed", "ns_compress_error_profile", "ns_fetch_compressed_error_profile", "ns_compress_bam", "ns_apply_variants",
           "ns_compress_bam_mapped", "ns_set_lift", "ns_set_splice", "ns_set_aln_tags", "ns_compress_bam_transcript"]


class NsReference(C.Structure):
    _fields_ = [("bases", C.c_void_p), ("n_bases", C.c_uint64), ("chrom_off", C.c_void_p), ("n_chrom", C.c_uint32),
                ("n_species", C.c_uint32), ("chrom_species", C.c_void_p), ("chrom_circular", C.c_void_p)]


class NsVariants(C.Structure):
    _fields_ = [("n_hap", C.c_uint32), ("hap_chrom", C.c_void_p), ("var_off", C.c_void_p), ("n_var", C.c_uint64),
                ("var_pos", C.c_void_p), ("var_ref_len", C.c_void_p), ("alt_off", C.c_void_p), ("alt_len", C.c_void_p),
                ("alt", C.c_void_p), ("alt_bytes", C.c_uint64), ("peak_bytes", C.POINTER(C.c_uint64)), ("alt_kind", C.c_void_p)]


NS_SPLICE_NO_GENOME = 0xffffffff


class NsSplice(C.Structure):
    _fields_ = [("n_trx", C.c_uint32), ("exon_off", C.c_void_p), ("exon_chrom", C.c_void_p), ("exon_start", C.c_void_p),
                ("exon_len", C.c_void_p), ("minus", C.c_void_p), ("n_genome", C.c_uint32), ("genome_len", C.c_void_p),
                ("genome_first", C.c_uint32), ("peak_bytes", C.POINTER(C.c_uint64))]


class NsAlnTags(C.Structure):
    _fields_ = [("n_ref", C.c_uint32), ("ref_names", C.c_void_p), ("ref_name_off", C.c_void_p), ("n_var", C.c_uint64),
                ("ref_paired", C.c_void_p), ("ref_paired_bytes", C.c_uint64), ("peak_bytes", C.POINTER(C.c_uint64))]


class NsKde(C.Structure):
    _fields_ = [("data", C.c_void_p), ("n", C.c_uint32), ("bandwidth", C.c_float)]


class NsModel(C.Structure):
    _fields_ = [
        ("kde_aligned", NsKde), ("kde_ht", NsKde), ("kde_ht_ratio", NsKde), ("kde_unaligned", NsKde), ("kde_gap", NsKde),
        ("kde2d_x", C.c_void_p), ("kde2d_y", C.c_void_p), ("n_kde2d", C.c_uint32), ("kde2d_bandwidth", C.c_float),
        ("alias_prob", C.c_void_p), ("alias_idx", C.c_void_p), ("alias_desc", C.c_void_p),
        ("n_tables", C.c_uint32), ("alias_len", C.c_uint32),
        ("match_bin_lo", C.c_void_p), ("match_bin_hi", C.c_void_p),
        ("n_match_bins", C.c_uint32), ("has_qual", C.c_uint32),
        ("trans", (C.c_uint32 * 3) * NS_N_ERR_STATES),
        ("qual_cdf", (C.c_uint32 * NS_QUAL_SLOTS) * NS_N_QUAL_STATES),
        ("hp", (C.c_double * 6) * 2), ("hp_mis_rate", C.c_double),
        ("has_hp", C.c_uint32), ("strandness_rate", C.c_float), ("segment_mean", C.c_float),
        ("mean_ref_per_event", C.c_float),
        ("ref_per_event_cv", C.c_float),
    ]


class NsRunConfig(C.Structure):
    _fields_ = [("mode", C.c_uint32), ("circular", C.c_uint32), ("perfect", C.c_uint32), ("fastq", C.c_uint32),
                ("chimeric", C.c_uint32), ("kmer_bias", C.c_uint32), ("min_len", C.c_uint32), ("max_len", C.c_uint32),
                ("median_len", C.c_double), ("sd_len", C.c_double), ("flags", C.c_uint32), ("kde2d_sample", C.c_uint32),
                ("polya_scale", C.c_double), ("trx_records", C.c_uint32), ("reserved", C.c_uint32)]


class NsExpression(C.Structure):
    _fields_ = [("alias_prob", C.c_void_p), ("alias_idx", C.c_void_p), ("expr_chrom", C.c_void_p),
                ("n_expressed", C.c_uint32), ("chrom_has_polya", C.c_void_p)]


NS_FLAG_UNALIGNED_SCRIPTS = 1
NS_FLAG_URACIL = 2
NS_FLAG_EMIT_EXACT = 4
NS_FLAG_EMIT_WHOLE = 8


class NsReadMeta(C.Structure):
    _fields_ = [("seq_off", C.c_uint64), ("seq_len", C.c_uint32), ("head", C.c_uint32), ("tail", C.c_uint32),
                ("piece_first", C.c_uint32), ("n_pieces", C.c_uint16), ("reversed", C.c_uint8), ("flags", C.c_uint8),
                ("attempts", C.c_uint32)]


class NsPieceMeta(C.Structure):
    _fields_ = [("op_off", C.c_uint64), ("n_ops", C.c_uint32), ("kind", C.c_uint32), ("chrom", C.c_uint32),
                ("pos", C.c_uint32), ("ref_len", C.c_uint32), ("out_len", C.c_uint32), ("out_rel", C.c_uint32),
                ("l_new", C.c_uint32), ("ref_req", C.c_uint32), ("read_slot", C.c_uint32),
                ("ev_off", C.c_uint64), ("ev_n_ops", C.c_uint32), ("polya_len", C.c_uint32)]


class NsBatchInfo(C.Structure):
    _fields_ = [("seq_bytes", C.c_uint64), ("n_ops", C.c_uint64), ("total_bases", C.c_uint64),
                ("n_reads", C.c_uint32), ("n_pieces", C.c_uint32), ("n_launches", C.c_uint32),
                ("ms_setup", C.c_float), ("ms_plan", C.c_float), ("ms_scan", C.c_float), ("ms_script", C.c_float),
                ("ms_emit", C.c_float), ("ms_total", C.c_float), ("t_begin_ms", C.c_double), ("t_end_ms", C.c_double),
                ("raw_ev_off", C.c_uint64)]


# numpy views of the two record types
import numpy as np  # noqa: E402

READ_DTYPE = np.dtype([("seq_off", "<u8"), ("seq_len", "<u4"), ("head", "<u4"), ("tail", "<u4"),
                       ("piece_first", "<u4"), ("n_pieces", "<u2"), ("reversed", "u1"), ("flags", "u1"),
                       ("attempts", "<u4")], align=True)
PIECE_DTYPE = np.dtype([("op_off", "<u8"), ("n_ops", "<u4"), ("kind", "<u4"), ("chrom", "<u4"), ("pos", "<u4"),
                        ("ref_len", "<u4"), ("out_len", "<u4"), ("out_rel", "<u4"), ("l_new", "<u4"),
                        ("ref_req", "<u4"), ("read_slot", "<u4"), ("ev_off", "<u8"), ("ev_n_ops", "<u4"),
                        ("polya_len", "<u4")], align=True)
assert READ_DTYPE.itemsize == C.sizeof(NsReadMeta) == 32
assert PIECE_DTYPE.itemsize == C.sizeof(NsPieceMeta) == 64

_lib = None


def lib():
    """Loads the CUDA library.  Fails loudly when it has not been built (python __graft_entry__.py build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("nanosim_b200: %s is missing -- build it with `python -c 'import __graft_entry__ as g; "
                           "g.build()'`; there is no CPU fallback" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    P = C.c_void_p
    L.ns_create.argtypes = [C.c_int, C.c_uint64, C.POINTER(P)]
    L.ns_create.restype = C.c_int
    L.ns_clone.argtypes = [P, C.POINTER(P)]
    L.ns_clone.restype = C.c_int
    L.ns_destroy.argtypes = [P]
    L.ns_destroy.restype = C.c_int
    L.ns_last_error.argtypes = [P]
    L.ns_last_error.restype = C.c_char_p
    L.ns_set_reference.argtypes = [P, C.POINTER(NsReference)]
    L.ns_set_reference.restype = C.c_int
    L.ns_apply_variants.argtypes = [P, C.POINTER(NsVariants)]
    L.ns_apply_variants.restype = C.c_int
    L.ns_set_lift.argtypes = [P, C.POINTER(NsVariants)]
    L.ns_set_lift.restype = C.c_int
    L.ns_set_splice.argtypes = [P, C.POINTER(NsSplice)]
    L.ns_set_splice.restype = C.c_int
    L.ns_set_aln_tags.argtypes = [P, C.POINTER(NsAlnTags)]
    L.ns_set_aln_tags.restype = C.c_int
    L.ns_set_model.argtypes = [P, C.POINTER(NsModel)]
    L.ns_set_model.restype = C.c_int
    L.ns_set_abundance.argtypes = [P, P, P, C.c_uint32]
    L.ns_set_abundance.restype = C.c_int
    L.ns_set_expression.argtypes = [P, C.POINTER(NsExpression)]
    L.ns_set_expression.restype = C.c_int
    L.ns_configure.argtypes = [P, C.POINTER(NsRunConfig)]
    L.ns_configure.restype = C.c_int
    L.ns_simulate.argtypes = [P, C.c_int, C.c_uint64, C.c_uint32, C.POINTER(NsBatchInfo)]
    L.ns_simulate.restype = C.c_int
    L.ns_fetch.argtypes = [P, P, P, P, P, P]
    L.ns_fetch.restype = C.c_int
    L.ns_device_buffers.argtypes = [P, C.POINTER(P), C.POINTER(P), C.POINTER(P), C.POINTER(P), C.POINTER(P)]
    L.ns_device_buffers.restype = C.c_int
    L.ns_op_stats.argtypes = [P, P]
    L.ns_op_stats.restype = C.c_int
    L.ns_format_records.argtypes = [P, P, P, C.c_uint32, P, P, C.c_int, P, C.c_uint64, C.c_int]
    L.ns_format_records.restype = C.c_int64
    L.ns_format_error_profile.argtypes = [P, P, P, P, C.c_uint32, P, P, P, P, C.c_uint64, C.c_uint64, P, C.c_uint64, C.c_int]
    L.ns_format_error_profile.restype = C.c_int64
    L.ns_format_names.argtypes = [P, P, C.c_uint32, C.c_int, C.c_uint32, C.c_uint64, P, P, P, C.c_uint64, P]
    L.ns_format_names.restype = C.c_int64
    L.ns_get_reference.argtypes = [P, P, C.c_uint64]
    L.ns_get_reference.restype = C.c_int
    L.ns_nccl_unique_id.argtypes = [P]
    L.ns_nccl_unique_id.restype = C.c_int
    L.ns_bcast_nccl.argtypes = [P, P, C.c_int, C.c_int, C.c_int]
    L.ns_bcast_nccl.restype = C.c_int
    L.ns_read_fasta.argtypes = [C.c_char_p, P, C.c_uint64, P, P, C.c_uint64, P, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64),
                                C.POINTER(C.c_uint64), C.c_int]
    L.ns_read_fasta.restype = C.c_int64
    L.ns_write_records.argtypes = [C.c_int, C.c_uint64, P, P, P, C.c_uint32, P, P, C.c_int, C.c_int]
    L.ns_write_records.restype = C.c_int64
    L.ns_write_error_profile.argtypes = [C.c_int, C.c_uint64, P, P, P, P, C.c_uint32, P, P, P, P, C.c_uint64, C.c_uint64, C.c_int]
    L.ns_write_error_profile.restype = C.c_int64
    L.ns_transfer_info.argtypes = [P, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    L.ns_transfer_info.restype = C.c_int
    L.ns_unpack_bases.argtypes = [P, P, C.c_uint64, C.c_int, C.c_int]
    L.ns_unpack_bases.restype = C.c_int
    L.ns_reemit.argtypes = [P, P, P, C.c_uint32, P, C.c_uint32, P, C.c_uint64]
    L.ns_reemit.restype = C.c_int
    L.ns_batch_info.argtypes = [P, C.POINTER(NsBatchInfo)]
    L.ns_batch_info.restype = C.c_int
    L.ns_compress_records.argtypes = [P, P, P, C.POINTER(C.c_uint64)]
    L.ns_compress_records.restype = C.c_int
    L.ns_compress_bam.argtypes = [P, P, P, C.POINTER(C.c_uint64)]
    L.ns_compress_bam.restype = C.c_int
    L.ns_compress_bam_mapped.argtypes = [P, P, P, C.POINTER(C.c_uint64)]
    L.ns_compress_bam_mapped.restype = C.c_int
    L.ns_compress_bam_transcript.argtypes = [P, P, P, C.POINTER(C.c_uint64)]
    L.ns_compress_bam_transcript.restype = C.c_int
    L.ns_fetch_compressed.argtypes = [P, P, C.c_uint64]
    L.ns_fetch_compressed.restype = C.c_int
    L.ns_compress_error_profile.argtypes = [P, P, P, C.POINTER(C.c_uint64)]
    L.ns_compress_error_profile.restype = C.c_int
    L.ns_fetch_compressed_error_profile.argtypes = [P, P, C.c_uint64]
    L.ns_fetch_compressed_error_profile.restype = C.c_int
    _lib = L
    return L
