/*
 * nanosim_b200 -- C ABI of the H100-native (sm_90a) per-read simulation path of NanoSim.
 *
 * The reference (bcgsc/NanoSim, pure Python) has no FFI: the seam this library replaces is the Python call
 *
 *     simulation(mode, out, dna_type, per, kmer_bias, basecaller, max_l, min_l, num_threads, fastq,
 *                median_l, sd_l, model_ir, uracil, polya, chimeric)            src/simulator.py:1571-1572
 *       -> simulation_aligned_genome(dna_type, min_l, max_l, median_l, sd_l, out_reads, out_error,
 *                                    kmer_bias, fastq, num_simulate, per, chimeric)      :1266-1267
 *       -> simulation_unaligned(dna_type, min_l, max_l, median_l, sd_l, out_reads, fastq,
 *                               num_simulate, uracil)                                    :1482
 *
 * whose inputs travel as module globals filled by read_profile() (:244-591).  Each entry point below names the
 * reference interface it stands in for.  Plain pointers and sizes only; all functions return 0 on success and a
 * negative NS_E* code otherwise, with a human-readable message available from ns_last_error().
 * Pointers passed to ns_set_* may be host or device pointers (unified addressing); the library copies what it
 * needs into its own HBM allocations before returning, so the caller keeps ownership of its buffers.
 */
#ifndef NANOSIM_B200_H
#define NANOSIM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NS_OK 0
#define NS_EINVAL (-1)
#define NS_ECUDA (-2)
#define NS_ESTATE (-3)
#define NS_ENOMEM (-4)

#define NS_MAX_SEGMENTS 16        /* segments per chimeric read (reference: unbounded Geometric, :1277) */
#define NS_N_ERR_STATES 7         /* start mis ins del mis0 ins0 del0        (:486-495, :1913-1914)      */
#define NS_N_QUAL_STATES 5        /* mis ins match ht unmapped               (:580-591)                  */
#define NS_QUAL_SLOTS 94          /* cdf over q = 0..93                                                   */

typedef struct NsContext NsContext;

/* seq_dict / seq_len / genome_len / dict_dna_type globals (simulator.py:279-356): all chromosomes concatenated,
 * one ASCII byte per base (case and IUPAC codes kept; case_convert :743-755 is applied per read on the device). */
typedef struct {
    const uint8_t* bases;
    uint64_t n_bases;
    const uint64_t* chrom_off;   /* n_chrom + 1 offsets into bases, file order */
    uint32_t n_chrom;
    /* metagenome mode (seq_dict[species][chrom], dict_dna_type, :284-339); NULL / 0 in genome mode.  The chromosomes of
     * one species must be contiguous, species in genome-list order. */
    uint32_t n_species;
    const uint32_t* chrom_species;   /* species index of every chromosome */
    const uint8_t* chrom_circular;   /* 1 = "circular" (the default for local files, :323), 0 = "linear" */
} NsReference;

/* transcriptome mode: dict_exp / ecdf_length_list / ecdf_weight_list (make_cdf :69-97) and trx_with_polya (:455-463).
 * The n_expressed transcripts present in both the expression profile and the reference, as a Walker alias table over
 * their TPM shares; expr_chrom[i] = index of transcript i among the reference's records. */
typedef struct {
    const uint32_t* alias_prob;
    const uint32_t* alias_idx;
    const uint32_t* expr_chrom;
    uint32_t n_expressed;
    const uint8_t* chrom_has_polya;  /* per reference record; NULL = no --polya list */
} NsExpression;

/* One joblib KernelDensity pickle (kde_aligned, kde_ht, ... :545-577): gaussian kernel, training samples + bandwidth.
 * A draw is data[floor(u*n)] + N(0, bandwidth)  (sklearn KernelDensity.sample; call site :235). */
typedef struct {
    const float* data;
    uint32_t n;
    float bandwidth;
} NsKde;

/* match_ht_list, match_markov_model, error_par, trans_error_pr, lognorm_base_qual, pw_hp_len/lr_hp_len/hp_mis_rate,
 * strandness_rate, segment_mean (:247-251, :473-591) as flat tables.  Every discrete distribution is a Walker alias
 * table over 0..n-1 (built exactly on the host, nanosim_b200/model.py): table t occupies
 * alias_prob/alias_idx[alias_desc[2t] .. +alias_desc[2t+1]).  Table ids: 0 first match, 1 mismatch length,
 * 2 insertion length, 3 deletion length, 4+b next-match length given previous-match bin b (last slot = "ECDF miss"). */
typedef struct {
    NsKde kde_aligned;        /* _aligned_region.pkl (or _aligned_reads.pkl with perfect=1) */
    NsKde kde_ht;             /* _ht_length.pkl, log10(x+1) domain */
    NsKde kde_ht_ratio;       /* _ht_ratio.pkl */
    NsKde kde_unaligned;      /* _unaligned_length.pkl (n = 0 if absent) */
    NsKde kde_gap;            /* _gap_length.pkl, log10(x+1) domain (n = 0 if absent) */
    /* _aligned_region_2d.pkl (transcriptome): training rows (transcript length, aligned length) sorted by transcript
     * length; n_kde2d = 0 if absent.  select_nearest_kde2d (:108-111) is sampled exactly from them, see plan_kernel.cuh */
    const float* kde2d_x;
    const float* kde2d_y;
    uint32_t n_kde2d;
    float kde2d_bandwidth;
    const uint32_t* alias_prob;
    const uint32_t* alias_idx;
    const uint32_t* alias_desc;
    uint32_t n_tables;
    uint32_t alias_len;
    const uint32_t* match_bin_lo;   /* previous-match-length bins [lo, hi) of _match_markov_model's header */
    const uint32_t* match_bin_hi;
    uint32_t n_match_bins;
    uint32_t has_qual;
    uint32_t trans[NS_N_ERR_STATES][3];                 /* r<t0: mis; r<t1: ins; r>=t2: del; else previous error */
    uint32_t qual_cdf[NS_N_QUAL_STATES][NS_QUAL_SLOTS]; /* q = first slot with r < cdf[q] (32-bit fixed point)   */
    double hp[2][6];          /* rows AT, CG: const, alpha1, beta1, breakpoint1, intercept, slope */
    double hp_mis_rate;
    uint32_t has_hp;
    float strandness_rate;
    float segment_mean;
    float mean_ref_per_event; /* sizing hint for op slots: reference bases per error event ... */
    float ref_per_event_cv;   /* ... and their coefficient of variation (slots hold mean + 6 sigma events) */
} NsModel;

/* The scalar arguments of simulation()/simulation_aligned_genome()/simulation_unaligned(). */
typedef struct {
    uint32_t mode;            /* 0 genome, 1 metagenome, 2 transcriptome */
    uint32_t circular;        /* dna_type == "circular" (single chromosome) */
    uint32_t perfect;
    uint32_t fastq;
    uint32_t chimeric;
    uint32_t kmer_bias;       /* 0 = off (-k) */
    uint32_t min_len;
    uint32_t max_len;         /* caller passes min(max_len, max_chrom) as simulator.py:2318 does */
    double median_len;        /* 0 = off (-med / -sd) */
    double sd_len;
    uint32_t flags;           /* NS_FLAG_* */
    uint32_t kde2d_sample;    /* transcriptome: size N of the 2-D KDE sample select_nearest_kde2d searches (:1072, :1090):
                                 the reference uses the number of aligned reads of the worker */
    double polya_scale;       /* transcriptome --polya: scale of expon(loc=2, scale) (:1046-1053); 0 = no polyA tails */
    uint32_t trx_records;     /* transcriptome with intron retention: the first trx_records reference records are the
                                 transcripts, the rest the genome ns_reemit reads introns from; 0 = every record is a transcript */
    uint32_t reserved;
} NsRunConfig;

/* Unaligned reads normally take the warp-per-read fast path, which writes bases directly and keeps no edit scripts.
 * With this flag they go through the same plan/script/emit pipeline as aligned reads (identical lengths, strands and
 * positions; used by the tests to check the fast path against re-applied edit scripts). */
#define NS_FLAG_UNALIGNED_SCRIPTS 1u
#define NS_FLAG_URACIL 2u            /* --uracil: T -> U in the emitted reads (:1247-1248) */
/* The emit kernel reads plain-ACGT stretches of the reference from a 2-bit copy (fast route) and everything else byte by
 * byte (exact route: IUPAC codes, circular wrap-around, minus-strand genome pieces).  Both give the same bytes; this flag
 * sends every piece down the exact route (tests compare the two). */
#define NS_FLAG_EMIT_EXACT 4u
/* Pieces longer than 16 kb are emitted as several work items (each resuming the script walk from a checkpoint), so that the
 * longest read of a batch does not keep one warp busy long after the rest has finished; long unaligned reads are walked by a
 * whole thread block instead of one warp for the same reason.  This flag emits every piece as one item and walks every
 * unaligned read with one warp (tests compare the two: same bytes). */
#define NS_FLAG_EMIT_WHOLE 8u

#define NS_KIND_ALIGNED 0
#define NS_KIND_UNALIGNED 1

#define NS_PIECE_SEGMENT 0    /* aligned segment (error_list + mutate_read)                  */
#define NS_PIECE_GAP 1        /* chimeric gap (simulation_gap :1552-1568)                    */
#define NS_PIECE_UNALIGNED 2  /* unaligned read body (simulation_unaligned :1482-1549)       */
/* NsPieceMeta.kind: the low 16 bits hold the kind above; intron-retention reads (ns_reemit) use three flags */
#define NS_PIECE_KIND(k) ((k) & 0xffffu)
#define NS_PIECE_REF_REV 0x80000000u  /* the piece reads its reference backwards and complemented (minus-strand transcript) */
#define NS_PIECE_CONT 0x40000000u     /* continues the previous segment of the read: error positions keep counting (:2006) */
#define NS_PIECE_RETAINED 0x20000000u /* the piece lies in a retained intron (read name, :1189-1192) */
#define NS_PIECE_GENOME 0x10000000u   /* every piece of a read laid out on the genome; ref_req = its transcript's record */

/* What the reference encodes in the read name and FASTQ record (:1390-1402, :1437-1443). */
typedef struct {
    uint64_t seq_off;         /* first base of this read in the seq / qual buffers (16-byte aligned slot) */
    uint32_t seq_len;
    uint32_t head;
    uint32_t tail;
    uint32_t piece_first;     /* index of the read's first piece */
    uint16_t n_pieces;        /* 2*n_segments-1 for aligned reads, 1 for unaligned */
    uint8_t reversed;         /* 1 = "_R" */
    uint8_t flags;            /* bit0 = op slot overflow (read is invalid), bit1 = chimeric */
    uint32_t attempts;        /* rejection-loop iterations used (:1367, :1429) */
} NsReadMeta;

typedef struct {
    uint64_t op_off;          /* first op of the piece in the op buffer */
    uint32_t n_ops;
    uint32_t kind;            /* NS_PIECE_* */
    uint32_t chrom;           /* index into NsReference.chrom_off */
    uint32_t pos;             /* 0-based start on that chromosome ("{chrom}_{pos}") */
    uint32_t ref_len;         /* middle_ref: reference bases the piece spans */
    uint32_t out_len;         /* bases this piece contributes (incl. head/tail carried by the edge pieces) */
    uint32_t out_rel;         /* offset of the piece inside the forward-strand read */
    uint32_t l_new;           /* error_list's nominal length (== out_len - head/tail unless an ins/ins collision) */
    uint32_t ref_req;         /* length drawn from the KDE before error_list extended it (m_ref) */
    uint32_t read_slot;       /* index of the owning read inside the batch */
    uint64_t ev_off;          /* the piece's ERROR-EVENT script (what mutate_read logs, :2006-2008): equal to op_off/n_ops */
    uint32_t ev_n_ops;        /* unless -hp/-k rewrote the emitted script (mutate_homo); then this is the script before it */
    uint32_t polya_len;       /* transcriptome: length of the simulated polyA tail (0 otherwise) */
} NsPieceMeta;

/* Edit script element: (type << 28) | length.  The op list of a piece, applied left to right to the reference
 * segment, is what mutate_read (:1919-2015) computes; it is also the content of <out>_aligned_error_profile. */
#define NS_OP_COPY 0u    /* copy n reference bases          (match quality)     */
#define NS_OP_MIS 1u     /* n substituted bases             (mis quality)       */
#define NS_OP_INS 2u     /* n random inserted bases         (ins quality)       */
#define NS_OP_DEL 3u     /* skip n reference bases                              */
#define NS_OP_HT 4u      /* n random head/tail bases        (ht quality)        */
#define NS_OP_LIT 5u     /* n copies of a literal base: bits [27:26] base (A C T G = 0 1 2 3), [25:24] quality state
                            (0 mis, 1 ins, 2 match, 3 ht), [23:0] n.  Scripts rewritten by the homopolymer pass; polyA tails. */
#define NS_OP_TYPE(op) ((op) >> 28)
#define NS_OP_LEN(op) (NS_OP_TYPE(op) == NS_OP_LIT ? ((op) & 0x00ffffffu) : ((op) & 0x0fffffffu))

typedef struct {
    uint64_t seq_bytes;       /* size of the seq (and qual) buffer for this batch */
    uint64_t n_ops;
    uint64_t total_bases;     /* sum of seq_len */
    uint32_t n_reads;
    uint32_t n_pieces;
    uint32_t n_launches;      /* launches for this batch (and ns_reemit on it): one per kernel of this library, one per CUB
                               * scan, one per CUB sort; memsets and copies are not counted */
    /* CUDA-event durations on the library's stream: set-up (segment counts, buffer growth), plan pass 1 (rejection
     * loops + counts), scans + host round trip of the totals, plan pass 2 (edit scripts), emit, and the whole batch */
    float ms_setup, ms_plan, ms_scan, ms_script, ms_emit, ms_total;
    /* begin / end of the batch on the device timeline, in ms since the first ns_create() of this process on this device;
     * comparable across contexts (streams) of one device, so overlapped pipelines can be timed on the device */
    double t_begin_ms, t_end_ms;
    /* -hp/-k with intron retention (kmer_bias != 0, trx_records != 0): the op buffer also holds a verbatim copy of the event
     * scripts as the plan wrote them, before the homopolymer pass filtered them; a segment's unfiltered script starts at
     * raw_ev_off + ev_off (ev_n_ops ops).  0 = no copy.  ns_reemit leaves it as it is. */
    uint64_t raw_ev_off;
} NsBatchInfo;

/* --- lifetime --------------------------------------------------------------------------------------------- */
/* replaces: process start + random.seed/np.random.seed (:2236-2238).  The stream of read `i` depends only on
 * (seed, kind, i), so output is invariant to batch size and GPU count. */
int ns_create(int device, uint64_t seed, NsContext** out);
int ns_destroy(NsContext* ctx);
const char* ns_last_error(const NsContext* ctx);
/* A second context on the same device that SHARES the parent's reference and model tables in HBM (no copy) but has its
 * own stream and batch buffers: two or more contexts driven from different host threads overlap one batch's kernels
 * with another batch's device->host copy.  The parent must outlive its clones. */
int ns_clone(NsContext* parent, NsContext** out);

/* --- read_profile() (:244-591): reference + model tables into HBM, once ------------------------------------- */
int ns_set_reference(NsContext* ctx, const NsReference* ref);
int ns_set_model(NsContext* ctx, const NsModel* model);
int ns_configure(NsContext* ctx, const NsRunConfig* cfg);
/* metagenome: dict_abun / dict_abun_inflated of the current sample (main() :2497-2514), one value per species in
 * genome-list order; resets the running per-species base counts that assign_species (:758-811) keeps per worker. */
int ns_set_abundance(NsContext* ctx, const double* abun, const double* abun_inflated, uint32_t n_species);
/* transcriptome: expression profile + polyA list (read_profile :383-463). */
int ns_set_expression(NsContext* ctx, const NsExpression* expr);

/* --- simulation_aligned_genome / simulation_unaligned worker bodies (:1266-1454, :1482-1549) ---------------- */
/* Simulates reads [first_read_id, first_read_id + n_reads) of `kind`; results stay in HBM until the next call. */
int ns_simulate(NsContext* ctx, int kind, uint64_t first_read_id, uint32_t n_reads, NsBatchInfo* info);

/* Device->host copy of the last batch into caller buffers (pinned memory recommended).  qual / pieces / ops may be
 * NULL.  seq and qual need info.seq_bytes bytes, reads n_reads entries, pieces n_pieces, ops n_ops uint32.
 * seq arrives as ASCII as always; on the wire large batches travel as 2 bits per base (packed by a kernel, expanded by
 * host threads inside this call: NANOSIM_B200_UNPACK_THREADS; default 16 when the host has >= 48 cores per GPU process
 * (cores / LOCAL_WORLD_SIZE), else 0 = plain ASCII copies). */
int ns_fetch(NsContext* ctx, uint8_t* seq, uint8_t* qual, NsReadMeta* reads, NsPieceMeta* pieces, uint32_t* ops);

/* Multi-GPU init (one process per GPU): the reference's forked workers inherit seq_dict from the parent
 * (simulator.py:1588-1622); here rank `root` reads the FASTA, calls ns_set_reference, and ONE NCCL broadcast hands bases,
 * chromosome offsets and the metagenome tables to the other ranks' HBM, where each rank builds its own 2-bit copy.  Rank
 * `root` obtains a communicator id with ns_nccl_unique_id() and passes it to the others by any host channel (the driver
 * uses torch.distributed's store); every rank then calls ns_bcast_nccl() (collective).  libnccl.so.2 is loaded at run time. */
/* Host copy of the resident reference bytes (ranks that received them by broadcast format the error profile's reference
 * column from it). */
int ns_get_reference(NsContext* ctx, uint8_t* bases, uint64_t cap);
#define NS_NCCL_ID_BYTES 128
int ns_nccl_unique_id(uint8_t* id /* NS_NCCL_ID_BYTES */);
int ns_bcast_nccl(NsContext* ctx, const uint8_t* id, int rank, int world, int root);

/* read_profile's reference reader (simulator.py:341-349, readfq :709-740) for FASTA and FASTQ files: sequence bytes of all
 * records back to back exactly as in the file (case and IUPAC codes kept, line ends dropped), record offsets, header lines.
 * Multi-threaded over an mmap of the file.  Two calls: with bases == NULL only the three counts are set (the caller sizes
 * its buffers: n_bases bytes, n_records + 1 offsets, header_bytes bytes, n_records header offsets), then the fill.  Returns
 * the number of bases or a negative NS_E* code. */
int64_t ns_read_fasta(const char* path, uint8_t* bases, uint64_t bases_cap, uint64_t* rec_off, char* headers, uint64_t headers_cap,
                      uint64_t* header_off, uint32_t* n_records, uint64_t* n_bases, uint64_t* header_bytes, int n_threads);

/* How ns_fetch moves the bases of large batches: *packed_bases = 1 when they cross PCIe as 2 bits each (every byte of the
 * reference is an IUPAC nucleotide code, so reads hold A C G T/U only, and the host has threads to expand them),
 * *unpack_threads = host threads ns_fetch uses for the expansion.  (No reference counterpart: its workers write files.) */
int ns_transfer_info(NsContext* ctx, uint32_t* packed_bases, uint32_t* unpack_threads);

/* The host half of that transfer, for consumers that copy the packed bases themselves: expands n_bases bases, 2 bits each
 * (base k in bits [2(k&3)+1 : 2(k&3)] of packed[k >> 2]; A C T G = 0 1 2 3, U for T when uracil), into ASCII with `threads`
 * host threads (AVX2 when the CPU has it).  Replaces nothing in the reference: its workers hold Python strings. */
int ns_unpack_bases(const uint8_t* packed, uint8_t* seq, uint64_t n_bases, int uracil, int threads);

/* Intron retention (simulator.py:1156-1183), second half: replaces the piece lists of `n_slots` reads of the last batch and
 * emits those reads again.  The host decides which reads retain introns (nanosim_b200/intron_retention.py) and lays each of
 * them out as pieces on the GENOME records of the reference, one per exon / retained-intron interval (NS_PIECE_REF_REV,
 * NS_PIECE_CONT, NS_PIECE_RETAINED), with the read's edit script cut at the interval boundaries.  new_reads[k] replaces
 * read read_slots[k]; new_pieces / new_ops are appended behind the batch's pieces / ops, and piece_first / op_off / ev_off
 * in the new metadata are absolute indices into the grown arrays.
 * Without -hp/-k: same seq_len, the bytes are overwritten in place.  All emit randomness is indexed by the position in the
 * read, so inserted, head/tail and polyA bases and every quality value come out as before; only bases taken from the
 * reference change.
 * With -hp/-k: new_ops are the UNFILTERED event scripts (NsBatchInfo.raw_ev_off) cut at the interval boundaries, and each
 * read's pieces must form one chain -- genome segments at even offsets, each after the first NS_PIECE_CONT, zero-op gaps
 * in between, one strand, op_off == ev_off.  The -k filter and mutate_homo run again over each chain as one sequence (the
 * genomic read); the filtered scripts stay the pieces' event scripts, the rewritten ones are appended behind them.  The
 * read length changes: each replaced read gets a new 16-byte-aligned slot behind the batch's bytes (the old slot is no
 * longer referenced), and the batch's totals grow (ns_batch_info).  As positions shift and emit randomness is keyed by
 * position, such reads keep neither their qualities nor their inserted bases. */
int ns_reemit(NsContext* ctx, const uint32_t* read_slots, const NsReadMeta* new_reads, uint32_t n_slots,
              const NsPieceMeta* new_pieces, uint32_t n_new_pieces, const uint32_t* new_ops, uint64_t n_new_ops);
/* The totals of the last batch as they stand now (ns_simulate's NsBatchInfo, updated by ns_reemit): what ns_fetch copies. */
int ns_batch_info(NsContext* ctx, NsBatchInfo* info);

/* Device pointers of the last batch (for consumers that stay on the GPU, e.g. torch tensors / NCCL gathers). */
int ns_device_buffers(NsContext* ctx, const uint8_t** seq, const uint8_t** qual, const NsReadMeta** reads,
                      const NsPieceMeta** pieces, const uint32_t** ops);

/* Histograms of the last batch's edit scripts, computed on the device (what tests compare with the statistics of
 * the reference's <out>_aligned_error_profile).  out must hold NS_STATS_WORDS uint64. */
#define NS_STATS_EV_CAP 64
#define NS_STATS_RUN_CAP 512
#define NS_STATS_EPR_CAP 131072   /* error events per aligned segment (mutate_read call), exact counts 0..cap-1, cap+ */
/* layout (uint64 words): [0..7] totals (segments, reference bases, segment output bases, head/tail bases, gaps, gap bases,
 * events, -), [8..15] events / event bases by type (mis ins del), 3 event-length histograms, match-run and first-match
 * histograms, then NS_STATS_EPR_OFF: events-per-segment histogram (segments with at least one event, as the error profile
 * shows them), NS_STATS_SUB_OFF: 4x4 reference base x read base of 1-base mismatches (A C G T order, read taken in the
 * reference's orientation), NS_STATS_INS_OFF: inserted bases by A C G T, NS_STATS_COMP_OFF: base composition of the reads */
#define NS_STATS_EPR_OFF (8 + 8 + 3 * (NS_STATS_EV_CAP + 1) + 2 * (NS_STATS_RUN_CAP + 1))
#define NS_STATS_SUB_OFF (NS_STATS_EPR_OFF + NS_STATS_EPR_CAP + 1)
#define NS_STATS_INS_OFF (NS_STATS_SUB_OFF + 16)
#define NS_STATS_COMP_OFF (NS_STATS_INS_OFF + 4)
#define NS_STATS_WORDS (NS_STATS_COMP_OFF + 4)
int ns_op_stats(NsContext* ctx, uint64_t* out);

/* Host-side record formatting of a fetched batch into the reference's FASTA/FASTQ text (:1437-1443); multi-threaded.
 * names: n_reads NUL-terminated strings laid out back to back, name_off[i] = start of read i's name. */
int64_t ns_format_records(const uint8_t* seq, const uint8_t* qual, const NsReadMeta* reads, uint32_t n_reads,
                          const char* names, const uint64_t* name_off, int fastq, char* out, uint64_t out_cap,
                          int n_threads);

/* Host-side rows of <out>_aligned_error_profile (mutate_read's log, :2006-2008; the caller writes the header line
 * :1634): for every aligned segment of every read, its error events right to left --
 * "name<TAB>position in the segment's reference<TAB>mis|ins|del<TAB>length<TAB>reference bases<TAB>read bases".
 * Needs the fetched ops (event scripts), the host copy of the reference (bases + chrom_off as passed to
 * ns_set_reference), the seed of the context and the id of the batch's first read.  Same two-call protocol and name
 * layout as ns_format_records; multi-threaded. */
int64_t ns_format_error_profile(const uint8_t* seq, const NsReadMeta* reads, const NsPieceMeta* pieces, const uint32_t* ops,
                                uint32_t n_reads, const uint8_t* ref_bases, const uint64_t* chrom_off, const char* names,
                                const uint64_t* name_off, uint64_t seed, uint64_t first_id, char* out, uint64_t out_cap,
                                int n_threads);

/* The two formatters above writing straight into a file (what the reference's workers do with out_reads.write /
 * out_error.write, simulator.py:1437-1443, 2006-2008): every thread formats its stretch of records into a private chunk and
 * pwrite()s it at byte `file_off` + its position, so no text buffer of the whole batch exists and the copy into the page
 * cache runs on n_threads cores.  Returns the bytes written (the caller advances its offset by it) or a negative NS_E*. */
int64_t ns_write_records(int fd, uint64_t file_off, const uint8_t* seq, const uint8_t* qual, const NsReadMeta* reads,
                         uint32_t n_reads, const char* names, const uint64_t* name_off, int fastq, int n_threads);
int64_t ns_write_error_profile(int fd, uint64_t file_off, const uint8_t* seq, const NsReadMeta* reads, const NsPieceMeta* pieces,
                               const uint32_t* ops, uint32_t n_reads, const uint8_t* ref_bases, const uint64_t* chrom_off,
                               const char* names, const uint64_t* name_off, uint64_t seed, uint64_t first_id, int n_threads);

/* The last batch's FASTA/FASTQ text (ns_format_records' bytes, after ns_reemit as well) as BGZF, built on the device: the
 * text is cut into blocks of 56 KiB (the last one shorter) and every block becomes one gzip member of at most 64 KiB with
 * the BGZF extra field, one dynamic-Huffman DEFLATE block each, so gzip, zcat and htslib read the members and their
 * concatenation.  The end-of-file block is not included.  names / name_off: the layout ns_format_records takes (uploaded
 * by this call).  The members stay in HBM until the next ns_simulate / ns_reemit; *nbytes = their size.  NS_ESTATE if a
 * member came out larger than 64 KiB (cannot happen: see nanosim_b200/csrc/bgzf_kernel.cuh). */
int ns_compress_records(NsContext* ctx, const char* names, const uint64_t* name_off, uint64_t* nbytes);
/* The last batch's reads as unaligned BAM records (after ns_reemit as well), BGZF-compressed on the device like
 * ns_compress_records: one record per read, in read order and orientation, with the name ns_format_records would write,
 * flag 4 (unmapped), refID / pos / next_refID / next_pos -1, mapq 255, bin 4680, no CIGAR and no aux data; the bases as
 * 4-bit codes ("=ACMGRSVTWYHKDBN" in either case, U as T, any other byte N), the qualities - 33 (0xff each without
 * --fastq).  Records straddle members where the 56 KiB cut falls.  Neither the BAM header nor the end-of-file block is
 * included.  The members replace those of the last ns_compress_records (and a later ns_compress_records replaces these);
 * ns_fetch_compressed copies them.  NS_EINVAL when a name is longer than 254 bytes (the message names the first such read
 * and its length); names are never truncated. */
int ns_compress_bam(NsContext* ctx, const char* names, const uint64_t* name_off, uint64_t* nbytes);
/* Device->host copy of those members; NS_ENOMEM when cap is smaller than ns_compress_records' (or ns_compress_bam's)
 * *nbytes. */
int ns_fetch_compressed(NsContext* ctx, uint8_t* out, uint64_t cap);
/* The rows of <out>_aligned_error_profile for the last aligned batch (ns_format_error_profile's bytes, after ns_reemit as
 * well; no header line) as BGZF, formatted and compressed on the device from the batch's reads, pieces, event scripts and
 * sequence and the resident reference: 56 KiB blocks, one member each, in which every row's read name is sent as a
 * back-reference to the row before it (the rule is in nanosim_b200/csrc/bgzf_kernel.cuh).  Same name layout as
 * ns_compress_records; the seed is the context's.  The members stay in HBM in a buffer of their own (ns_compress_records
 * before or after this call keeps its members) until the next ns_simulate / ns_reemit; *nbytes = their size, 0 for a
 * batch without error events.  NS_EINVAL when the last batch is not aligned. */
int ns_compress_error_profile(NsContext* ctx, const char* names, const uint64_t* name_off, uint64_t* nbytes);
/* Device->host copy of those members; NS_ENOMEM when cap is smaller than ns_compress_error_profile's *nbytes. */
int ns_fetch_compressed_error_profile(NsContext* ctx, uint8_t* out, uint64_t cap);

/* Host-side read names of a fetched batch in the reference's formats (genome :1390-1402, metagenome :965-969,
 * transcriptome :1188-1219, perfect :1332-1343, unaligned :1511/:1529-1534), written as NUL-terminated strings back to
 * back (name_off[i] = start of read i's name): the layout the two formatters above take.  flags: bit 0 perfect,
 * bit 1 metagenome, bit 2 transcriptome.  index_base = the reference's shared total_simulated counter at the batch's
 * first read.  chrom_names uses the same layout (one name per reference record).  Two-call protocol: out == NULL
 * returns the bytes needed. */
int64_t ns_format_names(const NsReadMeta* reads, const NsPieceMeta* pieces, uint32_t n_reads, int kind, uint32_t flags,
                        uint64_t index_base, const char* chrom_names, const uint64_t* chrom_name_off, char* out,
                        uint64_t out_cap, uint64_t* name_off);

#ifdef __cplusplus
}
#endif
#endif
