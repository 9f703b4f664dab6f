// C ABI of libnanosim_b200.so (include/nanosim_b200.h): context, HBM residency of reference + model tables,
// batch orchestration (plan -> scan -> script -> emit) on one CUDA stream, device->host fetch.  The entry points that need
// no context (formatters, FASTA reader, expansion of the 2-bit bases) are in host_io.cu.
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <dlfcn.h>
#include <string>
#include <memory>
#include <vector>

#if __has_include(<nccl.h>)
#include <nccl.h>
#define NS_HAVE_NCCL 1
#else
#define NS_HAVE_NCCL 0
#endif

#include "nanosim_b200.h"
#include "device_common.cuh"
#include "qual_table.h"
#include "plan_kernel.cuh"
#include "emit_kernel.cuh"
#include "uread_kernel.cuh"
#include "hp_kernel.cuh"
#include "bgzf_kernel.cuh"
#include "errprof_kernel.cuh"
#include "aln_kernel.cuh"
#include "haplotype.h"
#include "host_io.h"

namespace {

// Device memory, page-locked host memory and events belong to exactly one owner, which frees them: none of them is copied.
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() {
        if (p) cudaFree(p);
    }
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    // grow but keep the first `keep` bytes (rare path)
    cudaError_t ensure_keep(size_t bytes, size_t keep, cudaStream_t st) {
        if (bytes <= cap) return cudaSuccess;
        void* np = nullptr;
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMalloc(&np, want);
        if (e != cudaSuccess) return e;
        if (p && keep) {
            e = cudaMemcpyAsync(np, p, keep, cudaMemcpyDeviceToDevice, st);
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        }
        if (p) cudaFree(p);
        p = np;
        cap = want;
        return e;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct PinnedBuf {
    void* p = nullptr;
    size_t cap = 0;
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf&) = delete;
    PinnedBuf& operator=(const PinnedBuf&) = delete;
    ~PinnedBuf() {
        if (p) cudaFreeHost(p);
    }
    cudaError_t ensure(size_t bytes, unsigned flags) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
        size_t want = bytes + bytes / 8 + 4096;
        cudaError_t e = cudaHostAlloc(&p, want, flags);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct Event {
    cudaEvent_t e = nullptr;
    Event() = default;
    Event(const Event&) = delete;
    Event& operator=(const Event&) = delete;
    ~Event() {
        if (e) cudaEventDestroy(e);
    }
    operator cudaEvent_t() const { return e; }
};

// Reference and model tables in HBM.  A context and its clones (ns_clone) hold one copy; only the context that created
// it sets them.
struct Tables {
    bool have_ref = false, have_model = false, have_expr = false;
    DevBuf ref_bases, ref_off, ref_packed, ref_pk_off, ref_exc, ref_species, ref_circular, ref_sp_off;
    DevBuf kde[5], alias, qlut, kde2d_x, kde2d_y, expr_alias, expr_chrom, chrom_polya;
    std::vector<uint64_t> h_chrom_off;
    std::vector<uint32_t> h_sp_off;
    DevRef dref{};                  // without the transcript-length table: that one is per context (NsContext::trx)
    DevModel dmodel{};
    NsModel hmodel{};
    // ns_apply_variants: the record offsets of the haploid reference the haplotypes were built from (empty before)
    std::vector<uint64_t> h_haploid_off;
    // ns_set_lift: the lift table of the resident haplotype records (aln_kernel.cuh's AlnLift)
    DevBuf lift_seg, lift_kind, lift_first, lift_chrom, lift_hp;
    bool have_lift = false;
    // ns_set_splice: the transcripts' exons on the genome records (aln_kernel.cuh's AlnSplice)
    DevBuf splice_exon, splice_first, splice_minus;
    uint32_t splice_n_trx = 0, splice_genome_first = NS_SPLICE_NO_GENOME, splice_n_genome = 0;
    bool have_splice = false;
    // ns_set_lift, for ns_set_aln_tags: the lift's variant count and the REF bytes its ALTs pair with (prefix sum per variant)
    std::vector<uint64_t> h_lift_pair_off;
    // ns_set_aln_tags: the mapped header's SN names (aln_kernel.cuh's AlnAuxArgs) and, with a lift, the REF bytes
    // (AlnTagArgs::pair, pair_off)
    DevBuf tag_sn, tag_sn_off, tag_pair, tag_pair_off;
    uint32_t tag_n_sn = 0;
    bool have_aln_tags = false;
};

// transcript lengths ascending + their record indices (ns_configure, transcriptome mode); a clone that configures another
// record count builds its own
struct TrxTable {
    DevBuf buf;
    uint32_t n = 0;
};

// the packed BGZF members of one compressed output of the last batch: `bytes` of `buf`, fetchable while `valid`
struct MemberSlot {
    DevBuf buf;
    uint64_t bytes = 0;
    bool valid = false;
};

}  // namespace

struct NsContext {
    int device = 0;
    uint64_t seed = 0;
    cudaStream_t stream = nullptr;
    Event ev[6];
    std::string err;
    int sm_count = 0;               // ns_create: cudaDeviceProp::multiProcessorCount

    std::shared_ptr<Tables> tables = std::make_shared<Tables>();
    bool clone = false;             // ns_clone: the tables are the parent's, and only the parent sets them
    bool have_cfg = false;
    NsRunConfig hcfg{};
    DevCfg dcfg{};
    std::shared_ptr<const TrxTable> trx;
    std::vector<double> abun, abun_inflated, species_bases;     // metagenome: dict_abun, dict_abun_inflated, running totals
    DevBuf sp_bases_dev;

    // batch state
    DevBuf split_base, split_extra, split_ckpt, hp_keys;     // long pieces -> extra emit work items (emit_kernel.cuh:split_kernel)
    DevBuf reads, pieces, ops, seq, qual, nseg, npieces, piece_first, scan_in, scan_out, scan_tmp, counter, totals,
        stats, sort_keys, sort_vals, sort_tmp, hp_off;
    PinnedBuf h_totals;             // mapped
    uint64_t* h_totals_dev = nullptr;
    // ns_fetch sends bases over PCIe as 2 bits each: device pack buffer, pinned staging, event after its copy
    DevBuf pack_dev;
    PinnedBuf pack_host;
    Event ev_pack;
    Event ev_block;                 // cudaEventBlockingSync: long waits sleep instead of spinning (wait_stream)
    // ns_compress_records: the uploaded names, record layout, members as the deflate kernel leaves them, and the packed
    // BGZF members of the last batch
    DevBuf z_names, z_name_off, z_name_len, z_rec_off, z_stage, z_msize, z_moff, z_trailer;
    MemberSlot z_out;
    // ns_compress_error_profile: the rows of the last aligned batch and their BGZF members.  Names, layout and staging are
    // the z_ buffers above: only the members outlive a call.
    DevBuf ep_text;
    MemberSlot ep_out;
    // ns_compress_bam_mapped: per read its record and CIGAR-word counts (2n) and their offsets (2n), its primary alignment;
    // the records' descriptors and CIGAR words.  Its members go to z_out.
    DevBuf m_cnt, m_first, m_prim, m_aln, m_cig;
    // with NM and SA (ns_set_aln_tags): every record's NM, aux bytes, their offsets, and the aux bytes themselves
    DevBuf m_nm, m_aux_len, m_aux_off, m_aux;
    // Batches of one job have near-identical sizes: once a batch of a kind has run with host-sized buffers, the next ones
    // are submitted in one go (no host round trip between the first and the last kernel) against those capacities; a
    // kernel checks them on the device and a batch that does not fit is simply run again the sized way.
    bool opt_ok[2] = {false, false};
    uint32_t opt_n[2] = {0, 0};
    NsBatchInfo last{};
    int last_kind = 0;
    uint64_t last_first_id = 0;
    bool have_batch = false;

    ~NsContext() {
        if (stream) cudaStreamDestroy(stream);
    }
};

// NsContext::totals: the counters of a batch (ns_simulate zeroes them all) and of a compression (which zeroes its own, from
// NS_T_Z_TEXT on), published to h_totals by publish_totals_and_wait
enum TotalsSlot : int {
    NS_T_PIECES,                // pieces of the batch
    NS_T_OVERFLOW_OPS,          // script ops of the pieces of reads whose script overflowed its slot
    NS_T_SEQ_BYTES,             // sequence bytes (read_layout)
    NS_T_BASES,                 // bases (read_layout)
    NS_T_SLOT_OPS,              // script ops of the capped slots
    NS_T_FLAGGED,               // reads whose script overflowed its slot
    NS_T_HP_OPS,                // script ops the homopolymer pass writes
    NS_T_POOL_CURSOR,           // the bump pool of re-drawn unaligned reads (uread_kernel.cuh): its cursor,
    NS_T_POOL,                  // its base
    NS_T_POOL_SIZE,             // and its size
    NS_T_PRIMARY,               // script ops of the primary area
    NS_T_ABORT,                 // abort flags (bit 0: script area too small, bit 1: with the overflow area, bit 2: sequence
                                // buffers too small)
    NS_T_Z_TEXT,                // compression: text bytes
    NS_T_Z_BYTES,               // compression: member bytes
    NS_T_Z_OVERSIZE,            // compression: members above 64 KiB
    NS_T_Z_LONG_NAMES,          // compression: read names too long for BAM
    NS_T_COUNT,
    // ns_compress_bam_mapped's record and CIGAR-word totals borrow the text and member-bytes slots, which its later scans
    // overwrite
    NS_T_M_RECORDS = NS_T_Z_TEXT,
    NS_T_M_CIGAR_WORDS = NS_T_Z_BYTES,
    NS_T_M_AUX_BYTES = NS_T_Z_BYTES,    // with NM and SA, at the second wait: the records' aux bytes
};

// Wait for everything queued on the context's stream.  cudaStreamSynchronize spins: a host thread per overlapped context then
// burns a core for the whole of a big batch.  GPU processes that share a host under a CPU quota also need that CPU time for
// the expansion of the 2-bit bases in ns_fetch, so with several GPU processes on the host (torchrun's LOCAL_WORLD_SIZE > 1,
// or NANOSIM_B200_BLOCKING_SYNC=1) long waits sleep on a cudaEventBlockingSync event; a single process, and every short
// wait, spins as before.  Not measured on H100.
static bool blocking_sync_wanted() {
    static const bool want = [] {
        if (const char* e = getenv("NANOSIM_B200_BLOCKING_SYNC")) return atoi(e) != 0;
        const char* lw = getenv("LOCAL_WORLD_SIZE");
        return lw && atoi(lw) > 1;
    }();
    return want;
}
static cudaError_t wait_stream(NsContext* ctx, bool long_wait) {
    if (!long_wait || !blocking_sync_wanted()) return cudaStreamSynchronize(ctx->stream);
    cudaError_t e = cudaSuccess;
    if (!ctx->ev_block) e = cudaEventCreateWithFlags(&ctx->ev_block.e, cudaEventBlockingSync | cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventRecord(ctx->ev_block, ctx->stream);
    if (e == cudaSuccess) e = cudaEventSynchronize(ctx->ev_block);
    return e;
}


namespace {

cudaEvent_t g_base[64] = {};      // per device: origin of the device timeline reported in NsBatchInfo

int env_int(const char* name, int dflt) {
    const char* e = getenv(name);
    return (e && *e) ? atoi(e) : dflt;
}

int fail(NsContext* c, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (c) c->err = buf;
    return code;
}

#define CK(call)                                                                                      \
    do {                                                                                              \
        cudaError_t e_ = (call);                                                                      \
        if (e_ != cudaSuccess)                                                                        \
            return fail(ctx, NS_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

__global__ void scatter_piece_off(NsPieceMeta* pieces, uint32_t n, const uint64_t* off) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) pieces[i].op_off = off[i];
}
__global__ void set_sentinel_off(NsPieceMeta* pieces, uint32_t n, const uint64_t* total) {
    if (threadIdx.x == 0 && blockIdx.x == 0) pieces[n].op_off = *total;
}
// pieces of reads whose script overflowed its slot (NsReadMeta.flags bit 0) get exact offsets behind the primary area
__global__ void gather_flagged_ops(const NsPieceMeta* pieces, const NsReadMeta* reads, uint32_t n, uint64_t* out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (reads[pieces[i].read_slot].flags & 1u) ? pieces[i].n_ops : 0u;
}
__global__ void scatter_flagged_off(NsPieceMeta* pieces, const NsReadMeta* reads, uint32_t n, const uint64_t* off, const uint64_t* base) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && (reads[pieces[i].read_slot].flags & 1u)) pieces[i].op_off = *base + off[i];
}
__global__ void copy_ev_fields(NsPieceMeta* pieces, uint32_t n) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        pieces[i].ev_off = pieces[i].op_off;
        pieces[i].ev_n_ops = pieces[i].n_ops;
    }
}
__global__ void add_base_u64(uint64_t* v, uint32_t n, uint64_t base) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] += base;
}
// ns_set_reference: the 2-bit copy of the reference (DevRef::packed).  One thread per packed word; exceptions (bytes
// that are not a/c/g/t in either case) are counted per 256-word block, other[0] counts bytes that are not even an IUPAC
// nucleotide code (case_convert passes those through unchanged, so reads may then hold characters other than ACGT).
__global__ void pack_reference_kernel(const uint8_t* __restrict__ bases, const uint64_t* __restrict__ chrom_off,
                                      const uint64_t* __restrict__ pk_off, uint32_t n_chrom, uint32_t* __restrict__ packed,
                                      uint64_t n_words, uint32_t* __restrict__ exc_cnt, unsigned long long* other) {
    const uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= n_words) return;
    // chromosome of this word: last c with pk_off[c] <= w
    uint32_t lo = 0, hi = n_chrom;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (pk_off[mid] <= w) lo = mid; else hi = mid;
    }
    const uint64_t cstart = chrom_off[lo], clen = chrom_off[lo + 1] - cstart;
    const uint64_t first = (w - pk_off[lo]) * 16;
    uint32_t word = 0, n_exc = 0, n_other = 0;
    for (uint32_t j = 0; j < 16; ++j) {
        if (first + j >= clen) break;
        uint32_t c = bases[cstart + first + j];
        if (c - 'a' < 26u) c -= 32;
        if (acgt_fast(c)) {
            word |= base_idx(c) << (2 * j);
        } else {
            ++n_exc;
            if (resolve_iupac(c, 0u, 0u) == c) ++n_other;      // not in case_convert's table: passes through unchanged
        }
    }
    packed[w] = word;
    if (n_exc) atomicAdd(&exc_cnt[w >> REF_EXC_BLOCK_SHIFT], n_exc);
    if (n_other) atomicAdd(other, (unsigned long long)n_other);
}

// Bases leave the device as 2 bits each (the emit kernel only writes A C G T/U): 16 ASCII bytes -> one 32-bit word,
// base j of a byte quadruple in bits [2j, 2j+1], code = (c >> 1) & 3 (A 0, C 1, T/U 2, G 3).  ns_fetch expands them again
// on the host, so callers see the same ASCII buffers while the PCIe transfer of a FASTQ batch shrinks from 2 to 1.25 B/base.
__global__ void pack_bases_kernel(const uint4* __restrict__ seq, uint32_t* __restrict__ out, uint64_t n16) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n16) return;
    const uint4 v = seq[i];
    auto pk = [](uint32_t w) {
        const uint32_t t = (w >> 1) & 0x03030303u;
        return (t | (t >> 6) | (t >> 12) | (t >> 18)) & 0xffu;
    };
    out[i] = pk(v.x) | (pk(v.y) << 8) | (pk(v.z) << 16) | (pk(v.w) << 24);
}
// The batch totals the host needs mid-pipeline are written straight into mapped pinned host memory: a cudaMemcpy
// would queue behind another context's multi-GB device->host transfer on the copy engine and serialise the pipelines.
__global__ void publish_totals(const uint64_t* totals, volatile uint64_t* host) {
    if (threadIdx.x < NS_T_COUNT) host[threadIdx.x] = totals[threadIdx.x];
    __threadfence_system();
}
// sync-free batches: what the host would compute from the scans, computed and checked against the capacities on the device
__global__ void capacity_stage_a(uint64_t* totals, uint32_t fast_unaligned, uint64_t ops_cap) {
    if (threadIdx.x || blockIdx.x) return;
    const uint64_t slot_ops = totals[NS_T_SLOT_OPS];
    const uint64_t pool_ops = fast_unaligned ? slot_ops / 16 + (1u << 20) : 0;
    totals[NS_T_POOL] = slot_ops;
    totals[NS_T_POOL_SIZE] = pool_ops;
    totals[NS_T_PRIMARY] = slot_ops + pool_ops;
    if (slot_ops + pool_ops + 4 > ops_cap) totals[NS_T_ABORT] |= 1u;
}
__global__ void capacity_stage_b(uint64_t* totals, uint64_t ops_cap, uint64_t seq_cap) {
    if (threadIdx.x || blockIdx.x) return;
    if (totals[NS_T_PRIMARY] + totals[NS_T_OVERFLOW_OPS] + 4 > ops_cap) totals[NS_T_ABORT] |= 2u;
    if (totals[NS_T_SEQ_BYTES] + 16 > seq_cap) totals[NS_T_ABORT] |= 4u;
}
__global__ void gather_read_bytes(const NsReadMeta* reads, uint32_t n, uint64_t* out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = ((uint64_t)reads[i].seq_len + 15u) & ~(uint64_t)15u;
}
__global__ void scatter_read_off(NsReadMeta* reads, uint32_t n, const uint64_t* off) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) reads[i].seq_off = off[i];
}
__global__ void widen_u32(const uint32_t* in, uint32_t n, uint64_t* out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[i];
}
__global__ void narrow_u64(const uint64_t* in, uint32_t n, uint32_t* out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (uint32_t)in[i];
}
// totals[k] = off[n-1] + in[n-1]
__global__ void last_total(const uint64_t* in, const uint64_t* off, uint32_t n, uint64_t* totals, int k) {
    if (threadIdx.x == 0 && blockIdx.x == 0) totals[k] = n ? off[n - 1] + in[n - 1] : 0;
}
__global__ void sum_bases(const NsReadMeta* reads, uint32_t n, unsigned long long* out) {
    unsigned long long s = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) s += reads[i].seq_len;
    for (int d = 16; d > 0; d >>= 1) s += __shfl_down_sync(0xffffffffu, s, d);
    if ((threadIdx.x & 31) == 0 && s) atomicAdd(out, s);
}

// op-list histograms (ns_op_stats)
__device__ __forceinline__ int acgt_index(uint32_t c) {          // A C G T(U) -> 0 1 2 3, anything else -1
    if (c - 'a' < 26u) c -= 32;
    return c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : (c == 'T' || c == 'U') ? 3 : -1;
}
__global__ void op_stats_kernel(const NsPieceMeta* pieces, const NsReadMeta* reads, const uint32_t* ops, uint32_t n,
                                DevRef ref, const uint8_t* seq, unsigned long long* st) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const NsPieceMeta pm = pieces[i];
    const NsReadMeta rm = reads[pm.read_slot];
    // pieces a read no longer owns (its piece list was replaced by ns_reemit) are not counted
    if (i < rm.piece_first || i >= rm.piece_first + rm.n_pieces) return;
    unsigned long long* ev = st + 8;
    unsigned long long* evlen = st + 16;
    unsigned long long* run_h = evlen + 3 * (NS_STATS_EV_CAP + 1);
    unsigned long long* first_h = run_h + (NS_STATS_RUN_CAP + 1);
    if (NS_PIECE_KIND(pm.kind) != NS_PIECE_SEGMENT) {
        atomicAdd(&st[4], 1ull);
        atomicAdd(&st[5], (unsigned long long)pm.out_len);
        return;
    }
    atomicAdd(&st[0], 1ull);
    atomicAdd(&st[1], (unsigned long long)pm.ref_len);
    uint64_t run = 0, ht = 0, n_ev = 0;
    bool first = true;
    // substituted / inserted bases are read back from the sequence: only when the event script is the emitted script
    // (-hp rewrites it) and the piece reads the reference forwards
    const bool bases_ok = seq != nullptr && pm.ev_off == pm.op_off && !(pm.kind & NS_PIECE_REF_REV);
    const uint64_t cstart = ref.chrom_off[pm.chrom];
    const uint32_t clen = (uint32_t)(ref.chrom_off[pm.chrom + 1] - cstart);
    const uint8_t* rs = seq ? seq + rm.seq_off : nullptr;
    uint32_t sub[16], insb[4];
#pragma unroll
    for (int k = 0; k < 16; ++k) sub[k] = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) insb[k] = 0;
    auto read_base = [&](uint32_t x) -> int {                    // base x of the read in the reference's orientation
        if (!rm.reversed) return acgt_index(rs[x]);
        const int b = acgt_index(rs[rm.seq_len - 1u - x]);
        return b < 0 ? b : 3 - b;
    };
    uint32_t o = pm.out_rel, rf = 0;
    for (uint32_t k = 0; k < pm.ev_n_ops; ++k) {         // the event script (== op script unless -hp rewrote it)
        uint32_t op = ops[pm.ev_off + k];
        uint32_t ty = op >> 28, len = op_len(op);
        if (ty == NS_OP_HT) {
            ht += len;
        } else if (ty == NS_OP_COPY) {
            run += len;
        } else if (ty <= NS_OP_DEL) {
            uint32_t t = ty - 1;   // 0 mis 1 ins 2 del
            atomicAdd(&ev[t], 1ull);
            atomicAdd(&ev[3 + t], (unsigned long long)len);
            atomicAdd(&evlen[t * (NS_STATS_EV_CAP + 1) + (len < NS_STATS_EV_CAP ? len : NS_STATS_EV_CAP)], 1ull);
            unsigned long long* h = first ? first_h : run_h;
            atomicAdd(&h[run < NS_STATS_RUN_CAP ? run : NS_STATS_RUN_CAP], 1ull);
            first = false;
            run = 0;
            ++n_ev;
            if (bases_ok && ty == NS_OP_MIS && len == 1) {
                uint32_t ab = pm.pos + rf;
                if (ab >= clen) ab -= clen;
                const int a = acgt_index(ref.bases[cstart + ab]), b = read_base(o);
                if (a >= 0 && b >= 0) ++sub[a * 4 + b];
            } else if (bases_ok && ty == NS_OP_INS) {
                for (uint32_t t2 = 0; t2 < len; ++t2) {
                    const int b = read_base(o + t2);
                    if (b >= 0) ++insb[b];
                }
            }
        }
        if (ty != NS_OP_DEL) o += len;
        if (ty == NS_OP_COPY || ty == NS_OP_MIS || ty == NS_OP_DEL) rf += len;
    }
    atomicAdd(&st[2], (unsigned long long)(pm.out_len - ht));
    atomicAdd(&st[3], (unsigned long long)ht);
    atomicAdd(&st[6], (unsigned long long)n_ev);
    if (n_ev) atomicAdd(&st[NS_STATS_EPR_OFF + (n_ev < NS_STATS_EPR_CAP ? n_ev : NS_STATS_EPR_CAP)], 1ull);
#pragma unroll
    for (int k = 0; k < 16; ++k)
        if (sub[k]) atomicAdd(&st[NS_STATS_SUB_OFF + k], (unsigned long long)sub[k]);
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (insb[k]) atomicAdd(&st[NS_STATS_INS_OFF + k], (unsigned long long)insb[k]);
}
// base composition of the batch's reads (as emitted; U counts as T): one warp per read
__global__ void base_comp_kernel(const NsReadMeta* reads, uint32_t n, const uint8_t* seq, unsigned long long* st) {
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= n) return;
    const NsReadMeta rm = reads[w];
    const uint8_t* rs = seq + rm.seq_off;
    uint32_t c[4] = {0, 0, 0, 0};
    for (uint32_t x = lane; x < rm.seq_len; x += 32) {
        const int b = acgt_index(rs[x]);
        if (b >= 0) ++c[b];
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        uint32_t v = c[k];
        for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
        if (lane == 0 && v) atomicAdd(&st[NS_STATS_COMP_OFF + k], (unsigned long long)v);
    }
}

cudaError_t upload(DevBuf& b, const void* src, size_t bytes, cudaStream_t s) {
    cudaError_t e = b.ensure(bytes ? bytes : 16);
    if (e != cudaSuccess) return e;
    if (bytes == 0) return cudaSuccess;
    return cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyDefault, s);
}

// The steps of a batch.  Every kernel, CUB scan and CUB sort of a batch is counted in NsBatchInfo.n_launches here.
template <class... P, class... A>
cudaError_t launch(NsContext* ctx, void (*kernel)(P...), unsigned grid, unsigned block, size_t smem, A... args) {
    kernel<<<grid, block, smem, ctx->stream>>>(args...);
    ++ctx->last.n_launches;
    return cudaGetLastError();
}

// out = exclusive prefix sum of in[0, n); totals[slot] = the sum of all n
int scan_total(NsContext* ctx, const uint64_t* in, uint64_t* out, uint32_t n, int slot) {
    size_t tmp = 0;
    CK(cub::DeviceScan::ExclusiveSum(nullptr, tmp, in, out, (int)n, ctx->stream));
    CK(ctx->scan_tmp.ensure(tmp));
    CK(cub::DeviceScan::ExclusiveSum(ctx->scan_tmp.p, tmp, in, out, (int)n, ctx->stream));
    ++ctx->last.n_launches;
    CK(launch(ctx, last_total, 1, 32, 0, in, out, n, ctx->totals.as<uint64_t>(), slot));
    return NS_OK;
}

// a 16-byte aligned sequence slot per read: reads[i].seq_off, and the sequence bytes and bases in totals
int read_layout(NsContext* ctx, uint32_t n) {
    const unsigned gb = (n + 255) / 256;
    NsReadMeta* reads = ctx->reads.as<NsReadMeta>();
    uint64_t* totals = ctx->totals.as<uint64_t>();
    CK(launch(ctx, gather_read_bytes, gb, 256, 0, reads, n, ctx->scan_in.as<uint64_t>()));
    if (int rc = scan_total(ctx, ctx->scan_in.as<uint64_t>(), ctx->scan_out.as<uint64_t>(), n, NS_T_SEQ_BYTES)) return rc;
    CK(launch(ctx, scatter_read_off, gb, 256, 0, reads, n, ctx->scan_out.as<uint64_t>()));
    CK(cudaMemsetAsync(totals + NS_T_BASES, 0, sizeof(uint64_t), ctx->stream));
    CK(launch(ctx, sum_bases, std::min(gb, 1024u), 256, 0, reads, n, (unsigned long long*)(totals + NS_T_BASES)));
    return NS_OK;
}

int sort_pairs_descending(NsContext* ctx, const uint32_t* keys_in, uint32_t* keys_out, const uint32_t* vals_in, uint32_t* vals_out,
                          uint32_t n) {
    size_t tmp = 0;
    CK(cub::DeviceRadixSort::SortPairsDescending(nullptr, tmp, keys_in, keys_out, vals_in, vals_out, (int)n, 0, 32, ctx->stream));
    CK(ctx->sort_tmp.ensure(tmp));
    CK(cub::DeviceRadixSort::SortPairsDescending(ctx->sort_tmp.p, tmp, keys_in, keys_out, vals_in, vals_out, (int)n, 0, 32, ctx->stream));
    ++ctx->last.n_launches;
    return NS_OK;
}

// the host reads the batch totals (h_totals) after this
int publish_totals_and_wait(NsContext* ctx, bool long_wait = false) {
    CK(launch(ctx, publish_totals, 1, 32, 0, ctx->totals.as<uint64_t>(), ctx->h_totals_dev));
    CK(wait_stream(ctx, long_wait));
    return NS_OK;
}

// the reference as the kernels see it: the shared tables plus this context's transcript-length table
DevRef dev_ref(const NsContext* ctx) {
    DevRef r = ctx->tables->dref;
    if (ctx->trx) {
        r.trx_len_sorted = ctx->trx->buf.as<uint32_t>();
        r.trx_len_idx = r.trx_len_sorted + ctx->trx->n;
        r.n_trx_sorted = ctx->trx->n;
    }
    return r;
}

// emit_kernel over `n_pieces` pieces of the context's current batch (all of them, or the ones `order` lists)
int launch_emit(NsContext* ctx, int kind, uint64_t first_read_id, uint32_t n_pieces, const uint32_t* order,
                const uint32_t* abort_flag = nullptr, bool split = true, cudaEvent_t emit_begin = nullptr) {
    cudaStream_t st = ctx->stream;
    EmitArgs ea;
    ea.ref = dev_ref(ctx);
    ea.cfg = ctx->dcfg;
    ea.kind = (uint32_t)kind;
    ea.first_id = first_read_id;
    ea.reads = ctx->reads.as<NsReadMeta>();
    ea.pieces = ctx->pieces.as<NsPieceMeta>();
    ea.ops = ctx->ops.as<uint32_t>();
    ea.n_pieces = n_pieces;
    ea.seq = ctx->seq.as<uint8_t>();
    ea.qual = ctx->qual.as<uint8_t>();
    ea.qlut = ctx->tables->qlut.as<uint32_t>();
    ea.force_exact = (ctx->hcfg.flags & NS_FLAG_EMIT_EXACT) ? 1u : 0u;
    ea.abort = abort_flag;
    ea.counter = ctx->counter.as<uint32_t>();
    ea.order = order;
    CK(cudaMemsetAsync(ctx->counter.p, 0, 64, st));
    {   // long pieces become several work items.  Capacity: every extra item stands for EMIT_SPLIT - 16 or more output bytes
        // of its piece, and a batch's output fits the sequence buffer (checked on the device for sync-free batches).
        const uint32_t cap_extra = (uint32_t)std::min<size_t>(ctx->seq.cap / (EMIT_SPLIT - 16u) + 64u, 0x7fffffffu);
        ea.split_base = nullptr;
        ea.extra = nullptr;
        ea.ckpt = nullptr;
        ea.n_extra = ctx->counter.as<uint32_t>() + 4;
        ea.cap_extra = cap_extra;
        if (split && n_pieces && !(ctx->hcfg.flags & NS_FLAG_EMIT_WHOLE)) {     // (`order` lists pieces below n_pieces whenever split is asked for)
            CK(ctx->split_base.ensure((size_t)n_pieces * sizeof(uint32_t)));
            CK(ctx->split_extra.ensure((size_t)cap_extra * sizeof(uint2)));
            CK(ctx->split_ckpt.ensure((size_t)cap_extra * sizeof(uint4)));
            CK(cudaMemsetAsync(ctx->split_extra.p, 0xff, (size_t)cap_extra * sizeof(uint2), st));
            SplitArgs sa;
            sa.reads = ea.reads;
            sa.pieces = ea.pieces;
            sa.ops = ea.ops;
            sa.n_pieces = n_pieces;
            sa.split_base = ctx->split_base.as<uint32_t>();
            sa.extra = ctx->split_extra.as<uint2>();
            sa.ckpt = ctx->split_ckpt.as<uint4>();
            sa.n_extra = ctx->counter.as<uint32_t>() + 4;
            sa.cap_extra = cap_extra;
            sa.abort = abort_flag;
            const unsigned sblocks = std::min<unsigned>((n_pieces + 7u) / 8u, (unsigned)ctx->sm_count * 8u);
            CK(launch(ctx, split_kernel, sblocks, 256, 0, sa));
            if (emit_begin) CK(cudaEventRecord(emit_begin, st));     // the emit phase of the batch timings starts after the split
            ea.split_base = sa.split_base;
            ea.extra = sa.extra;
            ea.ckpt = sa.ckpt;
        }
    }
    // FASTQ: the quality tables go to shared memory as well
    // an unaligned batch holds unaligned read bodies only (NS_PIECE_UNALIGNED): the kernel with the longer ring
    const bool unal = kind == NS_KIND_UNALIGNED;
    void (*kernel)(EmitArgs) = ctx->hcfg.fastq ? (unal ? emit_kernel<true, EMIT_RING_UNAL> : emit_kernel<true, EMIT_RING>)
                                               : (unal ? emit_kernel<false, EMIT_RING_UNAL> : emit_kernel<false, EMIT_RING>);
    const size_t smem = ctx->hcfg.fastq ? (unal ? emit_smem_bytes<true, EMIT_RING_UNAL>() : emit_smem_bytes<true, EMIT_RING>())
                                        : (unal ? emit_smem_bytes<false, EMIT_RING_UNAL>() : emit_smem_bytes<false, EMIT_RING>());
    CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 1;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, EMIT_WARPS * 32, smem));
    const unsigned blocks = std::min<unsigned>((n_pieces + EMIT_WARPS - 1) / EMIT_WARPS, (unsigned)(ctx->sm_count * std::max(per_sm, 1)));
    CK(launch(ctx, kernel, blocks, EMIT_WARPS * 32, smem, ea));
    return NS_OK;
}

}  // namespace

extern "C" {

int ns_create(int device, uint64_t seed, NsContext** out) {
    if (!out) return NS_EINVAL;
    *out = nullptr;
    NsContext* ctx = new NsContext();
    ctx->device = device;
    ctx->seed = seed;
    cudaError_t e = cudaSetDevice(device);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
    for (int i = 0; i < 6 && e == cudaSuccess; ++i) e = cudaEventCreate(&ctx->ev[i].e);
    if (e == cudaSuccess) e = ctx->h_totals.ensure(NS_T_COUNT * sizeof(uint64_t), cudaHostAllocMapped);
    if (e == cudaSuccess) e = cudaHostGetDevicePointer((void**)&ctx->h_totals_dev, ctx->h_totals.p, 0);
    if (e == cudaSuccess && device >= 0 && device < 64 && !g_base[device]) {
        e = cudaEventCreate(&g_base[device]);
        if (e == cudaSuccess) e = cudaEventRecord(g_base[device], ctx->stream);
        if (e == cudaSuccess) e = cudaEventSynchronize(g_base[device]);
    }
    if (e == cudaSuccess) {
        cudaDeviceProp prop;
        e = cudaGetDeviceProperties(&prop, device);
        if (e == cudaSuccess) ctx->sm_count = prop.multiProcessorCount;
    }
    if (e != cudaSuccess) {
        fprintf(stderr, "nanosim_b200: ns_create failed: %s\n", cudaGetErrorString(e));
        delete ctx;
        return NS_ECUDA;
    }
    *out = ctx;
    return NS_OK;
}

int ns_destroy(NsContext* ctx) {
    if (!ctx) return NS_EINVAL;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    delete ctx;
    return NS_OK;
}

const char* ns_last_error(const NsContext* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int ns_clone(NsContext* parent, NsContext** out) {
    if (!parent || !out) return NS_EINVAL;
    NsContext* c = nullptr;
    int rc = ns_create(parent->device, parent->seed, &c);
    if (rc != NS_OK) return rc;
    c->tables = parent->tables;
    c->clone = true;
    c->have_cfg = parent->have_cfg;
    c->hcfg = parent->hcfg;
    c->dcfg = parent->dcfg;
    c->trx = parent->trx;
    c->abun = parent->abun;
    c->abun_inflated = parent->abun_inflated;
    c->species_bases.assign(parent->abun.size(), 0.0);      // every clone is its own worker (own running totals)
    *out = c;
    return NS_OK;
}

// ns_set_aln_tags' tables go with every table they were built against
static void drop_aln_tags(Tables& tab) {
    tab.have_aln_tags = false;
    tab.tag_n_sn = 0;
    for (DevBuf* b : {&tab.tag_sn, &tab.tag_sn_off, &tab.tag_pair, &tab.tag_pair_off}) b->release();
}

int ns_set_reference(NsContext* ctx, const NsReference* ref) {
    if (!ctx || !ref || !ref->bases || !ref->chrom_off || ref->n_chrom == 0)
        return fail(ctx, NS_EINVAL, "ns_set_reference: null argument or empty reference");
    if (ctx->clone) return fail(ctx, NS_ESTATE, "ns_set_reference: a cloned context shares its parent's reference");
    CK(cudaSetDevice(ctx->device));
    Tables& tab = *ctx->tables;
    tab.h_chrom_off.resize(ref->n_chrom + 1);
    CK(cudaMemcpy(tab.h_chrom_off.data(), ref->chrom_off, (ref->n_chrom + 1) * sizeof(uint64_t), cudaMemcpyDefault));
    if (tab.h_chrom_off[0] != 0 || tab.h_chrom_off[ref->n_chrom] != ref->n_bases)
        return fail(ctx, NS_EINVAL, "ns_set_reference: chrom_off must start at 0 and end at n_bases");
    for (uint32_t i = 0; i < ref->n_chrom; ++i) {
        uint64_t len = tab.h_chrom_off[i + 1] - tab.h_chrom_off[i];
        if (tab.h_chrom_off[i + 1] < tab.h_chrom_off[i] || len > 0xffffffffull)
            return fail(ctx, NS_EINVAL, "ns_set_reference: chromosome %u has an invalid length", i);
    }
    CK(upload(tab.ref_bases, ref->bases, ref->n_bases, ctx->stream));
    CK(upload(tab.ref_off, tab.h_chrom_off.data(), (ref->n_chrom + 1) * sizeof(uint64_t), ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    tab.dref.bases = tab.ref_bases.as<uint8_t>();
    tab.dref.chrom_off = tab.ref_off.as<uint64_t>();
    {   // 2-bit copy + exception counts for the emit kernel's fast path
        std::vector<uint64_t> pk(ref->n_chrom + 1);
        uint64_t words = 1;                                             // guard word in front
        for (uint32_t i = 0; i < ref->n_chrom; ++i) {
            pk[i] = words;
            words += (tab.h_chrom_off[i + 1] - tab.h_chrom_off[i] + 15) / 16;
        }
        pk[ref->n_chrom] = words;
        const uint64_t n_blocks = ((words + 2) >> REF_EXC_BLOCK_SHIFT) + 2;
        CK(tab.ref_packed.ensure((size_t)(words + 2 + 64) * 4));      // + slack: a 64-word window copy may start at the last word
        CK(tab.ref_exc.ensure((size_t)(2 * n_blocks + 2) * 4 + 16));
        CK(upload(tab.ref_pk_off, pk.data(), pk.size() * sizeof(uint64_t), ctx->stream));
        CK(cudaMemsetAsync(tab.ref_packed.p, 0, (size_t)(words + 2 + 64) * 4, ctx->stream));
        CK(cudaMemsetAsync(tab.ref_exc.p, 0, (size_t)(2 * n_blocks + 2) * 4 + 16, ctx->stream));
        uint32_t* cnt = tab.ref_exc.as<uint32_t>() + n_blocks + 1;     // counts behind the prefix array
        unsigned long long* other = (unsigned long long*)(tab.ref_exc.as<uint32_t>() + ((2 * n_blocks + 2 + 1) & ~1ull));
        pack_reference_kernel<<<(unsigned)((words + 255) / 256), 256, 0, ctx->stream>>>(
            tab.ref_bases.as<uint8_t>(), tab.ref_off.as<uint64_t>(), tab.ref_pk_off.as<uint64_t>(), ref->n_chrom,
            tab.ref_packed.as<uint32_t>(), words, cnt, other);
        CK(cudaGetLastError());
        size_t tmp = 0;
        CK(cub::DeviceScan::ExclusiveSum(nullptr, tmp, cnt, tab.ref_exc.as<uint32_t>(), (int)(n_blocks + 1), ctx->stream));
        CK(ctx->scan_tmp.ensure(tmp));
        CK(cub::DeviceScan::ExclusiveSum(ctx->scan_tmp.p, tmp, cnt, tab.ref_exc.as<uint32_t>(), (int)(n_blocks + 1), ctx->stream));
        unsigned long long h_other = 0;
        CK(cudaMemcpyAsync(&h_other, other, sizeof h_other, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        tab.dref.packed = tab.ref_packed.as<uint32_t>();
        tab.dref.pk_words = words + 2;
        tab.dref.pk_off = tab.ref_pk_off.as<uint64_t>();
        tab.dref.exc_pre = tab.ref_exc.as<uint32_t>();
        tab.dref.all_iupac = h_other == 0 ? 1u : 0u;
    }
    tab.dref.genome_len = ref->n_bases;
    tab.dref.n_chrom = ref->n_chrom;
    tab.dref.n_species = 0;
    tab.dref.chrom_species = nullptr;
    tab.dref.chrom_circular = nullptr;
    tab.dref.species_chrom_off = nullptr;
    tab.dref.expr_alias = nullptr;
    tab.dref.expr_chrom = nullptr;
    tab.dref.n_expressed = 0;
    tab.dref.chrom_has_polya = nullptr;
    ctx->trx.reset();
    tab.have_expr = false;
    if (ref->n_species > 0) {
        if (!ref->chrom_species || !ref->chrom_circular)
            return fail(ctx, NS_EINVAL, "ns_set_reference: n_species > 0 needs chrom_species and chrom_circular");
        std::vector<uint32_t> sp(ref->n_chrom);
        std::vector<uint8_t> circ(ref->n_chrom);
        CK(cudaMemcpy(sp.data(), ref->chrom_species, sp.size() * 4, cudaMemcpyDefault));
        CK(cudaMemcpy(circ.data(), ref->chrom_circular, circ.size(), cudaMemcpyDefault));
        tab.h_sp_off.assign(ref->n_species + 1, 0);
        for (uint32_t i = 0; i < ref->n_chrom; ++i) {
            if (sp[i] >= ref->n_species || (i > 0 && sp[i] < sp[i - 1]))
                return fail(ctx, NS_EINVAL, "ns_set_reference: chromosomes must be grouped by species in species order");
            tab.h_sp_off[sp[i] + 1] = i + 1;
        }
        for (uint32_t k = 1; k <= ref->n_species; ++k) {
            if (tab.h_sp_off[k] == 0) tab.h_sp_off[k] = tab.h_sp_off[k - 1];
            if (tab.h_sp_off[k] == tab.h_sp_off[k - 1]) return fail(ctx, NS_EINVAL, "ns_set_reference: species %u has no chromosome", k - 1);
        }
        CK(upload(tab.ref_species, sp.data(), sp.size() * 4, ctx->stream));
        CK(upload(tab.ref_circular, circ.data(), circ.size(), ctx->stream));
        CK(upload(tab.ref_sp_off, tab.h_sp_off.data(), tab.h_sp_off.size() * 4, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        tab.dref.n_species = ref->n_species;
        tab.dref.chrom_species = tab.ref_species.as<uint32_t>();
        tab.dref.chrom_circular = tab.ref_circular.as<uint8_t>();
        tab.dref.species_chrom_off = tab.ref_sp_off.as<uint32_t>();
    }
    tab.have_ref = true;
    tab.h_haploid_off.clear();
    tab.have_lift = false;
    for (DevBuf* b : {&tab.lift_seg, &tab.lift_kind, &tab.lift_first, &tab.lift_chrom, &tab.lift_hp}) b->release();
    tab.have_splice = false;
    for (DevBuf* b : {&tab.splice_exon, &tab.splice_first, &tab.splice_minus}) b->release();
    drop_aln_tags(tab);
    ctx->have_batch = false;
    ctx->opt_ok[0] = ctx->opt_ok[1] = false;
    return NS_OK;
}

// The checks ns_apply_variants and ns_set_lift make on the tables, against the haploid records' offsets `off`: *any_rc
// tells whether some variant is an inversion
static bool variants_given(const NsVariants* v) {
    return v && v->hap_chrom && v->var_off && v->n_hap != 0 && (!v->n_var || (v->var_pos && v->var_ref_len && v->alt_off && v->alt_len)) &&
           (!v->alt_bytes || v->alt);
}
static int check_variants(NsContext* ctx, const char* fname, const NsVariants* v, const std::vector<uint64_t>& off, bool* any_rc) {
    const uint32_t n_chrom = (uint32_t)(off.size() - 1);
    *any_rc = false;
    if (v->var_off[0] != 0 || v->var_off[v->n_hap] != v->n_var)
        return fail(ctx, NS_EINVAL, "%s: var_off must start at 0 and end at n_var", fname);
    for (uint32_t h = 0; h < v->n_hap; ++h) {
        const uint32_t c = v->hap_chrom[h];
        if (c >= n_chrom) return fail(ctx, NS_EINVAL, "%s: haplotype %u names record %u of %u", fname, h, c, n_chrom);
        if (v->var_off[h + 1] < v->var_off[h]) return fail(ctx, NS_EINVAL, "%s: var_off decreases at haplotype %u", fname, h);
        uint64_t end = 0;
        for (uint64_t j = v->var_off[h]; j < v->var_off[h + 1]; ++j) {
            const uint8_t kind = v->alt_kind ? v->alt_kind[j] : 0;
            if (kind > 2)
                return fail(ctx, NS_EINVAL, "%s: variant %llu of haplotype %u has ALT kind %u (0, 1 or 2)", fname, (unsigned long long)j, h,
                            (unsigned)kind);
            if (v->var_pos[j] < end || v->var_pos[j] + v->var_ref_len[j] > off[c + 1] - off[c])
                return fail(ctx, NS_EINVAL, "%s: variant %llu of haplotype %u overlaps the one before it or lies outside its record", fname,
                            (unsigned long long)j, h);
            const uint64_t src_bytes = kind ? off[c + 1] - off[c] : v->alt_bytes;      // kinds 1 and 2 read the source record
            if (v->alt_off[j] > src_bytes || v->alt_len[j] > src_bytes - v->alt_off[j])
                return fail(ctx, NS_EINVAL, "%s: the ALT of variant %llu of haplotype %u lies outside %s", fname, (unsigned long long)j, h,
                            kind ? "its source record" : "the ALT bytes");
            end = v->var_pos[j] + v->var_ref_len[j];
            *any_rc |= kind == 2;
        }
    }
    return NS_OK;
}

// The tables' uploads and hap_layout's segments (sources, lengths, output offsets) and record offsets, on the context's
// stream; the haploid records' offsets on the device are chrom_off.  ns_apply_variants and ns_set_lift share them.
struct VariantLayout {
    DevBuf hap_chrom, var_off, var_pos, var_ref_len, alt_off, alt_len, alt_kind, seg_src, seg_len, seg_out, hap_off;
    HapArgs args{};
    size_t bytes() const {
        return hap_chrom.cap + var_off.cap + var_pos.cap + var_ref_len.cap + alt_off.cap + alt_len.cap + alt_kind.cap + seg_src.cap +
               seg_len.cap + seg_out.cap + hap_off.cap;
    }
};
static cudaError_t variant_layout(NsContext* ctx, const NsVariants* v, const uint64_t* chrom_off, VariantLayout& L) {
    cudaStream_t st = ctx->stream;
    const uint64_t n_seg = 2 * v->n_var + v->n_hap;
    cudaError_t e = cudaSuccess;
    auto ok = [&](cudaError_t x) { return (e = x) == cudaSuccess; };
    if (!ok(upload(L.hap_chrom, v->hap_chrom, (size_t)v->n_hap * 4, st)) || !ok(upload(L.var_off, v->var_off, (size_t)(v->n_hap + 1) * 8, st)) ||
        !ok(upload(L.var_pos, v->var_pos, v->n_var * 8, st)) || !ok(upload(L.var_ref_len, v->var_ref_len, v->n_var * 4, st)) ||
        !ok(upload(L.alt_off, v->alt_off, v->n_var * 8, st)) || !ok(upload(L.alt_len, v->alt_len, v->n_var * 4, st)) ||
        (v->alt_kind && !ok(upload(L.alt_kind, v->alt_kind, v->n_var, st))) || !ok(L.seg_src.ensure(n_seg * 8)) ||
        !ok(L.seg_len.ensure((n_seg + 1) * 8)) || !ok(L.seg_out.ensure((n_seg + 1) * 8)) || !ok(L.hap_off.ensure((size_t)(v->n_hap + 1) * 8)))
        return e;
    L.args = HapArgs{L.hap_chrom.as<uint32_t>(), L.var_off.as<uint64_t>(), L.var_pos.as<uint64_t>(), L.var_ref_len.as<uint32_t>(),
                     L.alt_off.as<uint64_t>(), L.alt_len.as<uint32_t>(), v->alt_kind ? L.alt_kind.as<uint8_t>() : nullptr, chrom_off, v->n_hap,
                     n_seg, L.seg_src.as<uint64_t>(), L.seg_len.as<uint64_t>()};
    size_t tmp = 0;
    if (!ok(hap_layout(L.args, L.seg_out.as<uint64_t>(), L.hap_off.as<uint64_t>(), nullptr, &tmp, st)) || !ok(ctx->scan_tmp.ensure(tmp)))
        return e;
    return hap_layout(L.args, L.seg_out.as<uint64_t>(), L.hap_off.as<uint64_t>(), ctx->scan_tmp.p, &tmp, st);
}

int ns_apply_variants(NsContext* ctx, const NsVariants* v) {
    if (!ctx || !variants_given(v)) return fail(ctx, NS_EINVAL, "ns_apply_variants: null argument or no haplotype");
    if (ctx->clone) return fail(ctx, NS_ESTATE, "ns_apply_variants: a cloned context shares its parent's reference");
    Tables& tab = *ctx->tables;
    if (!tab.have_ref) return fail(ctx, NS_ESTATE, "ns_apply_variants: set the reference first (ns_set_reference or ns_bcast_nccl)");
    if (tab.dref.n_species) return fail(ctx, NS_EINVAL, "ns_apply_variants: a metagenome reference cannot carry variants");
    bool any_rc = false;                                            // an inversion: the gather's reverse-complement path
    if (int rc = check_variants(ctx, "ns_apply_variants", v, tab.h_chrom_off, &any_rc)) return rc;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const uint64_t n_seg = 2 * v->n_var + v->n_hap;
    DevBuf alt, out;
    VariantLayout lay;
    CK(variant_layout(ctx, v, tab.dref.chrom_off, lay));
    CK(alt.ensure(v->alt_bytes + 16));                              // hap_gather_kernel reads whole words behind the end
    if (v->alt_bytes) CK(cudaMemcpyAsync(alt.p, v->alt, v->alt_bytes, cudaMemcpyHostToDevice, st));
    const DevBuf &seg_src = lay.seg_src, &seg_out = lay.seg_out, &hap_off = lay.hap_off;
    uint64_t n_bases = 0;
    CK(cudaMemcpyAsync(&n_bases, seg_out.as<uint64_t>() + n_seg, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (n_bases == 0) return fail(ctx, NS_EINVAL, "ns_apply_variants: the haplotypes have no bases");
    CK(out.ensure(n_bases + 16));
    CK(hap_gather(tab.dref.bases, alt.as<uint8_t>(), seg_src.as<uint64_t>(), seg_out.as<uint64_t>(), n_seg, n_bases, any_rc, out.as<uint8_t>(),
                  st));
    CK(cudaStreamSynchronize(st));
    // accounted peak (sizes of the library's allocations, not a device reading) at the two high points: the haploid
    // reference beside the haplotypes, then the new resident copy (ns_set_reference's) beside them; the build's tables
    // and the scan's scratch space are held throughout
    const size_t build = lay.bytes() + alt.cap + out.cap + ctx->scan_tmp.cap;
    const size_t peak_a = build + tab.ref_bases.cap + tab.ref_off.cap + tab.ref_packed.cap + tab.ref_pk_off.cap + tab.ref_exc.cap;
    // the haploid bytes and their 2-bit copy go before ns_set_reference allocates the haplotypes' own
    tab.have_ref = false;
    tab.ref_bases.release();
    tab.ref_packed.release();
    std::vector<uint64_t> haploid_off = tab.h_chrom_off;
    NsReference r{};
    r.bases = out.as<uint8_t>();                    // device pointers: ns_set_reference copies from them
    r.n_bases = n_bases;
    r.chrom_off = hap_off.as<uint64_t>();
    r.n_chrom = v->n_hap;
    const int rc = ns_set_reference(ctx, &r);
    if (rc != NS_OK) return rc;
    tab.h_haploid_off = std::move(haploid_off);
    const size_t peak_b = build + tab.ref_bases.cap + tab.ref_off.cap + tab.ref_packed.cap + tab.ref_pk_off.cap + tab.ref_exc.cap;
    if (v->peak_bytes) *v->peak_bytes = std::max(peak_a, peak_b);
    return NS_OK;
}

int ns_set_lift(NsContext* ctx, const NsVariants* v) {
    static const char* fname = "ns_set_lift";
    if (!ctx || !variants_given(v)) return fail(ctx, NS_EINVAL, "%s: null argument or no haplotype", fname);
    if (ctx->clone) return fail(ctx, NS_ESTATE, "%s: a cloned context shares its parent's tables", fname);
    Tables& tab = *ctx->tables;
    if (!tab.have_ref || tab.h_haploid_off.empty())
        return fail(ctx, NS_ESTATE, "%s: the resident reference is not the haplotypes of ns_apply_variants", fname);
    bool any_rc = false;
    if (int rc = check_variants(ctx, fname, v, tab.h_haploid_off, &any_rc)) return rc;
    const std::vector<uint64_t>& off = tab.h_haploid_off;
    if (v->n_hap != tab.dref.n_chrom)
        return fail(ctx, NS_EINVAL, "%s: %u haplotypes for %u resident haplotype records", fname, v->n_hap, tab.dref.n_chrom);
    std::vector<uint64_t> first(v->n_hap + 1);                      // hap_seg_first: each record's first segment
    std::vector<uint8_t> hp(v->n_hap);                              // the haplotype's place among those of its source record
    for (uint32_t h = 0; h < v->n_hap; ++h) {
        const uint32_t c = v->hap_chrom[h];
        int64_t len = (int64_t)(off[c + 1] - off[c]);
        for (uint64_t j = v->var_off[h]; j < v->var_off[h + 1]; ++j) len += (int64_t)v->alt_len[j] - (int64_t)v->var_ref_len[j];
        const uint64_t resident = tab.h_chrom_off[h + 1] - tab.h_chrom_off[h];
        if ((uint64_t)len != resident)
            return fail(ctx, NS_EINVAL, "%s: haplotype %u has %lld bases by these tables, the resident record %u has %llu", fname, h,
                        (long long)len, h, (unsigned long long)resident);
        first[h] = 2 * v->var_off[h] + h;
        hp[h] = (uint8_t)(h > 0 && v->hap_chrom[h - 1] == c ? hp[h - 1] + 1 : 1);
    }
    first[v->n_hap] = 2 * v->n_var + v->n_hap;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    tab.have_lift = false;
    drop_aln_tags(tab);
    tab.h_lift_pair_off.assign(v->n_var + 1, 0);
    for (uint64_t j = 0; j < v->n_var; ++j)
        tab.h_lift_pair_off[j + 1] = tab.h_lift_pair_off[j] + ((v->alt_kind ? v->alt_kind[j] : 0) == HAP_LIFT_SEQ ? std::min(v->alt_len[j], v->var_ref_len[j]) : 0);
    DevBuf haploid;
    VariantLayout lay;
    CK(upload(haploid, off.data(), off.size() * 8, st));
    CK(variant_layout(ctx, v, haploid.as<uint64_t>(), lay));
    const uint64_t n_seg = lay.args.n_seg;
    CK(tab.lift_seg.ensure(n_seg * sizeof(HapLift)));
    CK(tab.lift_kind.ensure(n_seg));
    CK(hap_lift(lay.args, lay.seg_out.as<uint64_t>(), lay.hap_off.as<uint64_t>(), tab.lift_seg.as<HapLift>(), tab.lift_kind.as<uint8_t>(), st));
    CK(upload(tab.lift_first, first.data(), first.size() * 8, st));
    CK(upload(tab.lift_chrom, v->hap_chrom, (size_t)v->n_hap * 4, st));
    CK(upload(tab.lift_hp, hp.data(), hp.size(), st));
    CK(cudaStreamSynchronize(st));
    tab.have_lift = true;
    if (v->peak_bytes)
        *v->peak_bytes = tab.lift_seg.cap + tab.lift_kind.cap + tab.lift_first.cap + tab.lift_chrom.cap + tab.lift_hp.cap;
    return NS_OK;
}

int ns_set_splice(NsContext* ctx, const NsSplice* sp) {
    static const char* fname = "ns_set_splice";
    if (!ctx || !sp || !sp->exon_off || (sp->n_trx && !sp->minus) || (sp->n_genome && !sp->genome_len) ||
        (sp->exon_off[sp->n_trx] && (!sp->exon_chrom || !sp->exon_start || !sp->exon_len)))
        return fail(ctx, NS_EINVAL, "%s: null argument", fname);
    if (ctx->clone) return fail(ctx, NS_ESTATE, "%s: a cloned context shares its parent's tables", fname);
    Tables& tab = *ctx->tables;
    if (!tab.have_ref) return fail(ctx, NS_ESTATE, "%s: set the reference first (ns_set_reference or ns_bcast_nccl)", fname);
    const std::vector<uint64_t>& off = tab.h_chrom_off;
    const uint32_t n_res = tab.dref.n_chrom;
    if (sp->n_trx > n_res) return fail(ctx, NS_EINVAL, "%s: %u transcripts for %u resident records", fname, sp->n_trx, n_res);
    if (sp->genome_first != NS_SPLICE_NO_GENOME) {
        if (sp->genome_first < sp->n_trx || (uint64_t)sp->genome_first + sp->n_genome != n_res)
            return fail(ctx, NS_EINVAL, "%s: genome records %u .. %llu are not the resident records behind the %u transcripts", fname,
                        sp->genome_first, (unsigned long long)sp->genome_first + sp->n_genome, sp->n_trx);
        for (uint32_t g = 0; g < sp->n_genome; ++g) {
            const uint64_t res = off[sp->genome_first + g + 1] - off[sp->genome_first + g];
            if (sp->genome_len[g] != res)
                return fail(ctx, NS_EINVAL, "%s: genome record %u has %llu bases, the resident record %u has %llu", fname, g,
                            (unsigned long long)sp->genome_len[g], sp->genome_first + g, (unsigned long long)res);
        }
    }
    if (sp->exon_off[0] != 0) return fail(ctx, NS_EINVAL, "%s: exon_off must start at 0", fname);
    const uint64_t n_exon = sp->exon_off[sp->n_trx];
    if (n_exon > 0xffffffffull) return fail(ctx, NS_EINVAL, "%s: %llu exons are too many", fname, (unsigned long long)n_exon);
    std::vector<SpliceExon> ex(n_exon);
    for (uint32_t t = 0; t < sp->n_trx; ++t) {
        if (sp->exon_off[t + 1] < sp->exon_off[t]) return fail(ctx, NS_EINVAL, "%s: exon_off decreases at transcript %u", fname, t);
        const bool minus = sp->minus[t] != 0;
        uint64_t cum = 0;
        for (uint64_t j = sp->exon_off[t]; j < sp->exon_off[t + 1]; ++j) {
            const uint32_t c = sp->exon_chrom[j], s = sp->exon_start[j], l = sp->exon_len[j];
            if (c >= sp->n_genome || l == 0 || (uint64_t)s + l > sp->genome_len[c])
                return fail(ctx, NS_EINVAL, "%s: exon %llu of transcript %u leaves its genome record", fname,
                            (unsigned long long)(j - sp->exon_off[t]), t);
            if (j > sp->exon_off[t]) {
                const uint32_t pc = sp->exon_chrom[j - 1], ps = sp->exon_start[j - 1], pl = sp->exon_len[j - 1];
                if (c != pc || (minus ? s > ps : s < ps))
                    return fail(ctx, NS_EINVAL, "%s: the exons of transcript %u are not monotone in transcript order at exon %llu", fname,
                                t, (unsigned long long)(j - sp->exon_off[t]));
                if (minus ? (uint64_t)s + l > ps : s < (uint64_t)ps + pl)
                    return fail(ctx, NS_EINVAL, "%s: exons %llu and %llu of transcript %u overlap", fname,
                                (unsigned long long)(j - 1 - sp->exon_off[t]), (unsigned long long)(j - sp->exon_off[t]), t);
            }
            ex[j] = SpliceExon{c, s, l, (uint32_t)cum};
            cum += l;
        }
        const uint64_t res = off[t + 1] - off[t];
        if (sp->exon_off[t + 1] > sp->exon_off[t] && cum != res)
            return fail(ctx, NS_EINVAL, "%s: the exons of transcript %u add up to %llu bases, the resident record %u has %llu", fname, t,
                        (unsigned long long)cum, t, (unsigned long long)res);
    }
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    tab.have_splice = false;
    drop_aln_tags(tab);
    CK(upload(tab.splice_exon, ex.data(), std::max<size_t>(ex.size(), 1) * sizeof(SpliceExon), st));
    CK(upload(tab.splice_first, sp->exon_off, ((size_t)sp->n_trx + 1) * 8, st));
    CK(upload(tab.splice_minus, sp->minus, std::max<size_t>(sp->n_trx, 1), st));
    CK(cudaStreamSynchronize(st));
    tab.splice_n_trx = sp->n_trx;
    tab.splice_genome_first = sp->genome_first;
    tab.splice_n_genome = sp->n_genome;
    tab.have_splice = true;
    if (sp->peak_bytes) *sp->peak_bytes = tab.splice_exon.cap + tab.splice_first.cap + tab.splice_minus.cap;
    return NS_OK;
}

int ns_set_aln_tags(NsContext* ctx, const NsAlnTags* t) {
    static const char* fname = "ns_set_aln_tags";
    if (!ctx || !t || !t->ref_name_off || (t->ref_name_off[t->n_ref] && !t->ref_names) || (t->ref_paired_bytes && !t->ref_paired))
        return fail(ctx, NS_EINVAL, "%s: null argument", fname);
    if (ctx->clone) return fail(ctx, NS_ESTATE, "%s: a cloned context shares its parent's tables", fname);
    Tables& tab = *ctx->tables;
    if (!tab.have_ref) return fail(ctx, NS_ESTATE, "%s: set the reference first (ns_set_reference or ns_bcast_nccl)", fname);
    if (t->ref_name_off[0] != 0) return fail(ctx, NS_EINVAL, "%s: ref_name_off must start at 0", fname);
    for (uint32_t k = 0; k < t->n_ref; ++k)
        if (t->ref_name_off[k + 1] <= t->ref_name_off[k])
            return fail(ctx, NS_EINVAL, "%s: reference name %u is empty or ref_name_off decreases there", fname, k);
    const uint64_t n_var = tab.have_lift ? tab.h_lift_pair_off.size() - 1 : 0;
    const uint64_t paired = tab.have_lift ? tab.h_lift_pair_off.back() : 0;
    if (t->n_var != n_var)
        return fail(ctx, NS_EINVAL, "%s: the REF bytes table is for %llu variants, the lift has %llu", fname, (unsigned long long)t->n_var,
                    (unsigned long long)n_var);
    if (t->ref_paired_bytes != paired)
        return fail(ctx, NS_EINVAL, "%s: the REF bytes table has %llu bytes, the lift's ALTs pair %llu", fname,
                    (unsigned long long)t->ref_paired_bytes, (unsigned long long)paired);
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    drop_aln_tags(tab);
    CK(upload(tab.tag_sn, t->ref_names, t->ref_name_off[t->n_ref], st));
    CK(upload(tab.tag_sn_off, t->ref_name_off, ((size_t)t->n_ref + 1) * 8, st));
    CK(upload(tab.tag_pair, t->ref_paired, paired, st));
    if (tab.have_lift) CK(upload(tab.tag_pair_off, tab.h_lift_pair_off.data(), tab.h_lift_pair_off.size() * 8, st));
    CK(cudaStreamSynchronize(st));
    tab.tag_n_sn = t->n_ref;
    tab.have_aln_tags = true;
    if (t->peak_bytes) *t->peak_bytes = tab.tag_sn.cap + tab.tag_sn_off.cap + tab.tag_pair.cap + tab.tag_pair_off.cap;
    return NS_OK;
}

int ns_set_model(NsContext* ctx, const NsModel* m) {
    if (!ctx || !m) return fail(ctx, NS_EINVAL, "ns_set_model: null argument");
    if (ctx->clone) return fail(ctx, NS_ESTATE, "ns_set_model: a cloned context shares its parent's model");
    if (m->n_match_bins == 0 || m->n_match_bins > NS_MAX_BINS || m->n_tables != 4 + m->n_match_bins)
        return fail(ctx, NS_EINVAL, "ns_set_model: need 1..%d match bins and 4+bins alias tables", NS_MAX_BINS);
    if (!m->alias_prob || !m->alias_idx || !m->alias_desc || !m->match_bin_lo || !m->match_bin_hi)
        return fail(ctx, NS_EINVAL, "ns_set_model: null table pointer");
    CK(cudaSetDevice(ctx->device));
    Tables& tab = *ctx->tables;
    tab.hmodel = *m;
    DevModel& d = tab.dmodel;
    const NsKde* src[5] = {&m->kde_aligned, &m->kde_ht, &m->kde_ht_ratio, &m->kde_unaligned, &m->kde_gap};
    DevKde* dst[5] = {&d.aligned, &d.ht, &d.ratio, &d.unaligned, &d.gap};
    for (int i = 0; i < 5; ++i) {
        if (src[i]->n && !src[i]->data) return fail(ctx, NS_EINVAL, "ns_set_model: KDE %d has n>0 but no data", i);
        CK(upload(tab.kde[i], src[i]->data, (size_t)src[i]->n * sizeof(float), ctx->stream));
        dst[i]->data = tab.kde[i].as<float>();
        dst[i]->n = src[i]->n;
        dst[i]->bw = src[i]->bandwidth;
    }
    if ((m->kde_aligned.n == 0 && m->n_kde2d == 0) || m->kde_ht.n == 0 || m->kde_ht_ratio.n == 0)
        return fail(ctx, NS_EINVAL, "ns_set_model: aligned (or 2-D aligned) / ht / ht_ratio KDEs are required");
    d.kde2d_x = d.kde2d_y = nullptr;
    d.n_kde2d = 0;
    d.kde2d_bw = 0.f;
    if (m->n_kde2d > 0) {
        if (!m->kde2d_x || !m->kde2d_y) return fail(ctx, NS_EINVAL, "ns_set_model: n_kde2d > 0 needs kde2d_x / kde2d_y");
        std::vector<float> hx(m->n_kde2d);
        CK(cudaMemcpy(hx.data(), m->kde2d_x, hx.size() * sizeof(float), cudaMemcpyDefault));
        for (uint32_t i = 1; i < m->n_kde2d; ++i)
            if (hx[i] < hx[i - 1]) return fail(ctx, NS_EINVAL, "ns_set_model: kde2d_x must be sorted ascending");
        CK(upload(tab.kde2d_x, m->kde2d_x, (size_t)m->n_kde2d * sizeof(float), ctx->stream));
        CK(upload(tab.kde2d_y, m->kde2d_y, (size_t)m->n_kde2d * sizeof(float), ctx->stream));
        d.kde2d_x = tab.kde2d_x.as<float>();
        d.kde2d_y = tab.kde2d_y.as<float>();
        d.n_kde2d = m->n_kde2d;
        d.kde2d_bw = m->kde2d_bandwidth;
    }
    // interleave (prob, alias) so that one 8-byte load serves a draw
    std::vector<uint32_t> hp(m->alias_len), hi(m->alias_len), desc(2 * m->n_tables);
    CK(cudaMemcpy(hp.data(), m->alias_prob, hp.size() * 4, cudaMemcpyDefault));
    CK(cudaMemcpy(hi.data(), m->alias_idx, hi.size() * 4, cudaMemcpyDefault));
    CK(cudaMemcpy(desc.data(), m->alias_desc, desc.size() * 4, cudaMemcpyDefault));
    std::vector<uint2> inter(m->alias_len);
    for (uint32_t i = 0; i < m->alias_len; ++i) inter[i] = make_uint2(hp[i], hi[i]);
    CK(upload(tab.alias, inter.data(), inter.size() * sizeof(uint2), ctx->stream));
    d.alias = tab.alias.as<uint2>();
    for (uint32_t t = 0; t < m->n_tables; ++t) {
        d.tab_off[t] = desc[2 * t];
        d.tab_n[t] = desc[2 * t + 1];
        if (d.tab_n[t] == 0 || (uint64_t)d.tab_off[t] + d.tab_n[t] > m->alias_len)
            return fail(ctx, NS_EINVAL, "ns_set_model: alias table %u out of range", t);
    }
    std::vector<uint32_t> blo(m->n_match_bins), bhi(m->n_match_bins);
    CK(cudaMemcpy(blo.data(), m->match_bin_lo, blo.size() * 4, cudaMemcpyDefault));
    CK(cudaMemcpy(bhi.data(), m->match_bin_hi, bhi.size() * 4, cudaMemcpyDefault));
    d.n_bins = m->n_match_bins;
    for (uint32_t b = 0; b < d.n_bins; ++b) {
        d.bin_lo[b] = blo[b];
        d.bin_hi[b] = bhi[b];
    }
    memcpy(d.trans, m->trans, sizeof d.trans);
    d.strandness = m->strandness_rate;
    d.seg_p = m->segment_mean > 1.0f ? 1.0 / (double)m->segment_mean : 1.0;
    std::vector<uint32_t> lut;
    build_qlut(m->qual_cdf, lut);
    CK(upload(tab.qlut, lut.data(), lut.size() * 4, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    tab.have_model = true;
    ctx->have_batch = false;
    ctx->opt_ok[0] = ctx->opt_ok[1] = false;
    return NS_OK;
}

int ns_configure(NsContext* ctx, const NsRunConfig* cfg) {
    if (!ctx || !cfg) return fail(ctx, NS_EINVAL, "ns_configure: null argument");
    const Tables& tab = *ctx->tables;
    if (cfg->mode > 2) return fail(ctx, NS_EINVAL, "ns_configure: mode must be 0 (genome), 1 (metagenome) or 2 (transcriptome)");
    if (cfg->mode == 2 && cfg->chimeric) return fail(ctx, NS_EINVAL, "ns_configure: transcriptome reads are not chimeric");
    if (cfg->mode == 2 && tab.have_model && tab.dmodel.n_kde2d == 0)
        return fail(ctx, NS_ESTATE, "ns_configure: transcriptome mode needs _aligned_region_2d.pkl in the model");
    if (cfg->mode == 1 && tab.have_ref && tab.dref.n_species == 0)
        return fail(ctx, NS_ESTATE, "ns_configure: metagenome mode needs a reference with species information");
    if (cfg->mode == 1 && cfg->kmer_bias != 0) return fail(ctx, NS_EINVAL, "ns_configure: -hp/-k is not offered in metagenome mode");
    if (cfg->max_len < cfg->min_len) return fail(ctx, NS_EINVAL, "Maximum read length must be longer than Minimum read length!");
    if (cfg->perfect && cfg->chimeric) return fail(ctx, NS_EINVAL, "Perfect reads cannot be chimeric");
    if ((cfg->median_len != 0.0) != (cfg->sd_len != 0.0))
        return fail(ctx, NS_EINVAL, "Please provide both mean and standard deviation of read length!");
    if (cfg->median_len != 0.0 && cfg->chimeric) return fail(ctx, NS_EINVAL, "Lognormal distributed reads cannot be chimeric!");
    if (cfg->median_len < 0.0 || cfg->sd_len < 0.0) return fail(ctx, NS_EINVAL, "ns_configure: negative -med/-sd");
    if (cfg->kmer_bias != 0 && tab.have_model && !tab.hmodel.has_hp)
        return fail(ctx, NS_ESTATE, "ns_configure: -hp/-k needs _hp_lengths_model_parameters.tsv in the model");
    if (cfg->kmer_bias == 1) return fail(ctx, NS_EINVAL, "ns_configure: -k must be >= 2 (every base is a run of length 1)");
    ctx->hcfg = *cfg;
    ctx->dcfg.circular = cfg->circular;
    ctx->dcfg.perfect = cfg->perfect;
    ctx->dcfg.fastq = cfg->fastq;
    ctx->dcfg.chimeric = cfg->chimeric;
    ctx->dcfg.kmer_bias = cfg->kmer_bias;
    ctx->dcfg.metagenome = cfg->mode == 1 ? 1u : 0u;
    ctx->dcfg.transcriptome = cfg->mode == 2 ? 1u : 0u;
    ctx->dcfg.uracil = (cfg->flags & NS_FLAG_URACIL) ? 1u : 0u;
    ctx->dcfg.kde2d_n = cfg->kde2d_sample ? cfg->kde2d_sample : 1u;
    ctx->dcfg.trx_records = cfg->trx_records;
    if (cfg->mode == 2 && tab.have_ref) {
        // records sorted by length for the unaligned reads' transcript draw (plan_kernel.cuh:draw_position_trx)
        const uint32_t nrec = cfg->trx_records ? std::min(cfg->trx_records, tab.dref.n_chrom) : tab.dref.n_chrom;
        if (!ctx->trx || ctx->trx->n != nrec) {
            std::vector<uint32_t> idx(nrec), both(2 * (size_t)nrec);
            for (uint32_t i = 0; i < nrec; ++i) idx[i] = i;
            const std::vector<uint64_t>& off = tab.h_chrom_off;
            std::stable_sort(idx.begin(), idx.end(), [&](uint32_t x, uint32_t y) { return off[x + 1] - off[x] < off[y + 1] - off[y]; });
            for (uint32_t i = 0; i < nrec; ++i) {
                both[i] = (uint32_t)(off[idx[i] + 1] - off[idx[i]]);
                both[nrec + i] = idx[i];
            }
            CK(cudaSetDevice(ctx->device));
            auto trx = std::make_shared<TrxTable>();
            CK(upload(trx->buf, both.data(), both.size() * 4, ctx->stream));
            CK(cudaStreamSynchronize(ctx->stream));
            trx->n = nrec;
            ctx->trx = std::move(trx);
        }
    }
    ctx->dcfg.polya_scale = cfg->polya_scale;
    ctx->dcfg.min_len = cfg->min_len;
    ctx->dcfg.max_len = std::min(cfg->max_len, 0x0fffffffu);
    ctx->dcfg.seed = ctx->seed;
    ctx->dcfg.median_len = cfg->median_len;
    ctx->dcfg.sd_len = cfg->sd_len;
    ctx->have_cfg = true;
    ctx->have_batch = false;
    ctx->opt_ok[0] = ctx->opt_ok[1] = false;
    return NS_OK;
}

int ns_set_abundance(NsContext* ctx, const double* abun, const double* abun_inflated, uint32_t n_species) {
    if (!ctx || !abun || n_species == 0) return fail(ctx, NS_EINVAL, "ns_set_abundance: null argument");
    const Tables& tab = *ctx->tables;
    if (!tab.have_ref || tab.dref.n_species != n_species)
        return fail(ctx, NS_ESTATE, "ns_set_abundance: the reference has %u species, got %u", tab.dref.n_species, n_species);
    ctx->abun.assign(abun, abun + n_species);
    if (abun_inflated) ctx->abun_inflated.assign(abun_inflated, abun_inflated + n_species);
    else ctx->abun_inflated.assign(n_species, 0.0);
    ctx->species_bases.assign(n_species, 0.0);
    return NS_OK;
}

int ns_set_expression(NsContext* ctx, const NsExpression* ex) {
    if (!ctx || !ex || !ex->alias_prob || !ex->alias_idx || !ex->expr_chrom || ex->n_expressed == 0)
        return fail(ctx, NS_EINVAL, "ns_set_expression: null argument or no expressed transcript");
    Tables& tab = *ctx->tables;
    if (!tab.have_ref) return fail(ctx, NS_ESTATE, "ns_set_expression: set the reference transcriptome first");
    if (ctx->clone) return fail(ctx, NS_ESTATE, "ns_set_expression: a cloned context shares its parent's tables");
    CK(cudaSetDevice(ctx->device));
    const uint32_t n = ex->n_expressed;
    std::vector<uint32_t> hp(n), hi(n), hc(n);
    CK(cudaMemcpy(hp.data(), ex->alias_prob, n * 4, cudaMemcpyDefault));
    CK(cudaMemcpy(hi.data(), ex->alias_idx, n * 4, cudaMemcpyDefault));
    CK(cudaMemcpy(hc.data(), ex->expr_chrom, n * 4, cudaMemcpyDefault));
    std::vector<uint2> inter(n);
    for (uint32_t i = 0; i < n; ++i) {
        if (hi[i] >= n || hc[i] >= tab.dref.n_chrom) return fail(ctx, NS_EINVAL, "ns_set_expression: index out of range at %u", i);
        inter[i] = make_uint2(hp[i], hi[i]);
    }
    CK(upload(tab.expr_alias, inter.data(), inter.size() * sizeof(uint2), ctx->stream));
    CK(upload(tab.expr_chrom, hc.data(), hc.size() * 4, ctx->stream));
    tab.dref.expr_alias = tab.expr_alias.as<uint2>();
    tab.dref.expr_chrom = tab.expr_chrom.as<uint32_t>();
    tab.dref.n_expressed = n;
    tab.dref.chrom_has_polya = nullptr;
    if (ex->chrom_has_polya) {
        CK(upload(tab.chrom_polya, ex->chrom_has_polya, tab.dref.n_chrom, ctx->stream));
        tab.dref.chrom_has_polya = tab.chrom_polya.as<uint8_t>();
    }
    CK(cudaStreamSynchronize(ctx->stream));
    tab.have_expr = true;
    ctx->have_batch = false;
    return NS_OK;
}

// ---- assign_species (:758-811) on the host: a sequential greedy pass over the batch's segments.
namespace {
struct HostRng {       // splitmix64 stream keyed by (seed, batch id); only drives the species choices
    uint64_t s;
    uint64_t next() {
        uint64_t z = (s += 0x9E3779B97F4A7C15ull);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        return z ^ (z >> 31);
    }
    double uniform() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
    uint32_t below(uint32_t n) { return (uint32_t)(((unsigned __int128)next() * n) >> 64); }
};

// reads: order = reads with the most segments first (stable), then single-segment reads by decreasing length;
// quota[s] = total_bases * abun[s] / sum(abun) - current[s]; every segment takes a uniformly random species whose quota
// still fits it (else any species with quota left); later segments of a chimeric read stay in the previous species with
// probability abun_inflated[prev] % (:793-797).
// seg_len[j]: drawn length of segment j (segments of read i are first[i] .. first[i] + n_seg[i]); by_len: read slots by
// decreasing total drawn length (the device's stable radix sort, = decreasing segment length for single-segment reads).
// The species whose quota exceeds a length are a PREFIX of the species sorted by quota, so a pick is a binary search + one
// uniform draw, and charging a quota moves one species a few places down that order.
void assign_species_host(const std::vector<uint32_t>& n_seg, const std::vector<uint32_t>& first, const std::vector<uint32_t>& seg_len,
                         const std::vector<uint32_t>& by_len, std::vector<uint32_t>& seg_species, const std::vector<double>& abun,
                         const std::vector<double>& inflated, const std::vector<double>& current, HostRng& rng) {
    const uint32_t n = (uint32_t)n_seg.size(), S = (uint32_t)abun.size();
    std::vector<uint32_t> order;
    order.reserve(n);
    for (uint32_t k = NS_MAX_SEGMENTS; k >= 2; --k)                        // most segments first, stable
        for (uint32_t i = 0; i < n; ++i)
            if (n_seg[i] == k) order.push_back(i);
    for (uint32_t q = 0; q < n; ++q)
        if (n_seg[by_len[q]] <= 1) order.push_back(by_len[q]);
    double to_add = 0, cur = 0, tot_abun = 0;
    for (uint32_t v : seg_len) to_add += v;
    for (uint32_t s = 0; s < S; ++s) {
        cur += current[s];
        tot_abun += abun[s];
    }
    std::vector<double> quota(S);
    for (uint32_t s = 0; s < S; ++s) quota[s] = (to_add + cur) * abun[s] / tot_abun - current[s];
    std::vector<uint32_t> ord(S), where(S);                                // species by decreasing quota, and its inverse
    for (uint32_t s = 0; s < S; ++s) ord[s] = s;
    std::stable_sort(ord.begin(), ord.end(), [&](uint32_t x, uint32_t y) { return quota[x] > quota[y]; });
    for (uint32_t k = 0; k < S; ++k) where[ord[k]] = k;
    auto count_above = [&](double v) {                                      // species with quota > v
        uint32_t lo = 0, hi = S;
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (quota[ord[mid]] > v) lo = mid + 1; else hi = mid;
        }
        return lo;
    };
    auto pick_above = [&](double v, int exclude) -> uint32_t {              // uniform among them, `exclude` left out
        const uint32_t c = count_above(v);
        const bool ex_in = exclude >= 0 && where[exclude] < c;
        const uint32_t m = c - (ex_in ? 1u : 0u);
        if (m == 0) return 0xffffffffu;
        uint32_t r = rng.below(m);
        if (ex_in && r >= where[exclude]) ++r;
        return ord[r];
    };
    auto pick = [&](double len, int exclude) -> uint32_t {
        uint32_t sp = pick_above(len, exclude);                             // quota - len > 0
        if (sp == 0xffffffffu && exclude < 0) sp = pick_above(0.0, -1);     // else any species with quota left
        return sp;
    };
    auto charge = [&](uint32_t sp, double len) {
        quota[sp] -= len;
        uint32_t k = where[sp];
        while (k + 1 < S && quota[ord[k + 1]] > quota[sp]) {               // keeps `ord` sorted
            ord[k] = ord[k + 1];
            where[ord[k]] = k;
            ++k;
        }
        ord[k] = sp;
        where[sp] = k;
    };
    for (uint32_t oi = 0; oi < n; ++oi) {
        const uint32_t i = order[oi];
        int pre = -1;
        for (uint32_t q = 0; q < n_seg[i]; ++q) {
            const double len = seg_len[first[i] + q];
            uint32_t sp;
            if (q == 0) {
                sp = pick(len, -1);
            } else {
                const double p = rng.uniform() * 100.0;
                uint32_t other = pick(len, pre);
                if (p <= inflated[pre] && quota[pre] > 0) sp = (uint32_t)pre;
                else if (p > inflated[pre] && other != 0xffffffffu) sp = other;
                else sp = pick(len, -1);
            }
            if (sp == 0xffffffffu) sp = ord[0];           // cannot happen while sum(quota) >= len; keep it total anyway
            seg_species[first[i] + q] = sp;
            charge(sp, len);
            pre = (int)sp;
        }
    }
}

// segment lengths down / species up: 4 bytes per segment instead of whole NsPieceMeta records
__global__ void gather_segment_req(const NsPieceMeta* pieces, const uint32_t* piece_first, const uint32_t* n_seg, uint32_t n_reads,
                                   const uint32_t* seg_first, uint32_t* out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_reads) return;
    const uint32_t pf = piece_first ? piece_first[i] : i, ns = n_seg ? n_seg[i] : 1u, sf = seg_first ? seg_first[i] : i;
    for (uint32_t q = 0; q < ns; ++q) out[sf + q] = pieces[pf + 2 * q].ref_req;
}
__global__ void scatter_segment_species(NsPieceMeta* pieces, const uint32_t* piece_first, const uint32_t* n_seg, uint32_t n_reads,
                                        const uint32_t* seg_first, const uint32_t* species) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_reads) return;
    const uint32_t pf = piece_first ? piece_first[i] : i, ns = n_seg ? n_seg[i] : 1u, sf = seg_first ? seg_first[i] : i;
    for (uint32_t q = 0; q < ns; ++q) pieces[pf + 2 * q].chrom = species[sf + q];    // species id travels in `chrom` until the position is drawn
}

__global__ void species_bases_kernel(const NsPieceMeta* pieces, uint32_t n, const uint32_t* chrom_species, double* acc) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && NS_PIECE_KIND(pieces[i].kind) == NS_PIECE_SEGMENT) atomicAdd(&acc[chrom_species[pieces[i].chrom]], (double)pieces[i].ref_len);
}
}  // namespace

namespace {
__global__ void hp_piece_keys(const NsPieceMeta* pieces, uint32_t n, uint32_t* keys, uint32_t* vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    keys[i] = NS_PIECE_KIND(pieces[i].kind) == NS_PIECE_SEGMENT ? pieces[i].ref_len : 0u;
    vals[i] = i;
}

// keep_off: the read keeps its slot in the sequence buffer (its bytes are overwritten in place)
__global__ void replace_reads(NsReadMeta* reads, const uint32_t* slots, const NsReadMeta* repl, uint32_t n, uint32_t n_reads,
                              uint32_t keep_off) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && slots[i] < n_reads) {
        NsReadMeta r = repl[i];
        if (keep_off) r.seq_off = reads[slots[i]].seq_off;
        reads[slots[i]] = r;
    }
}
__global__ void gather_seq_len(const NsReadMeta* reads, const uint32_t* slots, uint32_t n, uint32_t n_reads, uint32_t* out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = slots[i] < n_reads ? reads[slots[i]].seq_len : 0u;
}
__global__ void iota_from(uint32_t* v, uint32_t n, uint32_t first) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = first + i;
}
}  // namespace

int ns_simulate(NsContext* ctx, int kind, uint64_t first_read_id, uint32_t n_reads, NsBatchInfo* info) {
    if (!ctx) return NS_EINVAL;
    const Tables& tab = *ctx->tables;
    if (!tab.have_ref || !tab.have_model || !ctx->have_cfg)
        return fail(ctx, NS_ESTATE, "ns_simulate: reference, model and run configuration must be set first");
    if (kind != NS_KIND_ALIGNED && kind != NS_KIND_UNALIGNED) return fail(ctx, NS_EINVAL, "ns_simulate: bad kind %d", kind);
    if (kind == NS_KIND_UNALIGNED && tab.dmodel.unaligned.n == 0 && ctx->hcfg.median_len == 0.0)
        return fail(ctx, NS_ESTATE, "ns_simulate: model has no unaligned-length KDE");
    if (kind == NS_KIND_ALIGNED && ctx->hcfg.chimeric && tab.dmodel.gap.n == 0)
        return fail(ctx, NS_ESTATE, "ns_simulate: chimeric simulation needs the gap-length KDE");
    if (ctx->dcfg.transcriptome && kind == NS_KIND_ALIGNED && !tab.have_expr)
        return fail(ctx, NS_ESTATE, "ns_simulate: transcriptome mode needs ns_set_expression");
    if (ctx->hcfg.fastq && !tab.hmodel.has_qual)
        return fail(ctx, NS_ESTATE, "ns_simulate: --fastq needs base-quality parameters in the model");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    ctx->have_batch = false;
    ctx->z_out.valid = ctx->ep_out.valid = false;
    memset(&ctx->last, 0, sizeof ctx->last);
    if (n_reads == 0) {
        if (info) *info = ctx->last;
        ctx->have_batch = true;
        ctx->last_kind = kind;
        return NS_OK;
    }
    const uint32_t n = n_reads;
    const bool chim = (kind == NS_KIND_ALIGNED) && ctx->hcfg.chimeric;
    const bool species = ctx->dcfg.metagenome && kind == NS_KIND_ALIGNED;
    const bool hp = ctx->hcfg.kmer_bias > 0 && kind == NS_KIND_ALIGNED;
    const bool fast_unaligned = kind == NS_KIND_UNALIGNED && !(ctx->hcfg.flags & NS_FLAG_UNALIGNED_SCRIPTS);
    // One submission, no host round trip (DESIGN §3): a kind of batch without a chimeric piece count, species assignment,
    // homopolymer pass or scripted unaligned reads in the way, of which a batch at least this large has run sized.
    const bool may_sync_free = !chim && !species && !hp && (kind == NS_KIND_ALIGNED || fast_unaligned);
    const bool sync_free = may_sync_free && ctx->opt_ok[kind] && n <= ctx->opt_n[kind] && ctx->ops.cap > 64 && ctx->seq.cap > 64 &&
                           (!ctx->hcfg.fastq || ctx->qual.cap >= ctx->seq.cap);
    const DevRef dref = dev_ref(ctx);
    const unsigned tb = 256, gb = (n + tb - 1) / tb;
    CK(ctx->reads.ensure((size_t)n * sizeof(NsReadMeta)));
    CK(ctx->counter.ensure(64));
    CK(ctx->totals.ensure(NS_T_COUNT * sizeof(uint64_t)));
    CK(ctx->scan_in.ensure((size_t)n * (2 * NS_MAX_SEGMENTS) * sizeof(uint64_t)));
    CK(ctx->scan_out.ensure((size_t)n * (2 * NS_MAX_SEGMENTS) * sizeof(uint64_t)));
    CK(cudaMemsetAsync(ctx->totals.p, 0, NS_T_COUNT * sizeof(uint64_t), st));
    CK(cudaEventRecord(ctx->ev[0], st));
    const uint64_t ops_cap = ctx->ops.cap / sizeof(uint32_t), seq_cap = ctx->seq.cap;
    uint64_t* d_totals = ctx->totals.as<uint64_t>();
    const uint64_t* h_totals = ctx->h_totals.as<uint64_t>();      // as of the last publish_totals_and_wait
    auto script_ops = [h_totals] { return h_totals[NS_T_PRIMARY] + h_totals[NS_T_OVERFLOW_OPS] + h_totals[NS_T_HP_OPS]; };
    uint64_t* scan_in = ctx->scan_in.as<uint64_t>();
    uint64_t* scan_out = ctx->scan_out.as<uint64_t>();
    const uint32_t* d_abort = sync_free ? (const uint32_t*)(d_totals + NS_T_ABORT) : nullptr;

    // ---- pieces per read
    uint32_t n_pieces = n;
    const uint32_t* d_nseg = nullptr;
    const uint32_t* d_pfirst = nullptr;
    if (chim) {
        CK(ctx->nseg.ensure((size_t)n * 4));
        CK(ctx->npieces.ensure((size_t)n * 4));
        CK(ctx->piece_first.ensure((size_t)n * 4));
        CK(launch(ctx, segments_kernel, gb, tb, 0, tab.dmodel, ctx->dcfg, (uint32_t)kind, first_read_id, n, ctx->nseg.as<uint32_t>(),
                  ctx->npieces.as<uint32_t>()));
        CK(launch(ctx, widen_u32, gb, tb, 0, ctx->npieces.as<uint32_t>(), n, scan_in));
        if (int rc = scan_total(ctx, scan_in, scan_out, n, NS_T_PIECES)) return rc;
        CK(launch(ctx, narrow_u64, gb, tb, 0, scan_out, n, ctx->piece_first.as<uint32_t>()));
        if (int rc = publish_totals_and_wait(ctx)) return rc;
        n_pieces = (uint32_t)h_totals[NS_T_PIECES];
        d_nseg = ctx->nseg.as<uint32_t>();
        d_pfirst = ctx->piece_first.as<uint32_t>();
    }
    CK(ctx->pieces.ensure((size_t)(n_pieces + 1) * sizeof(NsPieceMeta)));
    CK(cudaMemsetAsync(ctx->pieces.p, 0, (size_t)(n_pieces + 1) * sizeof(NsPieceMeta), st));
    const unsigned gp = (n_pieces + tb - 1) / tb;
    NsReadMeta* reads = ctx->reads.as<NsReadMeta>();
    NsPieceMeta* pieces = ctx->pieces.as<NsPieceMeta>();

    // ---- generation-0 lengths -> op-slot capacities (scan) and processing order (longest reads first)
    CK(ctx->sort_keys.ensure((size_t)n * 8));
    CK(ctx->sort_vals.ensure((size_t)n * 8));
    uint32_t* keys_in = ctx->sort_keys.as<uint32_t>();
    uint32_t* keys_out = keys_in + n;
    uint32_t* vals_in = ctx->sort_vals.as<uint32_t>();
    uint32_t* vals_out = vals_in + n;
    const bool exact_only = (kind == NS_KIND_UNALIGNED) && !fast_unaligned;
    CK(launch(ctx, lengths_kernel, gb, tb, 0, tab.dmodel, ctx->dcfg, (uint32_t)kind, first_read_id, n, d_nseg, d_pfirst, pieces,
              1.0f / std::max(1.0f, tab.hmodel.mean_ref_per_event), std::min(8.0f, std::max(1.0f, tab.hmodel.ref_per_event_cv)),
              exact_only ? 1u : 0u, scan_in, keys_in, vals_in));
    if (int rc = scan_total(ctx, scan_in, scan_out, n_pieces, NS_T_SLOT_OPS)) return rc;
    CK(launch(ctx, scatter_piece_off, gp, tb, 0, pieces, n_pieces, scan_out));
    CK(launch(ctx, set_sentinel_off, 1, 32, 0, pieces, n_pieces, d_totals + NS_T_SLOT_OPS));
    if (int rc = sort_pairs_descending(ctx, keys_in, keys_out, vals_in, vals_out, n)) return rc;
    // primary script area = the capped slots (+ a bump pool for re-drawn unaligned reads, uread_kernel.cuh)
    CK(launch(ctx, capacity_stage_a, 1, 32, 0, d_totals, fast_unaligned ? 1u : 0u, sync_free ? ops_cap : ~0ull));
    if (!sync_free) {
        if (int rc = publish_totals_and_wait(ctx)) return rc;
        CK(ctx->ops.ensure((size_t)(h_totals[NS_T_PRIMARY] + 4) * sizeof(uint32_t)));
    }
    uint32_t batch_reversed = 0;
    if (species) {
        // ---- assign_species (:758-811): sequential greedy quota fill over this batch's segments, on the host.  Down: the
        //      drawn segment lengths and the reads' order by length (4 B each); up: one species per segment.
        if (ctx->abun.size() != tab.dref.n_species) return fail(ctx, NS_ESTATE, "ns_simulate: call ns_set_abundance first");
        std::vector<uint32_t> hseg(n, 1u), hfirst(n), by_len(n);
        uint32_t n_segs = n;
        if (chim) {
            CK(cudaMemcpyAsync(hseg.data(), ctx->nseg.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            n_segs = 0;
            for (uint32_t i = 0; i < n; ++i) {
                hfirst[i] = n_segs;
                n_segs += hseg[i];
            }
        } else {
            for (uint32_t i = 0; i < n; ++i) hfirst[i] = i;
        }
        CK(ctx->hp_off.ensure((size_t)(n + n_segs) * 4));                 // scratch: segment starts + per-segment values
        uint32_t* d_sfirst = ctx->hp_off.as<uint32_t>();
        uint32_t* d_segval = d_sfirst + n;
        if (chim) CK(cudaMemcpyAsync(d_sfirst, hfirst.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
        CK(launch(ctx, gather_segment_req, gb, tb, 0, pieces, d_pfirst, d_nseg, n, chim ? d_sfirst : nullptr, d_segval));
        std::vector<uint32_t> seg_len(n_segs), seg_species(n_segs, 0u);
        CK(cudaMemcpyAsync(seg_len.data(), d_segval, (size_t)n_segs * 4, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(by_len.data(), vals_out, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        HostRng hr{ctx->seed * 0x9E3779B97F4A7C15ull ^ (first_read_id + 0x1234567ull)};
        batch_reversed = hr.uniform() > (double)tab.dmodel.strandness ? 1u : 0u;      // once per batch (:860)
        assign_species_host(hseg, hfirst, seg_len, by_len, seg_species, ctx->abun, ctx->abun_inflated, ctx->species_bases, hr);
        CK(cudaMemcpyAsync(d_segval, seg_species.data(), (size_t)n_segs * 4, cudaMemcpyHostToDevice, st));
        CK(launch(ctx, scatter_segment_species, gb, tb, 0, pieces, d_pfirst, d_nseg, n, chim ? d_sfirst : nullptr, d_segval));
        CK(cudaStreamSynchronize(st));                                    // seg_species must outlive the copy
    }
    CK(cudaEventRecord(ctx->ev[1], st));

    // ---- plan: rejection loops, positions, edit scripts (single pass)
    PlanArgs pa;
    pa.m = tab.dmodel;
    pa.ref = dref;
    pa.cfg = ctx->dcfg;
    pa.kind = (uint32_t)kind;
    pa.first_id = first_read_id;
    pa.n_reads = n;
    pa.n_seg = d_nseg;
    pa.piece_first = d_pfirst;
    pa.reads = reads;
    pa.pieces = pieces;
    pa.ops = ctx->ops.as<uint32_t>();
    pa.order = vals_out;
    pa.counter = ctx->counter.as<uint32_t>();
    pa.n_flagged = (uint32_t*)(d_totals + NS_T_FLAGGED);
    pa.batch_reversed = batch_reversed;
    pa.abort = d_abort;
    const unsigned plan_tb = 128;
    // 2 resident blocks per SM rather than 4 (the register limit): the lanes' scattered memory accesses (script stores,
    // alias loads) share one memory pipeline, which more warps only queue on, and another context's emit kernel still
    // finds room on every SM (transcripts are short -- 1-2 kb reads, no long tail, two passes: there the register limit
    // of 4 blocks is used).  NANOSIM_B200_PLAN_BLOCKS_PER_SM overrides the cap.  DESIGN.md §10 has the H100 sweep.
    static const int plan_per_sm_env = env_int("NANOSIM_B200_PLAN_BLOCKS_PER_SM", 0);
    const int plan_per_sm = plan_per_sm_env > 0 ? plan_per_sm_env : (ctx->dcfg.transcriptome ? 4 : 2);
    unsigned plan_blocks = std::min<unsigned>((n + plan_tb - 1) / plan_tb, (unsigned)ctx->sm_count * (unsigned)std::max(1, plan_per_sm));
    // unaligned reads without NS_FLAG_UNALIGNED_SCRIPTS: warp-per-read evaluation (uread_kernel.cuh), same outputs
    UreadArgs ua;
    ua.m = tab.dmodel;
    ua.ref = dref;
    ua.cfg = ctx->dcfg;
    ua.first_id = first_read_id;
    ua.n_reads = n;
    ua.reads = pa.reads;
    ua.pieces = pa.pieces;
    ua.ops = pa.ops;
    ua.order = vals_out;
    ua.counter = pa.counter;
    ua.n_flagged = pa.n_flagged;
    ua.pool_cursor = (unsigned long long*)(d_totals + NS_T_POOL_CURSOR);
    ua.pool = d_totals + NS_T_POOL;             // {base, size} of the bump pool, written by capacity_stage_a
    ua.abort = d_abort;
    const unsigned ublocks = std::min<unsigned>((n + UREAD_WARPS - 1) / UREAD_WARPS, (unsigned)ctx->sm_count * 8u);
    if (chim && !ctx->hcfg.perfect) {
        // chimeric gaps of every read's first attempt, a warp per read (uread_kernel.cuh:gap_kernel)
        GapArgs ga;
        ga.m = tab.dmodel;
        ga.cfg = ctx->dcfg;
        ga.kind = (uint32_t)kind;
        ga.first_id = first_read_id;
        ga.n_reads = n;
        ga.n_seg = d_nseg;
        ga.piece_first = d_pfirst;
        ga.pieces = pa.pieces;
        ga.ops = pa.ops;
        ga.counter = pa.counter;
        ga.abort = d_abort;
        CK(cudaMemsetAsync(ctx->counter.p, 0, 64, st));
        CK(launch(ctx, gap_kernel, ublocks, UREAD_WARPS * 32, 0, ga));
    }
    CK(cudaMemsetAsync(ctx->counter.p, 0, 64, st));
    if (fast_unaligned) CK(launch(ctx, uread_kernel<false>, ublocks, UREAD_WARPS * 32, 0, ua));
    else CK(launch(ctx, plan_kernel<false>, plan_blocks, plan_tb, 0, pa));
    CK(cudaEventRecord(ctx->ev[2], st));

    // ---- sequence slots per read (scan); exact offsets for scripts that overflowed their slot
    if (int rc = read_layout(ctx, n)) return rc;
    CK(launch(ctx, gather_flagged_ops, gp, tb, 0, pieces, reads, n_pieces, scan_in));
    if (int rc = scan_total(ctx, scan_in, scan_out, n_pieces, NS_T_OVERFLOW_OPS)) return rc;
    if (sync_free) {
        CK(launch(ctx, capacity_stage_b, 1, 32, 0, d_totals, ops_cap, seq_cap));
    } else {
        if (int rc = publish_totals_and_wait(ctx)) return rc;
        CK(ctx->seq.ensure((size_t)h_totals[NS_T_SEQ_BYTES] + 16));
        if (ctx->hcfg.fastq) CK(ctx->qual.ensure((size_t)h_totals[NS_T_SEQ_BYTES] + 16));
    }
    CK(cudaEventRecord(ctx->ev[3], st));
    // rare: replay the flagged reads and write their scripts behind the primary area.  A sync-free batch does not know
    // whether there are any, so it always submits the (normally empty) replay.
    if (sync_free || (uint32_t)h_totals[NS_T_FLAGGED] > 0) {
        if (!sync_free)
            CK(ctx->ops.ensure_keep((size_t)(script_ops() + 4) * sizeof(uint32_t), (size_t)h_totals[NS_T_PRIMARY] * sizeof(uint32_t), st));
        pa.ops = ua.ops = ctx->ops.as<uint32_t>();
        CK(launch(ctx, scatter_flagged_off, gp, tb, 0, pieces, reads, n_pieces, scan_out, d_totals + NS_T_PRIMARY));
        CK(cudaMemsetAsync(ctx->counter.p, 0, 64, st));
        if (fast_unaligned) CK(launch(ctx, uread_kernel<true>, ublocks, UREAD_WARPS * 32, 0, ua));
        else CK(launch(ctx, plan_kernel<true>, plan_blocks, plan_tb, 0, pa));
    }
    CK(launch(ctx, copy_ev_fields, gp, tb, 0, pieces, n_pieces));
    uint64_t raw_ev_off = 0, raw_ops = 0;
    if (hp && !ctx->hcfg.perfect) {
        // ---- homopolymer pass (hp_kernel.cuh): count, re-scan lengths and script offsets, write
        if (!tab.hmodel.has_hp) return fail(ctx, NS_ESTATE, "ns_simulate: -hp/-k needs homopolymer parameters in the model");
        const uint64_t event_ops = script_ops();
        HpArgs ha;
        ha.ref = dref;
        ha.cfg = ctx->dcfg;
        ha.first_id = first_read_id;
        ha.reads = reads;
        ha.pieces = pieces;
        ha.n_pieces = n_pieces;
        ha.ops = pa.ops;
        ha.out_n_ops = scan_in;
        ha.out_off = nullptr;
        memcpy(ha.hp, tab.hmodel.hp, sizeof ha.hp);
        ha.hp_mis_rate = tab.hmodel.hp_mis_rate;
        ha.counter = ctx->counter.as<uint32_t>();
        {   // segments longest first: the lanes of a warp walk segments of similar length, and the longest one starts first
            CK(ctx->hp_keys.ensure((size_t)n_pieces * 16));
            uint32_t* k_in = ctx->hp_keys.as<uint32_t>();
            uint32_t *k_out = k_in + n_pieces, *v_in = k_out + n_pieces, *v_out = v_in + n_pieces;
            CK(launch(ctx, hp_piece_keys, gp, tb, 0, pieces, n_pieces, k_in, v_in));
            if (int rc = sort_pairs_descending(ctx, k_in, k_out, v_in, v_out, n_pieces)) return rc;
            ha.order = v_out;
        }
        ha.force_exact = (ctx->hcfg.flags & NS_FLAG_EMIT_EXACT) ? 1u : 0u;
        ha.piece_base = 0;
        const unsigned hp_blocks = std::min<unsigned>((n_pieces + 127) / 128, (unsigned)ctx->sm_count * 16u);
        CK(cudaMemsetAsync(ctx->counter.p, 0, 64, st));
        CK(launch(ctx, hp_kernel<false>, hp_blocks, 128, 0, ha));
        CK(launch(ctx, hp_fix_reads, gb, tb, 0, reads, pieces, n));
        CK(ctx->hp_off.ensure((size_t)n_pieces * sizeof(uint64_t)));
        if (int rc = scan_total(ctx, scan_in, ctx->hp_off.as<uint64_t>(), n_pieces, NS_T_HP_OPS)) return rc;
        CK(launch(ctx, add_base_u64, gp, tb, 0, ctx->hp_off.as<uint64_t>(), n_pieces, event_ops));
        if (int rc = read_layout(ctx, n)) return rc;
        if (int rc = publish_totals_and_wait(ctx)) return rc;
        // with intron retention, a verbatim copy of the event scripts goes behind the rewritten ones before the WRITE pass
        // filters them in place: ns_reemit lays retaining reads out on the genome by cutting the unfiltered scripts
        raw_ops = ctx->hcfg.trx_records ? event_ops : 0;
        CK(ctx->ops.ensure_keep((size_t)(script_ops() + raw_ops + 4) * sizeof(uint32_t), (size_t)event_ops * sizeof(uint32_t), st));
        CK(ctx->seq.ensure((size_t)h_totals[NS_T_SEQ_BYTES] + 16));
        if (ctx->hcfg.fastq) CK(ctx->qual.ensure((size_t)h_totals[NS_T_SEQ_BYTES] + 16));
        if (raw_ops) {
            raw_ev_off = script_ops();
            CK(cudaMemcpyAsync(ctx->ops.as<uint32_t>() + raw_ev_off, ctx->ops.p, (size_t)raw_ops * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
        }
        ha.ops = ctx->ops.as<uint32_t>();
        ha.out_off = ctx->hp_off.as<uint64_t>();
        CK(cudaMemsetAsync(ctx->counter.p, 0, 64, st));
        CK(launch(ctx, hp_kernel<true>, hp_blocks, 128, 0, ha));
    }
    CK(cudaEventRecord(ctx->ev[4], st));

    // ---- emit (one piece per read: the plan's longest-first order serves the emit too)
    if (int rc = launch_emit(ctx, kind, first_read_id, n_pieces, chim ? nullptr : vals_out, d_abort, true, ctx->ev[4])) return rc;
    CK(cudaEventRecord(ctx->ev[5], st));
    if (species) {
        // current_species_bases[species] += len(new_seg) (:1004) for the next batch's quotas
        const uint32_t S = tab.dref.n_species;
        CK(ctx->sp_bases_dev.ensure((size_t)S * sizeof(double)));
        CK(cudaMemsetAsync(ctx->sp_bases_dev.p, 0, (size_t)S * sizeof(double), st));
        CK(launch(ctx, species_bases_kernel, gp, tb, 0, pieces, n_pieces, tab.dref.chrom_species, ctx->sp_bases_dev.as<double>()));
        std::vector<double> add(S);
        CK(cudaMemcpyAsync(add.data(), ctx->sp_bases_dev.p, (size_t)S * sizeof(double), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        for (uint32_t k = 0; k < S; ++k) ctx->species_bases[k] += add[k];
    }
    if (sync_free) {
        if (int rc = publish_totals_and_wait(ctx, n >= 16384u)) return rc;
        if (h_totals[NS_T_ABORT]) {
            // a buffer was too small for this batch: nothing was written past a capacity (the kernels saw the flag and
            // returned); run it again the sized way, which also re-establishes the capacities
            ctx->opt_ok[kind] = false;
            return ns_simulate(ctx, kind, first_read_id, n_reads, info);
        }
    } else {
        CK(wait_stream(ctx, n >= 16384u));
        if (may_sync_free) {
            ctx->opt_ok[kind] = true;
            ctx->opt_n[kind] = n;
        }
    }

    NsBatchInfo& bi = ctx->last;
    bi.seq_bytes = h_totals[NS_T_SEQ_BYTES];
    bi.n_ops = script_ops() + raw_ops;
    bi.raw_ev_off = raw_ev_off;
    bi.total_bases = h_totals[NS_T_BASES];
    bi.n_reads = n;
    bi.n_pieces = n_pieces;
    auto ms = [](cudaEvent_t a, cudaEvent_t b) {
        float t = 0;
        cudaEventElapsedTime(&t, a, b);
        return t;
    };
    bi.ms_setup = ms(ctx->ev[0], ctx->ev[1]);
    bi.ms_plan = ms(ctx->ev[1], ctx->ev[2]);
    bi.ms_scan = ms(ctx->ev[2], ctx->ev[3]);
    bi.ms_script = ms(ctx->ev[3], ctx->ev[4]);
    bi.ms_emit = ms(ctx->ev[4], ctx->ev[5]);
    bi.ms_total = ms(ctx->ev[0], ctx->ev[5]);
    bi.t_begin_ms = ms(g_base[ctx->device], ctx->ev[0]);
    bi.t_end_ms = ms(g_base[ctx->device], ctx->ev[5]);
    ctx->last_kind = kind;
    ctx->last_first_id = first_read_id;
    ctx->have_batch = true;
    if (info) *info = bi;
    return NS_OK;
}

int ns_fetch(NsContext* ctx, uint8_t* seq, uint8_t* qual, NsReadMeta* reads, NsPieceMeta* pieces, uint32_t* ops) {
    if (!ctx) return NS_EINVAL;
    if (!ctx->have_batch) return fail(ctx, NS_ESTATE, "ns_fetch: no simulated batch");
    CK(cudaSetDevice(ctx->device));
    const NsBatchInfo& bi = ctx->last;
    cudaStream_t st = ctx->stream;
    if (bi.n_reads == 0) return NS_OK;
    if (qual && !ctx->hcfg.fastq) return fail(ctx, NS_ESTATE, "ns_fetch: qualities requested but the run is not --fastq");
    // 2 bits per base only when reads cannot hold anything but A C G T/U: every reference byte is an IUPAC nucleotide code
    const int nt = ctx->tables->dref.all_iupac ? unpack_threads() : 0;
    const bool packed = seq && nt > 0 && bi.seq_bytes >= (1u << 20);
    if (packed) {
        // bases: pack on the device, copy a quarter of the bytes, expand on the host while the other copies run
        const uint64_t n16 = (bi.seq_bytes + 15) / 16;            // the seq buffer has 16 bytes of slack
        CK(ctx->pack_dev.ensure((size_t)n16 * 4));
        CK(ctx->pack_host.ensure((size_t)n16 * 4, cudaHostAllocDefault));
        if (!ctx->ev_pack) CK(cudaEventCreateWithFlags(&ctx->ev_pack.e, cudaEventDisableTiming | (blocking_sync_wanted() ? (unsigned)cudaEventBlockingSync : 0u)));
        pack_bases_kernel<<<(unsigned)((n16 + 255) / 256), 256, 0, st>>>(ctx->seq.as<uint4>(), ctx->pack_dev.as<uint32_t>(), n16);
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(ctx->pack_host.p, ctx->pack_dev.p, (size_t)n16 * 4, cudaMemcpyDeviceToHost, st));
        CK(cudaEventRecord(ctx->ev_pack, st));
    } else if (seq) {
        CK(cudaMemcpyAsync(seq, ctx->seq.p, bi.seq_bytes, cudaMemcpyDeviceToHost, st));
    }
    if (qual) CK(cudaMemcpyAsync(qual, ctx->qual.p, bi.seq_bytes, cudaMemcpyDeviceToHost, st));
    if (reads) CK(cudaMemcpyAsync(reads, ctx->reads.p, (size_t)bi.n_reads * sizeof(NsReadMeta), cudaMemcpyDeviceToHost, st));
    if (pieces) CK(cudaMemcpyAsync(pieces, ctx->pieces.p, (size_t)bi.n_pieces * sizeof(NsPieceMeta), cudaMemcpyDeviceToHost, st));
    if (ops) CK(cudaMemcpyAsync(ops, ctx->ops.p, (size_t)bi.n_ops * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    if (packed) {
        CK(cudaEventSynchronize(ctx->ev_pack));
        unpack_bases(ctx->pack_host.as<uint8_t>(), seq, bi.seq_bytes, ctx->dcfg.uracil != 0, nt);
    }
    CK(wait_stream(ctx, bi.seq_bytes >= (64u << 20)));
    return NS_OK;
}

extern "C++" {    // templates cannot have C linkage

// The checks every compression makes first, in this order: its arguments, a simulated batch and, where the entry needs
// aligned reads (`lacks`: what unaligned reads have none of), an aligned batch
static int check_compress(NsContext* ctx, const char* fname, const char* names, const uint64_t* name_off, const uint64_t* nbytes,
                          const char* lacks) {
    if (!ctx) return NS_EINVAL;
    if (!names || !name_off || !nbytes) return fail(ctx, NS_EINVAL, "%s: null argument", fname);
    if (!ctx->have_batch) return fail(ctx, NS_ESTATE, "%s: no simulated batch", fname);
    if (lacks && ctx->last_kind != NS_KIND_ALIGNED)
        return fail(ctx, NS_EINVAL, "%s: the last batch is unaligned reads, which have no %s", fname, lacks);
    return NS_OK;
}

// After those checks and the entry's own: `out` invalidated and *n the last batch's reads.  A batch without reads leaves
// `out` valid and empty.  Otherwise the n names (ns_format_records' layout) go into z_names / z_name_off, with room for the
// names' lengths, the per-read sizes (scan_in) and their offsets (z_rec_off), and the totals slots of a compression zeroed.
static int begin_members(NsContext* ctx, const char* names, const uint64_t* name_off, MemberSlot& out, uint64_t* nbytes,
                         uint32_t* n) {
    CK(cudaSetDevice(ctx->device));
    out.valid = false;
    out.bytes = 0;
    *n = ctx->last.n_reads;
    if (*n == 0) {
        out.valid = true;
        *nbytes = 0;
        return NS_OK;
    }
    cudaStream_t st = ctx->stream;
    uint64_t blob = 0;                      // the names' extent: every name with its NUL
    for (uint32_t i = 0; i < *n; ++i) blob = std::max<uint64_t>(blob, name_off[i] + strlen(names + name_off[i]) + 1);
    CK(upload(ctx->z_names, names, blob, st));
    CK(upload(ctx->z_name_off, name_off, (size_t)*n * sizeof(uint64_t), st));
    CK(ctx->z_name_len.ensure((size_t)*n * sizeof(uint32_t)));
    CK(ctx->z_rec_off.ensure((size_t)*n * sizeof(uint64_t)));
    CK(ctx->scan_in.ensure((size_t)*n * sizeof(uint64_t)));
    CK(cudaMemsetAsync(ctx->totals.as<uint64_t>() + NS_T_Z_TEXT, 0, (NS_T_COUNT - NS_T_Z_TEXT) * sizeof(uint64_t), st));
    return NS_OK;
}

// the host round trip after a size pass that counts the read names too long for BAM: NS_EINVAL names the first of them
static int publish_sizes(NsContext* ctx, const char* fname, const char* names, const uint64_t* name_off, uint32_t n) {
    if (int rc = publish_totals_and_wait(ctx)) return rc;
    const uint64_t n_long = ctx->h_totals.as<uint64_t>()[NS_T_Z_LONG_NAMES];
    if (n_long == 0) return NS_OK;
    uint32_t i = 0;                                             // the first such name, for the message
    while (i + 1 < n && strlen(names + name_off[i]) <= BAM_MAX_NAME) ++i;
    return fail(ctx, NS_EINVAL, "%s: read %u has a name of %zu bytes, more than the %u BAM holds (%llu such reads)", fname, i,
                strlen(names + name_off[i]), BAM_MAX_NAME, (unsigned long long)n_long);
}

// The back of every compression: the members of the `text` bytes of text that `src` brings into shared memory, staged
// where bgzf_deflate_kernel leaves them; their offsets and total (the last host round trip); the members packed into `out`,
// which becomes valid.  NS_EINVAL when the text is too much for one call.
template <class Source>
static int end_members(NsContext* ctx, const char* fname, uint64_t text, const Source& src, MemberSlot& out, uint64_t* nbytes) {
    const uint64_t n_blocks64 = (text + BGZF_BLOCK - 1) / BGZF_BLOCK;
    if (n_blocks64 > 0x7fffffffu) return fail(ctx, NS_EINVAL, "%s: %llu bytes of text is too much for one call", fname,
                                              (unsigned long long)text);
    const uint32_t n_blocks = (uint32_t)n_blocks64;
    CK(ctx->z_stage.ensure((size_t)n_blocks * BGZF_SLOT));
    CK(ctx->z_msize.ensure((size_t)n_blocks * sizeof(uint64_t)));
    CK(ctx->z_moff.ensure((size_t)n_blocks * sizeof(uint64_t)));
    CK(ctx->z_trailer.ensure((size_t)n_blocks * sizeof(uint2)));
    const BgzfMembers zm{text, ctx->z_stage.as<uint8_t>(), ctx->z_msize.as<uint64_t>(), ctx->z_trailer.as<uint2>(),
                         (unsigned long long*)(ctx->totals.as<uint64_t>() + NS_T_Z_OVERSIZE)};
    const int smem = (int)sizeof(typename Source::Smem);
    CK(cudaFuncSetAttribute(bgzf_deflate_kernel<Source>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CK(launch(ctx, bgzf_deflate_kernel<Source>, n_blocks, BGZF_THREADS, (size_t)smem, src, zm));
    if (int rc = scan_total(ctx, ctx->z_msize.as<uint64_t>(), ctx->z_moff.as<uint64_t>(), n_blocks, NS_T_Z_BYTES)) return rc;
    if (int rc = publish_totals_and_wait(ctx)) return rc;
    const uint64_t* h = ctx->h_totals.as<uint64_t>();
    if (h[NS_T_Z_OVERSIZE])
        return fail(ctx, NS_ESTATE, "%s: %llu BGZF members exceed %u bytes", fname, (unsigned long long)h[NS_T_Z_OVERSIZE],
                    BGZF_MAX_MEMBER);
    const uint64_t total = h[NS_T_Z_BYTES];
    CK(out.buf.ensure((size_t)total));
    CK(launch(ctx, bgzf_pack_kernel, n_blocks, 256, 0, (const uint8_t*)ctx->z_stage.p, (const uint64_t*)ctx->z_msize.p,
              (const uint64_t*)ctx->z_moff.p, (const uint2*)ctx->z_trailer.p, out.buf.as<uint8_t>()));
    CK(wait_stream(ctx, false));
    out.bytes = total;
    out.valid = true;
    *nbytes = total;
    return NS_OK;
}

static int fetch_members(NsContext* ctx, const char* fname, const MemberSlot& m, uint8_t* out, uint64_t cap) {
    if (!m.valid) return fail(ctx, NS_ESTATE, "%s: the last batch has not been compressed", fname);
    if (cap < m.bytes) return fail(ctx, NS_ENOMEM, "%s: %llu bytes do not fit in %llu", fname, (unsigned long long)m.bytes,
                                   (unsigned long long)cap);
    if (m.bytes == 0) return NS_OK;
    if (!out) return fail(ctx, NS_EINVAL, "%s: null argument", fname);
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(out, m.buf.p, m.bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CK(wait_stream(ctx, m.bytes >= (64u << 20)));
    return NS_OK;
}

// the last batch's reads with the names begin_members left on the device
static BgzfReadTable read_table(NsContext* ctx) {
    BgzfReadTable t;
    t.fastq = ctx->hcfg.fastq ? 1u : 0u;
    t.reads = ctx->reads.as<NsReadMeta>();
    t.seq = ctx->seq.as<uint8_t>();
    t.qual = t.fastq ? ctx->qual.as<uint8_t>() : nullptr;
    t.names = ctx->z_names.as<char>();
    t.name_off = ctx->z_name_off.as<uint64_t>();
    t.name_len = ctx->z_name_len.as<uint32_t>();
    return t;
}

// ns_compress_records (FASTA/FASTQ text) and ns_compress_bam (BAM records): the last batch's records in that layout as
// BGZF members in z_out
template <class Layout>
static int compress_records(NsContext* ctx, const char* fname, const char* names, const uint64_t* name_off, uint64_t* nbytes) {
    uint32_t n = 0;
    if (int rc = check_compress(ctx, fname, names, name_off, nbytes, nullptr)) return rc;
    if (int rc = begin_members(ctx, names, name_off, ctx->z_out, nbytes, &n)) return rc;
    if (n == 0) return NS_OK;
    const uint32_t fastq = ctx->hcfg.fastq ? 1u : 0u;
    CK(launch(ctx, record_size_kernel<Layout>, (n + 255) / 256, 256, 0, ctx->reads.as<NsReadMeta>(), n, ctx->z_names.as<char>(),
              ctx->z_name_off.as<uint64_t>(), fastq, ctx->z_name_len.as<uint32_t>(), ctx->scan_in.as<uint64_t>(),
              (unsigned long long*)(ctx->totals.as<uint64_t>() + NS_T_Z_LONG_NAMES)));
    if (int rc = scan_total(ctx, ctx->scan_in.as<uint64_t>(), ctx->z_rec_off.as<uint64_t>(), n, NS_T_Z_TEXT)) return rc;
    if (int rc = publish_sizes(ctx, fname, names, name_off, n)) return rc;
    BgzfRecords<Layout> src;
    src.tab = read_table(ctx);
    src.rec_off = ctx->z_rec_off.as<uint64_t>();
    src.n_recs = n;
    return end_members(ctx, fname, ctx->h_totals.as<uint64_t>()[NS_T_Z_TEXT], src, ctx->z_out, nbytes);
}

// ns_compress_bam_mapped and ns_compress_bam_transcript after their checks: the last aligned batch's records by the walk
// `mode` as BGZF members in z_out.  n_ids: the records' refIDs, for which NM and SA (ns_set_aln_tags) need one name each.
static int compress_aln(NsContext* ctx, const char* fname, AlnMode mode, uint64_t n_ids, const char* names, const uint64_t* name_off,
                        uint64_t* nbytes) {
    const Tables& tab = *ctx->tables;
    // NM and SA (ns_set_aln_tags): the header's names must be the records' refIDs
    const bool tags = tab.have_aln_tags;
    if (tags && tab.tag_n_sn != n_ids)
        return fail(ctx, NS_EINVAL, "%s: ns_set_aln_tags gave %u reference names for %llu reference records", fname, tab.tag_n_sn,
                    (unsigned long long)n_ids);
    uint32_t n = 0;
    if (int rc = begin_members(ctx, names, name_off, ctx->z_out, nbytes, &n)) return rc;
    if (n == 0) return NS_OK;
    CK(ctx->m_cnt.ensure((size_t)2 * n * sizeof(uint64_t)));
    CK(ctx->m_first.ensure((size_t)2 * n * sizeof(uint64_t)));
    CK(ctx->m_prim.ensure((size_t)n * sizeof(uint32_t)));
    AlnArgs aa{};
    aa.reads = ctx->reads.as<NsReadMeta>();
    aa.pieces = ctx->pieces.as<NsPieceMeta>();
    aa.ops = ctx->ops.as<uint32_t>();
    aa.chrom_off = tab.dref.chrom_off;
    aa.names = ctx->z_names.as<char>();
    aa.name_off = ctx->z_name_off.as<uint64_t>();
    aa.n_reads = n;
    aa.name_len = ctx->z_name_len.as<uint32_t>();
    aa.n_rec = ctx->m_cnt.as<uint64_t>();
    aa.n_cig = aa.n_rec + n;
    aa.primary = ctx->m_prim.as<uint32_t>();
    aa.long_names = (unsigned long long*)(ctx->totals.as<uint64_t>() + NS_T_Z_LONG_NAMES);
    uint64_t* rec_first = ctx->m_first.as<uint64_t>();
    const unsigned grid = (n + 255) / 256;
    // the rest, with the walk's kernels and record layout instantiated for that mode
    auto run = [&](auto walk) -> int {
        constexpr AlnMode kMode = decltype(walk)::value;
        using Layout = std::conditional_t<kMode == ALN_LIFT, BgzfLiftedLayout,
                                          std::conditional_t<kMode == ALN_SPLICE, BgzfSplicedLayout, BgzfMappedLayout>>;   // ALN_TRX: plain
        if constexpr (kMode == ALN_LIFT)
            aa.lift = AlnLift{tab.lift_seg.as<HapLift>(), tab.lift_kind.as<uint8_t>(), tab.lift_first.as<uint64_t>(),
                              tab.lift_chrom.as<uint32_t>(), tab.lift_hp.as<uint8_t>()};
        // ALN_TRX: only the chains of intron retention read the map; without it the walk sees none (n_trx 0)
        if constexpr (kMode == ALN_SPLICE || kMode == ALN_TRX) {
            if (kMode == ALN_SPLICE || ctx->hcfg.trx_records)
                aa.splice = AlnSplice{tab.splice_exon.as<SpliceExon>(), tab.splice_first.as<uint64_t>(), tab.splice_minus.as<uint8_t>(),
                                      tab.splice_n_trx, tab.splice_genome_first};
        }
        CK(launch(ctx, aln_count_kernel<kMode>, grid, 256, 0, aa));
        if (int rc = scan_total(ctx, aa.n_rec, rec_first, n, NS_T_M_RECORDS)) return rc;
        if (int rc = scan_total(ctx, aa.n_cig, rec_first + n, n, NS_T_M_CIGAR_WORDS)) return rc;
        if (int rc = publish_sizes(ctx, fname, names, name_off, n)) return rc;
        const uint64_t* h = ctx->h_totals.as<uint64_t>();
        const uint64_t n_rec = h[NS_T_M_RECORDS], n_words = h[NS_T_M_CIGAR_WORDS];
        if (n_rec > 0xffffffffu) return fail(ctx, NS_EINVAL, "%s: %llu records are too many for one call", fname, (unsigned long long)n_rec);
        CK(ctx->m_aln.ensure((size_t)n_rec * sizeof(BamAln)));
        CK(ctx->m_cig.ensure((size_t)std::max<uint64_t>(n_words, 1) * sizeof(uint32_t)));
        CK(ctx->scan_in.ensure((size_t)n_rec * sizeof(uint64_t)));
        CK(ctx->z_rec_off.ensure((size_t)n_rec * sizeof(uint64_t)));
        aa.rec_first = rec_first;
        aa.cig_first = rec_first + n;
        aa.aln = ctx->m_aln.as<BamAln>();
        aa.cigar = ctx->m_cig.as<uint32_t>();
        aa.rec_size = ctx->scan_in.as<uint64_t>();
        // with NM and SA: the tagged walk, the records' aux sizes (added to rec_size) and offsets before the same wait
        AlnAuxArgs ax{};
        if (tags) {
            CK(ctx->m_nm.ensure((size_t)n_rec * sizeof(uint32_t)));
            CK(ctx->m_aux_len.ensure((size_t)n_rec * sizeof(uint64_t)));
            CK(ctx->m_aux_off.ensure((size_t)n_rec * sizeof(uint64_t)));
            const AlnTagArgs tg{ctx->seq.as<uint8_t>(), tab.dref.bases, tab.dref.chrom_off, tab.dref.pk_off, tab.dref.exc_pre,
                                tab.tag_pair.as<uint8_t>(), tab.tag_pair_off.as<uint64_t>(), ctx->m_nm.as<uint32_t>()};
            CK(launch(ctx, aln_write_tags_kernel<kMode>, grid, 256, 0, aa, tg));
            ax.aln = aa.aln;
            ax.cigar = aa.cigar;
            ax.nm = tg.nm;
            ax.n_rec = aa.n_rec;
            ax.rec_first = rec_first;
            ax.sn = tab.tag_sn.as<char>();
            ax.sn_off = tab.tag_sn_off.as<uint64_t>();
            ax.n_reads = n;
            ax.mode = (uint32_t)kMode;
            ax.rec_size = aa.rec_size;
            ax.aux_len = ctx->m_aux_len.as<uint64_t>();
            ax.aux_off = ctx->m_aux_off.as<uint64_t>();
            CK(launch(ctx, aln_aux_size_kernel, grid, 256, 0, ax));
            if (int rc = scan_total(ctx, ax.aux_len, ctx->m_aux_off.as<uint64_t>(), (uint32_t)n_rec, NS_T_M_AUX_BYTES)) return rc;
        } else {
            CK(launch(ctx, aln_write_kernel<kMode>, grid, 256, 0, aa));
        }
        if (int rc = scan_total(ctx, aa.rec_size, ctx->z_rec_off.as<uint64_t>(), (uint32_t)n_rec, NS_T_Z_TEXT)) return rc;
        if (int rc = publish_totals_and_wait(ctx)) return rc;
        const BgzfMappedTable mt{read_table(ctx), aa.aln, aa.cigar};
        if (tags) {
            const uint64_t aux_total = h[NS_T_M_AUX_BYTES];
            CK(ctx->m_aux.ensure((size_t)std::max<uint64_t>(aux_total, 1)));
            ax.aux = ctx->m_aux.as<uint8_t>();
            CK(launch(ctx, aln_aux_write_kernel, grid, 256, 0, ax));
            BgzfRecords<BgzfTaggedLayout> src;
            src.tab = BgzfTaggedTable{mt, ax.aux, ax.aux_off, aux_total, (uint32_t)n_rec};
            src.rec_off = ctx->z_rec_off.as<uint64_t>();
            src.n_recs = (uint32_t)n_rec;
            return end_members(ctx, fname, h[NS_T_Z_TEXT], src, ctx->z_out, nbytes);
        }
        BgzfRecords<Layout> src;
        src.tab = mt;
        src.rec_off = ctx->z_rec_off.as<uint64_t>();
        src.n_recs = (uint32_t)n_rec;
        return end_members(ctx, fname, h[NS_T_Z_TEXT], src, ctx->z_out, nbytes);
    };
    // ALN_TRX last: the other walks keep their order of instantiation, on which ptxas' register allocation of the
    // deflate instantiations depends
    if (mode == ALN_SPLICE) return run(std::integral_constant<AlnMode, ALN_SPLICE>{});
    if (mode == ALN_LIFT) return run(std::integral_constant<AlnMode, ALN_LIFT>{});
    if (mode == ALN_PLAIN) return run(std::integral_constant<AlnMode, ALN_PLAIN>{});
    return run(std::integral_constant<AlnMode, ALN_TRX>{});
}

}  // extern "C++"

int ns_compress_records(NsContext* ctx, const char* names, const uint64_t* name_off, uint64_t* nbytes) {
    return compress_records<BgzfTextLayout>(ctx, "ns_compress_records", names, name_off, nbytes);
}

int ns_compress_bam(NsContext* ctx, const char* names, const uint64_t* name_off, uint64_t* nbytes) {
    return compress_records<BgzfBamLayout>(ctx, "ns_compress_bam", names, name_off, nbytes);
}

int ns_compress_bam_mapped(NsContext* ctx, const char* names, const uint64_t* name_off, uint64_t* nbytes) {
    static const char* fname = "ns_compress_bam_mapped";
    if (int rc = check_compress(ctx, fname, names, name_off, nbytes, "alignment")) return rc;
    const Tables& tab = *ctx->tables;
    // the walk: spliced onto the genome in transcriptome mode, lifted onto the haploid records after ns_set_lift, else plain
    const AlnMode mode = ctx->hcfg.mode == 2 ? ALN_SPLICE : tab.have_lift ? ALN_LIFT : ALN_PLAIN;
    if (mode == ALN_SPLICE && !tab.have_splice)
        return fail(ctx, NS_EINVAL, "%s: transcriptome reads are written as mapped records only with a splice map (ns_set_splice)", fname);
    if (mode == ALN_SPLICE && ctx->hcfg.trx_records && (tab.splice_n_trx != ctx->hcfg.trx_records || tab.splice_genome_first != ctx->hcfg.trx_records))
        return fail(ctx, NS_EINVAL, "%s: the splice map's transcripts and genome records are not the run's (trx_records %u)", fname,
                    ctx->hcfg.trx_records);
    if (mode == ALN_LIFT && ctx->hcfg.circular) return fail(ctx, NS_EINVAL, "%s: lifted records need linear haplotype records", fname);
    const uint64_t n_ids = mode == ALN_SPLICE ? tab.splice_n_genome : mode == ALN_LIFT ? tab.h_haploid_off.size() - 1 : tab.dref.n_chrom;
    return compress_aln(ctx, fname, mode, n_ids, names, name_off, nbytes);
}

int ns_compress_bam_transcript(NsContext* ctx, const char* names, const uint64_t* name_off, uint64_t* nbytes) {
    static const char* fname = "ns_compress_bam_transcript";
    if (int rc = check_compress(ctx, fname, names, name_off, nbytes, "alignment")) return rc;
    const Tables& tab = *ctx->tables;
    if (ctx->hcfg.mode != 2) return fail(ctx, NS_EINVAL, "%s: transcript-coordinate records need a transcriptome context", fname);
    // with intron retention the reads laid out on the genome are composed with the splice map, which must be the run's
    const uint32_t n_trx = ctx->hcfg.trx_records;
    if (n_trx && !tab.have_splice)
        return fail(ctx, NS_EINVAL, "%s: reads that retain an intron are written as mapped records only with a splice map (ns_set_splice)",
                    fname);
    if (n_trx && (tab.splice_n_trx != n_trx || tab.splice_genome_first != n_trx))
        return fail(ctx, NS_EINVAL, "%s: the splice map's transcripts and genome records are not the run's (trx_records %u)", fname, n_trx);
    return compress_aln(ctx, fname, ALN_TRX, n_trx ? n_trx : tab.dref.n_chrom, names, name_off, nbytes);
}

int ns_fetch_compressed(NsContext* ctx, uint8_t* out, uint64_t cap) {
    if (!ctx) return NS_EINVAL;
    return fetch_members(ctx, "ns_fetch_compressed", ctx->z_out, out, cap);
}

int ns_compress_error_profile(NsContext* ctx, const char* names, const uint64_t* name_off, uint64_t* nbytes) {
    static const char* fname = "ns_compress_error_profile";
    uint32_t n = 0;
    if (int rc = check_compress(ctx, fname, names, name_off, nbytes, "error profile")) return rc;
    if (int rc = begin_members(ctx, names, name_off, ctx->ep_out, nbytes, &n)) return rc;
    if (n == 0) return NS_OK;
    const Tables& tab = *ctx->tables;
    EpArgs ea;
    ea.reads = ctx->reads.as<NsReadMeta>();
    ea.pieces = ctx->pieces.as<NsPieceMeta>();
    ea.ops = ctx->ops.as<uint32_t>();
    ea.seq = ctx->seq.as<uint8_t>();
    ea.ref = tab.dref.bases;
    ea.chrom_off = tab.dref.chrom_off;
    ea.names = ctx->z_names.as<char>();
    ea.name_off = ctx->z_name_off.as<uint64_t>();
    ea.name_len = ctx->z_name_len.as<uint32_t>();
    ea.n_reads = n;
    ea.key = make_uint2((uint32_t)ctx->seed, (uint32_t)(ctx->seed >> 32));
    ea.first_id = ctx->last_first_id;
    ea.size = ctx->scan_in.as<uint64_t>();
    ea.off = ctx->z_rec_off.as<uint64_t>();
    const unsigned warps_grid = (n + 7) / 8;                    // one warp per read, 8 per block
    CK(launch(ctx, errprof_size_kernel, warps_grid, 256, 0, ea));
    if (int rc = scan_total(ctx, ctx->scan_in.as<uint64_t>(), ctx->z_rec_off.as<uint64_t>(), n, NS_T_Z_TEXT)) return rc;
    if (int rc = publish_totals_and_wait(ctx)) return rc;
    const uint64_t text = ctx->h_totals.as<uint64_t>()[NS_T_Z_TEXT];
    if (text == 0) {                                            // no error events
        ctx->ep_out.valid = true;
        *nbytes = 0;
        return NS_OK;
    }
    CK(ctx->ep_text.ensure((size_t)text));
    ea.text = ctx->ep_text.as<uint8_t>();
    CK(launch(ctx, errprof_write_kernel, warps_grid, 256, 0, ea));
    BgzfRows src;
    src.text = ea.text;
    return end_members(ctx, fname, text, src, ctx->ep_out, nbytes);
}

int ns_fetch_compressed_error_profile(NsContext* ctx, uint8_t* out, uint64_t cap) {
    if (!ctx) return NS_EINVAL;
    return fetch_members(ctx, "ns_fetch_compressed_error_profile", ctx->ep_out, out, cap);
}

int ns_transfer_info(NsContext* ctx, uint32_t* packed_bases, uint32_t* n_threads) {
    if (!ctx) return NS_EINVAL;
    const int nt = (!ctx->tables->have_ref || ctx->tables->dref.all_iupac) ? unpack_threads() : 0;
    if (packed_bases) *packed_bases = nt > 0 ? 1u : 0u;
    if (n_threads) *n_threads = (uint32_t)nt;
    return NS_OK;
}

// ns_reemit on a -hp context, after the new pieces, their event scripts and the staging copies (scan_in: replacement reads,
// scan_out: slots) are on the device: homopolymer pass over the chains, new sequence slots, emit, new totals
static int reemit_hp(NsContext* ctx, uint32_t n_slots, uint32_t n_new_pieces, uint64_t n_new_ops,
                     const std::vector<uint32_t>& heads) {
    cudaStream_t st = ctx->stream;
    const Tables& tab = *ctx->tables;
    NsBatchInfo& bi = ctx->last;
    const uint32_t old_np = bi.n_pieces, n_chains = (uint32_t)heads.size();
    const uint64_t ev_end = bi.n_ops + n_new_ops;            // the new pieces' event scripts end here
    const unsigned rb = (n_slots + 255) / 256;
    NsReadMeta* staged = ctx->scan_in.as<NsReadMeta>();
    const uint32_t* d_slots = ctx->scan_out.as<uint32_t>();
    uint32_t* d_old_len = ctx->scan_out.as<uint32_t>() + n_slots;
    CK(launch(ctx, gather_seq_len, rb, 256, 0, ctx->reads.as<NsReadMeta>(), d_slots, n_slots, bi.n_reads, d_old_len));
    // the pass looks the chains up through the batch's reads: they point at the new pieces from here on
    CK(launch(ctx, replace_reads, rb, 256, 0, ctx->reads.as<NsReadMeta>(), d_slots, staged, n_slots, bi.n_reads, 1u));
    CK(ctx->hp_keys.ensure((size_t)n_chains * sizeof(uint32_t)));
    CK(cudaMemcpyAsync(ctx->hp_keys.p, heads.data(), (size_t)n_chains * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    CK(ctx->hp_off.ensure((size_t)n_new_pieces * sizeof(uint64_t)));
    CK(cudaMemsetAsync(ctx->hp_off.p, 0, (size_t)n_new_pieces * sizeof(uint64_t), st));
    HpArgs ha;
    ha.ref = dev_ref(ctx);
    ha.cfg = ctx->dcfg;
    ha.first_id = ctx->last_first_id;
    ha.reads = ctx->reads.as<NsReadMeta>();
    ha.pieces = ctx->pieces.as<NsPieceMeta>();
    ha.n_pieces = n_chains;
    ha.ops = ctx->ops.as<uint32_t>();
    ha.out_n_ops = ctx->hp_off.as<uint64_t>();
    ha.out_off = nullptr;
    memcpy(ha.hp, tab.hmodel.hp, sizeof ha.hp);
    ha.hp_mis_rate = tab.hmodel.hp_mis_rate;
    ha.counter = ctx->counter.as<uint32_t>();
    ha.order = ctx->hp_keys.as<uint32_t>();
    ha.force_exact = 1u;                                      // (chains take the byte-exact route regardless)
    ha.piece_base = old_np;
    const unsigned hp_blocks = std::min<unsigned>((n_chains + 127) / 128, (unsigned)ctx->sm_count * 16u);
    CK(cudaMemsetAsync(ctx->counter.p, 0, 64, st));
    CK(launch(ctx, hp_kernel<false, true>, hp_blocks, 128, 0, ha));
    CK(launch(ctx, hp_fix_reads, rb, 256, 0, staged, ha.pieces, n_slots));
    // lay out on the host: the rewritten scripts behind the new event scripts, each replaced read in a new 16-byte-aligned
    // slot behind the batch's bytes (its old slot is left unreferenced)
    std::vector<NsReadMeta> hr(n_slots);
    std::vector<uint64_t> off(n_new_pieces);
    std::vector<uint32_t> old_len(n_slots);
    CK(cudaMemcpyAsync(hr.data(), staged, (size_t)n_slots * sizeof(NsReadMeta), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(off.data(), ctx->hp_off.p, (size_t)n_new_pieces * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(old_len.data(), d_old_len, (size_t)n_slots * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    uint64_t op_end = ev_end;
    for (uint32_t q = 0; q < n_new_pieces; ++q) {
        const uint64_t c = off[q];
        off[q] = op_end;
        op_end += c;
    }
    uint64_t seq_end = bi.seq_bytes, total = bi.total_bases;
    for (uint32_t k = 0; k < n_slots; ++k) {
        seq_end = (seq_end + 15u) & ~(uint64_t)15u;
        hr[k].seq_off = seq_end;
        seq_end += hr[k].seq_len;
        total += (uint64_t)hr[k].seq_len - old_len[k];
    }
    seq_end = (seq_end + 15u) & ~(uint64_t)15u;
    CK(ctx->ops.ensure_keep((size_t)(op_end + 4) * sizeof(uint32_t), (size_t)ev_end * sizeof(uint32_t), st));
    CK(ctx->seq.ensure_keep((size_t)seq_end + 16, (size_t)bi.seq_bytes, st));
    if (ctx->hcfg.fastq) CK(ctx->qual.ensure_keep((size_t)seq_end + 16, (size_t)bi.seq_bytes, st));
    CK(cudaMemcpyAsync(ctx->hp_off.p, off.data(), (size_t)n_new_pieces * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(staged, hr.data(), (size_t)n_slots * sizeof(NsReadMeta), cudaMemcpyHostToDevice, st));
    CK(launch(ctx, replace_reads, rb, 256, 0, ctx->reads.as<NsReadMeta>(), d_slots, staged, n_slots, bi.n_reads, 0u));
    ha.ops = ctx->ops.as<uint32_t>();
    ha.out_off = ctx->hp_off.as<uint64_t>();
    CK(cudaMemsetAsync(ctx->counter.p, 0, 64, st));
    CK(launch(ctx, hp_kernel<true, true>, hp_blocks, 128, 0, ha));
    CK(launch(ctx, iota_from, (n_new_pieces + 255) / 256, 256, 0, ctx->sort_vals.as<uint32_t>(), n_new_pieces, old_np));
    if (int rc = launch_emit(ctx, NS_KIND_ALIGNED, ctx->last_first_id, n_new_pieces, ctx->sort_vals.as<uint32_t>(), nullptr, false))
        return rc;
    CK(cudaStreamSynchronize(st));
    bi.n_pieces = old_np + n_new_pieces;
    bi.n_ops = op_end;
    bi.seq_bytes = seq_end;
    bi.total_bases = total;
    return NS_OK;
}

int ns_batch_info(NsContext* ctx, NsBatchInfo* info) {
    if (!ctx || !info) return NS_EINVAL;
    if (!ctx->have_batch) return fail(ctx, NS_ESTATE, "ns_batch_info: no simulated batch");
    *info = ctx->last;
    return NS_OK;
}

int ns_reemit(NsContext* ctx, const uint32_t* read_slots, const NsReadMeta* new_reads, uint32_t n_slots,
              const NsPieceMeta* new_pieces, uint32_t n_new_pieces, const uint32_t* new_ops, uint64_t n_new_ops) {
    if (!ctx) return NS_EINVAL;
    if (!ctx->have_batch || ctx->last_kind != NS_KIND_ALIGNED) return fail(ctx, NS_ESTATE, "ns_reemit: no aligned batch to patch");
    if (n_slots == 0 || n_new_pieces == 0) return NS_OK;
    if (!read_slots || !new_reads || !new_pieces || (n_new_ops && !new_ops)) return fail(ctx, NS_EINVAL, "ns_reemit: null argument");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    ctx->z_out.valid = ctx->ep_out.valid = false;
    NsBatchInfo& bi = ctx->last;
    const uint32_t old_np = bi.n_pieces;
    const uint64_t old_ops = bi.n_ops;
    // the host built absolute indices against these totals: check the ones that would corrupt memory
    for (uint32_t k = 0; k < n_slots; ++k) {
        if (read_slots[k] >= bi.n_reads) return fail(ctx, NS_EINVAL, "ns_reemit: read slot %u out of range", read_slots[k]);
        if (new_reads[k].piece_first < old_np || (uint64_t)new_reads[k].piece_first + new_reads[k].n_pieces > (uint64_t)old_np + n_new_pieces)
            return fail(ctx, NS_EINVAL, "ns_reemit: read %u does not point into the new pieces", read_slots[k]);
    }
    for (uint32_t k = 0; k < n_new_pieces; ++k) {
        const NsPieceMeta& p = new_pieces[k];
        const Tables& tab = *ctx->tables;
        if (p.read_slot >= bi.n_reads || p.chrom >= tab.dref.n_chrom || p.op_off < old_ops || p.op_off + p.n_ops > old_ops + n_new_ops ||
            (uint64_t)p.pos + p.ref_len > tab.h_chrom_off[p.chrom + 1] - tab.h_chrom_off[p.chrom])
            return fail(ctx, NS_EINVAL, "ns_reemit: piece %u is inconsistent with the batch or the reference", k);
    }
    // -hp: the homopolymer pass runs again over each replaced read's pieces, as one chain (hp_kernel.cuh, CHAIN): they must
    // be laid out as intron_retention.py lays them out -- genome segments two apart, every one but the first continuing the
    // one before, zero-op gaps in between, one strand, event script == emitted script, no piece shared between reads
    const bool hp = ctx->hcfg.kmer_bias > 0 && !ctx->hcfg.perfect;
    std::vector<uint32_t> heads;
    if (hp) {
        uint64_t prev_end = old_np;
        for (uint32_t k = 0; k < n_slots; ++k) {
            const NsReadMeta& r = new_reads[k];
            bool ok = r.piece_first >= prev_end && (r.n_pieces & 1u);
            prev_end = (uint64_t)r.piece_first + r.n_pieces;
            const NsPieceMeta* pc = new_pieces + (r.piece_first - old_np);
            for (uint32_t q = 0; ok && q < r.n_pieces; ++q) {
                const NsPieceMeta& p = pc[q];
                ok = p.read_slot == read_slots[k];
                if (q & 1u) {
                    ok = ok && NS_PIECE_KIND(p.kind) == NS_PIECE_GAP && p.n_ops == 0;
                } else {
                    ok = ok && NS_PIECE_KIND(p.kind) == NS_PIECE_SEGMENT && (p.kind & NS_PIECE_GENOME) &&
                         ((p.kind & NS_PIECE_CONT) != 0) == (q > 0) && (p.kind & NS_PIECE_REF_REV) == (pc[0].kind & NS_PIECE_REF_REV) &&
                         p.ev_off == p.op_off && p.ev_n_ops == p.n_ops && p.ref_len > 0;
                }
            }
            if (!ok) return fail(ctx, NS_EINVAL, "ns_reemit: the pieces of read %u do not form one chain of genome pieces", read_slots[k]);
            heads.push_back(r.piece_first);
        }
    }
    CK(ctx->pieces.ensure_keep((size_t)(old_np + n_new_pieces + 1) * sizeof(NsPieceMeta), (size_t)old_np * sizeof(NsPieceMeta), st));
    CK(ctx->ops.ensure_keep((size_t)(old_ops + n_new_ops + 4) * sizeof(uint32_t), (size_t)old_ops * sizeof(uint32_t), st));
    CK(cudaMemcpyAsync(ctx->pieces.as<NsPieceMeta>() + old_np, new_pieces, (size_t)n_new_pieces * sizeof(NsPieceMeta), cudaMemcpyHostToDevice, st));
    if (n_new_ops) CK(cudaMemcpyAsync(ctx->ops.as<uint32_t>() + old_ops, new_ops, (size_t)n_new_ops * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    // staging for the slots / replacement reads / piece order: the scan buffers are free between batches
    CK(ctx->scan_in.ensure((size_t)n_slots * sizeof(NsReadMeta)));
    CK(ctx->scan_out.ensure((size_t)n_slots * 2 * sizeof(uint32_t)));
    CK(ctx->sort_vals.ensure((size_t)n_new_pieces * sizeof(uint32_t)));
    CK(cudaMemcpyAsync(ctx->scan_in.p, new_reads, (size_t)n_slots * sizeof(NsReadMeta), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->scan_out.p, read_slots, (size_t)n_slots * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    if (hp) return reemit_hp(ctx, n_slots, n_new_pieces, n_new_ops, heads);
    CK(launch(ctx, replace_reads, (n_slots + 255) / 256, 256, 0, ctx->reads.as<NsReadMeta>(), ctx->scan_out.as<uint32_t>(),
              ctx->scan_in.as<NsReadMeta>(), n_slots, bi.n_reads, 1u));
    CK(launch(ctx, iota_from, (n_new_pieces + 255) / 256, 256, 0, ctx->sort_vals.as<uint32_t>(), n_new_pieces, old_np));
    if (int rc = launch_emit(ctx, NS_KIND_ALIGNED, ctx->last_first_id, n_new_pieces, ctx->sort_vals.as<uint32_t>(), nullptr, false))
        return rc;
    CK(cudaStreamSynchronize(st));
    bi.n_pieces = old_np + n_new_pieces;
    bi.n_ops = old_ops + n_new_ops;
    return NS_OK;
}

int ns_device_buffers(NsContext* ctx, const uint8_t** seq, const uint8_t** qual, const NsReadMeta** reads,
                      const NsPieceMeta** pieces, const uint32_t** ops) {
    if (!ctx) return NS_EINVAL;
    if (!ctx->have_batch) return fail(ctx, NS_ESTATE, "ns_device_buffers: no simulated batch");
    if (seq) *seq = ctx->seq.as<uint8_t>();
    if (qual) *qual = ctx->hcfg.fastq ? ctx->qual.as<uint8_t>() : nullptr;
    if (reads) *reads = ctx->reads.as<NsReadMeta>();
    if (pieces) *pieces = ctx->pieces.as<NsPieceMeta>();
    if (ops) *ops = ctx->ops.as<uint32_t>();
    return NS_OK;
}

int ns_op_stats(NsContext* ctx, uint64_t* out) {
    if (!ctx || !out) return NS_EINVAL;
    if (!ctx->have_batch) return fail(ctx, NS_ESTATE, "ns_op_stats: no simulated batch");
    CK(cudaSetDevice(ctx->device));
    const size_t bytes = (size_t)NS_STATS_WORDS * sizeof(uint64_t);
    CK(ctx->stats.ensure(bytes));
    CK(cudaMemsetAsync(ctx->stats.p, 0, bytes, ctx->stream));
    const uint32_t n = ctx->last.n_pieces;
    if (n) {
        op_stats_kernel<<<(n + 127) / 128, 128, 0, ctx->stream>>>(ctx->pieces.as<NsPieceMeta>(), ctx->reads.as<NsReadMeta>(),
                                                                   ctx->ops.as<uint32_t>(), n, dev_ref(ctx), ctx->seq.as<uint8_t>(),
                                                                   (unsigned long long*)ctx->stats.p);
        const uint32_t nr = ctx->last.n_reads;
        if (nr && ctx->seq.p)
            base_comp_kernel<<<(nr + 3) / 4, 128, 0, ctx->stream>>>(ctx->reads.as<NsReadMeta>(), nr, ctx->seq.as<uint8_t>(),
                                                                     (unsigned long long*)ctx->stats.p);
        CK(cudaGetLastError());
    }
    CK(cudaMemcpyAsync(out, ctx->stats.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return NS_OK;
}

// ---------------------------------------------------------------------------------------------------------
// One NCCL broadcast of the reference at init (the reference's workers inherit the parent's seq_dict through fork(),
// simulator.py:1588-1622; ranks on different GPUs get it over NVLink instead of each parsing the FASTA).  NCCL is
// loaded at run time (dlopen), so the library has no link-time dependency on it.
// ---------------------------------------------------------------------------------------------------------
#if NS_HAVE_NCCL
namespace {
struct NcclApi {
    void* h = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
};
NcclApi& nccl_api() {
    static NcclApi api = [] {
        NcclApi a;
        const char* override_path = getenv("NANOSIM_B200_NCCL_LIB");
        const char* names[] = {override_path, "libnccl.so.2", "libnccl.so"};
        for (const char* n : names) {
            if (!n || !*n) continue;
            a.h = dlopen(n, RTLD_NOW | RTLD_LOCAL);
            if (a.h) break;
        }
        if (!a.h) return a;
        a.GetUniqueId = (decltype(a.GetUniqueId))dlsym(a.h, "ncclGetUniqueId");
        a.CommInitRank = (decltype(a.CommInitRank))dlsym(a.h, "ncclCommInitRank");
        a.Broadcast = (decltype(a.Broadcast))dlsym(a.h, "ncclBroadcast");
        a.CommDestroy = (decltype(a.CommDestroy))dlsym(a.h, "ncclCommDestroy");
        a.GetErrorString = (decltype(a.GetErrorString))dlsym(a.h, "ncclGetErrorString");
        a.ok = a.GetUniqueId && a.CommInitRank && a.Broadcast && a.CommDestroy;
        return a;
    }();
    return api;
}
}  // namespace
#endif

int ns_get_reference(NsContext* ctx, uint8_t* bases, uint64_t cap) {
    if (!ctx || !bases) return NS_EINVAL;
    const Tables& tab = *ctx->tables;
    if (!tab.have_ref) return fail(ctx, NS_ESTATE, "ns_get_reference: no reference set");
    if (cap < tab.dref.genome_len) return fail(ctx, NS_ENOMEM, "ns_get_reference: buffer too small");
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpy(bases, tab.dref.bases, tab.dref.genome_len, cudaMemcpyDeviceToHost));
    return NS_OK;
}

int ns_nccl_unique_id(uint8_t* id) {
#if NS_HAVE_NCCL
    if (!id) return NS_EINVAL;
    NcclApi& api = nccl_api();
    if (!api.ok) return NS_ESTATE;
    ncclUniqueId u;
    if (api.GetUniqueId(&u) != ncclSuccess) return NS_ECUDA;
    static_assert(sizeof(ncclUniqueId) == NS_NCCL_ID_BYTES, "ncclUniqueId size");
    memcpy(id, &u, sizeof u);
    return NS_OK;
#else
    (void)id;
    return NS_ESTATE;
#endif
}

int ns_bcast_nccl(NsContext* ctx, const uint8_t* id, int rank, int world, int root) {
    if (!ctx || !id || world < 1 || rank < 0 || rank >= world || root < 0 || root >= world) return fail(ctx, NS_EINVAL, "ns_bcast_nccl: bad argument");
#if NS_HAVE_NCCL
    const Tables& tab = *ctx->tables;
    if (ctx->clone) return fail(ctx, NS_ESTATE, "ns_bcast_nccl: a cloned context shares its parent's reference");
    if (rank == root && !tab.have_ref) return fail(ctx, NS_ESTATE, "ns_bcast_nccl: the root rank sets its reference first (ns_set_reference)");
    if (world == 1) return NS_OK;
    NcclApi& api = nccl_api();
    if (!api.ok) return fail(ctx, NS_ESTATE, "ns_bcast_nccl: libnccl.so.2 could not be loaded (NANOSIM_B200_NCCL_LIB overrides the path)");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    ncclUniqueId u;
    memcpy(&u, id, sizeof u);
    ncclComm_t comm = nullptr;
    ncclResult_t nr = api.CommInitRank(&comm, world, u, rank);
    if (nr != ncclSuccess) return fail(ctx, NS_ECUDA, "ns_bcast_nccl: ncclCommInitRank failed: %s", api.GetErrorString ? api.GetErrorString(nr) : "?");
    auto bc = [&](void* p, size_t bytes) { return bytes ? api.Broadcast(p, p, bytes, ncclUint8, root, comm, st) : ncclSuccess; };
    int rc = NS_OK;
    uint64_t* d_head = nullptr;
    void *t_bases = nullptr, *t_off = nullptr, *t_sp = nullptr, *t_circ = nullptr;
    do {
        uint64_t head[4] = {tab.dref.genome_len, tab.dref.n_chrom, tab.dref.n_species, 0};
        if (cudaMalloc((void**)&d_head, sizeof head) != cudaSuccess) { rc = NS_ENOMEM; break; }
        cudaMemcpyAsync(d_head, head, sizeof head, cudaMemcpyHostToDevice, st);
        if (bc(d_head, sizeof head) != ncclSuccess) { rc = NS_ECUDA; break; }
        cudaMemcpyAsync(head, d_head, sizeof head, cudaMemcpyDeviceToHost, st);
        if (cudaStreamSynchronize(st) != cudaSuccess) { rc = NS_ECUDA; break; }
        const uint64_t n_bases = head[0];
        const uint32_t n_chrom = (uint32_t)head[1], n_species = (uint32_t)head[2];
        if (rank == root) {
            t_bases = tab.ref_bases.p; t_off = tab.ref_off.p; t_sp = tab.ref_species.p; t_circ = tab.ref_circular.p;
        } else {
            if (cudaMalloc(&t_bases, n_bases ? n_bases : 16) != cudaSuccess || cudaMalloc(&t_off, (n_chrom + 1) * sizeof(uint64_t)) != cudaSuccess ||
                (n_species && (cudaMalloc(&t_sp, n_chrom * 4) != cudaSuccess || cudaMalloc(&t_circ, n_chrom) != cudaSuccess))) { rc = NS_ENOMEM; break; }
        }
        if (bc(t_bases, n_bases) != ncclSuccess || bc(t_off, (n_chrom + 1) * sizeof(uint64_t)) != ncclSuccess ||
            (n_species && (bc(t_sp, (size_t)n_chrom * 4) != ncclSuccess || bc(t_circ, n_chrom) != ncclSuccess))) { rc = NS_ECUDA; break; }
        if (cudaStreamSynchronize(st) != cudaSuccess) { rc = NS_ECUDA; break; }
        if (rank != root) {
            NsReference r;
            r.bases = (const uint8_t*)t_bases;            // device pointers: ns_set_reference copies from them
            r.n_bases = n_bases;
            r.chrom_off = (const uint64_t*)t_off;
            r.n_chrom = n_chrom;
            r.n_species = n_species;
            r.chrom_species = (const uint32_t*)t_sp;
            r.chrom_circular = (const uint8_t*)t_circ;
            rc = ns_set_reference(ctx, &r);
        }
    } while (0);
    if (rank != root) {
        cudaFree(t_bases); cudaFree(t_off); cudaFree(t_sp); cudaFree(t_circ);
    }
    cudaFree(d_head);
    api.CommDestroy(comm);
    if (rc != NS_OK && ctx->err.empty()) ctx->err = "ns_bcast_nccl: broadcast failed";
    return rc;
#else
    (void)rank; (void)world; (void)root;
    return fail(ctx, NS_ESTATE, "ns_bcast_nccl: built without nccl.h");
#endif
}

}  // extern "C"
