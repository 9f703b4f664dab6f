// Shared device-side definitions: counter-based RNG, table samplers, device mirrors of the C-ABI structs.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "nanosim_b200.h"

#define NS_MAX_BINS 24
#define NS_MAX_TABLES (4 + NS_MAX_BINS)

struct DevKde {
    const float* data;
    uint32_t n;
    float bw;
};

struct DevModel {
    DevKde aligned, ht, ratio, unaligned, gap;
    const float* kde2d_x;               // transcriptome: (transcript length, aligned length) rows sorted by x
    const float* kde2d_y;
    uint32_t n_kde2d;
    float kde2d_bw;
    const uint2* alias;                 // interleaved (accept threshold, alias index)
    uint32_t tab_off[NS_MAX_TABLES];
    uint32_t tab_n[NS_MAX_TABLES];
    uint32_t n_bins;
    uint32_t bin_lo[NS_MAX_BINS];
    uint32_t bin_hi[NS_MAX_BINS];
    uint32_t trans[NS_N_ERR_STATES][3];
    float strandness;
    double seg_p;                       // 1 / segment_mean
};

struct DevRef {
    const uint8_t* bases;
    const uint64_t* chrom_off;          // n_chrom + 1
    uint64_t genome_len;
    uint32_t n_chrom;
    // metagenome
    uint32_t n_species;
    const uint32_t* chrom_species;      // per chromosome
    const uint8_t* chrom_circular;      // per chromosome
    const uint32_t* species_chrom_off;  // n_species + 1: chromosomes of species s are [off[s], off[s+1])
    // transcriptome
    const uint2* expr_alias;            // Walker alias over the expressed transcripts (TPM shares)
    const uint32_t* expr_chrom;         // expressed transcript -> reference record
    uint32_t n_expressed;
    const uint8_t* chrom_has_polya;     // per reference record (nullptr: no polyA list)
    // transcript records sorted by length (ns_configure, transcriptome mode): lengths ascending and the record of each
    const uint32_t* trx_len_sorted;
    const uint32_t* trx_len_idx;
    uint32_t n_trx_sorted;
    // 2-bit copy of the reference for the emit kernel's fast path (built once by ns_set_reference): 16 bases per 32-bit
    // word, base j of a word in bits [2j+1:2j], code (c >> 1) & 3 of the upper-cased base (A 0, C 1, T 2, G 3); every
    // chromosome starts at a word boundary (pk_off[chrom], in words); one guard word in front, two behind.  Bytes that
    // case_convert does not map to exactly one of ACGT (IUPAC codes, anything else) are "exceptions" and get code 0:
    // exc_pre[b] = exceptions in packed words [0, 256 b) -- a piece whose words touch none takes the fast path.
    const uint32_t* packed;
    uint64_t pk_words;                  // packed words incl. the guards (another 64 words of slack are allocated behind them)
    const uint64_t* pk_off;
    const uint32_t* exc_pre;
    uint32_t all_iupac;                 // every reference byte is a nucleotide code case_convert turns into A C G T
};
#define REF_EXC_BLOCK_SHIFT 8           // 256 packed words = 4096 bases per exception-count block

struct DevCfg {
    uint32_t circular, perfect, fastq, chimeric, kmer_bias, metagenome, transcriptome, uracil, kde2d_n, trx_records;
    double polya_scale;
    uint32_t min_len, max_len;
    uint64_t seed;
    double median_len, sd_len;          // -med / -sd (0 = lengths from the KDEs)
};

// ------------------------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al., SC'11).  Counter = (read id lo, read id hi, stream word, block index); key = seed.
// ------------------------------------------------------------------------------------------------------------
template <int ROUNDS>
__host__ __device__ __forceinline__ uint4 philox4x32(uint4 c, uint2 k) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < ROUNDS; ++r) {
        uint64_t p0 = (uint64_t)M0 * c.x;       // one IMAD.WIDE each
        uint64_t p1 = (uint64_t)M1 * c.z;
        c = make_uint4((uint32_t)(p1 >> 32) ^ c.y ^ k.x, (uint32_t)p1, (uint32_t)(p0 >> 32) ^ c.w ^ k.y, (uint32_t)p0);
        k.x += W0;
        k.y += W1;
    }
    return c;
}
// 10 rounds (the Random123 / cuRAND default) for every structural draw: lengths, error chain, positions.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) { return philox4x32<10>(c, k); }
// 7 rounds -- the smallest round count that passes BigCrush in Salmon et al. (SC'11, table 2) -- for the bulk
// per-base streams of the emit kernel (quality values, substituted / inserted bases).
__host__ __device__ __forceinline__ uint4 philox4x32_7(uint4 c, uint2 k) { return philox4x32<7>(c, k); }

// stream word layout: [31:28] purpose, [27] kind, [26:0] attempt / generation
enum : uint32_t { ST_SEG = 1, ST_LEN = 2, ST_ATT = 3, ST_POS = 4, ST_EMIT_Q = 5, ST_EMIT_B = 6, ST_IUPAC = 7, ST_HP = 8, ST_GAP = 9, ST_CHAIN = 10 };

__host__ __device__ __forceinline__ uint32_t stream_word(uint32_t purpose, uint32_t kind, uint32_t sub) {
    return (purpose << 28) | ((kind & 1u) << 27) | (sub & 0x07ffffffu);
}

struct Rng {
    uint2 key;
    uint4 ctr;
    uint4 buf;
    int have;
    __device__ __forceinline__ void init(uint64_t seed, uint64_t id, uint32_t stream) {
        key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
        ctr = make_uint4((uint32_t)id, (uint32_t)(id >> 32), stream, 0u);
        have = 0;
    }
    __device__ __forceinline__ uint32_t next() {
        if (have == 0) {
            buf = philox4x32_10(ctr, key);
            ctr.w++;
            have = 4;
        }
        uint32_t r = buf.x;
        buf.x = buf.y;
        buf.y = buf.z;
        buf.z = buf.w;
        --have;
        return r;
    }
    // fresh block of four words (drops leftovers); used by the event loop: one Philox call per event
    __device__ __forceinline__ uint4 next4() {
        uint4 r = philox4x32_10(ctr, key);
        ctr.w++;
        have = 0;
        return r;
    }
    __device__ __forceinline__ uint64_t next64() {
        uint64_t a = next();
        return (a << 32) | next();
    }
};

__device__ __forceinline__ float u01_open_low(uint32_t r) {   // (0, 1]
    return ((float)(r >> 8) + 1.0f) * (1.0f / 16777216.0f);
}
__device__ __forceinline__ double u01_double(uint64_t r) {    // [0, 1)
    return (double)(r >> 11) * (1.0 / 9007199254740992.0);
}

// Walker alias draw from table t with one 32-bit word.
__device__ __forceinline__ uint32_t alias_draw(const DevModel& m, uint32_t t, uint32_t r) {
    uint32_t n = m.tab_n[t];
    uint64_t p = (uint64_t)r * n;
    uint32_t j = (uint32_t)(p >> 32);
    uint32_t frac = (uint32_t)p;
    uint2 e = __ldg(&m.alias[m.tab_off[t] + j]);
    return (frac < e.x || e.x == 0xffffffffu) ? j : e.y;
}

// The same draw with the table directory (offsets, sizes) in shared memory: a warp whose lanes index the directory
// differently pays one constant-cache replay per distinct index when it sits in the kernel parameters.
__device__ __forceinline__ uint32_t alias_draw_s(const uint2* __restrict__ alias, const uint32_t* tab_off, const uint32_t* tab_n, uint32_t t,
                                                 uint32_t r) {
    const uint64_t p = (uint64_t)r * tab_n[t];
    const uint32_t j = (uint32_t)(p >> 32);
    const uint2 e = __ldg(&alias[tab_off[t] + j]);
    return ((uint32_t)p < e.x || e.x == 0xffffffffu) ? j : e.y;
}

// sklearn KernelDensity.sample (gaussian): data[floor(u*N)] + N(0, bw)
__device__ __forceinline__ double kde_draw(const DevKde& k, Rng& rng) {
    uint64_t r0 = rng.next64();
    uint32_t r1 = rng.next(), r2 = rng.next();
    uint32_t i = (uint32_t)__umul64hi(r0, (uint64_t)k.n);
    float u1 = u01_open_low(r1);
    float u2 = (float)(r2 >> 8) * (1.0f / 16777216.0f);
    float z = sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
    return (double)__ldg(&k.data[i]) + (double)k.bw * (double)z;
}

// numpy.random.lognormal(mean, sigma) = exp(mean + sigma * N(0,1))
__device__ __forceinline__ double lognormal_draw(double mean, double sigma, Rng& rng) {
    uint32_t r1 = rng.next(), r2 = rng.next();
    float z = sqrtf(-2.0f * logf(u01_open_low(r1))) * cospif(2.0f * ((float)(r2 >> 8) * (1.0f / 16777216.0f)));
    return exp(mean + sigma * (double)z);
}

// base <-> index helpers: A C G T -> 0 1 3 2 via (c >> 1) & 3 ; complement = idx ^ 2
__device__ __forceinline__ uint32_t base_idx(uint32_t c) { return (c >> 1) & 3u; }
__device__ __forceinline__ uint32_t idx_base(uint32_t i) { return (0x47544341u >> (8u * i)) & 0xffu; }
// emitted character of a base index; --uracil writes U for T (:1247-1248)
__device__ __forceinline__ uint32_t emit_char(uint32_t i, uint32_t uracil) {
    return ((uracil ? 0x47554341u : 0x47544341u) >> (8u * i)) & 0xffu;
}
__device__ __forceinline__ bool is_acgt(uint32_t c) { return c == 'A' || c == 'C' || c == 'G' || c == 'T'; }
// bit i of 0x80045 is set for i = 'A'-'A', 'C'-'A', 'G'-'A', 'T'-'A'
__device__ __forceinline__ bool acgt_fast(uint32_t c) {
    uint32_t d = c - 'A';
    return d < 26u && ((0x80045u >> d) & 1u);
}
// Base qualities: per quality state a Walker alias table with 2^QLUT_BITS slots over the state's 24-bit pmf (built on the
// host, nanosim_api.cu:build_qlut; sampled in emit_kernel.cuh:qual_pick).
#define QLUT_BITS 11
#define QLUT_SIZE (1 << QLUT_BITS)

__device__ __forceinline__ uint32_t op_len(uint32_t op) { return (op >> 28) == NS_OP_LIT ? (op & 0x00ffffffu) : (op & 0x0fffffffu); }

// IUPAC resolution of case_convert (:744-746): members in the reference's list order, picked uniformly.
// r8 is a uniform byte; t3 a uniform value in {0,1,2}.
__device__ __forceinline__ uint32_t resolve_iupac(uint32_t c, uint32_t r8, uint32_t t3) {
    uint32_t n, set;   // set: up to 4 members packed one byte each
    switch (c) {
    case 'Y': n = 2; set = 'C' | ('T' << 8); break;
    case 'R': n = 2; set = 'A' | ('G' << 8); break;
    case 'W': n = 2; set = 'A' | ('T' << 8); break;
    case 'S': n = 2; set = 'G' | ('C' << 8); break;
    case 'K': n = 2; set = 'T' | ('G' << 8); break;
    case 'M': n = 2; set = 'C' | ('A' << 8); break;
    case 'D': n = 3; set = 'A' | ('G' << 8) | ('T' << 16); break;
    case 'V': n = 3; set = 'A' | ('C' << 8) | ('G' << 16); break;
    case 'H': n = 3; set = 'A' | ('C' << 8) | ('T' << 16); break;
    case 'B': n = 3; set = 'C' | ('G' << 8) | ('T' << 16); break;
    case 'N':
    case 'X': n = 4; set = 'A' | ('T' << 8) | ('C' << 16) | ('G' << 24); break;
    default: return c;
    }
    uint32_t k = (n == 3) ? t3 : ((r8 >> 4) & (n - 1));
    return (set >> (8 * k)) & 0xffu;
}

// case_convert of ONE reference base of one read, as a pure function of (read, piece, forward offset in the segment):
// every kernel that looks at the same base of the same read (emit, homopolymer pass) sees the same resolution.
__device__ __forceinline__ uint32_t converted_ref_base(uint32_t c, uint64_t seed, uint64_t rid, uint32_t piece_in_read,
                                                       uint32_t fwd_off) {
    if (c - 'a' < 26u) c -= 32;
    if (acgt_fast(c)) return c;
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    uint4 w = philox4x32_7(make_uint4((uint32_t)rid, (uint32_t)(rid >> 32), stream_word(ST_IUPAC, 0, piece_in_read), fwd_off >> 3), key);
    uint32_t wd = (fwd_off & 4u) ? ((fwd_off & 2u) ? w.w : w.z) : ((fwd_off & 2u) ? w.y : w.x);
    uint32_t h = (fwd_off & 1u) ? (wd >> 16) : (wd & 0xffffu);
    uint32_t r8 = h & 0xffu, r3 = h >> 8;
    return resolve_iupac(c, r8, r3 == 255u ? 0u : r3 % 3u);
}

// Bases of a MIS / INS event that the homopolymer pass rewrites (hp_kernel.cuh, ST_BASE); the error-profile formatter
// (host_io.cu) gives those events the same bases.  Base t of the event comes from byte t % 16 of Philox-7 block
// (event index in the piece's event script << 8) + (t >> 4) on stream ST_EMIT_B of the piece (key: the seed).
__host__ __device__ __forceinline__ uint4 event_base_block(uint2 key, uint64_t rid, uint32_t piece_in_read, uint32_t event,
                                                           uint32_t t) {
    return philox4x32_7(make_uint4((uint32_t)rid, (uint32_t)(rid >> 32), stream_word(ST_EMIT_B, 0, piece_in_read), (event << 8) + (t >> 4)), key);
}
__host__ __device__ __forceinline__ uint32_t event_byte(const uint4& blk, uint32_t t) {
    const uint32_t wd = (t & 8u) ? ((t & 4u) ? blk.w : blk.z) : ((t & 4u) ? blk.y : blk.x);
    return (wd >> (8u * (t & 3u))) & 0xffu;
}
// base index (A 0, C 1, T 2, G 3) from that byte: an inserted base is r8 & 3, a substituted one differs from the original
// base index `orig`
__host__ __device__ __forceinline__ uint32_t event_base(uint32_t r8, bool mis, uint32_t orig) {
    if (!mis) return r8 & 3u;
    const uint32_t rr = r8 == 255u ? 0u : r8;
    return ((orig & 3u) + 1u + rr % 3u) & 3u;
}
