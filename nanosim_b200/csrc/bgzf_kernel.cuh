// BGZF output: text cut into blocks of BGZF_BLOCK bytes and compressed into one gzip member per block on the device.
// Every member holds one final dynamic-Huffman DEFLATE block (RFC 1951 BTYPE 2) and carries the BGZF extra field (SAM/BAM
// format specification §4.1), so plain gzip readers and htslib both read the concatenation.  One thread block builds one
// member; nothing is shared between blocks.  One kernel, bgzf_deflate_kernel<Source>, builds every member; its Source
// brings the block's text into shared memory and cuts it into tokens:
//   BgzfRecords<BgzfTextLayout>  ns_compress_records: the last batch's FASTA/FASTQ text, as ns_format_records lays it out
//   BgzfRecords<BgzfBamLayout>   ns_compress_bam: the last batch's BAM records
//   BgzfRecords<BgzfMappedLayout> ns_compress_bam_mapped: the last aligned batch's mapped BAM records (aln_kernel.cuh)
//   BgzfRows                     ns_compress_error_profile: the error profile's rows, flat in HBM
//
// Records are literals only: simulated bases and qualities leave LZ77 almost nothing to find.  Such a member is the
// general one with 257 literal/length symbols (256 literals + end-of-block) and 2 distance symbols that nothing uses, the
// <257, 2> case: both distance codes get length 1, as zlib declares for a block of literals (its inflate rejects other
// incomplete distance codes).
// Size bound.  With at most 257 symbols a complete code with lengths 8 and 9 exists, so the optimal code under DEFLATE's
// 15-bit limit (package-merge below) spends at most 9 bits per byte: a block's data takes at most 9 * (BGZF_BLOCK + 1)
// bits = 64 513 bytes.  The header sends 259 code lengths with a code-length code of at most 7 bits (no run-length
// symbols), 3 + 14 + 19 * 3 + 259 * 7 bits = 237 bytes, and the gzip framing is 26 bytes: 64 776 <= 65 536.  The bound
// does not depend on the bytes, so it holds for the binary BAM records as well.
//
// Error-profile rows: every row starts with the read's name and a read has hundreds of rows, so each row's name is sent as
// a back-reference to the row before it.  The rule, a pure function of the text and the block cut [b0, b1): take a row
// starting at s whose previous row starts at p >= b0, and let f be the number of bytes before the row's first TAB.  If
// text[p, p+f+1) == text[s, s+f+1) and s - p <= 32768, then text[s, min(s+f+1, b1)) is coded as back-references with
// distance s - p when that span is at least 4 bytes long: pieces of 258 bytes, except that a piece shorter than 4 at the
// end borrows from the one before it (bgzf_rows_piece).  Every other byte is a literal.  The literal/length alphabet has
// 286 symbols and the distance alphabet 30; both codes are built with package-merge (limit 15), and a block with fewer
// than two distance symbols gets a second one of length 1, as zlib does.
// Size bound.  A complete code of at most 9 bits exists for 286 literal/length symbols and one of 5 bits for 30
// distance codes; a match of 4 or more bytes then costs at most 9 + 5 + 5 + 13 = 32 bits, at most 8 bits per byte.  So
// the optimal codes still spend at most 9 bits per text byte: at most 64 513 bytes of data per block.  The header sends
// all 286 + 30 code lengths, at most (3 + 14 + 19 * 3 + 316 * 7) / 8 -> 286 bytes, and with the 26 bytes of framing a
// member takes at most 64 825 <= 65 536 bytes.
//
// The kernel still checks every member and reports a violation of either bound (there is no stored-block fallback).
#pragma once
#include <cub/block/block_scan.cuh>

constexpr uint32_t BGZF_BLOCK = 56u << 10;          // uncompressed text bytes per member (the last one may be shorter)
constexpr uint32_t BGZF_MAX_MEMBER = 65536u;        // BSIZE is a 16-bit field holding the member size - 1
constexpr uint32_t BGZF_SLOT = 65536u;              // staging bytes per member (raw DEFLATE data, word aligned)
constexpr uint32_t BGZF_FRAME = 26u;                // 18-byte header with the BC subfield + CRC32 + ISIZE
constexpr int BGZF_THREADS = 512;
constexpr int BGZF_SYMS = 257;                      // literals + end-of-block
constexpr int BGZF_LL_SYMS = 286;                   // literals, end-of-block, length codes 257..285
constexpr int BGZF_D_SYMS = 30;                     // distance codes
constexpr uint32_t BGZF_WINDOW = 32768u;
constexpr uint32_t BGZF_CRC_POLY = 0xedb88320u;     // CRC-32 (gzip), reflected
// order in which the header sends the code-length code's lengths (RFC 1951 §3.2.7)
__constant__ uint8_t kBgzfClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// where bgzf_deflate_kernel leaves the members of text_bytes of text, one per BGZF_BLOCK
struct BgzfMembers {
    uint64_t text_bytes;
    uint8_t* stage;                 // BGZF_SLOT bytes per member: its DEFLATE data
    uint64_t* member_size;          // BGZF_FRAME + DEFLATE bytes
    uint2* trailer;                 // CRC32, ISIZE
    unsigned long long* oversize;   // members above BGZF_MAX_MEMBER
};

// shared-memory layout for NLL literal/length and ND distance symbols
template <int NLL, int ND>
struct BgzfSmem {
    uint8_t text[BGZF_BLOCK];
    union {
        uint32_t hist[BGZF_THREADS / 32][NLL];                  // per-warp literal/length histograms
        struct {
            uint32_t w[2][2 * NLL];
            uint8_t pkg[15][2 * NLL];
        } pm;                                                   // package-merge lists (2n - 2 items are ever selected)
    } u;
    uint32_t crc_tab[256];
    uint32_t x2n[32];                                           // x^(2^k) mod P
    uint32_t span_crc[BGZF_THREADS];
    uint32_t span_len[BGZF_THREADS];
    uint32_t freq[NLL];
    uint32_t code[NLL];                                         // bit-reversed canonical codes (DEFLATE sends LSB first)
    uint16_t sorted[NLL];
    uint8_t len[NLL];
    uint8_t len_sorted[NLL];
    uint32_t dfreq[ND];
    uint32_t dcode[ND];
    uint8_t dlen[ND];
    uint32_t cl_code[19];                                       // code-length code
    uint8_t cl_len[19];
    uint32_t hclen;
    uint32_t hdr_bits;
    typename cub::BlockScan<uint32_t, BGZF_THREADS>::TempStorage scan;
};

// GF(2) product of two reflected polynomials mod P (zlib's multmodp)
__device__ __forceinline__ uint32_t bgzf_multmodp(uint32_t a, uint32_t b) {
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = (b & 1) ? (b >> 1) ^ BGZF_CRC_POLY : b >> 1;
    }
    return p;
}
// CRC-32 of A followed by B from crc(A), crc(B) and |B|: crc(A) * x^(8|B|) + crc(B)
__device__ __forceinline__ uint32_t bgzf_crc_combine(const uint32_t* x2n, uint32_t crc_a, uint32_t crc_b, uint32_t len_b) {
    uint32_t p = 1u << 31;                                      // x^0
    for (uint32_t n = len_b, k = 3; n; n >>= 1, ++k)
        if (n & 1) p = bgzf_multmodp(x2n[k & 31], p);
    return bgzf_multmodp(p, crc_a) ^ crc_b;
}

// Optimal code lengths under a length limit (package-merge) for n >= 2 weights sorted ascending; len[k] belongs to w[k].
// Level 0 lists the leaves; level j merges the leaves with the pairs of level j-1's list.  The first 2n - 2 items of the
// top level are the solution: every leaf among the first m items of a level gains one bit, and the packages among them
// select the first 2 * packages items of the level below.  S: the kernel's shared-memory layout (its u.pm lists).
// This and bgzf_canonical are inlined by force: left to the inliner, their code in a kernel depends on how many kernels
// call them, and a second instantiation of the records kernel left it with 40 registers and 20 B of spills instead of
// 57 and none.
template <class S>
__device__ __forceinline__ void bgzf_package_merge(S& s, const uint32_t* w, int n, int limit, uint8_t* len) {
    const int cap = 2 * n - 2;
    uint32_t* prev = s.u.pm.w[0];
    uint32_t* cur = s.u.pm.w[1];
    for (int k = 0; k < n; ++k) {
        prev[k] = w[k];
        s.u.pm.pkg[0][k] = 0;
        len[k] = 0;
    }
    int prev_n = n;
    for (int lev = 1; lev < limit; ++lev) {
        const int np = prev_n / 2;
        int i = 0, j = 0, m = 0;
        while (m < cap && (i < n || j < np)) {
            const uint32_t pw = j < np ? prev[2 * j] + prev[2 * j + 1] : 0xffffffffu;
            if (i < n && w[i] <= pw) {
                cur[m] = w[i++];
                s.u.pm.pkg[lev][m] = 0;
            } else {
                cur[m] = pw;
                ++j;
                s.u.pm.pkg[lev][m] = 1;
            }
            ++m;
        }
        prev_n = m;
        uint32_t* t = prev;
        prev = cur;
        cur = t;
    }
    int m = cap;
    for (int lev = limit - 1; lev >= 0 && m > 0; --lev) {
        int leaves = 0;
        for (int t = 0; t < m; ++t) leaves += s.u.pm.pkg[lev][t] ? 0 : 1;
        for (int k = 0; k < leaves; ++k) ++len[k];
        m = 2 * (m - leaves);
    }
}

// canonical codes (RFC 1951 §3.2.2), bit-reversed
__device__ __forceinline__ void bgzf_canonical(const uint8_t* len, int n, uint32_t* code) {
    uint32_t count[16] = {0}, next[16];
    for (int k = 0; k < n; ++k) ++count[len[k]];
    count[0] = 0;
    uint32_t c = 0;
    for (int b = 1; b < 16; ++b) {
        c = (c + count[b - 1]) << 1;
        next[b] = c;
    }
    for (int k = 0; k < n; ++k)
        code[k] = len[k] ? __brev(next[len[k]]++) >> (32 - len[k]) : 0u;
}

// OR `nb` bits of `v` into the zeroed word stream at bit `pos` (bits that other threads also touch)
__device__ __forceinline__ void bgzf_or_bits(uint32_t* out, uint64_t& pos, uint32_t v, int nb) {
    const uint64_t x = (uint64_t)v << (pos & 31);
    atomicOr(out + (pos >> 5), (uint32_t)x);
    if ((pos & 31) + nb > 32) atomicOr(out + (pos >> 5) + 1, (uint32_t)(x >> 32));
    pos += nb;
}

// ---------------------------------------------------------------------------------------------------------------------
// records: one per read of the last batch, in a layout's bytes
// ---------------------------------------------------------------------------------------------------------------------

// one read's record as the text and BAM layouts see it: its name (nl bytes), its bases and qualities (L each; ql null
// without --fastq)
struct BgzfReadRec {
    const char* nm;
    const uint8_t* sq;
    const uint8_t* ql;
    uint32_t nl, L, fastq;
};
// the records of the text and BAM layouts: one per read of the batch
struct BgzfReadTable {
    const NsReadMeta* reads;
    const uint8_t* seq;
    const uint8_t* qual;
    const char* names;
    const uint64_t* name_off;
    const uint32_t* name_len;
    uint32_t fastq;
    __device__ __forceinline__ BgzfReadRec operator[](uint32_t r) const {
        const NsReadMeta rm = reads[r];
        return BgzfReadRec{names + name_off[r], seq + rm.seq_off, fastq ? qual + rm.seq_off : nullptr, name_len[r], rm.seq_len, fastq};
    }
};

// FASTA/FASTQ text (host_io.cu:format_records_impl): '>' name '\n' seq '\n', FASTQ '@' name '\n' seq '\n' '+' '\n' qual '\n'
struct BgzfTextLayout {
    using Table = BgzfReadTable;
    static constexpr uint32_t max_name = 0;                     // names of any length
    static __device__ __forceinline__ uint64_t size(uint32_t nl, uint64_t L, uint32_t fastq) {
        return fastq ? 1 + nl + 1 + L + 1 + 2 + L + 1 : 1 + nl + 1 + L + 1;
    }
    // byte q of a record
    static __device__ __forceinline__ uint8_t byte(uint64_t q, const BgzfReadRec& rc) {
        const uint32_t nl = rc.nl, L = rc.L, fastq = rc.fastq;
        if (q == 0) return fastq ? '@' : '>';
        if (q <= nl) return (uint8_t)rc.nm[q - 1];
        q -= nl + 1;
        if (q == 0) return '\n';
        q -= 1;
        if (q < L) return rc.sq[q];
        q -= L;
        if (q == 0 || !fastq) return '\n';
        if (q == 1) return '+';
        if (q == 2) return '\n';
        q -= 3;
        return q < L ? rc.ql[q] : '\n';
    }
};

// BAM output (ns_compress_bam): one unmapped record per read in read orientation (SAM/BAM format specification §4.2):
// block_size, refID -1, pos -1, l_read_name, mapq 255, bin 4680 (reg2bin(-1, 0)), n_cigar_op 0, flag 4, l_seq,
// next_refID -1, next_pos -1, tlen 0 (36 bytes, little-endian), the name and its NUL, the bases as 4-bit codes (first
// base in the high nibble, the low nibble of an odd last byte 0), the qualities - 33 (FASTQ) or 0xff each (FASTA)
constexpr uint32_t BAM_FIXED = 36;
constexpr uint32_t BAM_MAX_NAME = 254;              // l_read_name is one byte and counts the NUL

// 4-bit codes of the letters a..z of either case ("=ACMGRSVTWYHKDBN" -> 0..15, U as T as htslib reads it, other letters
// N), 16 nibbles to a word, so that the per-byte lookup is register arithmetic
constexpr uint64_t bam_letter_nibbles(int first) {
    const char* abc = "=ACMGRSVTWYHKDBN";
    uint64_t w = 0;
    for (int k = 0; k < 16 && first + k < 26; ++k) {
        const char c = (char)('A' + first + k);
        uint64_t v = c == 'U' ? 8 : 15;
        for (int j = 1; j < 16; ++j)
            if (abc[j] == c) v = (uint64_t)j;
        w |= v << (4 * k);
    }
    return w;
}
constexpr uint64_t kBamNibblesAtoP = bam_letter_nibbles(0), kBamNibblesQtoZ = bam_letter_nibbles(16);

__device__ __forceinline__ uint32_t bam_base_code(uint8_t c) {
    if (c == '=') return 0;
    const uint32_t k = (uint32_t)(c | 0x20) - 'a';            // 0..25 exactly for the letters of either case
    if (k >= 26) return 15;
    return (uint32_t)(((k < 16 ? kBamNibblesAtoP : kBamNibblesQtoZ) >> (4 * (k & 15))) & 15u);
}

struct BgzfBamLayout {
    using Table = BgzfReadTable;
    static constexpr uint32_t max_name = BAM_MAX_NAME;          // a longer name fails the call
    static __device__ __forceinline__ uint64_t size(uint32_t nl, uint64_t L, uint32_t) {
        return BAM_FIXED + nl + 1 + (L + 1) / 2 + L;
    }
    // byte q of a read's BAM record
    static __device__ __forceinline__ uint8_t byte(uint64_t q, const BgzfReadRec& rc) {
        const uint32_t nl = rc.nl, L = rc.L;
        if (q < BAM_FIXED) {
            uint32_t w;
            switch ((uint32_t)q >> 2) {
            case 0: w = BAM_FIXED - 4 + nl + 1 + (L + 1) / 2 + L; break;          // block_size
            case 3: w = (nl + 1) | (255u << 8) | (4680u << 16); break;          // l_read_name, mapq, bin
            case 4: w = 4u << 16; break;                                        // n_cigar_op, flag
            case 5: w = L; break;                                               // l_seq
            case 8: w = 0; break;                                               // tlen
            default: w = 0xffffffffu;                                           // refID, pos, next_refID, next_pos
            }
            return (uint8_t)(w >> (8 * ((uint32_t)q & 3)));
        }
        q -= BAM_FIXED;
        if (q < nl) return (uint8_t)rc.nm[q];
        if (q == nl) return 0;
        q -= nl + 1;
        const uint64_t n_packed = (L + 1) / 2;
        if (q < n_packed) {
            const uint64_t b = 2 * q;
            return (uint8_t)((bam_base_code(rc.sq[b]) << 4) | (b + 1 < L ? bam_base_code(rc.sq[b + 1]) : 0u));
        }
        q -= n_packed;
        return rc.fastq ? (uint8_t)(rc.ql[q] - 33) : 0xffu;
    }
};

// one read's record size; the name length is taken on the device from the NUL-terminated name, and names longer than the
// layout's max_name (if it has one) are counted into *long_names (the call then fails)
template <class Layout>
__global__ void record_size_kernel(const NsReadMeta* __restrict__ reads, uint32_t n, const char* __restrict__ names,
                                   const uint64_t* __restrict__ name_off, uint32_t fastq, uint32_t* __restrict__ name_len,
                                   uint64_t* __restrict__ size, unsigned long long* long_names) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const char* nm = names + name_off[i];
    uint32_t nl = 0;
    while (nm[nl]) ++nl;
    name_len[i] = nl;
    if (Layout::max_name && nl > Layout::max_name) atomicAdd(long_names, 1ull);
    size[i] = Layout::size(nl, reads[i].seq_len, fastq);
}

// bgzf_deflate_kernel's source of records in `Layout`, every byte a literal.  Record r is tab[r] (Layout::Table), its
// bytes Layout::byte(q, tab[r]).
template <class Layout>
struct BgzfRecords {
    static constexpr int NLL = BGZF_SYMS, ND = 2;
    using Smem = BgzfSmem<NLL, ND>;
    typename Layout::Table tab;
    const uint64_t* rec_off;        // exclusive prefix sum of the record sizes
    uint32_t n_recs;

    // gather this thread's span [lo, hi) of the block at t0
    __device__ __forceinline__ void load(Smem& s, uint64_t t0, uint64_t text_bytes, uint32_t, uint32_t lo, uint32_t hi) {
        if (lo >= hi) return;
        uint64_t p = t0 + lo;
        uint32_t rl = 0, rh = n_recs;                           // last record with rec_off <= p
        while (rh - rl > 1) {
            const uint32_t mid = (rl + rh) >> 1;
            if (rec_off[mid] <= p) rl = mid; else rh = mid;
        }
        uint32_t k = lo;
        for (uint32_t r = rl; k < hi; ++r) {                    // the records this span overlaps
            const uint64_t r0 = rec_off[r], r1 = r + 1 < n_recs ? rec_off[r + 1] : text_bytes;
            const auto rc = tab[r];
            for (; k < hi && p < r1; ++k, ++p) s.text[k] = Layout::byte(p - r0, rc);
        }
    }
    // thread t's tokens start at its byte span
    __device__ __forceinline__ uint32_t cut(const Smem&, uint32_t t, uint32_t span, uint32_t blen) const { return min(t * span, blen); }
    template <class Fn>
    __device__ __forceinline__ void tokens(const Smem& s, uint32_t lo, uint32_t hi, uint32_t, Fn fn) const {
        for (uint32_t k = lo; k < hi; ++k) fn((uint32_t)s.text[k], 0u, 0u);
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// flat text of rows (the error profile) with one back-reference per row for the repeated read name; see the header
// ---------------------------------------------------------------------------------------------------------------------

// length symbol (RFC 1951 §3.2.5) of a match of 3..258 bytes: symbol, extra bits, their value
__device__ __forceinline__ uint3 bgzf_len_sym(uint32_t n) {
    if (n == 258) return make_uint3(285, 0, 0);
    const uint32_t v = n - 3;
    if (v < 8) return make_uint3(257 + v, 0, 0);
    const uint32_t e = 29 - __clz(v);                          // floor(log2 v) - 2
    return make_uint3(261 + 4 * e + ((v >> e) & 3u), e, v & ((1u << e) - 1));
}
// distance symbol of a distance of 1..32768
__device__ __forceinline__ uint3 bgzf_dist_sym(uint32_t d) {
    const uint32_t v = d - 1;
    if (v < 4) return make_uint3(v, 0, 0);
    const uint32_t e = 30 - __clz(v);                          // floor(log2 v) - 1
    return make_uint3(2 * e + 2 + ((v >> e) & 1u), e, v & ((1u << e) - 1));
}
// the next piece of a back-reference with `rem` >= 4 bytes left: 258 bytes, or fewer so that at least 4 remain
__device__ __forceinline__ uint32_t bgzf_rows_piece(uint32_t rem) { return rem <= 258 ? rem : (rem - 258 < 4 ? rem - 4 : 258); }

// where thread t's tokens start: the first row start at or after its byte span (thread 0: the block's first byte).  A
// back-reference never crosses a row, so every thread codes its rows on its own.
__device__ __forceinline__ uint32_t bgzf_rows_cut(const BgzfSmem<BGZF_LL_SYMS, BGZF_D_SYMS>& s, uint32_t t, uint32_t span,
                                                  uint32_t blen) {
    if (t == 0) return 0;
    uint32_t k = min(t * span, blen);
    while (k < blen && s.text[k - 1] != '\n') ++k;
    return k;
}

// The back-reference of the row starting at block offset k (k >= 1, text[k-1] == '\n'): (length, distance), length 0
// when there is none.  g: the text at the block's start (the row's name may run past the block); left: text bytes from
// there; row0: the block starts with a row.
__device__ uint2 bgzf_row_match(const BgzfSmem<BGZF_LL_SYMS, BGZF_D_SYMS>& s, const uint8_t* __restrict__ g, uint32_t k,
                                uint32_t blen, uint64_t left, bool row0) {
    uint32_t p = k - 1;                                         // the previous row's start
    while (p > 0 && s.text[p - 1] != '\n') --p;
    if ((p == 0 && !row0) || k - p > BGZF_WINDOW) return make_uint2(0, 0);
    uint32_t f = 0;                                             // bytes before the row's first TAB
    for (;; ++f) {
        if (k + f >= left) return make_uint2(0, 0);
        const uint8_t c = k + f < blen ? s.text[k + f] : g[k + f];
        if (c == '\t') break;
        if (c == '\n') return make_uint2(0, 0);
    }
    for (uint32_t t = 0; t <= f; ++t)                           // p + t < k <= blen: the previous row is in shared memory
        if (s.text[p + t] != (k + t < blen ? s.text[k + t] : g[k + t])) return make_uint2(0, 0);
    const uint32_t m = min(f + 1, blen - k);
    return m >= 4 ? make_uint2(m, k - p) : make_uint2(0, 0);
}

// the tokens of [lo, hi): fn(c, 0, 0) for a literal byte c, fn(0, n, d) for a back-reference piece of n bytes, distance d
template <class Fn>
__device__ __forceinline__ void bgzf_rows_tokens(const BgzfSmem<BGZF_LL_SYMS, BGZF_D_SYMS>& s, const uint8_t* __restrict__ g,
                                                 uint32_t lo, uint32_t hi, uint32_t blen, uint64_t left, bool row0, Fn fn) {
    for (uint32_t k = lo; k < hi;) {
        if (k > 0 && s.text[k - 1] == '\n') {
            const uint2 m = bgzf_row_match(s, g, k, blen, left, row0);
            if (m.x) {
                for (uint32_t rem = m.x; rem;) {
                    const uint32_t n = bgzf_rows_piece(rem);
                    fn(0u, n, m.y);
                    rem -= n;
                }
                k += m.x;
                continue;
            }
        }
        fn((uint32_t)s.text[k], 0u, 0u);
        ++k;
    }
}

// bgzf_deflate_kernel's source of error-profile rows
struct BgzfRows {
    static constexpr int NLL = BGZF_LL_SYMS, ND = BGZF_D_SYMS;
    using Smem = BgzfSmem<NLL, ND>;
    const uint8_t* text;
    // the block's, set by load: the text at its start, the text bytes from there, whether it starts with a row
    const uint8_t* g = nullptr;
    uint64_t left = 0;
    bool row0 = false;

    __device__ __forceinline__ void load(Smem& s, uint64_t t0, uint64_t text_bytes, uint32_t blen, uint32_t, uint32_t) {
        g = text + t0;
        left = text_bytes - t0;
        row0 = t0 == 0 || text[t0 - 1] == '\n';
        for (uint32_t k = threadIdx.x; k < blen; k += BGZF_THREADS) s.text[k] = g[k];
    }
    __device__ __forceinline__ uint32_t cut(const Smem& s, uint32_t t, uint32_t span, uint32_t blen) const {
        return bgzf_rows_cut(s, t, span, blen);
    }
    template <class Fn>
    __device__ __forceinline__ void tokens(const Smem& s, uint32_t lo, uint32_t hi, uint32_t blen, Fn fn) const {
        bgzf_rows_tokens(s, g, lo, hi, blen, left, row0, fn);
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// one member per block of 512 threads
// ---------------------------------------------------------------------------------------------------------------------
template <class Source>
__global__ void __launch_bounds__(BGZF_THREADS) bgzf_deflate_kernel(Source src, BgzfMembers a) {
    constexpr int NLL = Source::NLL, ND = Source::ND;
    using Smem = typename Source::Smem;
    extern __shared__ __align__(16) unsigned char bgzf_smem_raw[];
    Smem& s = *reinterpret_cast<Smem*>(bgzf_smem_raw);
    const uint32_t tid = threadIdx.x, warp = tid >> 5;
    const uint64_t t0 = (uint64_t)blockIdx.x * BGZF_BLOCK;
    const uint32_t blen = (uint32_t)min((uint64_t)BGZF_BLOCK, a.text_bytes - t0);
    const uint32_t span = (blen + BGZF_THREADS - 1) / BGZF_THREADS;
    const uint32_t lo = min(tid * span, blen), hi = min(lo + span, blen);

    if (tid < 256) {
        uint32_t c = tid;
        for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ BGZF_CRC_POLY : c >> 1;
        s.crc_tab[tid] = c;
    }
    if (tid == 0) {
        uint32_t p = 1u << 30;                                  // x^1
        s.x2n[0] = p;
        for (int k = 1; k < 32; ++k) s.x2n[k] = p = bgzf_multmodp(p, p);
    }
    for (uint32_t k = tid; k < (BGZF_THREADS / 32) * NLL; k += BGZF_THREADS) (&s.u.hist[0][0])[k] = 0;
    if (tid < ND) s.dfreq[tid] = 0;
    src.load(s, t0, a.text_bytes, blen, lo, hi);
    __syncthreads();

    // CRC of the byte span; symbols of this thread's tokens
    uint32_t crc = 0xffffffffu;
    for (uint32_t k = lo; k < hi; ++k) crc = s.crc_tab[(crc ^ s.text[k]) & 0xffu] ^ (crc >> 8);
    s.span_crc[tid] = lo < hi ? ~crc : 0u;
    s.span_len[tid] = hi - lo;
    const uint32_t tlo = src.cut(s, tid, span, blen), thi = src.cut(s, tid + 1, span, blen);
    src.tokens(s, tlo, thi, blen, [&](uint32_t c, uint32_t n, uint32_t d) {
        if (n == 0) {
            atomicAdd(&s.u.hist[warp][c], 1u);
        } else {
            atomicAdd(&s.u.hist[warp][bgzf_len_sym(n).x], 1u);
            atomicAdd(&s.dfreq[bgzf_dist_sym(d).x], 1u);
        }
    });
    __syncthreads();
    // spans combine pairwise, left to right: [i, i+d) and [i+d, i+2d)
    for (uint32_t d = 1; d < BGZF_THREADS; d <<= 1) {
        if ((tid & (2 * d - 1)) == 0 && s.span_len[tid + d])
            s.span_crc[tid] = bgzf_crc_combine(s.x2n, s.span_crc[tid], s.span_crc[tid + d], s.span_len[tid + d]);
        __syncthreads();
        if ((tid & (2 * d - 1)) == 0) s.span_len[tid] += s.span_len[tid + d];
        __syncthreads();
    }
    if (tid < NLL) {
        uint32_t f = 0;
        for (int w = 0; w < BGZF_THREADS / 32; ++w) f += s.u.hist[w][tid];
        s.freq[tid] = tid == 256 ? 1u : f;                      // end-of-block
    }
    __syncthreads();

    // literal/length symbols in use, ascending by (frequency, symbol)
    if (tid < NLL && s.freq[tid]) {
        const uint32_t f = s.freq[tid];
        uint32_t rank = 0;
        for (int t = 0; t < NLL; ++t) {
            const uint32_t g = s.freq[t];
            rank += (g && (g < f || (g == f && t < (int)tid))) ? 1u : 0u;
        }
        s.sorted[rank] = (uint16_t)tid;
    }
    const int n_used = __syncthreads_count(tid < NLL && s.freq[tid] != 0);

    if (tid == 0) {
        // literal/length code: package-merge over the used symbols (the histograms and the span lengths are dead: their
        // space holds the lists and the sorted weights)
        uint32_t* w = s.span_len;
        for (int k = 0; k < n_used; ++k) w[k] = s.freq[s.sorted[k]];
        bgzf_package_merge(s, w, n_used, 15, s.len_sorted);
        for (int k = 0; k < NLL; ++k) s.len[k] = 0;
        for (int k = 0; k < n_used; ++k) s.len[s.sorted[k]] = s.len_sorted[k];
        bgzf_canonical(s.len, NLL, s.code);
        // distance code: the used symbols by (frequency, symbol); fewer than two get a second symbol of length 1
        uint8_t dsym[ND], dlen_sorted[ND];
        int nd = 0;
        for (int v = 0; v < ND; ++v) {
            s.dlen[v] = 0;
            if (s.dfreq[v]) {
                int at = nd++;
                while (at > 0 && (w[at - 1] > s.dfreq[v])) {
                    w[at] = w[at - 1];
                    dsym[at] = dsym[at - 1];
                    --at;
                }
                w[at] = s.dfreq[v];
                dsym[at] = (uint8_t)v;
            }
        }
        if (nd >= 2) {
            bgzf_package_merge(s, w, nd, 15, dlen_sorted);
            for (int k = 0; k < nd; ++k) s.dlen[dsym[k]] = dlen_sorted[k];
        } else {
            const int c = nd ? dsym[0] : 0;
            s.dlen[c] = 1;
            s.dlen[c == 0 ? 1 : 0] = 1;
        }
        bgzf_canonical(s.dlen, ND, s.dcode);
        // code-length code over the NLL literal/length and the ND distance code lengths, limit 7
        uint32_t clf[16] = {0};
        for (int k = 0; k < NLL; ++k) ++clf[s.len[k]];
        for (int k = 0; k < ND; ++k) ++clf[s.dlen[k]];
        uint8_t cl_sym[16], cl_len_sorted[16];
        uint32_t cl_w[16];
        uint8_t* cl_len = s.cl_len;
        for (int k = 0; k < 19; ++k) cl_len[k] = 0;
        int nc = 0;
        for (int v = 0; v < 16; ++v)
            if (clf[v]) {
                int at = nc++;                                  // insertion by (frequency, symbol)
                while (at > 0 && cl_w[at - 1] > clf[v]) {
                    cl_w[at] = cl_w[at - 1];
                    cl_sym[at] = cl_sym[at - 1];
                    --at;
                }
                cl_w[at] = clf[v];
                cl_sym[at] = (uint8_t)v;
            }
        bgzf_package_merge(s, cl_w, nc, 7, cl_len_sorted);
        for (int k = 0; k < nc; ++k) cl_len[cl_sym[k]] = cl_len_sorted[k];
        bgzf_canonical(cl_len, 19, s.cl_code);
        int hclen = 19;
        while (hclen > 4 && cl_len[kBgzfClOrder[hclen - 1]] == 0) --hclen;
        s.hclen = (uint32_t)hclen;
        // BFINAL, BTYPE, HLIT, HDIST, HCLEN, the code-length code, the NLL + ND code lengths
        uint32_t bits = 3 + 5 + 5 + 4 + 3 * hclen;
        for (int k = 0; k < NLL; ++k) bits += cl_len[s.len[k]];
        for (int k = 0; k < ND; ++k) bits += cl_len[s.dlen[k]];
        s.hdr_bits = bits;
    }
    __syncthreads();

    // bit count of this thread's tokens, then their offset behind the header
    uint32_t nbits = 0;
    src.tokens(s, tlo, thi, blen, [&](uint32_t c, uint32_t n, uint32_t d) {
        if (n == 0) {
            nbits += s.len[c];
        } else {
            const uint3 l = bgzf_len_sym(n), q = bgzf_dist_sym(d);
            nbits += s.len[l.x] + l.y + s.dlen[q.x] + q.y;
        }
    });
    uint32_t off = 0, data_bits = 0;
    cub::BlockScan<uint32_t, BGZF_THREADS>(s.scan).ExclusiveSum(nbits, off, data_bits);
    const uint64_t total_bits = (uint64_t)s.hdr_bits + data_bits + s.len[256];
    const uint32_t payload = (uint32_t)((total_bits + 7) / 8);
    uint32_t* out = reinterpret_cast<uint32_t*>(a.stage + (uint64_t)blockIdx.x * BGZF_SLOT);
    const uint32_t n_words = min((uint32_t)((total_bits + 31) / 32), BGZF_SLOT / 4);
    for (uint32_t k = tid; k < n_words; k += BGZF_THREADS) out[k] = 0;
    __syncthreads();
    if (payload + BGZF_FRAME > BGZF_MAX_MEMBER) {              // cannot happen (see the bounds above); reported, not written
        if (tid == 0) {
            atomicAdd(a.oversize, 1ull);
            a.member_size[blockIdx.x] = 0;
            a.trailer[blockIdx.x] = make_uint2(0, 0);
        }
        return;
    }

    if (tid == 0) {
        uint64_t pos = 0;
        bgzf_or_bits(out, pos, 1u, 1);                          // BFINAL
        bgzf_or_bits(out, pos, 2u, 2);                          // BTYPE: dynamic Huffman
        bgzf_or_bits(out, pos, NLL - 257, 5);                   // HLIT: NLL literal/length codes
        bgzf_or_bits(out, pos, ND - 1, 5);                      // HDIST: ND distance codes
        bgzf_or_bits(out, pos, s.hclen - 4, 4);
        for (uint32_t k = 0; k < s.hclen; ++k) bgzf_or_bits(out, pos, s.cl_len[kBgzfClOrder[k]], 3);
        for (int k = 0; k < NLL; ++k) bgzf_or_bits(out, pos, s.cl_code[s.len[k]], s.cl_len[s.len[k]]);
        for (int k = 0; k < ND; ++k) bgzf_or_bits(out, pos, s.cl_code[s.dlen[k]], s.cl_len[s.dlen[k]]);
    }

    // this thread's codes: words wholly inside its stretch are stored, the two it shares with its neighbours are OR-ed
    {
        const uint64_t start = (uint64_t)s.hdr_bits + off;
        uint64_t acc = 0;
        uint32_t fill = (uint32_t)(start & 31), w = (uint32_t)(start >> 5);
        bool first = (start & 31) != 0;
        auto put = [&](uint32_t v, uint32_t nb) {              // nb <= 15: one word completes at most
            acc |= (uint64_t)v << fill;
            fill += nb;
            if (fill >= 32) {
                if (first) atomicOr(out + w, (uint32_t)acc);
                else out[w] = (uint32_t)acc;
                first = false;
                ++w;
                acc >>= 32;
                fill -= 32;
            }
        };
        src.tokens(s, tlo, thi, blen, [&](uint32_t c, uint32_t n, uint32_t d) {
            if (n == 0) {
                put(s.code[c], s.len[c]);
            } else {
                const uint3 l = bgzf_len_sym(n), q = bgzf_dist_sym(d);
                put(s.code[l.x], s.len[l.x]);
                if (l.y) put(l.z, l.y);
                put(s.dcode[q.x], s.dlen[q.x]);
                if (q.y) put(q.z, q.y);
            }
        });
        if (tid == BGZF_THREADS - 1) put(s.code[256], s.len[256]);     // end-of-block closes the stream
        if (fill > 0) atomicOr(out + w, (uint32_t)acc);
    }
    if (tid == 0) {
        a.member_size[blockIdx.x] = payload + BGZF_FRAME;
        a.trailer[blockIdx.x] = make_uint2(s.span_crc[0], blen);
    }
}

// members into one buffer at their scanned offsets: BGZF header, DEFLATE data, CRC32, ISIZE
__global__ void bgzf_pack_kernel(const uint8_t* __restrict__ stage, const uint64_t* __restrict__ member_size,
                                 const uint64_t* __restrict__ member_off, const uint2* __restrict__ trailer, uint8_t* __restrict__ out) {
    const uint32_t b = blockIdx.x;
    const uint32_t size = (uint32_t)member_size[b];
    if (size == 0) return;
    uint8_t* dst = out + member_off[b];
    const uint8_t* src = stage + (uint64_t)b * BGZF_SLOT;
    const uint32_t payload = size - BGZF_FRAME;
    if (threadIdx.x < 18) {
        const uint32_t bsize = size - 1;
        const uint8_t hdr[18] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, (uint8_t)bsize, (uint8_t)(bsize >> 8)};
        dst[threadIdx.x] = hdr[threadIdx.x];
    } else if (threadIdx.x < 26) {
        const uint32_t k = threadIdx.x - 18;
        const uint2 t = trailer[b];
        const uint32_t v = k < 4 ? t.x : t.y;
        dst[18 + payload + k] = (uint8_t)(v >> (8 * (k & 3)));
    }
    for (uint32_t k = threadIdx.x; k < payload; k += blockDim.x) dst[18 + k] = src[k];
}
