// Emit kernel: applies each piece's edit script to the reference and writes bases + base qualities.
//
// This is extract_read's slice (/root/reference/src/simulator.py:1750-1781), case_convert (:743-755), mutate_read's
// string edits and quality interleaving (:1957-2015), the head/tail synthesis (:1421-1427), reverse_complement
// (:1433-1435, :1675-1680) and the per-state quality draws (model_base_qualities.py:120-130) in ONE pass:
//
//   * a warp owns one piece (an aligned segment with its head/tail, a chimeric gap, or an unaligned read) and
//     streams its ops 32 at a time; a warp-wide scan turns them into ring entries {output start, reference offset
//     within the chromosome, length, per-op constants} in shared memory (deletions only advance the reference offset
//     and get no entry; a pad entry aligns the piece to its first 16-byte chunk, a sentinel closes it);
//   * every lane produces one 16-byte output chunk per step.  It binary-searches the ring for the entry covering its
//     first base and then takes one of two routes, chosen per piece (warp-uniform):
//       FAST  the piece's reference span holds plain a/c/g/t only (DevRef::exc_pre) and does not wrap: the lane walks
//             the ENTRIES that overlap its chunk.  For an entry that reads the reference it fetches the 16 bases that
//             start at its first base from the 2-bit copy of the reference (two 32-bit loads + one funnel shift; a BREV
//             and a pair swap for a backward walk), shifts them into place and merges them under a mask into a 32-bit
//             accumulator of 16 2-bit bases; inserted / head-tail bases are one AND with the chunk's random word;
//             substituted bases are collected in a bit mask and patched afterwards, all 16 positions at once, by a
//             carry-less 2-bit add of a word of offsets 1..3; the quality state of every base lives in a second 2-bit
//             word that starts as "match" everywhere.  Four PRMTs turn the accumulator into ASCII.
//       EXACT a branch-free 16-base walk over the reference BYTES (case, IUPAC codes, circular wrap-around, the
//             complemented backward walk of minus-strand genome pieces): a predicated ring advance, a predicated byte
//             load and one table lookup for the case / IUPAC class per base; IUPAC codes raise a flag and are
//             resolved by a per-base routine.
//     Both routes draw the same random bits for the same base, so a read's bytes do not depend on the route (tested
//     by forcing the exact route: NS_FLAG_EMIT_EXACT);
//   * base qualities: one shared-memory lookup per base in a 2048-slot Walker alias table per quality state, built on
//     the host from the state's 24-bit pmf (slot = 11 bits, acceptance threshold = 13 bits: exact to 2^-24);
//   * reverse-strand reads are produced directly in output order by walking the edit script and the reference
//     backwards with a complemented character table (no second pass over the read);
//   * all randomness is Philox-7 keyed by (seed, read id, chunk index): per chunk of 16 bases, FASTQ draws 16 quality
//     words (slot 11 bits | threshold 13 bits | 8 spare bits) + one block {2 bits per base for inserted bases, 3 x 2 bits
//     per base for substitutions}; the spare bytes are 4 x 2 more substitution bits per base.  FASTA draws that block
//     + one block of substitution bits.  The bytes of a read therefore do not depend on the batch, the launch geometry
//     or the GPU count.
#pragma once
#include "device_common.cuh"

#define EMIT_WARPS 8
#define EMIT_RING 256
// Unaligned batches: their scripts hold about 0.87 ops per base, so 256 entries cover only ~290 of a step's 512 bases and
// 14 of 32 lanes idle.  Every piece of such a batch is unmapped and draws its qualities from one state's alias table, so
// the 32 KB of the other four tables hold a ring twice as long instead (same shared memory, 3 blocks per SM).
#define EMIT_RING_UNAL 512
#ifndef EMIT_MIN_BLOCKS
#define EMIT_MIN_BLOCKS 3     // resident blocks per SM the register allocation aims for
#endif

// Reference window: at the start of every 512-base step one lane asks the TMA engine for the 64 packed words (1024
// bases) the step is about to walk (cp.async.bulk global -> shared, completion on an mbarrier); the walk then reads the
// 2-bit reference from shared memory, and from global memory only when a long deletion carried it out of the window.
#ifndef EMIT_TMA_WINDOW
#define EMIT_TMA_WINDOW 1
#endif
#define EMIT_WIN_WORDS 64
#define EMIT_WINDOW_SMEM (EMIT_TMA_WINDOW ? EMIT_WARPS * (EMIT_WIN_WORDS * 4 + 8) : 0)

#define EMIT_F_RND 1u        // info bit: random base (INS, HT, pad); bit 1 is set with it (info & 3 == 3)
#define EMIT_F_REF 4u        // info bit: the base is read from the reference (COPY, MIS)
#define EMIT_F_MIS 8u        // info bit: ... and substituted by one of the three other bases

struct EmitArgs {
    DevRef ref;
    DevCfg cfg;
    uint32_t kind;
    uint32_t force_exact;        // debugging / tests: every piece takes the exact route
    uint64_t first_id;
    const NsReadMeta* reads;
    const NsPieceMeta* pieces;
    const uint32_t* ops;
    uint32_t n_pieces;
    uint8_t* seq;
    uint8_t* qual;
    const uint32_t* qlut;        // [5][QLUT_SIZE] alias table entries (built on the host from qual_cdf)
    uint32_t* counter;
    const uint32_t* order;       // piece processing order (longest first) or null
    const uint32_t* abort;       // sync-free batches: non-zero = a capacity check failed upstream, do nothing (or null)
    // long pieces are emitted EMIT_SPLIT bases per work item (split_kernel below): a piece's later stretches are extra work
    // items, taken before everything else, each starting from a checkpoint of the script walk
    const uint32_t* split_base;  // [n_pieces] first checkpoint of the piece, 0xffffffff = not split (null: nothing is split)
    const uint2* extra;          // {piece, stretch >= 1}, piece 0xffffffff = unused slot
    const uint4* ckpt;           // {op index in walking order, output start of that op, reference bases before it, -}
    const uint32_t* n_extra;     // number of extra work items (device counter written by split_kernel)
    uint32_t cap_extra;
};

// Output bases per work item of a long piece.  One warp emits ~512 bases per step; the longest read of a batch (100-600 kb)
// would keep one warp busy for milliseconds after every other warp has run out of work.
#define EMIT_SPLIT 16384u

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += t;
    }
    return v;
}

// Per-op constants of a ring entry: [1:0] 3 when the base is random (INS, HT, pad), [2] EMIT_F_REF, [3] EMIT_F_MIS,
// [15:8] the character classified when the reference is not read ('A' -> index 0, or the literal base of a LIT op),
// [31:16] byte offset of the quality state's alias table (state << 13).
// ref_comp: the piece classifies reference bytes with the COMPLEMENTING table (NS_PIECE_REF_REV); the characters stored for
// ops that do not read the reference are then pre-complemented so that they classify to the intended base.
__device__ __forceinline__ uint32_t emit_op_info(uint32_t op, bool unmapped, bool ref_comp = false) {
    const uint32_t ty = op >> 28;
    // quality state: COPY->match(2) MIS->mis(0) INS->ins(1) HT->ht(3) LIT->its own; gap/unaligned -> unmapped(4)
    const uint32_t qs = unmapped ? 4u : (ty == NS_OP_LIT ? ((op >> 24) & 3u) : ((0x30102u >> (4u * ty)) & 7u));
    uint32_t info = (qs * QLUT_SIZE * 4u) << 16;
    const uint32_t zero = ref_comp ? (uint32_t)'T' : (uint32_t)'A';          // classifies to base index 0
    if (ty < 2u) info |= EMIT_F_REF | (ty == NS_OP_MIS ? EMIT_F_MIS : 0u) | (zero << 8);
    else if (ty == NS_OP_LIT) info |= idx_base(((op >> 26) & 3u) ^ (ref_comp ? 2u : 0u)) << 8;
    else info |= 3u | (zero << 8);
    return info;
}

// ---- the random bits of one 16-base chunk -------------------------------------------------------------------------
// Drawn in two parts so that the 16 quality words are not live while the chunk's entries are walked.
struct ChunkAux {
    uint32_t RB;                  // base i's random base index in bits [2i+1:2i] (inserted, head/tail, pad bases)
    uint32_t X[3];                // substitution draws 1..3 of base i in bits [2i+1:2i]
};
template <bool FASTQ>
struct ChunkQual {
    uint32_t W[FASTQ ? 16 : 1];   // FASTQ: base i's quality word (alias slot in bits [18:8], threshold draw in [31:19])
    uint32_t X[4];                // substitution draws 4..7 (FASTQ: the low bytes of the quality words, gathered)
};

template <bool FASTQ>
__device__ __forceinline__ void draw_chunk_aux(ChunkAux& r, uint32_t id_lo, uint32_t id_hi, uint32_t kind, uint32_t chunk, uint2 key) {
    const uint4 a = FASTQ ? philox4x32_7(make_uint4(id_lo, id_hi, stream_word(ST_EMIT_Q, kind, chunk), 4u), key)
                          : philox4x32_7(make_uint4(id_lo, id_hi, stream_word(ST_EMIT_B, kind, chunk), 0u), key);
    r.RB = a.x; r.X[0] = a.y; r.X[1] = a.z; r.X[2] = a.w;
}
template <bool FASTQ>
__device__ __forceinline__ void draw_chunk_qual(ChunkQual<FASTQ>& r, uint32_t id_lo, uint32_t id_hi, uint32_t kind, uint32_t chunk, uint2 key) {
    if (FASTQ) {
        const uint32_t sw = stream_word(ST_EMIT_Q, kind, chunk);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint4 t = philox4x32_7(make_uint4(id_lo, id_hi, sw, (uint32_t)j), key);
            r.W[4 * j] = t.x; r.W[4 * j + 1] = t.y; r.W[4 * j + 2] = t.z; r.W[4 * j + 3] = t.w;
            r.X[j] = __byte_perm(__byte_perm(t.x, t.y, 0x0040), __byte_perm(t.z, t.w, 0x0040), 0x5410);
        }
    } else {
        const uint4 b = philox4x32_7(make_uint4(id_lo, id_hi, stream_word(ST_EMIT_B, kind, chunk), 1u), key);
        r.X[0] = b.x; r.X[1] = b.y; r.X[2] = b.z; r.X[3] = b.w;
        r.W[0] = 0;
    }
}

// Substitution offsets of all 16 bases of a chunk at once: field i (2 bits) = 1 + uniform{0,1,2}, what is added (mod 4) to
// a base index to replace it by one of the three other bases (random.choice of the remaining bases,
// simulator.py:1968-1973).  Field i is the first non-zero one among the seven 2-bit draws X1[i] .. X7[i] -- uniform over
// {1,2,3} -- and 1 if all seven are zero (probability 4^-7: relative bias 1.2e-4).
__host__ __device__ __forceinline__ uint32_t sub_offsets(const uint32_t (&XA)[3], const uint32_t (&XB)[4]) {
    uint32_t sub = XA[0];
#pragma unroll
    for (int j = 1; j < 7; ++j) {
        const uint32_t z = ~(sub | (sub >> 1)) & 0x55555555u;        // low bit of every field that is still zero
        sub |= (j < 3 ? XA[j] : XB[j - 3]) & (z * 3u);
    }
    return sub | (~(sub | (sub >> 1)) & 0x55555555u);
}
// per-field (a + b) mod 4 of two words of 16 2-bit fields
__host__ __device__ __forceinline__ uint32_t add_fields_mod4(uint32_t a, uint32_t b) {
    return a ^ b ^ ((a & b & 0x55555555u) << 1);
}

// Base quality from an alias-table entry: [31:19] 13-bit acceptance threshold, [15:8] alias character, [7:0] primary
// character (qual_table.h:build_qlut).  The draw w carries the slot in bits [18:8] and the threshold draw in [31:19].
__host__ __device__ __forceinline__ uint32_t qual_pick(uint32_t e, uint32_t w) {
    return ((w | 0x7ffffu) < e) ? e : (e >> 8);          // the character is the low byte of the result
}

struct EmitPiece {
    const uint8_t* cbase;    // first base of the chromosome
    uint32_t pos, clen;      // piece start within the chromosome, chromosome length
    uint32_t rdir;           // the reference is walked backwards (reverse read XOR minus-strand piece)
    uint32_t ref_comp;       // reference bases are complemented on classification (minus-strand piece)
    uint32_t tbl;            // output characters of base indices 0..3 (complemented for reverse reads)
    uint32_t piece_in_read;
    uint64_t rid;
};

// Ring entry (uint4): .x = 2 * output start (padded piece coordinate), .z = 2 * output end, .w = emit_op_info, and
// .y = reference offset of the entry's first base (within the chromosome, in walking order) MINUS its output start for a
// forward walk, PLUS it for a backward walk: the reference offset of output position p is then .y + p resp. .y - p.
// (Doubled coordinates: chunk masks are bit positions of 2-bit fields.)
__device__ __forceinline__ uint32_t entry_ref(const uint4& e, uint32_t rdir, uint32_t p) { return rdir ? e.y - p : e.y + p; }

// Exact path for ONE base whose reference byte is not plain ACGT (IUPAC codes): locates the ring entry of padded piece
// coordinate x again and redoes the base with the same random bits.  Returns the character.
template <uint32_t RING>
__device__ __noinline__ uint32_t emit_fix_base(const EmitArgs& a, const EmitPiece& pc, const uint4* ring, uint32_t w_ret,
                                               uint32_t w_loaded, uint32_t x, uint32_t rb2, uint32_t misoff) {
    uint32_t l = w_ret, h = w_loaded;
    while (h - l > 1) {
        uint32_t mid = (l + h) >> 1;
        if (ring[mid & (RING - 1)].x <= 2u * x) l = mid; else h = mid;
    }
    const uint4 e = ring[l & (RING - 1)];
    const uint32_t info = e.w;
    uint32_t oi;
    if (info & EMIT_F_REF) {
        uint32_t rabs = entry_ref(e, pc.rdir, x);
        if (rabs >= pc.clen) rabs += pc.rdir ? pc.clen : 0u - pc.clen;
        uint32_t c = __ldg(pc.cbase + rabs);
        if (c - 'a' < 26u) c -= 32;
        if (!acgt_fast(c)) {
            const uint32_t f = rabs >= pc.pos ? rabs - pc.pos : rabs + pc.clen - pc.pos;
            c = converted_ref_base(c, a.cfg.seed, pc.rid, pc.piece_in_read, f);
        }
        oi = base_idx(c) ^ (pc.ref_comp ? 2u : 0u);
        if (info & EMIT_F_MIS) oi = (oi + misoff) & 3u;
    } else {
        oi = (info & 3u) ? rb2 : (base_idx((info >> 8) & 0xffu) ^ (pc.ref_comp ? 2u : 0u));
    }
    return (pc.tbl >> (8u * oi)) & 0xffu;
}

// ---- EXACT route: the branch-free 16-base walk of one chunk over the reference bytes.  WRAPS: the piece crosses the
// origin of a circular chromosome (:1756-1760).  COMP: complementing classification (minus-strand genome pieces).
// sub = the chunk's substitution offsets (sub_offsets).
// ONE_LUT: every piece is unmapped and `lut` holds only the unmapped state's alias table (the unaligned batches' kernel).
template <bool FASTQ, bool WRAPS, bool COMP, uint32_t RING, bool ONE_LUT>
__device__ __forceinline__ void emit_chunk16(const uint4* ring, const uint32_t* lut, const uint8_t* cvt_tables,
                                             const uint8_t* __restrict__ cbase, uint32_t RB, uint32_t sub, const ChunkQual<FASTQ>& Q,
                                             uint32_t& k, uint32_t& rem, uint32_t& rabs, uint32_t& info, uint32_t rdir, uint32_t clen,
                                             uint32_t wrap_fix, uint32_t tbl, uint32_t (&sb)[4], uint32_t (&sq)[4], uint32_t& bad) {
    const uint8_t* cvt = cvt_tables + (COMP ? 256 : 0);    // compile-time offset: the lookup stays [register + immediate]
    const uint32_t dir = rdir ? 0xffffffffu : 1u;
    uint32_t sel = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        if (rem == 0) {                                    // next entry (never empty, never a deletion)
            ++k;
            const uint4 e = ring[k & (RING - 1)];
            rem = (e.z - e.x) >> 1;
            rabs = entry_ref(e, rdir, e.x >> 1);
            info = e.w;
        }
        --rem;
        uint32_t c = (info >> 8) & 0xffu;
        if (info & EMIT_F_REF) {
            c = __ldg(cbase + rabs);
            rabs += dir;
            if (WRAPS && rabs >= clen) rabs += wrap_fix;
        }
        const uint32_t code = cvt[c];
        bad |= code;
        uint32_t v = code | ((RB >> (2 * i)) & info & 3u);
        if (info & EMIT_F_MIS) v += (sub >> (2 * i)) & 3u;
        sel += v << (4 * (i & 3));
        if (FASTQ) {
            const uint32_t w = Q.W[i];
            const uint32_t e = *reinterpret_cast<const uint32_t*>(reinterpret_cast<const char*>(lut) + (ONE_LUT ? 0u : info >> 16) +
                                                                  ((w >> 6) & 0x1ffcu));
            sq[i >> 2] |= (qual_pick(e, w) & 0xffu) << (8 * (i & 3));
        }
        if ((i & 3) == 3) {
            sb[i >> 2] = __byte_perm(tbl, 0, sel & 0x3333u);
            sel = 0;
        }
    }
}

// 16 2-bit fields -> reversed order (field 15 first)
__device__ __forceinline__ uint32_t reverse_pairs(uint32_t x) {
    x = __brev(x);
    return ((x & 0x55555555u) << 1) | ((x >> 1) & 0x55555555u);
}
// the low 16 bits hold 8 2-bit base indices -> one index per nibble (PRMT selectors for two output words)
__device__ __forceinline__ uint32_t spread_pairs(uint32_t h) {
    uint32_t t = (h | (h << 8)) & 0x00ff00ffu;
    t = (t | (t << 4)) & 0x0f0f0f0fu;
    return (t | (t << 2)) & 0x33333333u;
}
__device__ __forceinline__ uint32_t bit_mask(uint32_t pos, uint32_t width) {     // `width` ones from bit `pos` (width <= 32)
    uint32_t m;
    asm("bmsk.clamp.b32 %0, %1, %2;" : "=r"(m) : "r"(pos), "r"(width));
    return m;
}

// ---- FAST route: one chunk from the 2-bit reference copy, entry by entry (see the header comment).
// pk = the packed reference, pk0w = the chromosome's first word in it; ring_s = shared-memory address of the warp's ring;
// k = ring index of the entry covering the chunk's first base; cs = padded piece coordinate of that base.  RDIR: the
// reference is walked backwards.  Returns the accumulator of 16 2-bit base indices; S = their 2-bit quality states
// ("match" unless an entry says otherwise; substituted bases are cleared to "mis" = 0 by the caller), mism = mask of the
// substituted bases.
// two consecutive packed words: from the step's window in shared memory when they are in it, else from global memory
__device__ __forceinline__ void load_packed_pair(const uint32_t* __restrict__ pk, uint32_t widx, uint32_t win_s, uint32_t win_w0,
                                                 uint32_t& w0, uint32_t& w1) {
#if EMIT_TMA_WINDOW
    const uint32_t rel = widx - win_w0;
    if (rel < EMIT_WIN_WORDS - 1u) {
        asm("ld.shared.u32 %0, [%2];\n\tld.shared.u32 %1, [%2+4];" : "=r"(w0), "=r"(w1) : "r"(win_s + 4u * rel));
        return;
    }
#endif
    w0 = __ldg(pk + widx);
    w1 = __ldg(pk + widx + 1);
}

template <bool RDIR, uint32_t RING>
__device__ __forceinline__ uint32_t emit_walk_entries(uint32_t ring_s, const uint32_t* __restrict__ pk, uint32_t pk0w, uint32_t win_s,
                                                      uint32_t win_w0, uint32_t RB, uint32_t& k, uint32_t cs, uint32_t& S, uint32_t& mism) {
    uint32_t acc = 0;
    S = 0xaaaaaaaau;                                                        // quality state 2 = match
    mism = 0;
    const uint32_t cs2 = 2u * cs;
    for (;;) {
        uint4 e;
        asm("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(e.x), "=r"(e.y), "=r"(e.z), "=r"(e.w) : "r"(ring_s + ((k & (RING - 1)) << 4)));
        const uint32_t info = e.w;
        const int32_t d0 = (int32_t)(e.x - cs2);
        const uint32_t lo2 = (uint32_t)(d0 > 0 ? d0 : 0);                   // 2 * first chunk position of the entry
        const uint32_t d1 = e.z - cs2;                                      // 2 * (entry end - chunk start) > 0
        const uint32_t hi2 = d1 < 32u ? d1 : 32u;
        const uint32_t m = bit_mask(lo2, hi2 - lo2);
        if (info & EMIT_F_REF) {
            const uint32_t p = cs + (lo2 >> 1);                             // output position of the first base taken here
            uint32_t r16;
            // packed word index = first word of the chromosome + base offset / 16 (32-bit: < 2^32 words = 68 Gbases)
            if (!RDIR) {
                const uint32_t l = e.y + p;
                uint32_t w0, w1;
                load_packed_pair(pk, pk0w + (l >> 4), win_s, win_w0, w0, w1);
                r16 = __funnelshift_r(w0, w1, (l + l) & 30u);
            } else {
                // the 16 bases ENDING at l = e.y - p, i.e. starting at l - 15 = (l + 1) - 16; for l < 15 the window reaches
                // into the guard word / the previous chromosome's padding: those bases are masked out
                const uint32_t l1 = e.y - p + 1u;
                uint32_t w0, w1;
                load_packed_pair(pk, pk0w + (l1 >> 4) - 1u, win_s, win_w0, w0, w1);
                r16 = reverse_pairs(__funnelshift_r(w0, w1, (l1 + l1) & 30u));
            }
            acc = (acc & ~m) | ((r16 << lo2) & m);
            if (info & EMIT_F_MIS) mism |= m;
        } else {
            const uint32_t v = (info & EMIT_F_RND) ? RB : ((info >> 9) & 3u) * 0x55555555u;   // random / literal run
            acc = (acc & ~m) | (v & m);
            S = (S & ~m) | (((info >> 29) * 0x55555555u) & m);
        }
        if (d1 >= 32u) break;
        ++k;
    }
    return acc;
}

template <bool FASTQ, uint32_t RING>
__device__ __forceinline__ void emit_chunk16_fast(uint32_t ring_s, const char* lut_s, const uint32_t* __restrict__ pk, uint32_t pk0w,
                                                  uint32_t win_s, uint32_t win_w0, uint32_t& k,
                                                  uint32_t cs, bool rdir, bool unmapped, uint32_t tbl, uint32_t id_lo, uint32_t id_hi,
                                                  uint32_t kind, uint32_t chunk, uint2 key, uint32_t (&sb)[4], uint32_t (&sq)[4]) {
    ChunkAux R;
    draw_chunk_aux<FASTQ>(R, id_lo, id_hi, kind, chunk, key);
    uint32_t S, mism;
    uint32_t acc = rdir ? emit_walk_entries<true, RING>(ring_s, pk, pk0w, win_s, win_w0, R.RB, k, cs, S, mism)
                        : emit_walk_entries<false, RING>(ring_s, pk, pk0w, win_s, win_w0, R.RB, k, cs, S, mism);
    ChunkQual<FASTQ> Q;                                                     // after the walk: 16 fewer live registers in it
    draw_chunk_qual<FASTQ>(Q, id_lo, id_hi, kind, chunk, key);
    // substituted bases: index + 1 + uniform{0,1,2} (mod 4), quality state "mis" (0)
    acc = add_fields_mod4(acc, sub_offsets(R.X, Q.X) & mism);
    S &= ~mism;
    {
        const uint32_t s0 = spread_pairs(acc & 0xffffu), s1 = spread_pairs(acc >> 16);
        sb[0] = __byte_perm(tbl, 0, s0);
        sb[1] = __byte_perm(tbl, 0, s0 >> 16);
        sb[2] = __byte_perm(tbl, 0, s1);
        sb[3] = __byte_perm(tbl, 0, s1 >> 16);
    }
    if (FASTQ) {
        if (unmapped) S = 0;                                                // the piece's lut_s is the unmapped state's table
        uint32_t q[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const uint32_t w = Q.W[i];
            // state << 13 | slot << 2
            const uint32_t st = (2 * i <= 13) ? (S << (13 - 2 * i)) : (S >> (2 * i - 13));
            const uint32_t off = (st & 0x6000u) | ((w >> 6) & 0x1ffcu);
            q[i] = qual_pick(*reinterpret_cast<const uint32_t*>(lut_s + off), w);
        }
#pragma unroll
        for (int g = 0; g < 4; ++g)
            sq[g] = __byte_perm(__byte_perm(q[4 * g], q[4 * g + 1], 0x0040), __byte_perm(q[4 * g + 2], q[4 * g + 3], 0x0040), 0x5410);
    }
}

// Shared memory of one block: the alias tables, the classification tables, the rings, the reference windows.
template <bool FASTQ, uint32_t RING>
constexpr size_t emit_smem_bytes() {
    return (FASTQ ? (size_t)(RING == EMIT_RING ? NS_N_QUAL_STATES : 1) * QLUT_SIZE * 4 : 0) + 512 +
           (size_t)EMIT_WARPS * RING * sizeof(uint4) + EMIT_WINDOW_SMEM;
}

// RING = EMIT_RING_UNAL: a batch of unaligned reads (every piece unmapped; NS_PIECE_UNALIGNED).
template <bool FASTQ, uint32_t RING>
__global__ void __launch_bounds__(EMIT_WARPS * 32, EMIT_MIN_BLOCKS) emit_kernel(const __grid_constant__ EmitArgs a) {
    if (a.abort && *a.abort) return;
    constexpr bool UNAL = RING != EMIT_RING;
    extern __shared__ uint4 smem4[];
    uint32_t* lut = reinterpret_cast<uint32_t*>(smem4);                          // FASTQ only
    uint8_t* cvt_tables = reinterpret_cast<uint8_t*>(lut + (FASTQ ? (UNAL ? 1 : NS_N_QUAL_STATES) * QLUT_SIZE : 0));
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint4* ring = reinterpret_cast<uint4*>(cvt_tables + 512) + warp * RING;
    const uint32_t ring_s = (uint32_t)__cvta_generic_to_shared(ring);
#if EMIT_TMA_WINDOW
    // per warp: a 64-word window of the packed reference + the mbarrier its TMA copy completes on
    const uint32_t win_s = (uint32_t)__cvta_generic_to_shared(reinterpret_cast<uint4*>(cvt_tables + 512) + EMIT_WARPS * RING) +
                           warp * (EMIT_WIN_WORDS * 4);
    const uint32_t mbar_s = win_s + (EMIT_WARPS - warp) * (EMIT_WIN_WORDS * 4) + warp * 8;
    uint32_t win_phase = 0;
    if (lane == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mbar_s));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
#else
    const uint32_t win_s = 0;
#endif
    if (FASTQ)
        for (int i = threadIdx.x; i < (UNAL ? 1 : NS_N_QUAL_STATES) * QLUT_SIZE; i += blockDim.x) lut[i] = a.qlut[(UNAL ? 4 * QLUT_SIZE : 0) + i];   // UNAL: state 4 (unmapped) only
    {   // case_convert classification: base index 0..3 (A C T G), 4 = needs the IUPAC path
        uint32_t c = threadIdx.x;
        uint32_t u = (c - 'a' < 26u) ? c - 32u : c;
        cvt_tables[c] = (uint8_t)(acgt_fast(u) ? base_idx(u) : 4u);
        cvt_tables[256 + c] = (uint8_t)(acgt_fast(u) ? base_idx(u) ^ 2u : 4u);     // complementing twin (NS_PIECE_REF_REV)
    }
    __syncthreads();
    const uint2 key = make_uint2((uint32_t)a.cfg.seed, (uint32_t)(a.cfg.seed >> 32));
    const uint32_t lane_lt = (1u << lane) - 1u;

    uint32_t n_extra = a.split_base ? *a.n_extra : 0u;
    if (n_extra > a.cap_extra) n_extra = a.cap_extra;
    for (;;) {
        uint32_t piece = 0, sub = 0;
        if (lane == 0) piece = atomicAdd(a.counter, 1u);
        piece = __shfl_sync(0xffffffffu, piece, 0);
        if (piece >= n_extra + a.n_pieces) break;
        if (piece < n_extra) {                   // a later stretch of a long piece
            const uint2 x = a.extra[piece];
            if (x.x == 0xffffffffu) continue;
            piece = x.x;
            sub = x.y;
        } else {
            piece -= n_extra;
            if (a.order) piece = __ldg(&a.order[piece]);
        }
        const NsPieceMeta pm = a.pieces[piece];
        if (pm.out_len == 0) continue;
        const NsReadMeta rm = a.reads[pm.read_slot];
        const bool rev = rm.reversed != 0;
        // a minus-strand piece (intron retention, ns_reemit) reads the genome backwards and complemented: together with the
        // read's own orientation that fixes the walking direction, and the complement moves into the classification table
        const bool ref_comp = (pm.kind & NS_PIECE_REF_REV) != 0;
        const bool rdir = rev != ref_comp;
        const uint32_t n_ops = pm.n_ops, ref_len = pm.ref_len;
        const uint32_t A = rev ? rm.seq_len - pm.out_rel - pm.out_len : pm.out_rel;    // piece start in read coordinates
        uint32_t pad = A & 15u;                              // x = read coordinate - P0: chunks are x/16
        const uint32_t P0 = A - pad;
        uint32_t x_end = pad + pm.out_len;
        // a stretch of a split piece: [sub * EMIT_SPLIT, (sub + 1) * EMIT_SPLIT) of x, the walk resumed from its checkpoint
        uint32_t t_first = 0, out_first = pad, ref_first = 0, x_first = 0;
        {
            const uint32_t sbase = a.split_base ? __ldg(&a.split_base[piece]) : 0xffffffffu;
            if (sbase != 0xffffffffu) {
                if (sub) {
                    const uint4 ck = a.ckpt[sbase + sub - 1u];
                    t_first = ck.x;
                    out_first = ck.y;
                    ref_first = ck.z;
                    x_first = sub * EMIT_SPLIT;
                    pad = 0;
                }
                if (x_end > (sub + 1u) * EMIT_SPLIT) x_end = (sub + 1u) * EMIT_SPLIT;
            }
        }
        const uint64_t cstart = a.ref.chrom_off[pm.chrom];
        EmitPiece pc;
        pc.cbase = a.ref.bases + cstart;
        pc.pos = pm.pos;
        pc.clen = (uint32_t)(a.ref.chrom_off[pm.chrom + 1] - cstart);
        pc.rdir = rdir;
        pc.ref_comp = ref_comp;
        {
            const uint32_t t = a.cfg.uracil ? 0x47554341u : 0x47544341u;             // "ACTG" / "ACUG"
            pc.tbl = rev ? __byte_perm(t, 0, 0x1032) : t;                            // complement: A<->T, C<->G
        }
        pc.piece_in_read = piece - rm.piece_first;
        pc.rid = a.first_id + pm.read_slot;
        const uint8_t* __restrict__ cbase = pc.cbase;
        const uint32_t clen = pc.clen, tbl = pc.tbl;
        const bool wraps = (uint64_t)pm.pos + ref_len > clen;                        // circular wrap (:1756-1760)
        const uint32_t wrap_fix = rdir ? clen : 0u - clen;
        const uint32_t* __restrict__ ops = a.ops + pm.op_off;
        uint8_t* seq_out = a.seq + rm.seq_off + P0;
        uint8_t* qual_out = FASTQ ? a.qual + rm.seq_off + P0 : nullptr;
        const bool unmapped = UNAL || NS_PIECE_KIND(pm.kind) != NS_PIECE_SEGMENT;
        const uint32_t id_lo = (uint32_t)pc.rid, id_hi = (uint32_t)(pc.rid >> 32);
        const uint32_t info_pad = emit_op_info(NS_OP_HT << 28, unmapped, ref_comp);
        // route: the fast one needs a forward-complement piece that stays inside its chromosome and whose packed words hold
        // no exception (IUPAC code, other character)
        const uint64_t pk0 = a.ref.pk_off[pm.chrom];
        bool fast = !wraps && !ref_comp && !a.force_exact;
        if (fast && ref_len) {
            const uint64_t w_lo = pk0 + (pm.pos >> 4), w_hi = pk0 + ((pm.pos + ref_len - 1u) >> 4);
            fast = __ldg(&a.ref.exc_pre[(w_hi >> REF_EXC_BLOCK_SHIFT) + 1]) == __ldg(&a.ref.exc_pre[w_lo >> REF_EXC_BLOCK_SHIFT]);
        }
        const char* lut_s = reinterpret_cast<const char*>(lut) + (unmapped && !UNAL ? 4u * QLUT_SIZE * 4u : 0u);

        uint32_t t_loaded = t_first, w_loaded = 0, w_ret = 0, out_loaded = out_first, ref_loaded = ref_first, prog = x_first;
        bool closed = false;
        if (pad) {
            if (lane == 0) ring[0] = make_uint4(0u, 0u, 2u * pad, info_pad);
            w_loaded = 1;
        }
        // ring entry of an op that starts at output position xo after rstart reference bases
        auto put_entry = [&](uint32_t slot, uint32_t xo, uint32_t rstart, uint32_t len, uint32_t op) {
            uint32_t ab = pm.pos + (rdir ? ref_len - 1u - rstart : rstart);           // first base in walking order
            if (wraps && ab >= clen) ab -= clen;
            ring[slot & (RING - 1)] = make_uint4(2u * xo, rdir ? ab + xo : ab - xo, 2u * (xo + len), emit_op_info(op, unmapped, ref_comp));
        };
        // the lane's two ops of the next round of the ring build, loaded one round ahead: the load of a step's first round
        // is in flight while the previous step produces its chunks
        uint32_t pf0 = 0, pf1 = 0;
        {
            const uint32_t t = t_loaded + 2u * lane;
            if (t < n_ops) pf0 = __ldg(&ops[rev ? n_ops - 1u - t : t]);
            if (t + 1u < n_ops) pf1 = __ldg(&ops[rev ? n_ops - 2u - t : t + 1u]);
        }
        while (prog < x_end) {
            // ---- 1. stream ops into the ring, two per lane, until the next 32 chunks are covered or the ring is full
            uint32_t target = prog + 512u < x_end ? prog + 512u : x_end;
            while (out_loaded < target && t_loaded < n_ops && (w_loaded - w_ret) + 65u <= RING) {
                const uint32_t t = t_loaded + 2u * lane;
                const uint32_t op0 = pf0, op1 = pf1;
                pf0 = pf1 = 0;
                if (t + 64u < n_ops) pf0 = __ldg(&ops[rev ? n_ops - 65u - t : t + 64u]);
                if (t + 65u < n_ops) pf1 = __ldg(&ops[rev ? n_ops - 66u - t : t + 65u]);
                const uint32_t ty0 = op0 >> 28, len0 = op_len(op0), ty1 = op1 >> 28, len1 = op_len(op1);
                const uint32_t o0 = (ty0 == NS_OP_DEL) ? 0u : len0, o1 = (ty1 == NS_OP_DEL) ? 0u : len1;
                const uint32_t r0 = (ty0 < 2u || ty0 == NS_OP_DEL) ? len0 : 0u, r1 = (ty1 < 2u || ty1 == NS_OP_DEL) ? len1 : 0u;
                const uint32_t so = warp_incl_scan(o0 + o1, lane), sr = warp_incl_scan(r0 + r1, lane);
                const uint32_t bal0 = __ballot_sync(0xffffffffu, o0 != 0u), bal1 = __ballot_sync(0xffffffffu, o1 != 0u);
                const uint32_t slot = w_loaded + __popc(bal0 & lane_lt) + __popc(bal1 & lane_lt);
                const uint32_t xo = out_loaded + so - (o0 + o1), rs = ref_loaded + sr - (r0 + r1);
                if (o0) put_entry(slot, xo, rs, len0, op0);
                if (o1) put_entry(slot + (o0 ? 1u : 0u), xo + o0, rs + r0, len1, op1);
                out_loaded += __shfl_sync(0xffffffffu, so, 31);
                ref_loaded += __shfl_sync(0xffffffffu, sr, 31);
                w_loaded += __popc(bal0) + __popc(bal1);
                t_loaded += (n_ops - t_loaded < 64u) ? n_ops - t_loaded : 64u;
            }
            if (!closed && (t_loaded == n_ops || out_loaded >= x_end)) {
                // sentinel: walking past the end of the piece stays inside the ring (ops left over are deletions)
                if (lane == 0) ring[w_loaded & (RING - 1)] = make_uint4(2u * out_loaded, 0u, 2u * out_loaded + 0x7ffffffeu, info_pad);
                ++w_loaded;
                closed = true;
            }
            __syncwarp();
            uint32_t win_w0 = (uint32_t)a.ref.pk_words + 4096u;                       // no word index is within 64 of this: no window
#if EMIT_TMA_WINDOW
            if (fast) {
                // the first entry at or after the step's first base that reads the reference tells where the step starts on it
                uint32_t kk = w_ret;
                uint4 e = ring[kk & (RING - 1)];
                while (!(e.w & EMIT_F_REF) && kk + 1u < w_loaded) {
                    ++kk;
                    e = ring[kk & (RING - 1)];
                }
                if (e.w & EMIT_F_REF) {
                    const uint32_t x0 = e.x >> 1;
                    const uint32_t w = (uint32_t)pk0 + (entry_ref(e, rdir, x0 > prog ? x0 : prog) >> 4);
                    // forward: words w .. ; backward: words .. w + 1 (16-byte aligned start)
                    win_w0 = !rdir ? (w & ~3u) : (w + 1u >= EMIT_WIN_WORDS - 1u ? (w + 1u - (EMIT_WIN_WORDS - 4u)) & ~3u : 0u);
                    if (lane == 0) {
                        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar_s), "r"(EMIT_WIN_WORDS * 4) : "memory");
                        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                     ::"r"(win_s), "l"(a.ref.packed + win_w0), "r"(EMIT_WIN_WORDS * 4), "r"(mbar_s) : "memory");
                    }
                }
            }
            const bool win_on = win_w0 < (uint32_t)a.ref.pk_words;
#endif
            // ---- 2. what can be produced now: whole chunks up to the loaded frontier (or the piece end)
            uint32_t lim = out_loaded < target ? out_loaded : target;
            if (lim < x_end) lim &= ~15u;
            // (the ring holds >= RING - 66 entries of >= 1 base beyond w_ret, so lim > prog whenever ops remain)
            // ---- 3. one 16-byte chunk per lane
            const uint32_t cs = prog + 16u * lane;
            uint32_t k = w_ret;
            if (cs < lim) {
                uint32_t l = w_ret, h = w_loaded;     // last entry whose output start <= cs
                while (h - l > 1) {
                    uint32_t mid = (l + h) >> 1;
                    if (ring[mid & (RING - 1)].x <= 2u * cs) l = mid; else h = mid;
                }
                k = l;
                // ---- all randomness of the chunk is position-indexed: (read id, chunk index in read coordinates)
                const uint32_t chunk = (P0 + cs) >> 4;
                uint32_t sb[4], sq[4] = {0, 0, 0, 0};
                if (fast) {
#if EMIT_TMA_WINDOW
                    if (win_on) {                  // the window's bytes have landed (phase parity of this warp's barrier)
                        asm volatile("{\n\t.reg .pred p;\n\tWIN_WAIT:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra WIN_DONE;\n\tbra WIN_WAIT;\n\tWIN_DONE:\n\t}"
                                     ::"r"(mbar_s), "r"(win_phase) : "memory");
                    }
#endif
                    emit_chunk16_fast<FASTQ, RING>(ring_s, lut_s, a.ref.packed, (uint32_t)pk0, win_s, win_w0, k, cs, rdir, unmapped, tbl, id_lo, id_hi, a.kind, chunk, key, sb, sq);
                } else {
                    ChunkAux R;
                    ChunkQual<FASTQ> Q;
                    draw_chunk_aux<FASTQ>(R, id_lo, id_hi, a.kind, chunk, key);
                    draw_chunk_qual<FASTQ>(Q, id_lo, id_hi, a.kind, chunk, key);
                    const uint32_t sub = sub_offsets(R.X, Q.X);
                    uint32_t rem, rabs, info;
                    {
                        const uint4 e = ring[k & (RING - 1)];
                        rem = (e.z >> 1) - cs;
                        info = e.w;
                        rabs = entry_ref(e, rdir, cs);
                        if (wraps && rabs >= clen) rabs += wrap_fix;
                    }
                    uint32_t bad = 0;
                    // three instantiations: plain, circular wrap, complementing (minus-strand genome pieces; keeps the wrap check)
                    if (ref_comp) emit_chunk16<FASTQ, true, true, RING, UNAL>(ring, lut, cvt_tables, cbase, R.RB, sub, Q, k, rem, rabs, info, rdir, clen, wrap_fix, tbl, sb, sq, bad);
                    else if (wraps) emit_chunk16<FASTQ, true, false, RING, UNAL>(ring, lut, cvt_tables, cbase, R.RB, sub, Q, k, rem, rabs, info, rdir, clen, wrap_fix, tbl, sb, sq, bad);
                    else emit_chunk16<FASTQ, false, false, RING, UNAL>(ring, lut, cvt_tables, cbase, R.RB, sub, Q, k, rem, rabs, info, rdir, clen, wrap_fix, tbl, sb, sq, bad);
                    // ---- rare: IUPAC codes, one base at a time
                    if (bad & 4u) {
#pragma unroll
                        for (int i = 0; i < 16; ++i) {
                            const uint32_t f = emit_fix_base<RING>(a, pc, ring, w_ret, w_loaded, cs + i, (R.RB >> (2 * i)) & 3u, (sub >> (2 * i)) & 3u);
                            const uint32_t m = 0xffu << (8 * (i & 3));
                            sb[i >> 2] = (sb[i >> 2] & ~m) | (f << (8 * (i & 3)));
                        }
                    }
                }
                if (cs >= pad && cs + 16u <= x_end) {
                    *reinterpret_cast<uint4*>(seq_out + cs) = make_uint4(sb[0], sb[1], sb[2], sb[3]);
                    if (FASTQ) *reinterpret_cast<uint4*>(qual_out + cs) = make_uint4(sq[0], sq[1], sq[2], sq[3]);
                } else {
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        if (cs + i >= pad && cs + i < x_end) {
                            seq_out[cs + i] = (uint8_t)(sb[i >> 2] >> (8 * (i & 3)));
                            if (FASTQ) qual_out[cs + i] = (uint8_t)(sq[i >> 2] >> (8 * (i & 3)));
                        }
                    }
                }
            }
            // ---- 4. retire: the entry the last active lane stopped in starts before the new frontier
            {
                const uint32_t n_act = (lim - prog + 15u) >> 4;
                const uint32_t k_last = __shfl_sync(0xffffffffu, k, n_act ? n_act - 1u : 0u);
                if (n_act) w_ret = k_last;
            }
            prog = lim;
            __syncwarp();
#if EMIT_TMA_WINDOW
            if (win_on) win_phase ^= 1u;           // every lane is past the window: the next step may overwrite it
#endif
        }
    }
}

// ---- long pieces -> extra work items + checkpoints (one warp per long piece; everything else costs one 64-byte read)
struct SplitArgs {
    const NsReadMeta* reads;
    const NsPieceMeta* pieces;
    const uint32_t* ops;
    uint32_t n_pieces;
    uint32_t* split_base;
    uint2* extra;
    uint4* ckpt;
    uint32_t* n_extra;
    uint32_t cap_extra;
    const uint32_t* abort;
};

__global__ void __launch_bounds__(256) split_kernel(const __grid_constant__ SplitArgs a) {
    if (a.abort && *a.abort) return;
    const int lane = threadIdx.x & 31;
    const uint32_t lane_lt = (1u << lane) - 1u;
    (void)lane_lt;
    const uint32_t n_warps = gridDim.x * (blockDim.x >> 5);
    for (uint32_t piece = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); piece < a.n_pieces; piece += n_warps) {
        const NsPieceMeta* pmp = a.pieces + piece;
        const uint32_t out_len = pmp->out_len;
        if (out_len <= EMIT_SPLIT - 16u) {                    // pad < 16: fits one work item
            if (lane == 0) a.split_base[piece] = 0xffffffffu;
            continue;
        }
        const NsPieceMeta pm = *pmp;
        const NsReadMeta rm = a.reads[pm.read_slot];
        const bool rev = rm.reversed != 0;
        const uint32_t A = rev ? rm.seq_len - pm.out_rel - pm.out_len : pm.out_rel;
        const uint32_t pad = A & 15u, x_end = pad + out_len;
        const uint32_t n_sub = (x_end + EMIT_SPLIT - 1u) / EMIT_SPLIT;
        if (n_sub < 2u) {
            if (lane == 0) a.split_base[piece] = 0xffffffffu;
            continue;
        }
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(a.n_extra, n_sub - 1u);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base + (n_sub - 1u) > a.cap_extra) {              // cannot happen with the capacity launch_emit reserves; stay whole
            if (lane == 0) a.split_base[piece] = 0xffffffffu;
            continue;
        }
        if (lane == 0) a.split_base[piece] = base;
        for (uint32_t j = 1u + lane; j < n_sub; j += 32u) a.extra[base + j - 1u] = make_uint2(piece, j);
        // The walk of the emit kernel's ring build (ops in walking order, output / reference prefix sums), 2048 ops per step:
        // every lane adds up 64 consecutive ops, one warp scan gives each lane its start, and a lane looks at its ops again
        // only when a boundary falls among them (a boundary every 16 kb, a lane's ops span a few hundred bases).
        const uint32_t* __restrict__ ops = a.ops + pm.op_off;
        const uint32_t n_ops = pm.n_ops;
        uint32_t out_loaded = pad, ref_loaded = 0;
        for (uint32_t t_tile = 0; t_tile < n_ops && out_loaded < x_end; t_tile += 2048u) {
            const uint32_t t0 = t_tile + 64u * lane, t1 = t0 + 64u < n_ops ? t0 + 64u : n_ops;
            uint32_t so = 0, sr = 0;
            for (uint32_t t = t0; t < t1; t += 8u) {            // eight loads in flight (an empty op counts for nothing)
                uint32_t v[8];
#pragma unroll
                for (uint32_t q = 0; q < 8u; ++q) v[q] = t + q < t1 ? __ldg(&ops[rev ? n_ops - 1u - (t + q) : t + q]) : 0u;
#pragma unroll
                for (uint32_t q = 0; q < 8u; ++q) {
                    const uint32_t ty = v[q] >> 28, len = op_len(v[q]);
                    so += (ty == NS_OP_DEL) ? 0u : len;
                    sr += (ty < 2u || ty == NS_OP_DEL) ? len : 0u;
                }
            }
            const uint32_t io = warp_incl_scan(so, lane), ir = warp_incl_scan(sr, lane);
            uint32_t xo = out_loaded + io - so, rs = ref_loaded + ir - sr;
            // boundaries j * EMIT_SPLIT in [xo, xo + so)
            if (so && (xo + so - 1u) / EMIT_SPLIT != (xo ? (xo - 1u) / EMIT_SPLIT : 0u)) {
                for (uint32_t t = t0; t < t1; ++t) {
                    const uint32_t op = __ldg(&ops[rev ? n_ops - 1u - t : t]);
                    const uint32_t ty = op >> 28, len = op_len(op);
                    const uint32_t o = (ty == NS_OP_DEL) ? 0u : len;
                    if (o) {
                        for (uint32_t j = (xo + EMIT_SPLIT - 1u) / EMIT_SPLIT; j < n_sub && j * EMIT_SPLIT < xo + o; ++j)
                            if (j) a.ckpt[base + j - 1u] = make_uint4(t, xo, rs, 0u);
                    }
                    xo += o;
                    rs += (ty < 2u || ty == NS_OP_DEL) ? len : 0u;
                }
            }
            out_loaded += __shfl_sync(0xffffffffu, io, 31);
            ref_loaded += __shfl_sync(0xffffffffu, ir, 31);
        }
    }
}
