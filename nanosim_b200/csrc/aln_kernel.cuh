// Mapped BAM (ns_compress_bam_mapped): the true alignment of every aligned read of the last batch, built from the pieces'
// emitted scripts (op_off / n_ops, forward-strand order) as BAM records for bgzf_deflate_kernel<BgzfRecords<BgzfMappedLayout>>.
// The rules are in DESIGN §3 "Mapped BAM"; tests/test_mapped_bam.py restates them in Python.
//   pass 1 (aln_count_kernel): per read its records (its alignments, or one unmapped record) and CIGAR words, and which
//          alignment is primary; CUB scans of both give every read its first record and first CIGAR word
//   pass 2 (aln_write_kernel): the same walk writes the records' descriptors, CIGAR words and sizes
// One thread per read: the rules (LIT groups, merging, trimming, the cut at a circular record's origin) are a sequential
// state machine over the script, and each read's ops are contiguous in HBM.
// ALN_LIFT (ns_set_lift, DESIGN §3 "Lifted mapped BAM"): the same walk composes every op with the haplotype record's lift
// segments on the way, so the records are against the haploid reference the VCF describes.
// ALN_SPLICE (ns_set_splice, DESIGN §3 "Spliced mapped BAM"): transcriptome reads, the walk composed with the transcript's
// exons (or, for a read that retains an intron, with its chain of genome pieces), so the records are against the genome
// with an N for every intron the read skips.
// ALN_TRX (ns_compress_bam_transcript, DESIGN §3 "Transcript-coordinate mapped BAM"): transcriptome reads against the
// transcripts they came from: a transcript piece takes the plain walk, a read that retains an intron walks its chain of
// genome pieces composed with its transcript's exons (ns_set_splice), the retained bases as insertions.
// NM and SA (ns_set_aln_tags, DESIGN §3 "NM and SA tags"): aln_write_tags_kernel is the same write walk counting every
// record's NM on the way (AlnWrite<kMode, true>::bases); aln_aux_size_kernel and aln_aux_write_kernel then lay out and
// fill each record's aux fields (HP/XS, NM, SA) for bgzf_deflate_kernel<BgzfRecords<BgzfTaggedLayout>>.
#pragma once

#include <type_traits>

#include "haplotype.h"

// which walk an aln kernel instantiation runs
enum AlnMode : int { ALN_PLAIN = 0, ALN_LIFT = 1, ALN_SPLICE = 2, ALN_TRX = 3 };
// the walks whose mapped records have a leading aux field (HP:C, XS:A); ALN_TRX records have the plain layout
__host__ __device__ constexpr bool aln_lead_aux(uint32_t mode) { return mode == ALN_LIFT || mode == ALN_SPLICE; }

// CIGAR operations (SAM/BAM specification §4.2.2: MIDNSHP=X -> 0..8)
enum : uint32_t { CIG_M = 0, CIG_I = 1, CIG_D = 2, CIG_N = 3, CIG_S = 4, CIG_H = 5 };
constexpr uint32_t ALN_CUT = 15;                    // the origin of a circular record: one alignment ends, the next starts
constexpr uint32_t BAM_MAX_CIGAR = 65535;           // n_cigar_op is 16 bits; more ops go into a CG:B,I field
constexpr uint32_t BAM_MAPQ = 60;
// where an M of aln_script comes from (the third argument of its fn): a COPY op, a MIS op, or the M part of a LIT group
// followed by a DEL; every other kind passes ALN_SRC_COPY
enum : uint32_t { ALN_SRC_COPY = 0, ALN_SRC_MIS = 1, ALN_SRC_LIT = 2 };

// one mapped record (or, flag 4, the unmapped record ns_compress_bam writes)
struct BamAln {
    uint32_t read;                  // slot of the read in the batch
    uint32_t q0;                    // first stored base, forward-strand offset in the read
    uint32_t l_seq;                 // stored bases
    uint32_t ref_id, pos, span;
    uint32_t n_cig;                 // CIGAR ops with the clips
    uint16_t bin, flag;
    uint64_t cig_off;               // first CIGAR word
};

// reg2bin (specification §5.3) of [beg, end); 4680 past 2^29, which BAI cannot index (CSI recomputes bins)
__host__ __device__ __forceinline__ uint32_t bam_reg2bin(uint64_t beg, uint64_t end) {
    if (end > (1ull << 29)) return 4680;
    --end;
    if (beg >> 14 == end >> 14) return ((1u << 15) - 1) / 7 + (uint32_t)(beg >> 14);
    if (beg >> 17 == end >> 17) return ((1u << 12) - 1) / 7 + (uint32_t)(beg >> 17);
    if (beg >> 20 == end >> 20) return ((1u << 9) - 1) / 7 + (uint32_t)(beg >> 20);
    if (beg >> 23 == end >> 23) return ((1u << 6) - 1) / 7 + (uint32_t)(beg >> 23);
    if (beg >> 26 == end >> 26) return ((1u << 3) - 1) / 7 + (uint32_t)(beg >> 26);
    return 0;
}

// A lifted record keeps its HP value (1 or 2) in BamAln::flag's bits 12-15, above the BAM flag bits; a spliced one its
// transcript's strand there (0 +, 1 -)
constexpr uint32_t BAM_FLAG_BITS = 0xfff, BAM_HP_SHIFT = 12;

// bytes of a mapped record: the fixed fields, name, CIGAR (kSmN when it does not fit), bases, qualities, hp (4: a lifted
// record's HP:C field or a spliced one's XS:A field), CG:B,I
__host__ __device__ __forceinline__ uint64_t bam_mapped_size(uint32_t nl, const BamAln& a, uint32_t hp = 0) {
    const bool cg = a.n_cig > BAM_MAX_CIGAR;
    return BAM_FIXED + nl + 1 + 4ull * (cg ? 2 : a.n_cig) + (a.l_seq + 1) / 2 + a.l_seq + hp + (cg ? 8 + 4ull * a.n_cig : 0);
}

// the complement of a 4-bit base code: its bits reversed (A 1 <-> T 8, C 2 <-> G 4, M <-> K, R <-> Y, V <-> B, H <-> D;
// =, S, W, N fixed)
__device__ __forceinline__ uint32_t bam_code_comp(uint32_t c) { return __brev(c) >> 28; }

struct BgzfMappedRec {
    BgzfReadRec rd;                 // the read
    BamAln a;
    const uint32_t* cig;
    uint32_t rev;
};
struct BgzfMappedTable {
    BgzfReadTable reads;
    const BamAln* aln;
    const uint32_t* cigar;
    __device__ __forceinline__ BgzfMappedRec operator[](uint32_t r) const {
        const BamAln a = aln[r];
        return BgzfMappedRec{reads[a.read], a, cigar + a.cig_off, a.flag & 16u};       // the record's strand
    }
};

// ALN_LIFT: a mapped record also has the HP:C field of its haplotype (BamAln::flag >> BAM_HP_SHIFT) as its first aux
// field; ALN_SPLICE: the XS:A field of its transcript's strand
template <AlnMode kMode>
struct BgzfMappedLayoutOf {
    using Table = BgzfMappedTable;
    static constexpr uint32_t hp = aln_lead_aux(kMode) ? 4 : 0;
    static __device__ __forceinline__ uint8_t byte(uint64_t q, const BgzfMappedRec& rc) {
        const BamAln& a = rc.a;
        if (a.flag & 4) return BgzfBamLayout::byte(q, rc.rd);
        const uint32_t nl = rc.rd.nl, ls = a.l_seq, L = rc.rd.L;
        const bool cg = a.n_cig > BAM_MAX_CIGAR;
        const uint32_t nc = cg ? 2 : a.n_cig;
        if (q < BAM_FIXED) {
            uint32_t w;
            switch ((uint32_t)q >> 2) {
            case 0: w = (uint32_t)bam_mapped_size(nl, a, hp) - 4; break;                    // block_size
            case 1: w = a.ref_id; break;
            case 2: w = a.pos; break;
            case 3: w = (nl + 1) | (BAM_MAPQ << 8) | ((uint32_t)a.bin << 16); break;       // l_read_name, mapq, bin
            case 4: w = nc | ((uint32_t)(aln_lead_aux(kMode) ? a.flag & BAM_FLAG_BITS : a.flag) << 16); break;   // n_cigar_op, flag
            case 5: w = ls; break;                                                          // l_seq
            case 8: w = 0; break;                                                           // tlen
            default: w = 0xffffffffu;                                                       // next_refID, next_pos
            }
            return (uint8_t)(w >> (8 * ((uint32_t)q & 3)));
        }
        q -= BAM_FIXED;
        if (q < nl) return (uint8_t)rc.rd.nm[q];
        if (q == nl) return 0;
        q -= nl + 1;
        if (q < 4ull * nc) {
            const uint32_t k = (uint32_t)q >> 2;
            const uint32_t w = !cg ? rc.cig[k] : k == 0 ? (ls << 4) | CIG_S : (a.span << 4) | CIG_N;
            return (uint8_t)(w >> (8 * ((uint32_t)q & 3)));
        }
        q -= 4ull * nc;
        // stored base b is forward-strand base q0 + b: a reversed read's is the complement of its mirror in the read
        auto code = [&](uint32_t b) -> uint32_t {
            const uint32_t f = a.q0 + b;
            return rc.rev ? bam_code_comp(bam_base_code(rc.rd.sq[L - 1 - f])) : bam_base_code(rc.rd.sq[f]);
        };
        const uint64_t n_packed = (ls + 1) / 2;
        if (q < n_packed) {
            const uint32_t b = 2 * (uint32_t)q;
            return (uint8_t)((code(b) << 4) | (b + 1 < ls ? code(b + 1) : 0u));
        }
        q -= n_packed;
        if (q < ls) {
            const uint32_t f = a.q0 + (uint32_t)q;
            return rc.rd.fastq ? (uint8_t)(rc.rd.ql[rc.rev ? L - 1 - f : f] - 33) : 0xffu;
        }
        q -= ls;
        if (kMode == ALN_LIFT) {
            if (q < 3) return (uint8_t)"HPC"[q];
            if (q == 3) return (uint8_t)(a.flag >> BAM_HP_SHIFT);
            q -= 4;
        }
        if (kMode == ALN_SPLICE) {
            if (q < 3) return (uint8_t)"XSA"[q];
            if (q == 3) return (uint8_t)(a.flag >> BAM_HP_SHIFT ? '-' : '+');
            q -= 4;
        }
        if (q < 4) return (uint8_t)"CGBI"[q];
        const uint32_t k = (uint32_t)(q - 4) >> 2;             // the count, then the words
        const uint32_t w = k == 0 ? a.n_cig : rc.cig[k - 1];
        return (uint8_t)(w >> (8 * ((uint32_t)q & 3)));
    }
};
struct BgzfMappedLayout : BgzfMappedLayoutOf<ALN_PLAIN> {};
struct BgzfLiftedLayout : BgzfMappedLayoutOf<ALN_LIFT> {};
struct BgzfSplicedLayout : BgzfMappedLayoutOf<ALN_SPLICE> {};

// With NM and SA (every walk): a mapped record's aux fields up to CG (HP/XS, NM, SA) are aux_len bytes that
// aln_aux_write_kernel left at aux; CG:B,I follows as in BgzfMappedLayoutOf
struct BgzfTaggedRec {
    BgzfMappedRec m;
    const uint8_t* aux;
    uint32_t aux_len;
};
struct BgzfTaggedTable {
    BgzfMappedTable m;
    const uint8_t* aux;
    const uint64_t* aux_off;        // exclusive prefix sum of the records' aux bytes
    uint64_t aux_total;
    uint32_t n_recs;
    __device__ __forceinline__ BgzfTaggedRec operator[](uint32_t r) const {
        const uint64_t o = aux_off[r], e = r + 1 < n_recs ? aux_off[r + 1] : aux_total;
        return BgzfTaggedRec{m[r], aux + o, (uint32_t)(e - o)};
    }
};
struct BgzfTaggedLayout {
    using Table = BgzfTaggedTable;
    static __device__ __forceinline__ uint8_t byte(uint64_t q, const BgzfTaggedRec& rc) {
        const BamAln& a = rc.m.a;
        if (a.flag & 4) return BgzfBamLayout::byte(q, rc.m.rd);
        const uint32_t nl = rc.m.rd.nl;
        if (q < 4) return (uint8_t)(((uint32_t)bam_mapped_size(nl, a, rc.aux_len) - 4) >> (8 * (uint32_t)q));     // block_size
        const bool cg = a.n_cig > BAM_MAX_CIGAR;
        const uint64_t core = bam_mapped_size(nl, a, 0) - (cg ? 8 + 4ull * a.n_cig : 0);        // up to the qualities
        // the fixed fields (flag without the HP/strand bits), name, CIGAR, bases and qualities
        if (q < core) return BgzfMappedLayoutOf<ALN_LIFT>::byte(q, rc.m);
        q -= core;
        if (q < rc.aux_len) return rc.aux[q];
        q -= rc.aux_len;
        if (q < 4) return (uint8_t)"CGBI"[q];
        const uint32_t k = (uint32_t)(q - 4) >> 2;
        const uint32_t w = k == 0 ? a.n_cig : rc.m.cig[k - 1];
        return (uint8_t)(w >> (8 * ((uint32_t)q & 3)));
    }
};

// ns_set_lift's table in HBM: haplotype record h's segments are seg[first[h] .. first[h + 1]) in haplotype order, their
// kinds kind[...]; hap_chrom[h] its source record and hap_number[h] its HP value
struct AlnLift {
    const HapLift* seg;
    const uint8_t* kind;
    const uint64_t* first;
    const uint32_t* hap_chrom;
    const uint8_t* hap_number;
};

// Where the lift walk stands: haplotype base t of segment s (s_last: the record's last segment); d_done once the
// reference-only bases of s are emitted.  Before each M or D it hands to fn: at, the reference coordinate of its first
// base (inv = false), or one past it in reference order (inv = true: inside an <INV>, the bases run backwards).
struct LiftWalk {
    const HapLift* seg;
    const uint8_t* kind;
    uint64_t s, s_last;
    uint32_t t;
    bool d_done, inv;
    uint32_t at;
};

// Past the end of segment s: its reference-only bases (a sequence ALT with ref_len > hap_len: a deletion) as D, then the
// next segment, with an ALN_CUT where the reference stops advancing forward (into a <DUP> copy, into or out of an <INV>)
template <class Fn>
__device__ __forceinline__ void lift_advance(LiftWalk& w, Fn& fn) {
    for (;;) {
        const HapLift g = w.seg[w.s];
        if (w.t < g.hap_len) return;
        const uint8_t k = w.kind[w.s];
        if (k == HAP_LIFT_SEQ && g.ref_len > g.hap_len && !w.d_done) {
            w.d_done = true;
            w.at = g.ref0 + g.hap_len;
            w.inv = false;
            fn(CIG_D, g.ref_len - g.hap_len, ALN_SRC_COPY);
        }
        if (w.s == w.s_last) return;
        ++w.s;
        w.t = 0;
        w.d_done = false;
        if (k == HAP_LIFT_INV || w.kind[w.s] != HAP_LIFT_SEQ) fn(ALN_CUT, 0u, ALN_SRC_COPY);
    }
}

// A read op (M, I or D over the haplotype) composed with the lift: I stays I; M and D over 1:1 bases stay M and D; over
// the inserted bases of a sequence ALT an M becomes I and a D vanishes
template <class Fn>
__device__ __forceinline__ void lift_put(LiftWalk& w, uint32_t kind, uint32_t len, uint32_t src, Fn& fn) {
    if (kind == CIG_I) {
        fn(CIG_I, len, src);
        return;
    }
    while (len) {
        const HapLift g = w.seg[w.s];
        const uint8_t k = w.kind[w.s];
        uint32_t n = len, out = kind;
        w.inv = k == HAP_LIFT_INV;
        if (w.t >= g.hap_len) {                                 // past the record's last base: no segment of a linear record
            w.at = g.ref0 + g.ref_len;                          // gets here; 1:1 so that the walk ends
            w.inv = false;
        } else if (w.inv) {
            n = min(len, g.hap_len - w.t);
            w.at = g.ref0 + g.ref_len - w.t;
        } else {
            const uint32_t m = k == HAP_LIFT_SEQ ? min(g.hap_len, g.ref_len) : g.hap_len;        // the 1:1 bases
            if (w.t < m) {
                n = min(len, m - w.t);
                w.at = g.ref0 + w.t;
            } else {
                n = min(len, g.hap_len - w.t);
                out = kind == CIG_M ? CIG_I : ~0u;
            }
        }
        if (out != ~0u) fn(out, n, src);
        w.t += n;
        len -= n;
        lift_advance(w, fn);
    }
}

// ns_set_splice's table in HBM: transcript t's exons are exon[first[t] .. first[t + 1]) in transcript order (none: no
// map), minus[t] its strand; genome_first the resident index of genome record 0 (the chains' pieces lie on those records)
struct SpliceExon {
    uint32_t chrom, start, len;     // genome record (0 = the first -rg record), first base on it, bases
    uint32_t cum;                   // transcript offset of its first base in transcript order
};
struct AlnSplice {
    const SpliceExon* exon;
    const uint64_t* first;
    const uint8_t* minus;
    uint32_t n_trx, genome_first;
};

// Where the splice walk stands: offset t in interval k of n_iv (a transcript's exons, or a chain's genome pieces), which is
// bases [start, start + len) of genome record chrom, walked backwards when inv (minus strand).  The ops walked are those of
// src[0], src[2], ... (n_src pieces: one transcript piece, or a chain's segments with their gap pieces between them).
// Before each M or D: at, the genome coordinate of its first base (inv = false) or one past it (inv = true).
struct SpliceWalk {
    const SpliceExon* exon;         // the transcript's exons; nullptr: the intervals are the chain's pieces
    const NsPieceMeta* src;
    const uint32_t* ops;
    uint32_t n_src, n_iv, k, t, genome_first;
    uint32_t chrom, start, len, at;
    bool inv;
};

__device__ __forceinline__ void splice_interval(const SpliceWalk& w, uint32_t k, uint32_t& chrom, uint32_t& start, uint32_t& len) {
    if (w.exon) {
        const SpliceExon e = w.exon[k];
        chrom = e.chrom;
        start = e.start;
        len = e.len;
    } else {
        const NsPieceMeta& pc = w.src[2 * k];
        chrom = pc.chrom - w.genome_first;
        start = pc.pos;
        len = pc.ref_len;
    }
}

// A read op (M, I or D over the transcript, or over the chain's pieces back to back) composed with the intervals: I stays
// I; an M or D that reaches the next interval's first base first emits the distance to it in the walk's direction as N
// (nothing when it is 0: an exon and the retained intron beside it), or an ALN_CUT when that interval is on another record
// or does not lie further on
template <class Fn>
__device__ __forceinline__ void splice_put(SpliceWalk& w, uint32_t kind, uint32_t len, uint32_t src, Fn& fn) {
    if (kind == CIG_I) {
        fn(CIG_I, len, src);
        return;
    }
    while (len) {
        if (w.t >= w.len && w.k + 1 < w.n_iv) {
            uint32_t c, s, l;
            splice_interval(w, w.k + 1, c, s, l);
            const int64_t gap = w.inv ? (int64_t)w.start - ((int64_t)s + l) : (int64_t)s - ((int64_t)w.start + w.len);
            if (c != w.chrom || gap < 0) fn(ALN_CUT, 0u, ALN_SRC_COPY);
            else if (gap) fn(CIG_N, (uint32_t)gap, ALN_SRC_COPY);
            ++w.k;
            w.t = 0;
            w.chrom = c;
            w.start = s;
            w.len = l;
        }
        const uint32_t n = w.t < w.len ? min(len, w.len - w.t) : len;     // past the last interval (no valid map gets here)
        w.at = w.inv ? w.start + w.len - w.t : w.start + w.t;
        fn(kind, n, src);
        w.t += n;
        len -= n;
    }
}

// ALN_TRX: where the walk of a read that retains an intron stands: offset t in piece k (of len bases) of its chain, the
// segments src[0], src[2], ... (n_src of them) back to back.  off is the transcript offset of piece k's first base in
// chain order (TRX_RETAINED: the piece lies in a retained intron), end one past the transcript offset of the last exon
// piece entered (~0u: none yet).  Before each M or D: at, the transcript offset of its first base.
constexpr uint32_t TRX_RETAINED = ~0u;
struct TrxWalk {
    const NsPieceMeta* src;
    const uint32_t* ops;
    const SpliceExon* exon;         // the transcript's exons in transcript order (n_exon)
    uint32_t n_src, n_exon, genome_first;
    uint32_t k, t, len, off, end, at;
    bool minus;                     // the transcript's strand
};

// The transcript offset of the first base in transcript order of the genome bases [pos, pos + len) of genome record
// chrom, when they lie in one exon of the transcript: the exons' starts ascend in transcript order on the plus strand and
// descend on the minus strand (ns_set_splice checks that), so a binary search finds the one that starts last at or
// before pos.  false when no exon holds them.
__device__ __forceinline__ bool trx_offset(const TrxWalk& w, uint32_t chrom, uint32_t pos, uint32_t len, uint32_t& off) {
    uint32_t lo = 0, hi = w.n_exon;                 // ends at the first exon starting after pos (plus), at or before it (minus)
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if ((w.exon[mid].start <= pos) != w.minus) lo = mid + 1; else hi = mid;
    }
    if (w.minus ? lo == w.n_exon : lo == 0) return false;
    const SpliceExon e = w.exon[w.minus ? lo : lo - 1];
    if (e.chrom != chrom || (uint64_t)pos + len > (uint64_t)e.start + e.len) return false;
    off = e.cum + (w.minus ? e.start + e.len - (pos + len) : pos - e.start);
    return true;
}

// Into piece k of the chain: an exon piece that does not start where the last one entered ended (in transcript offsets)
// ends the alignment (ALN_CUT)
template <class Fn>
__device__ __forceinline__ void trx_enter(TrxWalk& w, uint32_t k, Fn& fn) {
    const NsPieceMeta& pc = w.src[2 * k];
    w.k = k;
    w.t = 0;
    w.len = pc.ref_len;
    if (pc.kind & NS_PIECE_RETAINED) {
        w.off = TRX_RETAINED;
        return;
    }
    trx_offset(w, pc.chrom - w.genome_first, pc.pos, pc.ref_len, w.off);      // aln_read_chain checked that it finds one
    if (w.end != ~0u && w.off != w.end) fn(ALN_CUT, 0u, ALN_SRC_COPY);
    w.end = w.off + w.len;
}

// A read op (M, I or D over the chain's pieces back to back) composed with the transcript: I stays I; M and D over an exon
// piece stay M and D; over a retained intron an M becomes I and a D vanishes
template <class Fn>
__device__ __forceinline__ void trx_put(TrxWalk& w, uint32_t kind, uint32_t len, uint32_t src, Fn& fn) {
    if (kind == CIG_I) {
        fn(CIG_I, len, src);
        return;
    }
    while (len) {
        while (w.t >= w.len && w.k + 1 < w.n_src) trx_enter(w, w.k + 1, fn);
        const uint32_t n = w.t < w.len ? min(len, w.len - w.t) : len;     // past the chain's last base (no chain gets here)
        if (w.off != TRX_RETAINED) {
            w.at = w.off + w.t;
            fn(kind, n, src);
        } else if (kind == CIG_M) {
            fn(CIG_I, n, src);
        }
        w.t += n;
        len -= n;
    }
}

template <AlnMode kMode>
using AlnWalk = std::conditional_t<kMode == ALN_SPLICE, SpliceWalk, std::conditional_t<kMode == ALN_TRX, TrxWalk, LiftWalk>>;

struct AlnArgs {
    const NsReadMeta* reads;
    const NsPieceMeta* pieces;
    const uint32_t* ops;
    const uint64_t* chrom_off;
    const char* names;              // NUL-terminated, at name_off[i]
    const uint64_t* name_off;
    uint32_t n_reads;
    uint32_t* name_len;             // pass 1 writes, pass 2 reads
    uint64_t* n_rec;                // pass 1: records of every read
    uint64_t* n_cig;                // pass 1: CIGAR words of every read
    uint32_t* primary;              // pass 1: the primary alignment's index in the read
    unsigned long long* long_names; // pass 1: names longer than BAM_MAX_NAME
    const uint64_t* rec_first;      // pass 2: exclusive prefix sums of n_rec and n_cig
    const uint64_t* cig_first;
    BamAln* aln;                    // pass 2 writes
    uint32_t* cigar;
    uint64_t* rec_size;
    AlnLift lift;                   // ALN_LIFT only
    AlnSplice splice;               // ALN_SPLICE; ALN_TRX (the chains' transcripts; n_trx = 0: no map)
};

// fn(kind, len) over a segment's script: CIGAR kinds M I D (HT as I: it only stands at a read's edges), a LIT group followed
// by a DEL as |n - r| I or D and then min(n, r) M, zero lengths dropped, and an ALN_CUT (len 0) before the reference base
// at offset `cut` and every `period` bases behind it (a circular record's origin, each time the segment passes it; ~0:
// none), an M or D across one split there
// ALN_LIFT: every op goes through lift_put on walk w instead (no circular record: cut is ~0)
// ALN_SPLICE: the scripts of w's n_src pieces back to back (sc, n_ops unused), every op through splice_put
// ALN_TRX (a chain only): the same, every op through trx_put
template <AlnMode kMode, class Walk, class Fn>
__device__ __forceinline__ void aln_script(const uint32_t* __restrict__ sc, uint32_t n_ops, uint64_t cut, uint64_t period, Walk& w,
                                           Fn fn) {
    uint64_t rf = 0;
    uint32_t lit = 0;
    auto put = [&](uint32_t kind, uint32_t len, uint32_t src = ALN_SRC_COPY) {
        if (len == 0) return;
        if constexpr (kMode == ALN_LIFT) {
            lift_put(w, kind, len, src, fn);
            return;
        } else if constexpr (kMode == ALN_SPLICE) {
            splice_put(w, kind, len, src, fn);
            return;
        } else if constexpr (kMode == ALN_TRX) {
            trx_put(w, kind, len, src, fn);
            return;
        }
        if (kind != CIG_I) {
            while (rf <= cut && rf + len > cut) {
                const uint32_t a = (uint32_t)(cut - rf);
                if (a) fn(kind, a, src);
                fn(ALN_CUT, 0u, ALN_SRC_COPY);
                rf += a;
                len -= a;
                cut += period;
            }
            rf += len;
        }
        fn(kind, len, src);
    };
    uint32_t n_src = 1;
    if constexpr (kMode == ALN_SPLICE || kMode == ALN_TRX) n_src = w.n_src;
    for (uint32_t p = 0; p < n_src; ++p) {
        if constexpr (kMode == ALN_SPLICE || kMode == ALN_TRX) {
            sc = w.ops + w.src[2 * p].op_off;
            n_ops = w.src[2 * p].n_ops;
        }
        for (uint32_t j = 0; j < n_ops; ++j) {
            const uint32_t op = sc[j], ty = NS_OP_TYPE(op), ln = NS_OP_LEN(op);
            if (ty == NS_OP_LIT) {
                lit += ln;
                continue;
            }
            if (lit && ty == NS_OP_DEL) {
                put(lit > ln ? CIG_I : CIG_D, lit > ln ? lit - ln : ln - lit);
                put(CIG_M, min(lit, ln), ALN_SRC_LIT);
                lit = 0;
                continue;
            }
            put(CIG_I, lit);
            lit = 0;
            put(ty == NS_OP_DEL ? CIG_D : (ty == NS_OP_COPY || ty == NS_OP_MIS) ? CIG_M : CIG_I, ln, ty == NS_OP_MIS ? ALN_SRC_MIS : ALN_SRC_COPY);
        }
    }
    put(CIG_I, lit);
}

// The alignments of one segment (n_parts of them at most: the cuts split it), its ops starting at read offset q_start: for
// each, sink.begin(q0, rf0) at its first M, sink.op(kind, len) for its merged ops, sink.end(q1, rf1) after its last M
// (read offsets in the forward read, reference offsets in the segment).  Ops before the first M and after the last one
// are outside the alignment: their I is clip, their D (or N) moves the start or is dropped.  Two walks per part: the first
// finds the part's first and last M, the second emits what lies between them.  ALN_LIFT, ALN_SPLICE, ALN_TRX: every walk
// starts from `start`, the first one counts the parts (n_parts = 1 on entry), and sink.place(w) follows sink.begin with the
// walk as it stands at the first M (its position there).
template <AlnMode kMode, class Sink>
__device__ __forceinline__ void aln_segment(const uint32_t* sc, uint32_t n_ops, uint64_t cut, uint64_t period, uint32_t n_parts,
                                            uint32_t q_start, const AlnWalk<kMode>& start, Sink& sink) {
    for (uint32_t want = 0; want < n_parts; ++want) {
        uint32_t first = ~0u, last = 0, idx = 0, part = 0;
        AlnWalk<kMode> w = start;
        aln_script<kMode>(sc, n_ops, cut, period, w, [&](uint32_t kind, uint32_t, uint32_t) {
            if (kind == ALN_CUT) {
                ++part;
            } else if (kind == CIG_M && part == want) {
                if (first == ~0u) first = idx;
                last = idx;
            }
            ++idx;
        });
        if constexpr (kMode != ALN_PLAIN) n_parts = part + 1;
        if (first == ~0u) continue;
        idx = 0;
        uint32_t q = q_start, rf = 0, ck = 0, cl = 0;
        w = start;
        aln_script<kMode>(sc, n_ops, cut, period, w, [&](uint32_t kind, uint32_t len, uint32_t src) {
            if (idx >= first && idx <= last) {
                if (idx == first) {
                    sink.begin(q, rf);
                    if constexpr (kMode != ALN_PLAIN) sink.place(w);
                    ck = kind;
                    cl = 0;
                }
                sink.bases(kind, len, src, q, rf, w);
                if (kind == ck) {
                    cl += len;
                } else {
                    sink.op(ck, cl);
                    ck = kind;
                    cl = len;
                }
                if (idx == last) {
                    sink.op(ck, cl);
                    sink.end(q + len, rf + len);
                }
            }
            if (kind != CIG_D && (kMode != ALN_SPLICE || kind != CIG_N)) q += len;     // an N (splice walk) takes no read bases
            if (kind != CIG_I) rf += len;
            ++idx;
        });
    }
}

// ALN_SPLICE: read r's one alignment walk.  A read laid out on the genome (NS_PIECE_GENOME, it retains an intron) walks its
// chain of genome pieces; any other read its transcript piece over the transcript's exons, starting in the exon that holds
// its first base (binary search over the exons' transcript offsets).  A transcript without a map gives no alignment.
template <class Sink>
__device__ __forceinline__ void aln_read_spliced(const AlnArgs& a, const NsReadMeta& r, Sink& sink) {
    if (r.n_pieces == 0) return;
    const NsPieceMeta pc = a.pieces[r.piece_first];
    if (NS_PIECE_KIND(pc.kind) != NS_PIECE_SEGMENT) return;
    SpliceWalk w{};
    w.src = a.pieces + r.piece_first;
    w.ops = a.ops;
    w.genome_first = a.splice.genome_first;
    if (pc.kind & NS_PIECE_GENOME) {
        w.n_src = w.n_iv = (r.n_pieces + 1u) / 2u;
        w.inv = (pc.kind & NS_PIECE_REF_REV) != 0;
    } else {
        if (pc.chrom >= a.splice.n_trx) return;
        uint64_t lo = a.splice.first[pc.chrom], hi = a.splice.first[pc.chrom + 1];
        if (lo == hi) return;
        w.exon = a.splice.exon + lo;
        w.n_src = 1;
        w.n_iv = (uint32_t)(hi - lo);
        const uint64_t e0 = lo;
        while (hi - lo > 1) {
            const uint64_t mid = (lo + hi) >> 1;
            if (a.splice.exon[mid].cum <= pc.pos) lo = mid; else hi = mid;
        }
        w.k = (uint32_t)(lo - e0);
        w.t = pc.pos - a.splice.exon[lo].cum;
        w.inv = a.splice.minus[pc.chrom] != 0;
    }
    splice_interval(w, w.k, w.chrom, w.start, w.len);
    sink.segment(pc, 0);
    aln_segment<ALN_SPLICE>(nullptr, 0, ~0ull, 0, 1, pc.out_rel, w, sink);
}

// ALN_TRX: read r laid out on the genome (NS_PIECE_GENOME: it retains an intron) walks its chain of pieces back to back,
// its exon pieces composed with its transcript's exons, from the first piece.  No alignment when the transcript (ref_req)
// has no map or one of its exon pieces lies in none of the map's exons.
template <class Sink>
__device__ __forceinline__ void aln_read_chain(const AlnArgs& a, const NsReadMeta& r, Sink& sink) {
    const NsPieceMeta pc = a.pieces[r.piece_first];
    if (pc.ref_req >= a.splice.n_trx) return;
    const uint64_t e0 = a.splice.first[pc.ref_req], e1 = a.splice.first[pc.ref_req + 1];
    if (e0 == e1) return;
    TrxWalk w{};
    w.src = a.pieces + r.piece_first;
    w.ops = a.ops;
    w.exon = a.splice.exon + e0;
    w.n_src = (r.n_pieces + 1u) / 2u;
    w.n_exon = (uint32_t)(e1 - e0);
    w.genome_first = a.splice.genome_first;
    w.minus = a.splice.minus[pc.ref_req] != 0;
    for (uint32_t k = 0; k < w.n_src; ++k) {
        const NsPieceMeta& p = w.src[2 * k];
        uint32_t off;
        if (!(p.kind & NS_PIECE_RETAINED) && !trx_offset(w, p.chrom - w.genome_first, p.pos, p.ref_len, off)) return;
    }
    w.end = ~0u;
    auto none = [](uint32_t, uint32_t, uint32_t) {};
    trx_enter(w, 0, none);
    sink.segment(pc, 0);
    aln_segment<ALN_TRX>(nullptr, 0, ~0ull, 0, 1, pc.out_rel, w, sink);
}

// every alignment of read r, in the order of its segments: sink.segment(piece, record length) before each segment's.
// ALN_LIFT: the walk of a segment starts in the lift segment holding its first haplotype base, the last of its record's
// segments that starts at or before it (binary search).  ALN_TRX: a chain (aln_read_chain), else the plain walk.
template <AlnMode kMode, class Sink>
__device__ __forceinline__ void aln_read(const AlnArgs& a, const NsReadMeta& r, Sink& sink) {
    if constexpr (kMode == ALN_SPLICE) {
        aln_read_spliced(a, r, sink);
    } else {
        if constexpr (kMode == ALN_TRX) {
            if (r.n_pieces && (a.pieces[r.piece_first].kind & NS_PIECE_GENOME)) {
                aln_read_chain(a, r, sink);
                return;
            }
        }
        constexpr AlnMode kSeg = kMode == ALN_TRX ? ALN_PLAIN : kMode;
        for (uint32_t k = 0; k < r.n_pieces; ++k) {
            const NsPieceMeta pc = a.pieces[r.piece_first + k];
            if (NS_PIECE_KIND(pc.kind) != NS_PIECE_SEGMENT) continue;
            const uint64_t clen = a.chrom_off[pc.chrom + 1] - a.chrom_off[pc.chrom];
            // a segment that runs past its record's end (circular records only) is cut at the origin, as often as it passes it
            uint64_t cut = ~0ull;
            uint32_t n_parts = 1;
            LiftWalk w{};
            if constexpr (kMode == ALN_LIFT) {
                uint64_t lo = a.lift.first[pc.chrom], hi = a.lift.first[pc.chrom + 1];
                w.s_last = hi - 1;
                while (hi - lo > 1) {
                    const uint64_t mid = (lo + hi) >> 1;
                    if (a.lift.seg[mid].hap0 <= pc.pos) lo = mid; else hi = mid;
                }
                w.seg = a.lift.seg;
                w.kind = a.lift.kind;
                w.s = lo;
                w.t = pc.pos - a.lift.seg[lo].hap0;
            } else if ((uint64_t)pc.pos + pc.ref_len > clen) {
                cut = clen > pc.pos ? clen - pc.pos : 0;
                n_parts = 2 + (uint32_t)((pc.ref_len - 1 - cut) / clen);
            }
            sink.segment(pc, clen);
            aln_segment<kSeg>(a.ops + pc.op_off, pc.n_ops, cut, clen, n_parts, pc.out_rel, w, sink);
        }
    }
}

struct AlnCount {
    uint32_t L;
    uint32_t n_aln = 0, prim = 0, best = 0, q0 = 0, rf0 = 0, body = 0;
    uint64_t words = 0;
    __device__ void segment(const NsPieceMeta&, uint64_t) {}
    __device__ void begin(uint32_t q, uint32_t rf) {
        q0 = q;
        rf0 = rf;
        body = 0;
    }
    template <class Walk>
    __device__ void place(const Walk&) {}
    template <class Walk>
    __device__ void bases(uint32_t, uint32_t, uint32_t, uint32_t, uint32_t, const Walk&) {}
    __device__ void op(uint32_t, uint32_t) { ++body; }
    __device__ void end(uint32_t q1, uint32_t rf1) {
        words += body + (q0 > 0) + (q1 < L);
        if (rf1 - rf0 > best) {                                 // the longest span; the first of equal ones
            best = rf1 - rf0;
            prim = n_aln;
        }
        ++n_aln;
    }
};

template <AlnMode kMode>
__global__ void aln_count_kernel(AlnArgs a) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n_reads) return;
    const char* nm = a.names + a.name_off[i];
    uint32_t nl = 0;
    while (nm[nl]) ++nl;
    a.name_len[i] = nl;
    if (nl > BAM_MAX_NAME) atomicAdd(a.long_names, 1ull);
    const NsReadMeta r = a.reads[i];
    AlnCount c;
    c.L = r.seq_len;
    aln_read<kMode>(a, r, c);
    a.n_rec[i] = c.n_aln ? c.n_aln : 1;                         // no alignment: the unmapped record
    a.n_cig[i] = c.words;
    a.primary[i] = c.prim;
}

// With NM (aln_write_tags_kernel): where the walk finds the bases an M is compared with
struct AlnTagArgs {
    const uint8_t* seq;             // the batch's bases (NsReadMeta::seq_off)
    const uint8_t* bases;           // the resident reference (DevRef: bases, chrom_off, pk_off, exc_pre)
    const uint64_t* chrom_off;
    const uint64_t* pk_off;
    const uint32_t* exc_pre;
    const uint8_t* pair;            // ALN_LIFT: the REF bytes the ALT of variant v pairs with its first bases, at pair_off[v]
    const uint64_t* pair_off;
    uint32_t* nm;                   // every record's NM
};

// bases [off, off + n) of resident record rec lie in 4096-base blocks without an exception (DevRef::exc_pre): every byte is
// one of a/c/g/t in either case
__device__ __forceinline__ bool aln_ref_plain(const AlnTagArgs& g, uint32_t rec, uint32_t off, uint32_t n) {
    const uint64_t pk0 = g.pk_off[rec], w_lo = pk0 + (off >> 4), w_hi = pk0 + ((off + n - 1) >> 4);
    return __ldg(&g.exc_pre[(w_hi >> REF_EXC_BLOCK_SHIFT) + 1]) == __ldg(&g.exc_pre[w_lo >> REF_EXC_BLOCK_SHIFT]);
}

// ALN_LIFT: refID is the haplotype's source record and POS the lifted one; a part inside an <INV> is a record on the other
// strand, its CIGAR words (written in haplotype order) reversed in place and its stored bases mirrored.  ALN_SPLICE: refID
// is the genome record and POS the leftmost genome base; a minus-strand transcript's part is a record on the other strand
// as an <INV> part is, and the strand goes into the XS field.  ALN_TRX: a transcript piece's records are the plain ones; a
// chain's refID is its transcript (ref_req) and POS the transcript offset of its first M.
// kTags: every record's NM into tg.nm: its I and D lengths and the M bases whose 4-bit code differs from the reference
// byte's, or either is N (DESIGN §3 "NM and SA tags").  An M of a COPY (MIS) op over blocks without an exception matches
// (differs) base for base; any other M, and every M of an ALN_TRX chain (the read was copied from the genome, the record is
// against the transcript), compares the read's bases with the reference bytes.
template <AlnMode kMode, bool kTags = false>
struct AlnWrite {
    uint32_t i, L, nl, prim, rev;
    BamAln* rec;                    // the read's records
    uint32_t* cig;                  // its CIGAR words
    uint64_t* size;
    uint64_t cig_off;
    AlnLift lift;
    uint32_t n_aln = 0, w = 0, w0 = 0, q0 = 0, rf0 = 0, chrom = 0, pos = 0, at = 0;
    bool inv = false;
    uint64_t clen = 0;
    AlnTagArgs tg;                  // kTags only
    const uint8_t* sq = nullptr;    // the read's bases
    uint32_t* nm_out = nullptr;     // its records' NM
    uint32_t nm = 0, piece_rec = 0; // NM of the alignment so far; the segment's resident record
    bool chain = false;             // ALN_TRX: the read is a chain
    __device__ void segment(const NsPieceMeta& pc, uint64_t len) {
        chrom = pc.chrom;
        pos = pc.pos;
        clen = len;
        piece_rec = pc.chrom;
        if constexpr (kMode == ALN_TRX) {
            if (pc.kind & NS_PIECE_GENOME) {
                chain = true;
                chrom = piece_rec = pc.ref_req;
            }
        }
    }
    __device__ void begin(uint32_t q, uint32_t rf) {
        q0 = q;
        rf0 = rf;
        w0 = w;
        nm = 0;
        if (q > 0) cig[w++] = (q << 4) | (n_aln == prim ? CIG_S : CIG_H);
    }
    template <class Walk>
    __device__ void place(const Walk& w) {
        at = w.at;
        if constexpr (kMode != ALN_TRX) inv = w.inv;
        if constexpr (kMode == ALN_SPLICE) chrom = w.chrom;
    }
    // an op of the alignment, its first base at read offset q and segment reference offset rf, the walk as it stands
    template <class Walk>
    __device__ void bases(uint32_t kind, uint32_t len, uint32_t src, uint32_t q, uint32_t rf, const Walk& wk) {
        if constexpr (kTags) {
            if (kind == CIG_I || kind == CIG_D) nm += len;
            if (kind != CIG_M) return;
            uint32_t rc = piece_rec, off;                       // resident record and lowest offset of the M's bases
            bool comp = false;                                  // the bases run backwards there, complemented
            const uint8_t* paired = nullptr;                    // the REF bytes of an ALT
            bool inv_u = false;                                 // inside an <INV>: a U/u byte stands for the haploid's U
            bool exact = false;                                 // compared byte by byte whatever the M's source
            if constexpr (kMode == ALN_PLAIN || (kMode == ALN_TRX && !std::is_same_v<Walk, TrxWalk>)) {
                const uint64_t x = (uint64_t)pos + rf;
                off = (uint32_t)(x < clen ? x : x % clen);      // behind a circular record's origin only
            } else if constexpr (kMode == ALN_TRX) {            // a chain's exon piece: the transcript's bases
                off = wk.at;
                exact = true;
            } else if constexpr (kMode == ALN_LIFT) {
                // haplotype h's segments alternate stretch, variant, ..., stretch from lift.first[h] = 2 var_off[h] + h, so
                // segment s is a variant when s - h is odd, and then it is variant (s - h - 1) / 2 in NsVariants order (the
                // global index pair_off takes)
                off = wk.seg[wk.s].hap0 + wk.t;
                const uint64_t s2 = wk.s - piece_rec;            // 2 var_off[h] + the segment's place in its record
                if (wk.kind[wk.s] == HAP_LIFT_SEQ && (s2 & 1)) paired = tg.pair + tg.pair_off[(s2 - 1) >> 1] + wk.t;
                inv_u = wk.inv;
            } else if (wk.exon) {                               // a transcript piece: the transcript's own bases
                off = wk.exon[wk.k].cum + wk.t;
            } else {                                            // a chain piece: the genome record's
                rc = wk.genome_first + wk.chrom;
                comp = wk.inv;
                off = wk.inv ? wk.start + wk.len - wk.t - len : wk.start + wk.t;
            }
            if (!paired && !exact && src != ALN_SRC_LIT && aln_ref_plain(tg, rc, off, len)) {
                if (src == ALN_SRC_MIS) nm += len;
                return;
            }
            const uint8_t* g = paired ? paired : tg.bases + tg.chrom_off[rc] + off;
            for (uint32_t j = 0; j < len; ++j) {
                const uint32_t f = q + j;
                const uint32_t b = rev ? bam_code_comp(bam_base_code(sq[L - 1 - f])) : bam_base_code(sq[f]);
                uint32_t r = comp ? bam_code_comp(bam_base_code(g[len - 1 - j])) : bam_base_code(g[j]);
                // an <INV> segment holds the haploid bytes complemented by hap_complement, which keeps U/u: the haploid
                // base there is a U (read as T), whose complement is A
                if (inv_u && (g[j] | 0x20) == 'u') r = 1;
                nm += b != r || b == 15 || r == 15;
            }
        }
    }
    __device__ void op(uint32_t kind, uint32_t len) { cig[w++] = (len << 4) | kind; }
    __device__ void end(uint32_t q1, uint32_t rf1) {
        const bool primary = n_aln == prim;
        if (q1 < L) cig[w++] = ((L - q1) << 4) | (primary ? CIG_S : CIG_H);
        BamAln b;
        b.read = i;
        b.q0 = primary ? 0 : q0;
        b.l_seq = primary ? L : q1 - q0;
        b.ref_id = chrom;
        b.span = rf1 - rf0;
        b.n_cig = w - w0;
        uint64_t p;
        if constexpr (kMode == ALN_LIFT || kMode == ALN_SPLICE) {
            b.ref_id = kMode == ALN_LIFT ? lift.hap_chrom[chrom] : chrom;
            p = inv ? at - b.span : at;
            if (inv) {
                if (!primary) b.q0 = L - q1;
                for (uint32_t x = w0, y = w - 1; x < y; ++x, --y) {
                    const uint32_t c = cig[x];
                    cig[x] = cig[y];
                    cig[y] = c;
                }
            }
        } else if (kMode == ALN_TRX && chain) {
            p = at;
        } else {
            p = ((uint64_t)pos + rf0) % clen;                   // a part behind a circular record's origin starts past it
        }
        b.pos = (uint32_t)p;
        b.bin = (uint16_t)bam_reg2bin(p, p + b.span);
        b.flag = (uint16_t)(((rev ^ (uint32_t)inv) ? 16u : 0u) | (primary ? 0u : 0x800u));
        if constexpr (kMode == ALN_LIFT) b.flag |= (uint16_t)(lift.hap_number[chrom] << BAM_HP_SHIFT);
        if constexpr (kMode == ALN_SPLICE) b.flag |= (uint16_t)((uint32_t)inv << BAM_HP_SHIFT);
        b.cig_off = cig_off + w0;
        rec[n_aln] = b;
        size[n_aln] = bam_mapped_size(nl, b, aln_lead_aux(kMode) ? 4 : 0);
        if constexpr (kTags) nm_out[n_aln] = nm;
        ++n_aln;
    }
};

template <AlnMode kMode, bool kTags>
__device__ __forceinline__ void aln_write(const AlnArgs& a, const AlnTagArgs& tg) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n_reads) return;
    const NsReadMeta r = a.reads[i];
    const uint64_t r0 = a.rec_first[i];
    AlnWrite<kMode, kTags> s;
    s.lift = a.lift;
    s.i = i;
    s.L = r.seq_len;
    s.nl = a.name_len[i];
    s.prim = a.primary[i];
    s.rev = r.reversed;
    s.rec = a.aln + r0;
    s.cig_off = a.cig_first[i];
    s.cig = a.cigar + s.cig_off;
    s.size = a.rec_size + r0;
    if constexpr (kTags) {
        s.tg = tg;
        s.sq = tg.seq + r.seq_off;
        s.nm_out = tg.nm + r0;
    }
    aln_read<kMode>(a, r, s);
    if (s.n_aln == 0) {                                         // the unmapped record of ns_compress_bam
        BamAln b{};
        b.read = i;
        b.l_seq = r.seq_len;
        b.flag = 4;
        a.aln[r0] = b;
        a.rec_size[r0] = BgzfBamLayout::size(s.nl, r.seq_len, 0);
    }
}

template <AlnMode kMode>
__global__ void aln_write_kernel(AlnArgs a) {
    aln_write<kMode, false>(a, AlnTagArgs{});
}

template <AlnMode kMode>
__global__ void aln_write_tags_kernel(AlnArgs a, AlnTagArgs tg) {
    aln_write<kMode, true>(a, tg);
}

// ---------------------------------------------------------------------------------------------------------------------
// aux fields with NM and SA, one thread per read over its records (DESIGN §3 "NM and SA tags"): a mapped record's are
// HP:C (lift) or XS:A (splice) when aln_lead_aux, NM:I, and SA:Z when the read has more than one record, with one entry
// "rname,pos,strand,CIGAR,60,NM;" for each of its other records in record order.  CG:B,I follows in BgzfTaggedLayout.
// ---------------------------------------------------------------------------------------------------------------------
struct AlnAuxArgs {
    const BamAln* aln;
    const uint32_t* cigar;
    const uint32_t* nm;
    const uint64_t* n_rec;          // per read: its records and its first record
    const uint64_t* rec_first;
    const char* sn;                 // the header's @SQ SN names back to back, name k at sn_off[k] .. sn_off[k + 1]
    const uint64_t* sn_off;
    uint32_t n_reads, mode;         // mode: the AlnMode of the records
    uint64_t* rec_size;             // size pass: every mapped record's size grows by its NM and SA fields
    uint64_t* aux_len;              // size pass: every record's aux bytes before CG
    const uint64_t* aux_off;        // write pass: their exclusive prefix sum, and where they go
    uint8_t* aux;
};

__device__ __forceinline__ uint32_t aln_dec_len(uint32_t v) {
    uint32_t n = 1;
    for (; v >= 10; v /= 10) ++n;
    return n;
}
__device__ __forceinline__ uint8_t* aln_put_dec(uint8_t* p, uint32_t v) {
    const uint32_t n = aln_dec_len(v);
    for (uint32_t k = n; k-- > 0; v /= 10) p[k] = (uint8_t)('0' + v % 10);
    return p + n;
}

// bytes of record b's SA entry
__device__ __forceinline__ uint64_t aln_sa_len(const AlnAuxArgs& x, const BamAln& b, uint32_t nm) {
    uint64_t n = x.sn_off[b.ref_id + 1] - x.sn_off[b.ref_id] + aln_dec_len(b.pos + 1) + aln_dec_len(nm) + 9;      // ,,+/-,,60,;
    const uint32_t* c = x.cigar + b.cig_off;
    for (uint32_t k = 0; k < b.n_cig; ++k) n += aln_dec_len(c[k] >> 4) + 1;
    return n;
}
__device__ __forceinline__ uint8_t* aln_sa_put(const AlnAuxArgs& x, uint8_t* p, const BamAln& b, uint32_t nm) {
    for (uint64_t k = x.sn_off[b.ref_id]; k < x.sn_off[b.ref_id + 1]; ++k) *p++ = (uint8_t)x.sn[k];
    *p++ = ',';
    p = aln_put_dec(p, b.pos + 1);
    *p++ = ',';
    *p++ = (b.flag & 16) ? '-' : '+';
    *p++ = ',';
    const uint32_t* c = x.cigar + b.cig_off;
    for (uint32_t k = 0; k < b.n_cig; ++k) {
        p = aln_put_dec(p, c[k] >> 4);
        *p++ = (uint8_t)"MIDNSHP=X"[c[k] & 15];
    }
    *p++ = ',';
    *p++ = '6';
    *p++ = '0';
    *p++ = ',';
    p = aln_put_dec(p, nm);
    *p++ = ';';
    return p;
}

__global__ void aln_aux_size_kernel(AlnAuxArgs x) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= x.n_reads) return;
    const uint64_t r0 = x.rec_first[i], k = x.n_rec[i];
    if (x.aln[r0].flag & 4) {                                   // the unmapped record: no aux field
        x.aux_len[r0] = 0;
        return;
    }
    const uint32_t hp = aln_lead_aux(x.mode) ? 4 : 0;
    uint64_t all = 0;                                           // every record's SA entry
    if (k > 1)
        for (uint64_t j = 0; j < k; ++j) all += x.aux_len[r0 + j] = aln_sa_len(x, x.aln[r0 + j], x.nm[r0 + j]);
    for (uint64_t j = 0; j < k; ++j) {
        const uint64_t sa = k > 1 ? 3 + all - x.aux_len[r0 + j] + 1 : 0;
        x.rec_size[r0 + j] += 7 + sa;
        x.aux_len[r0 + j] = hp + 7 + sa;
    }
}

__global__ void aln_aux_write_kernel(AlnAuxArgs x) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= x.n_reads) return;
    const uint64_t r0 = x.rec_first[i], k = x.n_rec[i];
    if (x.aln[r0].flag & 4) return;
    for (uint64_t j = 0; j < k; ++j) {
        const BamAln b = x.aln[r0 + j];
        uint8_t* p = x.aux + x.aux_off[r0 + j];
        if (aln_lead_aux(x.mode)) {
            const uint32_t v = b.flag >> BAM_HP_SHIFT;
            p[0] = x.mode == ALN_LIFT ? 'H' : 'X';
            p[1] = x.mode == ALN_LIFT ? 'P' : 'S';
            p[2] = x.mode == ALN_LIFT ? 'C' : 'A';
            p[3] = (uint8_t)(x.mode == ALN_LIFT ? v : v ? '-' : '+');
            p += 4;
        }
        const uint32_t nm = x.nm[r0 + j];
        p[0] = 'N';
        p[1] = 'M';
        p[2] = 'I';
        for (int s = 0; s < 4; ++s) p[3 + s] = (uint8_t)(nm >> (8 * s));
        p += 7;
        if (k == 1) continue;
        p[0] = 'S';
        p[1] = 'A';
        p[2] = 'Z';
        p += 3;
        for (uint64_t o = 0; o < k; ++o)
            if (o != j) p = aln_sa_put(x, p, x.aln[r0 + o], x.nm[r0 + o]);
        *p = 0;
    }
}
