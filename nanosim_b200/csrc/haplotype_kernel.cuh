// ns_apply_variants: the haplotype records of a VCF sample, built in HBM from the resident reference.
// Haplotype h with variants j = var_off[h] .. var_off[h+1]-1 is a list of 2 n_h + 1 segments: the reference stretch before
// each variant, the variant's ALT bytes, and the stretch behind the last one.  Its segments are seg_first(h) = 2 var_off[h]
// + h onwards, so segment s of haplotype h is the stretch before variant var_off[h] + (s - seg_first(h)) / 2 when
// s - seg_first(h) is even, and that variant's ALT when it is odd.
//   hap_segments_kernel: one thread per segment, its source and length
//   (CUB exclusive sum over the lengths: every segment's offset in the output, and the total)
//   hap_offsets_kernel:  the haplotype records' offsets (chrom_off of the new reference)
//   hap_gather_kernel:   one thread per 16-byte unit of the output; see there
//   hap_lift_kernel:     (ns_set_lift, after hap_segments_kernel and the scan) one thread per segment, its HapLift
// Included only by haplotype.cu, which launches them: a translation unit of their own, so the host code that drives them
// leaves the code generated for nanosim_api.cu's kernels as it is.
#pragma once

#include "haplotype.h"

__device__ __forceinline__ uint64_t hap_seg_first(const uint64_t* var_off, uint32_t h) { return 2 * var_off[h] + h; }

// the haplotype of segment s: the last h with seg_first(h) <= s
__device__ __forceinline__ uint32_t hap_of_segment(const HapArgs& a, uint64_t s) {
    uint32_t lo = 0, hi = a.n_hap;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (hap_seg_first(a.var_off, mid) <= s) lo = mid; else hi = mid;
    }
    return lo;
}

__global__ void hap_segments_kernel(HapArgs a) {
    const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s > a.n_seg) return;
    if (s == a.n_seg) {
        a.seg_len[s] = 0;
        return;
    }
    const uint32_t lo = hap_of_segment(a, s);
    const uint64_t local = s - hap_seg_first(a.var_off, lo);
    const uint64_t j = a.var_off[lo] + local / 2;
    const uint32_t c = a.hap_chrom[lo];
    if (local & 1) {
        const uint8_t kind = a.alt_kind ? a.alt_kind[j] : 0;
        const uint64_t from = a.chrom_off[c] + a.alt_off[j];        // kinds 1 and 2: a span of the source record
        a.seg_src[s] = kind == 0 ? HAP_SRC_ALT | a.alt_off[j] : kind == 1 ? from : HAP_SRC_RC | (from + a.alt_len[j]);
        a.seg_len[s] = a.alt_len[j];
        return;
    }
    const uint64_t begin = j == a.var_off[lo] ? 0 : a.var_pos[j - 1] + a.var_ref_len[j - 1];
    const uint64_t end = j < a.var_off[lo + 1] ? a.var_pos[j] : a.chrom_off[c + 1] - a.chrom_off[c];
    a.seg_src[s] = a.chrom_off[c] + begin;
    a.seg_len[s] = end - begin;
}

// ns_set_lift: segment s as a HapLift (offsets in its haplotype record and in the source record) and its kind.  A stretch
// maps onto its own source span; an ALT onto [var_pos, var_pos + var_ref_len), except a <DUP> copy (kind 1), whose
// reference span is the source span [alt_off, alt_off + alt_len) it repeats.  (An <INV> has var_pos = alt_off.)
__global__ void hap_lift_kernel(HapArgs a, const uint64_t* __restrict__ seg_out, const uint64_t* __restrict__ hap_off,
                                HapLift* __restrict__ lift, uint8_t* __restrict__ kind) {
    const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.n_seg) return;
    const uint32_t h = hap_of_segment(a, s);
    const uint64_t local = s - hap_seg_first(a.var_off, h);
    const uint64_t j = a.var_off[h] + local / 2;
    HapLift g;
    g.hap0 = (uint32_t)(seg_out[s] - hap_off[h]);
    g.hap_len = (uint32_t)a.seg_len[s];
    uint8_t k = HAP_LIFT_SEQ;
    if (local & 1) {
        k = a.alt_kind ? a.alt_kind[j] : 0;
        g.ref0 = (uint32_t)(k == HAP_LIFT_DUP ? a.alt_off[j] : a.var_pos[j]);
        g.ref_len = k == HAP_LIFT_DUP ? a.alt_len[j] : a.var_ref_len[j];
    } else {
        g.ref0 = (uint32_t)(a.seg_src[s] - a.chrom_off[a.hap_chrom[h]]);
        g.ref_len = g.hap_len;
    }
    lift[s] = g;
    kind[s] = k;
}

// hap_off[h] = output offset of haplotype h's first segment; hap_off[n_hap] = the total
__global__ void hap_offsets_kernel(const uint64_t* __restrict__ var_off, const uint64_t* __restrict__ seg_out, uint32_t n_hap,
                                   uint64_t* __restrict__ hap_off) {
    const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h <= n_hap) hap_off[h] = seg_out[hap_seg_first(var_off, h)];
}

// The complement of a base for an inversion: A-T, C-G, R-Y, K-M, B-V and D-H swap, in either case (each case kept); S, W,
// N and every other byte stay as they are.  A 256-byte table built at compile time, read through the read-only data
// cache, where it stays resident: a copy in shared memory would need a fill and a barrier in every block (or a vote and
// a fill in every warp), for a table most blocks never read.
struct HapComplement {
    uint8_t b[256];
    constexpr HapComplement() : b() {
        const char pairs[] = "ATCGRYKMBVDH";
        for (int i = 0; i < 256; ++i) b[i] = (uint8_t)i;
        for (int i = 0; i < 12; ++i) {
            const int x = pairs[i], y = pairs[i ^ 1];
            b[x] = (uint8_t)y;
            b[x | 0x20] = (uint8_t)(y | 0x20);
        }
    }
};
__device__ const HapComplement hap_complement{};

// The 16 bytes at p (any alignment) as five aligned 32-bit loads funnel-shifted into place.  The aligned-down start is
// readable because p lies inside its buffer and every buffer starts 256-byte aligned (cudaMalloc), so it is never below
// the buffer's first byte, even for p at the very start of the reference; the last word ends at most 3 bytes behind
// p + 16, and the reference and the ALT bytes each have at least 4 readable bytes behind their end.
__device__ __forceinline__ uint4 hap_load16(const uint8_t* p) {
    const uint32_t* q = reinterpret_cast<const uint32_t*>(reinterpret_cast<uintptr_t>(p) & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 3) * 8;
    uint32_t w[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) w[i] = __ldg(q + i);
    uint4 v;
    v.x = __funnelshift_r(w[0], w[1], sh);
    v.y = __funnelshift_r(w[1], w[2], sh);
    v.z = __funnelshift_r(w[2], w[3], sh);
    v.w = __funnelshift_r(w[3], w[4], sh);
    return v;
}

__device__ __forceinline__ uint32_t hap_comp(uint32_t b) { return __ldg(hap_complement.b + b); }

// w with its bytes in reverse order, each complemented
__device__ __forceinline__ uint32_t hap_rc_word(uint32_t w) {
    const uint32_t r = __byte_perm(w, 0, 0x0123);
    const uint32_t lo = __byte_perm(hap_comp(r & 0xFF), hap_comp((r >> 8) & 0xFF), 0x0040);
    const uint32_t hi = __byte_perm(hap_comp((r >> 16) & 0xFF), hap_comp(r >> 24), 0x0040);
    return __byte_perm(lo, hi, 0x5410);
}

// Output unit u = bytes [16u, 16u + 16).  Its thread finds the segment holding byte 16u by binary search over the segment
// offsets.  A unit inside one forward segment is read with hap_load16 from its source and written as one 16-byte store.
// A unit inside one reverse-complement segment (seg_src = HAP_SRC_RC | the end E of its reference span) holds the source
// bytes E - t - 16 .. E - t - 1 in reverse, t being the unit's offset in the segment: they are loaded the same way,
// reversed with byte permutes, complemented through hap_complement and written with one 16-byte store.  A unit that a
// segment boundary or the end of the output splits is written byte by byte, walking the segments it spans, through the
// same table.  Haplotype records follow each other without padding, so a record end is a segment boundary.
// kRC = false (no inversion in the tables) compiles to the kernel without the reverse-complement path: that path, even
// never taken, made the forward units 7.6 % slower on an H100 (14.4 against 13.4 ms for config 2's haplotypes).
template <bool kRC>
__global__ void hap_gather_kernel(const uint8_t* __restrict__ ref, const uint8_t* __restrict__ alt, const uint64_t* __restrict__ seg_src,
                                  const uint64_t* __restrict__ seg_out, uint64_t n_seg, uint8_t* __restrict__ out) {
    const uint64_t u = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t total = seg_out[n_seg];
    const uint64_t p0 = u * 16;
    if (p0 >= total) return;
    uint64_t lo = 0, hi = n_seg;        // last s with seg_out[s] <= p0 (it is not empty: seg_out[s + 1] > p0)
    while (hi - lo > 1) {
        const uint64_t mid = (lo + hi) >> 1;
        if (seg_out[mid] <= p0) lo = mid; else hi = mid;
    }
    uint64_t s = lo;
    auto src = [&](uint64_t v) { return (v & HAP_SRC_ALT) ? alt + (v & ~HAP_SRC_ALT) : ref + v; };
    if (p0 + 16 <= seg_out[s + 1]) {
        const uint64_t v = seg_src[s];
        if (kRC && (v & HAP_SRC_RC)) {
            const uint4 f = hap_load16(ref + (v & ~HAP_SRC_RC) - (p0 - seg_out[s]) - 16);
            *reinterpret_cast<uint4*>(out + p0) = make_uint4(hap_rc_word(f.w), hap_rc_word(f.z), hap_rc_word(f.y), hap_rc_word(f.x));
        } else {
            *reinterpret_cast<uint4*>(out + p0) = hap_load16(src(v) + (p0 - seg_out[s]));
        }
        return;
    }
    for (uint64_t p = p0; p < p0 + 16 && p < total; ++p) {
        while (seg_out[s + 1] <= p) ++s;
        const uint64_t v = seg_src[s], t = p - seg_out[s];
        out[p] = (kRC && (v & HAP_SRC_RC)) ? hap_comp(ref[(v & ~HAP_SRC_RC) - 1 - t]) : src(v)[t];
    }
}
