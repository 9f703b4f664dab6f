// ns_apply_variants: the haplotype records of a VCF sample, built in HBM from the resident reference.
// Haplotype h with variants j = var_off[h] .. var_off[h+1]-1 is a list of 2 n_h + 1 segments: the reference stretch before
// each variant, the variant's ALT bytes, and the stretch behind the last one.  Its segments are seg_first(h) = 2 var_off[h]
// + h onwards, so segment s of haplotype h is the stretch before variant var_off[h] + (s - seg_first(h)) / 2 when
// s - seg_first(h) is even, and that variant's ALT when it is odd.
//   hap_segments_kernel: one thread per segment, its source and length
//   (CUB exclusive sum over the lengths: every segment's offset in the output, and the total)
//   hap_offsets_kernel:  the haplotype records' offsets (chrom_off of the new reference)
//   hap_gather_kernel:   one thread per 16-byte unit of the output; see there
// Included only by haplotype.cu, which launches them: a translation unit of their own, so the host code that drives them
// leaves the code generated for nanosim_api.cu's kernels as it is.
#pragma once

#include "haplotype.h"

__device__ __forceinline__ uint64_t hap_seg_first(const uint64_t* var_off, uint32_t h) { return 2 * var_off[h] + h; }

__global__ void hap_segments_kernel(HapArgs a) {
    const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s > a.n_seg) return;
    if (s == a.n_seg) {
        a.seg_len[s] = 0;
        return;
    }
    uint32_t lo = 0, hi = a.n_hap;      // haplotype of this segment: last h with seg_first(h) <= s
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (hap_seg_first(a.var_off, mid) <= s) lo = mid; else hi = mid;
    }
    const uint64_t local = s - hap_seg_first(a.var_off, lo);
    const uint64_t j = a.var_off[lo] + local / 2;
    if (local & 1) {
        a.seg_src[s] = HAP_SRC_ALT | a.alt_off[j];
        a.seg_len[s] = a.alt_len[j];
        return;
    }
    const uint32_t c = a.hap_chrom[lo];
    const uint64_t begin = j == a.var_off[lo] ? 0 : a.var_pos[j - 1] + a.var_ref_len[j - 1];
    const uint64_t end = j < a.var_off[lo + 1] ? a.var_pos[j] : a.chrom_off[c + 1] - a.chrom_off[c];
    a.seg_src[s] = a.chrom_off[c] + begin;
    a.seg_len[s] = end - begin;
}

// hap_off[h] = output offset of haplotype h's first segment; hap_off[n_hap] = the total
__global__ void hap_offsets_kernel(const uint64_t* __restrict__ var_off, const uint64_t* __restrict__ seg_out, uint32_t n_hap,
                                   uint64_t* __restrict__ hap_off) {
    const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h <= n_hap) hap_off[h] = seg_out[hap_seg_first(var_off, h)];
}

// Output unit u = bytes [16u, 16u + 16).  Its thread finds the segment holding byte 16u by binary search over the segment
// offsets.  A unit inside one segment is read as five aligned 32-bit words from its source (the reference and the ALT
// bytes each have at least 4 readable bytes behind their end) shifted into place, and written as one 16-byte store.  A
// unit that a segment boundary or the end of the output splits is written byte by byte, walking the segments it spans.
// Haplotype records follow each other without padding, so a record end is a segment boundary.
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
    auto src = [&](uint64_t seg) {
        const uint64_t v = seg_src[seg];
        return (v & HAP_SRC_ALT) ? alt + (v & ~HAP_SRC_ALT) : ref + v;
    };
    if (p0 + 16 <= seg_out[s + 1]) {
        const uint8_t* p = src(s) + (p0 - seg_out[s]);
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
        *reinterpret_cast<uint4*>(out + p0) = v;
        return;
    }
    for (uint64_t p = p0; p < p0 + 16 && p < total; ++p) {
        while (seg_out[s + 1] <= p) ++s;
        out[p] = src(s)[p - seg_out[s]];
    }
}
