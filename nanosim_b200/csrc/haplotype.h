// ns_apply_variants' device work (haplotype.cu, kernels in haplotype_kernel.cuh), callable from nanosim_api.cu.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>

#define HAP_SRC_ALT (1ull << 63)        // seg_src: offset into the ALT bytes, else into the reference bases
#define HAP_SRC_RC (1ull << 62)         // seg_src: the END of a reference span, read backwards and complemented

struct HapArgs {
    const uint32_t* hap_chrom;          // n_hap: source record of each haplotype
    const uint64_t* var_off;            // n_hap + 1
    const uint64_t* var_pos;            // 0-based start of the replaced span in the source record
    const uint32_t* var_ref_len;
    const uint64_t* alt_off;
    const uint32_t* alt_len;
    const uint8_t* alt_kind;            // NULL: all 0.  0 ALT bytes, 1 the source record's [alt_off, +alt_len), 2 that span
                                        // reverse-complemented
    const uint64_t* chrom_off;          // of the resident (haploid) reference
    uint32_t n_hap;
    uint64_t n_seg;                     // 2 n_var + n_hap
    uint64_t* seg_src;                  // n_seg
    uint64_t* seg_len;                  // n_seg + 1 (the last one 0: the scan's total lands behind the segments)
};

// Segments, their output offsets seg_out[0 .. n_seg] (seg_out[n_seg] = the haplotypes' bytes) and the haplotype records'
// offsets hap_off[0 .. n_hap], on `st`.  With tmp == nullptr only *tmp_bytes is set (the scan's scratch space).
cudaError_t hap_layout(const HapArgs& a, uint64_t* seg_out, uint64_t* hap_off, void* tmp, size_t* tmp_bytes, cudaStream_t st);
// The n_bases haplotype bytes into out (16-byte aligned, n_bases + 16 bytes), on `st`.  reverse_complement: some segment
// is HAP_SRC_RC (an ALT of kind 2).
cudaError_t hap_gather(const uint8_t* ref, const uint8_t* alt, const uint64_t* seg_src, const uint64_t* seg_out, uint64_t n_seg,
                       uint64_t n_bases, bool reverse_complement, uint8_t* out, cudaStream_t st);
