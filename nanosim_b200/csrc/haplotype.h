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

// One segment of a haplotype record as ns_set_lift keeps it: haplotype bases [hap0, hap0 + hap_len) of the record and
// the reference span [ref0, ref0 + ref_len) of its source record, with the segment's kind (HapLiftKind) beside it
struct HapLift {
    uint32_t hap0, hap_len, ref0, ref_len;
};
// the kind of a segment: a stretch between variants or a sequence ALT (min(hap_len, ref_len) bases 1:1, then the rest
// inserted or deleted), a <DUP> copy (1:1 onto [ref0, ref0 + ref_len) again), an <INV> (1:1, reversed); = alt_kind
enum : uint8_t { HAP_LIFT_SEQ = 0, HAP_LIFT_DUP = 1, HAP_LIFT_INV = 2 };

// Segments, their output offsets seg_out[0 .. n_seg] (seg_out[n_seg] = the haplotypes' bytes) and the haplotype records'
// offsets hap_off[0 .. n_hap], on `st`.  With tmp == nullptr only *tmp_bytes is set (the scan's scratch space).
cudaError_t hap_layout(const HapArgs& a, uint64_t* seg_out, uint64_t* hap_off, void* tmp, size_t* tmp_bytes, cudaStream_t st);
// The n_bases haplotype bytes into out (16-byte aligned, n_bases + 16 bytes), on `st`.  reverse_complement: some segment
// is HAP_SRC_RC (an ALT of kind 2).
cudaError_t hap_gather(const uint8_t* ref, const uint8_t* alt, const uint64_t* seg_src, const uint64_t* seg_out, uint64_t n_seg,
                       uint64_t n_bases, bool reverse_complement, uint8_t* out, cudaStream_t st);
// Every segment's HapLift and kind (n_seg of each) from the arrays hap_layout left, on `st`.
cudaError_t hap_lift(const HapArgs& a, const uint64_t* seg_out, const uint64_t* hap_off, HapLift* lift, uint8_t* kind, cudaStream_t st);
