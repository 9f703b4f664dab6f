// Launches of ns_apply_variants' kernels (haplotype_kernel.cuh) and its CUB scan.
#include <cub/device/device_scan.cuh>

#include "haplotype_kernel.cuh"

cudaError_t hap_layout(const HapArgs& a, uint64_t* seg_out, uint64_t* hap_off, void* tmp, size_t* tmp_bytes, cudaStream_t st) {
    const int64_t n = (int64_t)(a.n_seg + 1);
    if (!tmp) return cub::DeviceScan::ExclusiveSum(nullptr, *tmp_bytes, a.seg_len, seg_out, n, st);
    hap_segments_kernel<<<(unsigned)((a.n_seg + 1 + 255) / 256), 256, 0, st>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(tmp, *tmp_bytes, a.seg_len, seg_out, n, st);
    if (e != cudaSuccess) return e;
    hap_offsets_kernel<<<(a.n_hap + 1 + 255) / 256, 256, 0, st>>>(a.var_off, seg_out, a.n_hap, hap_off);
    return cudaGetLastError();
}

cudaError_t hap_gather(const uint8_t* ref, const uint8_t* alt, const uint64_t* seg_src, const uint64_t* seg_out, uint64_t n_seg,
                       uint64_t n_bases, bool reverse_complement, uint8_t* out, cudaStream_t st) {
    const unsigned blocks = (unsigned)((n_bases + 16 * 256 - 1) / (16 * 256));
    if (reverse_complement) hap_gather_kernel<true><<<blocks, 256, 0, st>>>(ref, alt, seg_src, seg_out, n_seg, out);
    else hap_gather_kernel<false><<<blocks, 256, 0, st>>>(ref, alt, seg_src, seg_out, n_seg, out);
    return cudaGetLastError();
}

cudaError_t hap_lift(const HapArgs& a, const uint64_t* seg_out, const uint64_t* hap_off, HapLift* lift, uint8_t* kind, cudaStream_t st) {
    hap_lift_kernel<<<(unsigned)((a.n_seg + 255) / 256), 256, 0, st>>>(a, seg_out, hap_off, lift, kind);
    return cudaGetLastError();
}
