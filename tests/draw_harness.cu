// Test harness for the device's random draw primitives (tests/test_device_draws.py).  It includes the library's own
// headers and restates nothing: every entry point runs one primitive over the inputs it is given, or over its whole input
// space, on the host (dev == 0) or on the current CUDA device (dev != 0, buffers are device pointers), and returns a
// cudaError_t after the device has finished.  Built with -DDRAW_HARNESS_HOST_ONLY the device entry points return
// cudaErrorNoDevice, so the host paths of the integer primitives are tested on machines without a GPU.
#include <cuda_runtime.h>
#include <stdint.h>

#include "device_common.cuh"
#include "emit_kernel.cuh"
#include "qual_table.h"

namespace {

#ifndef DRAW_HARNESS_HOST_ONLY
template <class F>
__global__ void each_kernel(F f, uint64_t n) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) f(i);
}

cudaError_t finish() {
    cudaError_t e = cudaGetLastError();
    return e != cudaSuccess ? e : cudaDeviceSynchronize();
}

template <class F>
cudaError_t each_device(const F& f, uint64_t n) {
    if (n) each_kernel<<<1024, 256>>>(f, n);
    return finish();
}
#endif

template <class F>
cudaError_t each(int dev, const F& f, uint64_t n) {
    if (!dev) {
        for (uint64_t i = 0; i < n; ++i) f(i);
        return cudaSuccess;
    }
#ifndef DRAW_HARNESS_HOST_ONLY
    return each_device(f, n);
#else
    return cudaErrorNoDevice;
#endif
}

template <int R>
struct PhiloxOp {
    const uint32_t* ctr;     // [n][4]
    const uint32_t* key;     // [n][2]
    uint32_t* out;           // [n][4]
    __host__ __device__ void operator()(uint64_t i) const {
        const uint4 c = philox4x32<R>(make_uint4(ctr[4 * i], ctr[4 * i + 1], ctr[4 * i + 2], ctr[4 * i + 3]),
                                      make_uint2(key[2 * i], key[2 * i + 1]));
        out[4 * i] = c.x; out[4 * i + 1] = c.y; out[4 * i + 2] = c.z; out[4 * i + 3] = c.w;
    }
};

struct SubOffsetsOp {
    const uint32_t* x;       // [n][7]: the draws X1..X7 of a chunk
    uint32_t* out;
    __host__ __device__ void operator()(uint64_t i) const {
        const uint32_t XA[3] = {x[7 * i], x[7 * i + 1], x[7 * i + 2]};
        const uint32_t XB[4] = {x[7 * i + 3], x[7 * i + 4], x[7 * i + 5], x[7 * i + 6]};
        out[i] = sub_offsets(XA, XB);
    }
};

struct AddFieldsOp {
    const uint32_t *a, *b;
    uint32_t* out;
    __host__ __device__ void operator()(uint64_t i) const { out[i] = add_fields_mod4(a[i], b[i]); }
};

// i = mis << 18 | orig << 16 | h: MIS for every (orig, h), INS for every h (i < 2^18 + 2^16)
struct EventBaseOp {
    uint8_t* out;
    __host__ __device__ void operator()(uint64_t i) const {
        out[i] = (uint8_t)event_base((uint32_t)i & 0xffffu, i < (1u << 18), (uint32_t)(i >> 16) & 3u);
    }
};

// the bases of event `event` of piece `piece` of read `rid` through the library's block layout
struct EventBasesOp {
    uint2 key;
    uint64_t rid;
    uint32_t piece, event, mis;
    const uint8_t* orig;
    uint8_t* out;
    __host__ __device__ void operator()(uint64_t t) const {
        const uint4 blk = event_base_block(key, rid, piece, event, (uint32_t)t);
        out[t] = (uint8_t)event_base(event_draw(blk, (uint32_t)t), mis != 0, orig[t]);
    }
};

// i = c << 16 | h: every byte c with every 16-bit draw h
struct Iupac16Op {
    uint8_t* out;
    __host__ __device__ void operator()(uint64_t i) const { out[i] = (uint8_t)resolve_iupac16((uint32_t)(i >> 16), (uint32_t)i & 0xffffu); }
};

struct ConvertedRefOp {
    uint64_t seed, rid;
    uint32_t piece;
    const uint8_t* c;
    const uint32_t* off;
    uint8_t* out;
    __host__ __device__ void operator()(uint64_t i) const { out[i] = (uint8_t)converted_ref_base(c[i], seed, rid, piece, off[i]); }
};

// i = state << 24 | u << 11 | slot: every 24-bit draw of every quality state; the 8 spare bits of the word are filled
// with a pattern (qual_pick must ignore them)
struct QualOp {
    const uint32_t* lut;     // [NS_N_QUAL_STATES][QLUT_SIZE]
    uint8_t* out;
    __host__ __device__ void operator()(uint64_t i) const {
        const uint32_t s = (uint32_t)(i >> 24), slot = (uint32_t)i & (QLUT_SIZE - 1u), u = ((uint32_t)i >> QLUT_BITS) & 0x1fffu;
        const uint32_t w = (u << 19) | (slot << 8) | (((uint32_t)i * 0x9e3779b9u) >> 24);
        out[i] = (uint8_t)(qual_pick(lut[(size_t)s * QLUT_SIZE + ((w >> 8) & (QLUT_SIZE - 1u))], w) & 0xffu);
    }
};

#ifndef DRAW_HARNESS_HOST_ONLY
// Both Walker alias samplers for words r[i] from tables t[i]: alias_draw reads the table directory from a DevModel,
// alias_draw_s (as plan_kernel calls it) from shared memory.
__global__ void alias_kernel(DevModel m, const uint32_t* t, const uint32_t* r, uint32_t* out_plain, uint32_t* out_shared, uint64_t n) {
    __shared__ uint32_t s_tab_off[NS_MAX_TABLES], s_tab_n[NS_MAX_TABLES];
    for (int i = threadIdx.x; i < NS_MAX_TABLES; i += blockDim.x) {
        s_tab_off[i] = m.tab_off[i];
        s_tab_n[i] = m.tab_n[i];
    }
    __syncthreads();
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        out_plain[i] = alias_draw(m, t[i], r[i]);
        out_shared[i] = alias_draw_s(m.alias, s_tab_off, s_tab_n, t[i], r[i]);
    }
}

// Every one of the 2^32 words through alias_draw on table t, counted per outcome.  A thread takes 2^12 consecutive words;
// the outcome changes at most twice per table slot along them, so the counts are kept as runs.
__global__ void alias_all_words_kernel(DevModel m, uint32_t t, unsigned long long* counts) {
    const uint64_t first = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) << 12;
    uint32_t cur = alias_draw(m, t, (uint32_t)first), run = 0;
    for (uint32_t k = 0; k < 4096u; ++k) {
        const uint32_t v = alias_draw(m, t, (uint32_t)(first + k));
        if (v != cur) {
            atomicAdd(&counts[cur], (unsigned long long)run);
            cur = v;
            run = 0;
        }
        ++run;
    }
    atomicAdd(&counts[cur], (unsigned long long)run);
}

DevModel alias_model(const uint2* alias, const uint32_t* tab_off, const uint32_t* tab_n, uint32_t n_tab) {
    DevModel m = {};
    m.alias = alias;
    for (uint32_t i = 0; i < n_tab && i < NS_MAX_TABLES; ++i) {
        m.tab_off[i] = tab_off[i];
        m.tab_n[i] = tab_n[i];
    }
    return m;
}

struct NormalOp {
    float *radius, *cosv;    // [2^24]: the two Box-Muller factors for word (v << 8) | spare bits
    __device__ void operator()(uint64_t v) const {
        const uint32_t w = ((uint32_t)v << 8) | ((uint32_t)v & 0xffu);
        radius[v] = nf32_radius(w);
        cosv[v] = nf32_cos(w);
    }
};
#endif

}  // namespace

extern "C" {

cudaError_t dh_philox(int dev, int rounds, const uint32_t* ctr, const uint32_t* key, uint32_t* out, uint64_t n) {
    if (rounds == 10) return each(dev, PhiloxOp<10>{ctr, key, out}, n);
    if (rounds == 7) return each(dev, PhiloxOp<7>{ctr, key, out}, n);
    return cudaErrorInvalidValue;
}

cudaError_t dh_sub_offsets(int dev, const uint32_t* x, uint32_t* out, uint64_t n) { return each(dev, SubOffsetsOp{x, out}, n); }

cudaError_t dh_add_fields_mod4(int dev, const uint32_t* a, const uint32_t* b, uint32_t* out, uint64_t n) {
    return each(dev, AddFieldsOp{a, b, out}, n);
}

// out: (1 << 18) + (1 << 16) bytes
cudaError_t dh_event_base_all(int dev, uint8_t* out) { return each(dev, EventBaseOp{out}, (1u << 18) + (1u << 16)); }

cudaError_t dh_event_bases(int dev, uint64_t seed, uint64_t rid, uint32_t piece, uint32_t event, uint32_t mis, const uint8_t* orig,
                           uint8_t* out, uint64_t n) {
    return each(dev, EventBasesOp{make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)), rid, piece, event, mis, orig, out}, n);
}

// out: 1 << 24 bytes
cudaError_t dh_iupac16_all(int dev, uint8_t* out) { return each(dev, Iupac16Op{out}, 1u << 24); }

cudaError_t dh_converted_ref_base(int dev, uint64_t seed, uint64_t rid, uint32_t piece, const uint8_t* c, const uint32_t* off, uint8_t* out,
                                  uint64_t n) {
    return each(dev, ConvertedRefOp{seed, rid, piece, c, off, out}, n);
}

// host only: the library's quality tables from a [NS_N_QUAL_STATES][NS_QUAL_SLOTS] 32-bit cdf
cudaError_t dh_build_qlut(const uint32_t* cdf32, uint32_t* lut) {
    std::vector<uint32_t> v;
    build_qlut(reinterpret_cast<const uint32_t(*)[NS_QUAL_SLOTS]>(cdf32), v);
    std::copy(v.begin(), v.end(), lut);
    return cudaSuccess;
}

// out: NS_N_QUAL_STATES << 24 bytes
cudaError_t dh_qual_all(int dev, const uint32_t* lut, uint8_t* out) { return each(dev, QualOp{lut, out}, (uint64_t)NS_N_QUAL_STATES << 24); }

// device only from here on.  alias: interleaved (accept threshold, alias index); tab_off / tab_n: host arrays of n_tab
cudaError_t dh_alias(const uint2* alias, const uint32_t* tab_off, const uint32_t* tab_n, uint32_t n_tab, const uint32_t* t, const uint32_t* r,
                     uint32_t* out_plain, uint32_t* out_shared, uint64_t n) {
#ifndef DRAW_HARNESS_HOST_ONLY
    if (n_tab > NS_MAX_TABLES) return cudaErrorInvalidValue;
    if (n) alias_kernel<<<1024, 256>>>(alias_model(alias, tab_off, tab_n, n_tab), t, r, out_plain, out_shared, n);
    return finish();
#else
    return cudaErrorNoDevice;
#endif
}

// counts: tab_n[t] zeroed device words
cudaError_t dh_alias_all_words(const uint2* alias, const uint32_t* tab_off, const uint32_t* tab_n, uint32_t n_tab, uint32_t t,
                               unsigned long long* counts) {
#ifndef DRAW_HARNESS_HOST_ONLY
    if (n_tab > NS_MAX_TABLES || t >= n_tab) return cudaErrorInvalidValue;
    alias_all_words_kernel<<<(1u << 20) / 256, 256>>>(alias_model(alias, tab_off, tab_n, n_tab), t, counts);
    return finish();
#else
    return cudaErrorNoDevice;
#endif
}

// radius, cosv: 1 << 24 floats each
cudaError_t dh_normal_factors(float* radius, float* cosv) {
#ifndef DRAW_HARNESS_HOST_ONLY
    return each_device(NormalOp{radius, cosv}, 1u << 24);
#else
    return cudaErrorNoDevice;
#endif
}

}  // extern "C"
