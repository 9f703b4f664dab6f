// Plan kernel: the per-read control flow of simulation_aligned_genome / simulation_unaligned
// (/root/reference/src/simulator.py:1266-1454, 1482-1549) with error_list (:1833-1916) and
// unaligned_error_list (:1784-1830) inside, run as a flattened per-lane state machine.
//
// One LANE owns one read at a time and fetches the next read from a global counter as soon as its read is
// accepted (persistent threads), so lanes of a warp are always in the same hot phase (one error/match event
// per loop iteration) regardless of how different their read lengths are.
//
// Reads are taken in order of decreasing drawn reference length (lengths_kernel + a radix sort), so the 32 lanes of
// a warp work on reads of almost equal length and finish together, and the longest chains start first.
//
//   REPLAY=false : runs the rejection loops (:1367, :1429, :1503, :1517), draws positions (extract_read :1750-1781),
//                  fills NsReadMeta / NsPieceMeta and writes every edit script into a slot sized from the drawn
//                  length (mean + 6 sigma of the op count).  A script that does not fit is only counted and the read is
//                  flagged;
//   REPLAY=true  : for flagged reads only (normally none; always for unaligned reads in NS_FLAG_UNALIGNED_SCRIPTS
//                  mode): replays the accepted attempt with identical random streams and writes the script at the
//                  exact offset an exclusive scan of the counts produced.
#pragma once
#include "device_common.cuh"

struct PlanArgs {
    DevModel m;
    DevRef ref;
    DevCfg cfg;
    uint32_t kind;              // NS_KIND_*
    uint64_t first_id;
    uint32_t n_reads;
    const uint32_t* n_seg;      // per read (nullptr => 1)
    const uint32_t* piece_first;// per read (nullptr => read index)
    NsReadMeta* reads;
    NsPieceMeta* pieces;
    uint32_t* ops;
    const uint32_t* order;      // read slots by decreasing drawn length (nullptr => identity)
    uint32_t* counter;          // work-fetch counter (zeroed before launch)
    uint32_t* n_flagged;        // REPLAY=false: number of reads whose script overflowed its slot
    uint32_t batch_reversed;    // metagenome: is_reversed is drawn once per batch (:860)
    const uint32_t* abort;      // sync-free batches: non-zero = the script area is too small, do nothing (or null)
};

#define NS_MAX_SAME_LEN_RETRIES 64

enum Phase : int { PH_FETCH = 0, PH_LEN, PH_ATT, PH_PIECE, PH_EVENT, PH_UEVENT, PH_PIECE_END, PH_CHECK, PH_DONE };

// VEC (first pass): slots are whole groups of 4 ops (lengths_kernel), 16-byte aligned, and each group goes out as ONE
// 16-byte store once it is full (finish() writes a partial last group).  The lanes of a warp write to 32 different slots,
// so a 4-byte store per op costs a memory transaction per op; a group costs one per 4 ops.  A group is written only when it
// lies wholly inside the slot; `n` keeps counting past `cap` (the read is then flagged and replayed).
// !VEC (replay): exact, unaligned slots, one 4-byte store per op.
template <bool VEC>
struct OpSink {
    uint32_t* base;       // start of this piece's op slot
    uint32_t cap;         // slot capacity in ops (VEC: a multiple of 4)
    uint32_t n;           // ops emitted so far (flushed)
    uint32_t n0;          // VEC: ops [0, n0) were written by another kernel (gap_kernel) and are not in `grp`
    uint4 grp;            // VEC: the open group, ops 4 * (n / 4) .. n - 1
    uint32_t pend_type;   // pending (mergeable) op
    uint32_t pend_len;
    uint32_t out_len;     // bases produced by flushed + pending ops
    __device__ __forceinline__ void begin(uint32_t* slot, uint32_t capacity) {
        base = slot;
        cap = capacity;
        n = 0;
        n0 = 0;
        pend_type = 0xffffffffu;
        pend_len = 0;
        out_len = 0;
    }
    __device__ __forceinline__ void set_word(uint32_t k, uint32_t w) {
        grp.x = k == 0 ? w : grp.x;
        grp.y = k == 1 ? w : grp.y;
        grp.z = k == 2 ? w : grp.z;
        grp.w = k == 3 ? w : grp.w;
    }
    __device__ __forceinline__ void emit(uint32_t w) {
        if (VEC) {
            set_word(n & 3u, w);
            if ((n & 3u) == 3u && n < cap) *reinterpret_cast<uint4*>(base + (n - 3u)) = grp;
        } else if (n < cap) {
            base[n] = w;
        }
        ++n;
    }
    // VEC: write the open, partial group (where it is inside the slot)
    __device__ __forceinline__ void finish() {
        if (!VEC) return;
        const uint32_t g = n & ~3u;
        if (g >= cap) return;
        const uint32_t w[4] = {grp.x, grp.y, grp.z, grp.w};
#pragma unroll
        for (uint32_t k = 0; k < 3; ++k)
            if (g + k < n && g + k >= n0) base[g + k] = w[k];
    }
    __device__ __forceinline__ void flush() {
        if (pend_type != 0xffffffffu && pend_len > 0) emit((pend_type << 28) | pend_len);
        pend_type = 0xffffffffu;
        pend_len = 0;
    }
    // merge == true: fold into the pending op when the type matches (used where event boundaries carry no meaning)
    __device__ __forceinline__ void push(uint32_t type, uint32_t len, bool merge) {
        if (len == 0) return;
        if (type != NS_OP_DEL) out_len += len;
        if (merge && type == pend_type) {
            pend_len += len;
            return;
        }
        flush();
        pend_type = type;
        pend_len = len;
    }
    // unmerged append (aligned segments: every error event keeps its own op, as in the reference's e_dict)
    __device__ __forceinline__ void put(uint32_t type, uint32_t len) {
        if (len == 0) return;
        if (type != NS_OP_DEL) out_len += len;
        emit((type << 28) | len);
    }
    // literal run (polyA): `len` copies of base index `base` with quality state `state`
    __device__ __forceinline__ void put_lit(uint32_t base_idx, uint32_t state, uint32_t len) {
        if (len == 0) return;
        out_len += len;
        emit((NS_OP_LIT << 28) | (base_idx << 26) | (state << 24) | len);
    }
    // the reference's e_dict[pos - 0.5] overwrite: a second insertion at the same position replaces the first (:1882)
    __device__ __forceinline__ void replace_last_ins(uint32_t old_len, uint32_t len) {
        out_len = out_len - old_len + len;
        const uint32_t i = n - 1, w = (NS_OP_INS << 28) | len;
        if (VEC && (i & 3u) != 3u) set_word(i & 3u, w);     // still in the open group
        else if (i < cap) base[i] = w;                      // its group was already written
    }
};

__device__ __forceinline__ uint32_t match_bin_scan(const DevModel& m, uint32_t prev_match) {
    uint32_t b = m.n_bins - 1;          // falls through to the last bin (:1891-1893)
    for (uint32_t i = 0; i < m.n_bins; ++i) {
        if (m.bin_lo[i] <= prev_match && prev_match < m.bin_hi[i]) {
            b = i;
            break;
        }
    }
    return b;
}
#define BIN_LUT_SIZE 1024
// bin of the previous match length: shared-memory table for short matches, header scan for the rest
__device__ __forceinline__ uint32_t match_bin(const DevModel& m, const uint8_t* lut, uint32_t prev_match) {
    return prev_match < BIN_LUT_SIZE ? (uint32_t)lut[prev_match] : match_bin_scan(m, prev_match);
}

// extract_read, genome branches (:1750-1781): uniform start over the concatenated genome, redrawn until the
// segment fits inside one chromosome (linear) / wrap-around on the single chromosome (circular).
__device__ __forceinline__ void draw_position(const DevRef& ref, const DevCfg& cfg, Rng& rng, uint32_t length,
                                              uint32_t& chrom, uint32_t& pos) {
    if (cfg.circular) {
        chrom = 0;
        pos = (uint32_t)__umul64hi(rng.next64(), ref.genome_len + 1);
        return;
    }
    for (int iter = 0; iter < 100000; ++iter) {
        uint64_t p = __umul64hi(rng.next64(), ref.genome_len + 1);
        if (p >= ref.genome_len) continue;          // walks off the last chromosome -> redraw
        uint32_t lo = 0, hi = ref.n_chrom;          // chrom_off[lo] <= p < chrom_off[hi]
        while (hi - lo > 1) {
            uint32_t mid = (lo + hi) >> 1;
            if (__ldg(&ref.chrom_off[mid]) <= p) lo = mid; else hi = mid;
        }
        uint64_t off = p - __ldg(&ref.chrom_off[lo]);
        uint64_t clen = __ldg(&ref.chrom_off[lo + 1]) - __ldg(&ref.chrom_off[lo]);
        if (off + length <= clen && length > 0) {
            chrom = lo;
            pos = (uint32_t)off;
            return;
        }
    }
    chrom = 0;
    pos = 0;
}

// extract_read, metagenome branch (:1704-1749): uniform chromosome of the species (species < 0: uniform species
// first, :1705-1706); a chromosome shorter than the segment is replaced by a uniformly chosen longer one, same species
// first; circular chromosomes start anywhere in [0, len] and wrap, linear ones in [0, len - length].
__device__ __forceinline__ void draw_position_meta(const DevRef& ref, Rng& rng, int species, uint32_t length, uint32_t& chrom,
                                                   uint32_t& pos) {
    uint32_t sp = species >= 0 ? (uint32_t)species : (uint32_t)__umul64hi(rng.next64(), (uint64_t)ref.n_species);
    const uint32_t c0 = __ldg(&ref.species_chrom_off[sp]), c1 = __ldg(&ref.species_chrom_off[sp + 1]);
    uint32_t c = c0 + (uint32_t)__umul64hi(rng.next64(), (uint64_t)(c1 - c0));
    uint64_t clen = __ldg(&ref.chrom_off[c + 1]) - __ldg(&ref.chrom_off[c]);
    if ((uint64_t)length > clen) {
        uint32_t n_same = 0, n_all = 0;
        for (uint32_t q = 0; q < ref.n_chrom; ++q) {
            const uint64_t l = __ldg(&ref.chrom_off[q + 1]) - __ldg(&ref.chrom_off[q]);
            if ((uint64_t)length < l) {
                ++n_all;
                if (q >= c0 && q < c1) ++n_same;
            }
        }
        const bool same = n_same > 0;
        const uint32_t n_pick = same ? n_same : n_all - n_same;   // the reference's `longer_chroms` excludes the species
        if (n_pick > 0) {
            uint32_t r = (uint32_t)__umul64hi(rng.next64(), (uint64_t)n_pick);
            for (uint32_t q = 0; q < ref.n_chrom; ++q) {
                const uint64_t l = __ldg(&ref.chrom_off[q + 1]) - __ldg(&ref.chrom_off[q]);
                const bool in_sp = q >= c0 && q < c1;
                if ((uint64_t)length < l && in_sp == same) {
                    if (r == 0) {
                        c = q;
                        break;
                    }
                    --r;
                }
            }
            clen = __ldg(&ref.chrom_off[c + 1]) - __ldg(&ref.chrom_off[c]);
        }
    }
    chrom = c;
    if (__ldg(&ref.chrom_circular[c])) {
        pos = (uint32_t)__umul64hi(rng.next64(), clen + 1);
    } else {
        pos = clen >= length ? (uint32_t)__umul64hi(rng.next64(), clen - length + 1) : 0u;
    }
}

// extract_read, transcriptome branch (:1695-1703, unaligned reads): a uniformly chosen transcript, drawn again until it is
// longer than the read, then a uniform start.  Redrawing until the condition holds == one uniform draw among the
// transcripts that satisfy it: they are a suffix of the records sorted by length (DevRef::trx_len_sorted), so the
// rejection loop (thousands of draws for a read close to the longest transcript) becomes one binary search.
__device__ __forceinline__ void draw_position_trx(const DevRef& ref, uint32_t n_records, Rng& rng, uint32_t length, uint32_t& chrom,
                                                  uint32_t& pos) {
    if (ref.trx_len_sorted && ref.n_trx_sorted == n_records) {
        uint32_t lo = 0, hi = n_records;                     // first sorted record longer than the read
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (__ldg(&ref.trx_len_sorted[mid]) > length) hi = mid; else lo = mid + 1;
        }
        if (lo < n_records) {
            const uint32_t j = lo + (uint32_t)__umul64hi(rng.next64(), (uint64_t)(n_records - lo));
            chrom = __ldg(&ref.trx_len_idx[j]);
            pos = (uint32_t)__umul64hi(rng.next64(), (uint64_t)(__ldg(&ref.trx_len_sorted[j]) - length + 1u));
            return;
        }
        chrom = 0;                                           // no transcript is long enough (the reference would spin forever)
        pos = 0;
        return;
    }
    for (int it = 0; it < 1000000; ++it) {
        const uint32_t c = (uint32_t)__umul64hi(rng.next64(), (uint64_t)n_records);
        const uint64_t clen = __ldg(&ref.chrom_off[c + 1]) - __ldg(&ref.chrom_off[c]);
        if ((uint64_t)length < clen) {
            chrom = c;
            pos = (uint32_t)__umul64hi(rng.next64(), clen - length + 1);
            return;
        }
    }
    chrom = 0;
    pos = 0;
}

// select_nearest_kde2d (:108-111) on a size-N sample of the 2-D KDE (:1072, :1090), sampled EXACTLY without drawing the
// N points: the KDE adds N(0, bw ~ 0.1) to integer training rows (x_i, y_i), so the sample point nearest to the
// transcript length L is a training row at some integer distance d; with p(d) = #{|x_i - L| <= d} / M,
// P(min distance <= d) = 1 - (1 - p(d))^N.  Inverting with one uniform gives d* = min{d: p(d) >= 1 - (1-u)^(1/N)};
// by symmetry the nearest point is uniform over the rows at distance exactly d*, and its aligned length is
// int(y_i + N(0, bw)).  O(log^2 M) instead of the reference's O(N) argmin per read.
__device__ __forceinline__ uint32_t lower_bound_f(const float* x, uint32_t n, float v) {     // first i with x[i] >= v
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        uint32_t mid = (lo + hi) >> 1;
        if (__ldg(&x[mid]) < v) lo = mid + 1; else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ uint32_t nearest_aligned_length(const DevModel& m, uint32_t n_sample, uint32_t L, Rng& rng) {
    const uint32_t M = m.n_kde2d;
    const double u = u01_double(rng.next64());
    const double q = -expm1(log1p(-u) / (double)(n_sample > 0 ? n_sample : 1));     // 1 - (1-u)^(1/N)
    const double need = q * (double)M;
    const float fl = (float)L;
    const float xmin = __ldg(&m.kde2d_x[0]), xmax = __ldg(&m.kde2d_x[M - 1]);
    uint32_t dlo = 0, dhi = (uint32_t)fmaxf(fabsf(fl - xmin), fabsf(xmax - fl)) + 1;    // count(dhi) == M
    while (dlo < dhi) {                                                                // smallest d with count(d) >= need
        const uint32_t d = (dlo + dhi) >> 1;
        const uint32_t a = lower_bound_f(m.kde2d_x, M, fl - (float)d);
        const uint32_t b = lower_bound_f(m.kde2d_x, M, fl + (float)d + 0.5f);
        if ((double)(b - a) >= need && b > a) dhi = d; else dlo = d + 1;
    }
    const uint32_t d = dlo;
    // rows at distance exactly d: x == L - d and (d > 0) x == L + d
    const uint32_t a0 = lower_bound_f(m.kde2d_x, M, fl - (float)d), a1 = lower_bound_f(m.kde2d_x, M, fl - (float)d + 0.5f);
    uint32_t b0 = 0, b1 = 0;
    if (d > 0) {
        b0 = lower_bound_f(m.kde2d_x, M, fl + (float)d);
        b1 = lower_bound_f(m.kde2d_x, M, fl + (float)d + 0.5f);
    }
    const uint32_t cnt = (a1 - a0) + (b1 - b0);
    uint32_t r = (uint32_t)__umul64hi(rng.next64(), (uint64_t)(cnt > 0 ? cnt : 1));
    const uint32_t row = cnt == 0 ? (a0 < M ? a0 : M - 1) : (r < a1 - a0 ? a0 + r : b0 + (r - (a1 - a0)));
    const uint32_t r1 = rng.next(), r2 = rng.next();
    const float z = sqrtf(-2.0f * logf(u01_open_low(r1))) * cospif(2.0f * ((float)(r2 >> 8) * (1.0f / 16777216.0f)));
    const double y = (double)__ldg(&m.kde2d_y[row]) + (double)m.kde2d_bw * (double)z;
    return y > 0.0 ? (uint32_t)y : 0u;
}

// ref_lengths / gap_lengths of generation `gen` for one aligned read (:1285-1299, :1309-1310) -> pieces[].ref_req
__device__ __forceinline__ void draw_lengths(const DevModel& m, const DevCfg& cfg, uint32_t kind, uint64_t rid, uint32_t gen,
                                             uint32_t n_seg, NsPieceMeta* pieces) {
    Rng lr;
    lr.init(cfg.seed, rid, stream_word(ST_LEN, kind, gen));
    for (uint32_t s = 0; s < n_seg; ++s) {
        uint32_t len = 0;
        for (int it = 0; it < 100000; ++it) {
            double x;
            if (cfg.median_len > 0.0) {
                // -med/-sd (:1285-1295): perfect reads take the log-normal length itself; otherwise the reference
                // subtracts a head/tail remainder from a log-normal TOTAL length.  Its list filtering (:1296) breaks
                // the pairing between that remainder and the one the read later gets, so the subtracted remainder is
                // an independent kde_ht draw here.
                if (cfg.perfect) {
                    x = lognormal_draw(log(cfg.median_len), cfg.sd_len, lr);
                } else {
                    double t = lognormal_draw(log(cfg.median_len + cfg.sd_len * cfg.sd_len / 2.0), cfg.sd_len, lr);
                    double rem = -1.0;
                    for (int jt = 0; jt < 100000 && rem < 0.0; ++jt) rem = pow(10.0, kde_draw(m.ht, lr)) - 1.0;
                    x = t - rem;
                }
            } else {
                x = kde_draw(m.aligned, lr);
            }
            bool ok = cfg.perfect ? (x >= (double)cfg.min_len && x <= (double)cfg.max_len)
                                  : (x > 0.0 && x <= (double)cfg.max_len);
            if (cfg.metagenome) {                        // int(round(x)) (:871); a zero-length segment is legal there
                if (ok) {
                    len = (uint32_t)rint(x);
                    break;
                }
                continue;
            }
            // int(x) == 0 makes the reference's extract_read spin forever (:1767-1780); redraw instead
            if (ok && (uint32_t)x > 0) {
                len = (uint32_t)x;
                break;
            }
        }
        pieces[2 * s].ref_req = len;
        if (s + 1 < n_seg) {
            double g = pow(10.0, kde_draw(m.gap, lr)) - 1.0;
            int64_t gi = (int64_t)g;
            pieces[2 * s + 1].ref_req = gi > 0 ? (uint32_t)gi : 0u;
        }
    }
}

// Generation-0 lengths of every read of the batch, op-slot capacities per piece and the sort key (total drawn length).
// cap = 2 * (E + 6 cv sqrt(E) + 8) + 4 ops for a segment expected to hold E = m_ref / mean_ref_per_event error events
// (cv = coefficient of variation of the reference advance per event: the event count of a renewal process has variance E cv^2).
__global__ void lengths_kernel(DevModel m, DevCfg cfg, uint32_t kind, uint64_t first_id, uint32_t n, const uint32_t* n_seg,
                               const uint32_t* piece_first, NsPieceMeta* pieces, float ev_per_base, float ev_cv, uint32_t exact_only,
                               uint64_t* caps, uint32_t* keys, uint32_t* vals) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t ns = n_seg ? n_seg[i] : 1u;
    const uint32_t pf = piece_first ? piece_first[i] : i;
    uint64_t total = 0;
    if (kind == NS_KIND_ALIGNED && cfg.transcriptome) {
        caps[pf] = 0;                   // the aligned length depends on the transcript drawn inside the attempt: exact pass
    } else if (kind == NS_KIND_ALIGNED) {
        draw_lengths(m, cfg, kind, first_id + i, 0, ns, pieces + pf);
        for (uint32_t q = 0; q < 2 * ns - 1; ++q) {
            const uint32_t len = pieces[pf + q].ref_req;
            total += len;
            uint64_t cap;
            if (q & 1u) cap = 2ull * len + 64;                           // gap: unaligned-type script
            else if (cfg.perfect) cap = 4;
            else {
                float e = (float)len * ev_per_base;
                cap = (uint64_t)(2.0f * (e + 6.0f * ev_cv * sqrtf(e) + 8.0f)) + 4;
            }
            caps[pf + q] = exact_only ? 0 : (cap + 3) & ~3ull;          // whole 16-byte groups (OpSink<true>)
        }
    } else if (exact_only) {
        caps[pf] = 0;                                                    // scripted unaligned reads: exact pass only
    } else {
        // unaligned fast path (uread_kernel.cuh): slot from the attempt-0 length (block 0 of the attempt stream); an
        // unmerged unaligned script has at most 4 ops per reference base, in practice ~0.7
        Rng r0;
        r0.init(cfg.seed, first_id + i, stream_word(ST_ATT, NS_KIND_UNALIGNED, 0));
        const double x = cfg.median_len > 0.0 ? lognormal_draw(log(cfg.median_len), cfg.sd_len, r0) : kde_draw(m.unaligned, r0);
        const uint64_t len = x >= 1.0 ? (x < 268435455.0 ? (uint64_t)x : 268435455ull) : 0ull;
        caps[pf] = len + (len >> 1) + 64;
        total = len;
    }
    keys[i] = total > 0xffffffffull ? 0xffffffffu : (uint32_t)total;
    vals[i] = i;
}

#ifndef PLAN_MIN_BLOCKS
#define PLAN_MIN_BLOCKS 4     // resident 128-thread blocks per SM the register allocation aims for
#endif
template <bool REPLAY>
__global__ void __launch_bounds__(128, PLAN_MIN_BLOCKS) plan_kernel(const __grid_constant__ PlanArgs a) {
    const DevModel& m = a.m;
    const DevCfg& cfg = a.cfg;
    const bool unal_kind = (a.kind == NS_KIND_UNALIGNED);
    if (a.abort && *a.abort) return;
    __shared__ uint8_t bin_lut[BIN_LUT_SIZE];
    // table directory and error-type thresholds: the lanes of a warp index them differently (bin of the previous match, error
    // state), which costs one constant-cache replay per distinct index when read from the kernel parameters
    __shared__ uint32_t s_tab_off[NS_MAX_TABLES], s_tab_n[NS_MAX_TABLES], s_trans[NS_N_ERR_STATES * 3];
    for (uint32_t i = threadIdx.x; i < BIN_LUT_SIZE; i += blockDim.x) bin_lut[i] = (uint8_t)match_bin_scan(m, i);
    for (uint32_t i = threadIdx.x; i < NS_MAX_TABLES; i += blockDim.x) {
        s_tab_off[i] = m.tab_off[i];
        s_tab_n[i] = m.tab_n[i];
    }
    for (uint32_t i = threadIdx.x; i < NS_N_ERR_STATES * 3; i += blockDim.x) s_trans[i] = m.trans[i / 3][i % 3];
    __syncthreads();

    int phase = PH_FETCH;
    uint32_t slot = 0;            // read index inside the batch
    uint64_t rid = 0;             // global read id
    uint32_t n_seg = 1, n_pieces = 1, piece_first = 0;
    uint32_t attempt = 0, gen = 0, gen_fails = 0;
    Rng rng;                      // attempt stream
    // attempt state
    uint32_t remainder = 0, head = 0, tail = 0, reversed = 0;
    uint64_t total = 0, actual = 0;
    uint32_t p = 0;               // piece cursor
    // chain state
    uint32_t pos = 0, middle_ref = 0, prev_match = 0, err_state = 0, last_err = 3;
    int64_t l_new = 0;
    uint32_t pending_ins = 0;     // unaligned chain: insertion waiting for the next non-ins step
    uint4 ev_r = make_uint4(0, 0, 0, 0);  // random block of the next error event (PH_EVENT)
    uint32_t gap_sw = 0, gap_draw = 0;   // chimeric gap / segment chain: its own stream (a gap's is shared with gap_kernel), draw k = Philox block k + 1
    bool last_op_was_ins_same_pos = false;
    uint32_t last_ins_len = 0;
    OpSink<!REPLAY> sink;
    sink.begin(nullptr, 0);
    bool overflow = false;

    for (;;) {
        switch (phase) {
        case PH_FETCH: {
            slot = atomicAdd(a.counter, 1u);
            if (slot >= a.n_reads) {
                phase = PH_DONE;
                break;
            }
            if (a.order) slot = a.order[slot];
            if (REPLAY && !(a.reads[slot].flags & 1u)) break;      // only flagged reads are replayed
            rid = a.first_id + slot;
            n_seg = a.n_seg ? a.n_seg[slot] : 1u;
            piece_first = a.piece_first ? a.piece_first[slot] : slot;
            n_pieces = unal_kind ? 1u : 2u * n_seg - 1u;
            overflow = false;
            if (REPLAY) {
                attempt = a.reads[slot].attempts;
            } else {
                attempt = 0;
                gen = 0;                   // generation-0 lengths were drawn by lengths_kernel
                gen_fails = 0;
            }
            phase = PH_ATT;
            break;
        }
        case PH_LEN: {   // aligned: new ref_lengths / gap_lengths after a :1429 rejection (generation >= 1)
            draw_lengths(m, cfg, a.kind, rid, gen, n_seg, a.pieces + piece_first);
            phase = PH_ATT;
            break;
        }
        case PH_ATT: {
            rng.init(cfg.seed, rid, stream_word(ST_ATT, a.kind, attempt));
            overflow = false;
            p = 0;
            total = 0;
            actual = 0;
            if (unal_kind) {
                // ref = int(kde_unaligned.sample()) (:1494-1499); <= 0 can never pass the min_l test (:1503)
                double x = cfg.median_len > 0.0 ? lognormal_draw(log(cfg.median_len), cfg.sd_len, rng)
                                                : kde_draw(m.unaligned, rng);
                int64_t r = (int64_t)x;
                if (!REPLAY) a.pieces[piece_first].ref_req = r > 0 ? (uint32_t)r : 0u;
                head = tail = 0;
                remainder = 0;
                if (r <= 0 && !REPLAY) {
                    ++attempt;                      // rejected: middle_ref < min_l
                    break;
                }
            } else if (cfg.transcriptome) {
                // transcript by TPM (random.choices over make_cdf, :1084), aligned length from the 2-D KDE nearest the
                // transcript length, redrawn until it is shorter than the transcript (:1085-1109)
                uint32_t trx = 0, tlen = 0, alen = 0;
                for (int it = 0; it < 1000000; ++it) {
                    const uint32_t r = rng.next();
                    const uint64_t pp = (uint64_t)r * a.ref.n_expressed;
                    const uint32_t j = (uint32_t)(pp >> 32);
                    const uint2 e = __ldg(&a.ref.expr_alias[j]);
                    const uint32_t k = ((uint32_t)pp < e.x || e.x == 0xffffffffu) ? j : e.y;
                    trx = __ldg(&a.ref.expr_chrom[k]);
                    tlen = (uint32_t)(__ldg(&a.ref.chrom_off[trx + 1]) - __ldg(&a.ref.chrom_off[trx]));
                    alen = nearest_aligned_length(m, cfg.kde2d_n, tlen, rng);
                    if (alen < tlen) break;
                }
                NsPieceMeta& pm0 = a.pieces[piece_first];
                pm0.ref_req = alen;
                pm0.chrom = trx;                                           // the transcript travels in `chrom`
                reversed = u01_double(rng.next64()) > (double)m.strandness;
                head = tail = 0;
                remainder = 0;
                if (!cfg.perfect) {
                    // remainder_l[simulated], head_vs_ht_ratio_l[simulated] (:1066-1070): one draw per ACCEPTED read, no
                    // filtering (a negative 10^x-1 truncates to 0, the ratio is clamped to [0,1])
                    Rng hr;
                    hr.init(cfg.seed, rid, stream_word(ST_LEN, a.kind, 0));
                    const double rem = pow(10.0, kde_draw(m.ht, hr)) - 1.0;
                    double ratio = kde_draw(m.ratio, hr);
                    ratio = ratio > 1.0 ? 1.0 : (ratio < 0.0 ? 0.0 : ratio);
                    remainder = rem > 0.0 ? (uint32_t)rem : 0u;
                    if (remainder > 0) {
                        head = (uint32_t)rint((double)remainder * ratio);
                        tail = remainder - head;
                    }
                }
            } else if (cfg.perfect) {
                head = tail = 0;
                remainder = 0;
                reversed = u01_double(rng.next64()) > (double)m.strandness;
                if (cfg.metagenome) reversed = a.batch_reversed;
            } else {
                // remainder = 10^x - 1 >= 0, ratio in [0,1] (:1456-1479), strand (:1312)
                double rem = -1.0;
                for (int it = 0; it < 100000 && rem < 0.0; ++it) rem = pow(10.0, kde_draw(m.ht, rng)) - 1.0;
                double ratio = -1.0;
                for (int it = 0; it < 100000 && (ratio < 0.0 || ratio > 1.0); ++it) ratio = kde_draw(m.ratio, rng);
                remainder = cfg.metagenome ? (uint32_t)rint(rem) : (uint32_t)rem;       // int(round()) (:916) vs int() (:1351)
                reversed = u01_double(rng.next64()) > (double)m.strandness;
                if (cfg.metagenome) reversed = a.batch_reversed;
                if (remainder == 0) {
                    head = tail = 0;
                } else {
                    head = (uint32_t)rint((double)remainder * ratio);     // Python round(): half to even (:1381)
                    tail = remainder - head;
                }
                total = remainder;
            }
            phase = PH_PIECE;
            break;
        }
        case PH_PIECE: {
            NsPieceMeta& pm = a.pieces[piece_first + p];
            uint32_t m_ref = pm.ref_req;
            // slot = [op_off, next piece's op_off) ; a replayed (flagged) piece has an exact slot
            sink.begin(a.ops + pm.op_off, REPLAY ? 0xffffffffu : (uint32_t)(a.pieces[piece_first + p + 1].op_off - pm.op_off));
            pos = 0;
            middle_ref = m_ref;
            l_new = (int64_t)m_ref;
            pending_ins = 0;
            last_op_was_ins_same_pos = false;
            bool is_gap = unal_kind || (p & 1u);
            if (!unal_kind && p == 0 && head > 0) sink.put(NS_OP_HT, head);
            if (is_gap && !unal_kind) {
                // a chimeric gap draws from its own stream (device_common.cuh ST_GAP); the first attempt was already walked
                // by gap_kernel, 32 draws at a time, and left its result in the piece record
                gap_sw = stream_word(ST_GAP, a.kind, (attempt << 5) | (p & 31u));
                gap_draw = 0;
                if (!REPLAY && attempt == 0 && pm.polya_len == 1u) {
                    pm.polya_len = 0;
                    sink.n = sink.n0 = pm.n_ops;        // no op follows: a gap gets no head or tail
                    sink.out_len = pm.out_len;
                    middle_ref = pm.ref_len;
                    l_new = (int64_t)pm.out_len;
                    phase = PH_PIECE_END;
                    break;
                }
                pm.polya_len = 0;
            }
            if (is_gap) {
                phase = (m_ref == 0) ? PH_PIECE_END : PH_UEVENT;
            } else if (cfg.perfect) {
                sink.put(NS_OP_COPY, m_ref);
                phase = PH_PIECE_END;
            } else {
                // the error chain of a segment draws from its own stream, keyed by (attempt, piece): block 0 = first match,
                // block k + 1 = event k (so that an event's block can be computed while the previous event is still waiting
                // for its table lookups)
                gap_sw = stream_word(ST_CHAIN, a.kind, (attempt << 5) | (p & 31u));
                gap_draw = 0;
                // first match from _first_match.hist, floor 2 (:1843-1850); no extension when it overshoots
                uint32_t fm = alias_draw(m, 0, philox4x32_10(make_uint4((uint32_t)rid, (uint32_t)(rid >> 32), gap_sw, 0u), rng.key).x);
                ev_r = philox4x32_10(make_uint4((uint32_t)rid, (uint32_t)(rid >> 32), gap_sw, 1u), rng.key);
                prev_match = fm;
                err_state = 0;     // "start"
                last_err = 3;
                pos = fm;
                sink.put(NS_OP_COPY, fm < middle_ref ? fm : middle_ref);
                phase = (pos < middle_ref) ? PH_EVENT : PH_PIECE_END;
            }
            break;
        }
        case PH_EVENT: {   // one pass of the while-loop body of error_list (:1858-1914)
            // this event's random block was computed during the previous event; the next one's is requested now, so that its
            // ten rounds run while this event waits for its table lookups (the lookups, not the arithmetic, are the chain)
            const uint4 r = ev_r;
            ++gap_draw;
            ev_r = philox4x32_10(make_uint4((uint32_t)rid, (uint32_t)(rid >> 32), gap_sw, gap_draw + 1u), rng.key);
            // the next match length only depends on the previous one (:1891-1903): its table lookup is issued first so
            // that it overlaps the error-length lookup below
            const uint32_t b = match_bin(m, bin_lut, prev_match);
            uint32_t mt = alias_draw_s(m.alias, s_tab_off, s_tab_n, 4 + b, r.z);
            // error type from the Markov chain keyed by prev_error[+"0"] (:1860-1864)
            uint32_t e;
            if (r.x < s_trans[3 * err_state]) e = 1;
            else if (r.x < s_trans[3 * err_state + 1]) e = 2;
            else if (r.x >= s_trans[3 * err_state + 2]) e = 3;
            else e = last_err;                        // dead gap of the (1-p_del, 1) interval: stale value
            last_err = e;
            uint32_t step = alias_draw_s(m.alias, s_tab_off, s_tab_n, e, r.y);    // tables 1..3: mis / ins / del lengths (:1866-1873)
            if (e == 2) {
                l_new += step;
                if (last_op_was_ins_same_pos) sink.replace_last_ins(last_ins_len, step);
                else sink.put(NS_OP_INS, step);
                last_ins_len = step;
            } else {
                if (e == 3) l_new -= step;
                sink.put(e == 1 ? NS_OP_MIS : NS_OP_DEL, step);
                pos += step;
                if (pos >= middle_ref) {
                    l_new += pos - middle_ref;
                    middle_ref = pos;
                }
            }
            if (mt == s_tab_n[4 + b] - 1) mt = step;  // ECDF miss: `step` keeps the error length (:1895-1898)
            if (prev_match == 0 && mt == 0) mt = 1;
            prev_match = mt;
            if (pos + mt > middle_ref) {
                l_new += pos + mt - middle_ref;
                middle_ref = pos + mt;
            }
            pos += mt;
            sink.put(NS_OP_COPY, mt);
            last_op_was_ins_same_pos = (e == 2 && mt == 0);
            err_state = e + (mt == 0 ? 3u : 0u);      // prev_error += "0" (:1913-1914)
            if (pos >= middle_ref) phase = PH_PIECE_END;
            break;
        }
        case PH_UEVENT: {  // one pass of unaligned_error_list's loop (:1794-1828) + its effect in mutate_read
            uint4 r;
            if (unal_kind) {
                r = rng.next4();
            } else {               // chimeric gap: block k + 1 of the gap's stream for draw k, as gap_kernel / uread_kernel count them
                r = philox4x32_10(make_uint4((uint32_t)rid, (uint32_t)(rid >> 32), gap_sw, ++gap_draw), rng.key);
            }
            // fixed type cdf 0.4 / 0.7 / 0.85 / 1 (:1787)
            uint32_t kind_u = r.x < 1717986918u ? 0u : (r.x < 3006477107u ? 1u : (r.x < 3650722201u ? 2u : 3u));
            if (kind_u == 2) {                       // ins: merged at key pos+0.1 (:1808-1815)
                uint32_t step = alias_draw(m, 2, r.y);
                pending_ins += step;
                l_new += step;
                break;
            }
            // mutate_read applies keys right to left; ceil(pos+0.1) = pos+1 puts the insertion AFTER the first
            // base of the step at `pos`, so a mis/del of length s at pos also eats min(a, s-1) inserted bases.
            uint32_t a_ins = pending_ins;
            pending_ins = 0;
            uint32_t s;
            if (kind_u == 0) {
                s = 1;
                sink.push(NS_OP_COPY, 1, true);
                sink.push(NS_OP_INS, a_ins, true);
            } else {
                s = alias_draw_s(m.alias, s_tab_off, s_tab_n, kind_u == 1 ? 1 : 3, r.y);
                uint32_t covered = a_ins < s - 1 ? a_ins : s - 1;     // inserted bases inside [pos, pos+s)
                uint32_t rest = (s - 1) - covered;                     // reference bases still hit after them
                if (kind_u == 1) {
                    sink.push(NS_OP_MIS, 1, true);
                    sink.push(NS_OP_INS, a_ins, true);                 // re-randomised inserted bases stay random
                    sink.push(NS_OP_MIS, rest, true);
                    sink.push(NS_OP_COPY, covered, true);
                } else {
                    l_new -= s;
                    sink.push(NS_OP_DEL, 1, true);
                    sink.push(NS_OP_INS, a_ins - covered, true);
                    sink.push(NS_OP_DEL, rest, true);
                    sink.push(NS_OP_COPY, covered, true);
                }
            }
            pos += s;
            if (pos > middle_ref) {
                l_new += pos - middle_ref;
                middle_ref = pos;
            }
            if (pos >= middle_ref) phase = PH_PIECE_END;
            break;
        }
        case PH_PIECE_END: {
            NsPieceMeta& pm = a.pieces[piece_first + p];
            bool is_gap = unal_kind || (p & 1u);
            sink.flush();
            if (cfg.transcriptome && !unal_kind) {
                // the polyA tail sits between the mutated transcript piece and the tail (:1229-1241); its length is only
                // known after the position draw, so the first pass appends it in PH_CHECK and the replay reads it back
                if (REPLAY) {
                    sink.put_lit(0u, 3u, pm.polya_len);
                    sink.put(NS_OP_HT, tail);
                }
            } else if (!unal_kind && p + 1 == n_pieces && tail > 0) {
                sink.put(NS_OP_HT, tail);
            }
            sink.finish();
            if (!REPLAY) {
                if (sink.n > sink.cap) overflow = true;
                pm.n_ops = sink.n;
                pm.read_slot = slot;
                pm.kind = unal_kind ? NS_PIECE_UNALIGNED : (is_gap ? NS_PIECE_GAP : NS_PIECE_SEGMENT);
                pm.ref_len = middle_ref;
                pm.out_len = sink.out_len;
                pm.out_rel = (uint32_t)actual;
                pm.l_new = (uint32_t)(l_new < 0 ? 0 : l_new);
            }
            // a replayed gap was first walked by gap_kernel, whose script merges less: the exact slot is at least as large
            if (REPLAY && is_gap && !unal_kind) pm.n_ops = sink.n;
            actual += sink.out_len;
            if (cfg.metagenome && !unal_kind) {
                // metagenome: total = remainder + middle_ref of the segments + mutated gap lengths (:924-943)
                total += is_gap ? (uint64_t)sink.out_len : (uint64_t)middle_ref;
            } else if (!is_gap) {
                total += (uint64_t)(l_new < 0 ? 0 : l_new);               // `total += middle` (:1362): segments only
            }
            ++p;
            phase = (p < n_pieces) ? PH_PIECE : PH_CHECK;
            break;
        }
        case PH_CHECK: {
            if (REPLAY) {
                phase = PH_FETCH;
                break;
            }
            bool ok1, ok2;
            if (cfg.transcriptome && !unal_kind) {
                NsPieceMeta& pm = a.pieces[piece_first];
                const uint32_t trx = pm.chrom;
                const uint32_t tlen = (uint32_t)(__ldg(&a.ref.chrom_off[trx + 1]) - __ldg(&a.ref.chrom_off[trx]));
                if (!cfg.perfect && pm.ref_len > tlen) {                  // `if middle_ref > ref_trx_len: continue` (:1148)
                    ++attempt;
                    phase = PH_ATT;
                    break;
                }
                // extract_read_trx (:1683-1691): uniform start; the read keeps a polyA tail when it ends within 10 bases
                // of the transcript's 3' end and the transcript is in the --polya list
                Rng pr;
                pr.init(cfg.seed, rid, stream_word(ST_POS, a.kind, attempt));
                const uint32_t ppos = (uint32_t)__umul64hi(pr.next64(), (uint64_t)(tlen - pm.ref_len) + 1);
                uint32_t polya_len = 0;
                const bool has = a.ref.chrom_has_polya && cfg.polya_scale > 0.0 && __ldg(&a.ref.chrom_has_polya[trx]);
                if (has && (uint64_t)ppos + pm.ref_len + 10 >= tlen) {
                    const double uu = 1.0 - u01_double(pr.next64());     // (0,1]
                    polya_len = (uint32_t)(2.0 - cfg.polya_scale * log(uu));   // int(expon(loc=2, scale).rvs()) (:1053)
                }
                sink.put_lit(0u, 3u, polya_len);
                sink.put(NS_OP_HT, tail);
                sink.finish();
                if (sink.n > sink.cap) overflow = true;
                pm.pos = ppos;
                pm.polya_len = polya_len;
                pm.n_ops = sink.n;
                pm.out_len = sink.out_len;
                actual = sink.out_len;
                NsReadMeta rm;
                rm.seq_off = 0;
                rm.seq_len = (uint32_t)actual;
                rm.head = head;
                rm.tail = tail;
                rm.piece_first = piece_first;
                rm.n_pieces = 1;
                rm.reversed = (uint8_t)reversed;
                rm.flags = (uint8_t)(overflow ? 1 : 0);
                rm.attempts = attempt;
                if (overflow) atomicAdd(a.n_flagged, 1u);
                a.reads[slot] = rm;
                phase = PH_FETCH;
                break;
            }
            if (unal_kind) {
                // :1503 middle_ref in range, :1517 len(read_mutated) in range
                ok1 = middle_ref >= cfg.min_len && middle_ref <= cfg.max_len;
                ok2 = actual >= cfg.min_len && actual <= cfg.max_len;
                if (!(ok1 && ok2)) {
                    ++attempt;
                    phase = PH_ATT;
                    break;
                }
                reversed = u01_double(rng.next64()) > (double)m.strandness;    // :1526-1527
            } else if (cfg.perfect) {
                ok2 = actual >= cfg.min_len && actual <= cfg.max_len;          // :1429
                if (!ok2) {
                    ++attempt;
                    ++gen;
                    phase = PH_LEN;
                    break;
                }
            } else {
                ok1 = total >= cfg.min_len && total <= cfg.max_len;            // :1367 keeps the ref lengths
                if (!ok1) {
                    ++attempt;
                    // The reference retries the same lengths with the following reads of its batch and only redraws
                    // them when the batch is exhausted (:1283-1299); lengths that can (almost) never pass would
                    // otherwise spin here, so they are redrawn after NS_MAX_SAME_LEN_RETRIES rejections.
                    if (++gen_fails >= NS_MAX_SAME_LEN_RETRIES) {
                        gen_fails = 0;
                        ++gen;
                        phase = PH_LEN;
                    } else {
                        phase = PH_ATT;
                    }
                    break;
                }
                ok2 = actual >= cfg.min_len && actual <= cfg.max_len;          // :1429 consumes them
                if (!ok2) {
                    ++attempt;
                    ++gen;
                    gen_fails = 0;
                    phase = PH_LEN;
                    break;
                }
            }
            // accepted: positions (extract_read) for every piece, then the read record
            Rng pr;
            pr.init(cfg.seed, rid, stream_word(ST_POS, a.kind, attempt));
            for (uint32_t q = 0; q < n_pieces; ++q) {
                NsPieceMeta& pm = a.pieces[piece_first + q];
                uint32_t chrom = 0, ppos = 0;
                if (cfg.metagenome) {
                    // segments carry the species assign_species gave them (in `chrom`); gaps and unaligned reads take a
                    // uniformly random species (:1705-1706)
                    const bool seg = !unal_kind && !(q & 1u);
                    draw_position_meta(a.ref, pr, seg ? (int)pm.chrom : -1, pm.ref_len, chrom, ppos);
                } else if (cfg.transcriptome) {
                    draw_position_trx(a.ref, cfg.trx_records ? cfg.trx_records : a.ref.n_chrom, pr, pm.ref_len, chrom, ppos);
                } else if (pm.ref_len > 0) {
                    draw_position(a.ref, cfg, pr, pm.ref_len, chrom, ppos);
                }
                pm.chrom = chrom;
                pm.pos = ppos;
            }
            NsReadMeta rm;
            rm.seq_off = 0;
            rm.seq_len = (uint32_t)actual;
            rm.head = head;
            rm.tail = tail;
            rm.piece_first = piece_first;
            rm.n_pieces = (uint16_t)n_pieces;
            rm.reversed = (uint8_t)reversed;
            rm.flags = (uint8_t)(((n_seg > 1) ? 2 : 0) | (overflow ? 1 : 0));
            if (overflow) atomicAdd(a.n_flagged, 1u);
            rm.attempts = attempt;
            a.reads[slot] = rm;
            phase = PH_FETCH;
            break;
        }
        default:
            break;
        }
        if (phase == PH_DONE) break;
    }
}

// n_seg ~ Geometric(1/segment_mean) per read (:1276-1279), fixed across rejection retries.
__global__ void segments_kernel(DevModel m, DevCfg cfg, uint32_t kind, uint64_t first_id, uint32_t n, uint32_t* n_seg,
                                uint32_t* n_pieces) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Rng r;
    r.init(cfg.seed, first_id + i, stream_word(ST_SEG, kind, 0));
    double u = 1.0 - u01_double(r.next64());        // (0, 1]
    uint32_t k = 1;
    if (m.seg_p < 1.0) {
        double v = ceil(log(u) / log1p(-m.seg_p));
        k = v < 1.0 ? 1u : (v > (double)NS_MAX_SEGMENTS ? (uint32_t)NS_MAX_SEGMENTS : (uint32_t)v);
    }
    n_seg[i] = k;
    n_pieces[i] = 2 * k - 1;
}
