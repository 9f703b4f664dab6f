// Unaligned reads (simulation_unaligned, /root/reference/src/simulator.py:1482-1549), one WARP per read.
//
// unaligned_error_list (:1784-1830) draws an i.i.d. step per loop iteration (type with fixed cdf 0.4/0.7/0.85/1,
// length from the mixed models), so -- unlike the Markov chain of aligned reads -- the walk can be evaluated 32
// draws at a time: lane j takes draw (base + j), a warp prefix sum over the reference advance gives every draw its
// position, the first non-insertion draw that reaches m_ref ends the read exactly where the sequential loop would,
// and consecutive insertions are folded into the following step with a ballot/shuffle.  Draw k uses Philox block
// k+1 of the attempt's stream, i.e. exactly the words the sequential state machine in plan_kernel.cuh consumes for
// its k-th loop iteration, so both paths produce the same read lengths, rejections, strands, positions and bytes
// (tests/test_gpu_parity.py::test_unaligned_fast_path_equals_scripted_path).
//
// Every lane writes the ops of its own draw into the read's edit script; emit_kernel turns the script into bases and
// "unmapped"-state qualities (:1521).  With mutate_read's right-to-left string edits (:1957-1995) a step of length s at
// `pos` preceded by `a` inserted bases (key ceil(pos + 0.1) = pos + 1) becomes
//     match : COPY 1, INS a
//     mis   : MIS 1,  INS a,           MIS rest, COPY covered
//     del   : DEL 1,  INS a - covered, DEL rest, COPY covered
// with covered = min(a, s - 1) and rest = s - 1 - covered (the substitution / deletion also hits the inserted bases
// that sit inside its span; re-randomised random bases stay uniform).  Empty ops are dropped, equal neighbours inside
// a draw are merged, and a run of plain matches becomes one COPY.
//
// Like plan_kernel, the first pass writes into a slot sized from the attempt-0 length (lengths_kernel) and flags the
// read when the script does not fit (or a later attempt was longer); flagged reads are replayed into exact slots.
#pragma once
#include "device_common.cuh"
#include "emit_kernel.cuh"
#include "plan_kernel.cuh"

struct UreadArgs {
    DevModel m;
    DevRef ref;
    DevCfg cfg;
    uint64_t first_id;
    uint32_t n_reads;
    NsReadMeta* reads;
    NsPieceMeta* pieces;     // [n_reads + 1]: op_off of piece i+1 bounds the slot of piece i (first pass)
    uint32_t* ops;
    const uint32_t* order;   // processing order (longest first), may be null
    uint32_t* counter;
    uint32_t* n_flagged;
    // slots for re-drawn reads (a rejected attempt draws a new length, :1503): bump-allocated behind the primary area
    unsigned long long* pool_cursor;
    const uint64_t* pool;    // {base, size} of the pool, in ops (device memory: written by capacity_stage_a)
    const uint32_t* abort;   // sync-free batches: non-zero = the script area is too small, do nothing (or null)
    uint32_t cta_min_len;    // reads whose first drawn length exceeds this are walked by a whole block (0: none, NS_FLAG_EMIT_WHOLE)
};

#define UREAD_WARPS 8

// unaligned_error_list (:1784-1830) + its effect in mutate_read for ONE read / chimeric gap of drawn length m_ref, evaluated by
// a whole warp 32 draws at a time (see the header comment).  Draw k uses Philox block k + 1 of stream `sw`.  Ops go to
// ops[0 .. cap) (counted beyond that).
// inclusive warp prefix sums of the reference advance (non-insertion steps) and of the inserted bases of 32 draws: one scan
// over both packed in a word when every step is short enough for the sums to fit 16 bits (always, with the shipped models)
__device__ __forceinline__ void scan_advance_and_insertions(bool nonins, uint32_t s, int lane, uint32_t& adv_incl, uint32_t& ins_incl) {
    if (__all_sync(0xffffffffu, s < 2048u)) {
        const uint32_t both = warp_incl_scan(nonins ? s : (s << 16), lane);
        adv_incl = both & 0xffffu;
        ins_incl = both >> 16;
    } else {
        adv_incl = warp_incl_scan(nonins ? s : 0u, lane);
        ins_incl = warp_incl_scan(nonins ? 0u : s, lane);
    }
}

struct UChain {
    uint32_t n_ops, middle_ref, n_draws;
    int64_t l_new;
};
__device__ __forceinline__ UChain unaligned_chain_warp(const DevModel& m, uint2 key, uint32_t id_lo, uint32_t id_hi, uint32_t sw,
                                                       uint32_t m_ref, uint32_t* ops, uint32_t cap, int lane) {
    const uint32_t lane_lt = (1u << lane) - 1u;
    uint32_t base = 0, pos_base = 0, carry_a = 0, middle_ref = m_ref, n_draws = 0, n_ops = 0;
    int64_t l_new = (int64_t)m_ref;
    bool done = false;
    // draw `d` of the attempt: its type and step length (independent of everything before it: the next 32 draws are
    // issued before the scans of the current 32, so that the Philox rounds and the table loads overlap the shuffles)
    auto draw = [&](uint32_t d, uint32_t& kd, uint32_t& sd) {
        const uint4 r = philox4x32_10(make_uint4(id_lo, id_hi, sw, d + 1u), key);
        kd = r.x < 1717986918u ? 0u : (r.x < 3006477107u ? 1u : (r.x < 3650722201u ? 2u : 3u));
        sd = 1;
        if (kd != 0) sd = alias_draw(m, kd == 1 ? 1u : (kd == 2 ? 2u : 3u), r.y);
    };
    uint32_t kind_next, s_next;
    draw(lane, kind_next, s_next);
    while (!done) {
        const uint32_t kind = kind_next, s = s_next;
        draw(base + 32u + lane, kind_next, s_next);
        const bool nonins = kind != 2;
        uint32_t Pl, I;
        scan_advance_and_insertions(nonins, s, lane, Pl, I);
        const uint32_t P = pos_base + Pl;
        const uint32_t stop_mask = __ballot_sync(0xffffffffu, nonins && P >= m_ref);
        const int jstop = stop_mask ? __ffs(stop_mask) - 1 : 32;
        const bool valid = lane <= jstop;
        const uint32_t nonins_mask = __ballot_sync(0xffffffffu, nonins);
        // inserted bases pending in front of a non-insertion draw = I - I(previous non-insertion draw)
        const uint32_t below = nonins_mask & lane_lt;
        const int pn = below ? 31 - __clz(below) : -1;
        const uint32_t I_pn = __shfl_sync(0xffffffffu, I, pn < 0 ? 0 : pn);
        const uint32_t a_ins = nonins ? (pn >= 0 ? I - I_pn : I + carry_a) : 0u;
        int32_t delta = 0;
        if (valid) delta = kind == 2 ? (int32_t)s : (kind == 3 ? -(int32_t)s : 0);
        delta = __reduce_add_sync(0xffffffffu, delta);
        l_new += delta;

        // ---- this draw's ops (at most four), empty ones dropped and equal neighbours merged
        uint32_t o0 = 0, o1 = 0, o2 = 0, o3 = 0;          // an empty op is the zero word (COPY of length 0)
        const bool emits = valid && nonins;
        // a run of plain matches (no pending insertion) is written once, by its first lane
        const uint32_t plain_mask = __ballot_sync(0xffffffffu, emits && kind == 0 && a_ins == 0);
        if (emits) {
            if (kind == 0) {
                if (a_ins == 0) {
                    if (!(lane > 0 && ((plain_mask >> (lane - 1)) & 1u))) {
                        const uint32_t run = __ffs(~(plain_mask >> lane)) - 1;       // consecutive set bits from `lane`
                        o0 = (NS_OP_COPY << 28) | (run == 0xffffffffu ? 32u - lane : run);
                    }
                } else {
                    o0 = (NS_OP_COPY << 28) | 1u;
                    o1 = (NS_OP_INS << 28) | a_ins;
                }
            } else {
                const uint32_t covered = a_ins < s - 1 ? a_ins : s - 1;
                const uint32_t rest = s - 1 - covered;
                const uint32_t T = kind == 1 ? NS_OP_MIS : NS_OP_DEL;
                const uint32_t n_ins = kind == 1 ? a_ins : a_ins - covered;
                if (n_ins == 0) {
                    o0 = (T << 28) | (1u + rest);
                } else {
                    o0 = (T << 28) | 1u;
                    o1 = (NS_OP_INS << 28) | n_ins;
                    if (rest) o2 = (T << 28) | rest;
                }
                if (covered) o3 = (NS_OP_COPY << 28) | covered;
            }
        }
        const uint32_t p1 = o0 ? 1u : 0u, p2 = p1 + (o1 ? 1u : 0u), p3 = p2 + (o2 ? 1u : 0u);
        const uint32_t cnt = p3 + (o3 ? 1u : 0u);
        const uint32_t incl = warp_incl_scan(cnt, lane);
        const uint32_t at = n_ops + incl - cnt;
        if (o0 && at < cap) ops[at] = o0;
        if (o1 && at + p1 < cap) ops[at + p1] = o1;
        if (o2 && at + p2 < cap) ops[at + p2] = o2;
        if (o3 && at + p3 < cap) ops[at + p3] = o3;
        n_ops += __shfl_sync(0xffffffffu, incl, 31);

        if (jstop < 32) {
            const uint32_t Pstop = __shfl_sync(0xffffffffu, P, jstop);
            if (Pstop > middle_ref) {                      // overrun extends the segment (:1826-1828)
                l_new += Pstop - middle_ref;
                middle_ref = Pstop;
            }
            n_draws = base + (uint32_t)jstop + 1u;
            done = true;
        } else {
            pos_base = __shfl_sync(0xffffffffu, P, 31);
            const uint32_t I31 = __shfl_sync(0xffffffffu, I, 31);
            if (nonins_mask) {
                const int last = 31 - __clz(nonins_mask);
                carry_a = I31 - __shfl_sync(0xffffffffu, I, last);
            } else {
                carry_a += I31;
            }
            base += 32;
        }
    }
    UChain c;
    c.n_ops = n_ops;
    c.middle_ref = middle_ref;
    c.n_draws = n_draws;
    c.l_new = l_new;
    return c;
}


// The same walk by a whole thread block: warp w takes draws base + 32 w .. + 31 of a round of 32 * UREAD_WARPS draws.  What a
// warp needs from the warps before it -- the reference advance (position of its first draw, for the stopping rule), the
// inserted bases still pending (they join its first non-insertion draw) and the number of ops -- travels through shared
// memory, two barriers per round.  Every warp treats its 32 draws exactly as unaligned_chain_warp treats one iteration, so
// both produce the same ops word for word; a 200 kb read takes 1/8 of the time.
struct UCtaShared {
    uint32_t A[2][UREAD_WARPS], I[2][UREAD_WARPS], non[2][UREAD_WARPS], trail[2][UREAD_WARPS];      // after the scans
    uint32_t stop[2][UREAD_WARPS], cnt[2][UREAD_WARPS], pstop[2][UREAD_WARPS];                      // after the ops
    int32_t delta[2][UREAD_WARPS];
    uint32_t bc32;
    unsigned long long bc64;
};
__device__ __forceinline__ UChain unaligned_chain_cta(const DevModel& m, uint2 key, uint32_t id_lo, uint32_t id_hi, uint32_t sw,
                                                      uint32_t m_ref, uint32_t* ops, uint32_t cap, UCtaShared& sh) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const uint32_t lane_lt = (1u << lane) - 1u;
    uint32_t base = 0, pos_base = 0, carry_round = 0, middle_ref = m_ref, n_draws = 0, n_ops = 0;
    int64_t l_new = (int64_t)m_ref;
    auto draw = [&](uint32_t d, uint32_t& kd, uint32_t& sd) {
        const uint4 r = philox4x32_10(make_uint4(id_lo, id_hi, sw, d + 1u), key);
        kd = r.x < 1717986918u ? 0u : (r.x < 3006477107u ? 1u : (r.x < 3650722201u ? 2u : 3u));
        sd = 1;
        if (kd != 0) sd = alias_draw(m, kd == 1 ? 1u : (kd == 2 ? 2u : 3u), r.y);
    };
    uint32_t kind_next, s_next;
    draw(32u * (uint32_t)w + lane, kind_next, s_next);
    for (uint32_t par = 0;; par ^= 1u) {
        const uint32_t kind = kind_next, s = s_next;
        draw(base + 32u * UREAD_WARPS + 32u * (uint32_t)w + lane, kind_next, s_next);
        const bool nonins = kind != 2;
        uint32_t Pl, I;
        scan_advance_and_insertions(nonins, s, lane, Pl, I);
        const uint32_t nonins_mask = __ballot_sync(0xffffffffu, nonins);
        const uint32_t P31 = __shfl_sync(0xffffffffu, Pl, 31), I31 = __shfl_sync(0xffffffffu, I, 31);
        const uint32_t I_last = __shfl_sync(0xffffffffu, I, nonins_mask ? 31 - __clz(nonins_mask) : 0);
        if (lane == 0) {
            sh.A[par][w] = P31;
            sh.I[par][w] = I31;
            sh.non[par][w] = nonins_mask != 0u;
            sh.trail[par][w] = nonins_mask ? I31 - I_last : I31;
        }
        __syncthreads();
        uint32_t pos_off = 0, carry_in = carry_round, A_tot = 0, carry_out = carry_round;
#pragma unroll
        for (int v = 0; v < UREAD_WARPS; ++v) {
            const uint32_t Av = sh.A[par][v];
            const uint32_t c = sh.non[par][v] ? sh.trail[par][v] : carry_out + sh.I[par][v];
            if (v < w) {
                pos_off += Av;
                carry_in = c;
            }
            carry_out = c;
            A_tot += Av;
        }
        const uint32_t P = pos_base + pos_off + Pl;
        const uint32_t stop_mask = __ballot_sync(0xffffffffu, nonins && P >= m_ref);
        const int jstop = stop_mask ? __ffs(stop_mask) - 1 : 32;
        const bool valid = lane <= jstop;
        // inserted bases pending in front of a non-insertion draw = I - I(previous non-insertion draw)
        const uint32_t below = nonins_mask & lane_lt;
        const int pn = below ? 31 - __clz(below) : -1;
        const uint32_t I_pn = __shfl_sync(0xffffffffu, I, pn < 0 ? 0 : pn);
        const uint32_t a_ins = nonins ? (pn >= 0 ? I - I_pn : I + carry_in) : 0u;
        int32_t delta = 0;
        if (valid) delta = kind == 2 ? (int32_t)s : (kind == 3 ? -(int32_t)s : 0);
        delta = __reduce_add_sync(0xffffffffu, delta);

        // ---- this draw's ops (at most four), exactly as in unaligned_chain_warp
        uint32_t o0 = 0, o1 = 0, o2 = 0, o3 = 0;
        const bool emits = valid && nonins;
        const uint32_t plain_mask = __ballot_sync(0xffffffffu, emits && kind == 0 && a_ins == 0);
        if (emits) {
            if (kind == 0) {
                if (a_ins == 0) {
                    if (!(lane > 0 && ((plain_mask >> (lane - 1)) & 1u))) {
                        const uint32_t run = __ffs(~(plain_mask >> lane)) - 1;
                        o0 = (NS_OP_COPY << 28) | (run == 0xffffffffu ? 32u - lane : run);
                    }
                } else {
                    o0 = (NS_OP_COPY << 28) | 1u;
                    o1 = (NS_OP_INS << 28) | a_ins;
                }
            } else {
                const uint32_t covered = a_ins < s - 1 ? a_ins : s - 1;
                const uint32_t rest = s - 1 - covered;
                const uint32_t T = kind == 1 ? NS_OP_MIS : NS_OP_DEL;
                const uint32_t n_ins = kind == 1 ? a_ins : a_ins - covered;
                if (n_ins == 0) {
                    o0 = (T << 28) | (1u + rest);
                } else {
                    o0 = (T << 28) | 1u;
                    o1 = (NS_OP_INS << 28) | n_ins;
                    if (rest) o2 = (T << 28) | rest;
                }
                if (covered) o3 = (NS_OP_COPY << 28) | covered;
            }
        }
        const uint32_t p1 = o0 ? 1u : 0u, p2 = p1 + (o1 ? 1u : 0u), p3 = p2 + (o2 ? 1u : 0u);
        const uint32_t cnt = p3 + (o3 ? 1u : 0u);
        const uint32_t incl = warp_incl_scan(cnt, lane);
        const uint32_t cnt_w = __shfl_sync(0xffffffffu, incl, 31);
        const uint32_t Pstop_w = __shfl_sync(0xffffffffu, P, jstop & 31);
        if (lane == 0) {
            sh.stop[par][w] = (uint32_t)jstop;
            sh.cnt[par][w] = cnt_w;
            sh.delta[par][w] = delta;
            sh.pstop[par][w] = Pstop_w;
        }
        __syncthreads();
        int ws = UREAD_WARPS;                                // first warp of the round that holds the stopping draw
#pragma unroll
        for (int v = UREAD_WARPS - 1; v >= 0; --v)
            if (sh.stop[par][v] < 32u) ws = v;
        uint32_t off = 0, tot = 0;
        int32_t dsum = 0;
#pragma unroll
        for (int v = 0; v < UREAD_WARPS; ++v) {
            if (v <= ws) {
                const uint32_t c = sh.cnt[par][v];
                if (v < w) off += c;
                tot += c;
                dsum += sh.delta[par][v];
            }
        }
        if (w <= ws) {
            const uint32_t at = n_ops + off + incl - cnt;
            if (o0 && at < cap) ops[at] = o0;
            if (o1 && at + p1 < cap) ops[at + p1] = o1;
            if (o2 && at + p2 < cap) ops[at + p2] = o2;
            if (o3 && at + p3 < cap) ops[at + p3] = o3;
        }
        n_ops += tot;
        l_new += dsum;
        if (ws < UREAD_WARPS) {
            const uint32_t Pstop = sh.pstop[par][ws];
            if (Pstop > middle_ref) {                      // overrun extends the segment (:1826-1828)
                l_new += Pstop - middle_ref;
                middle_ref = Pstop;
            }
            n_draws = base + 32u * (uint32_t)ws + sh.stop[par][ws] + 1u;
            break;
        }
        pos_base += A_tot;
        carry_round = carry_out;
        base += 32u * UREAD_WARPS;
    }
    UChain c;
    c.n_ops = n_ops;
    c.middle_ref = middle_ref;
    c.n_draws = n_draws;
    c.l_new = l_new;
    return c;
}

// reads whose first drawn length exceeds this are walked by a whole block, the rest by one warp each: a block covers 256
// draws per round but pays two barriers for it, so per draw it is slower than eight independent warps
#define UREAD_CTA_MIN_LEN 32768u

// One read (its rejection loop :1503, :1517), by one warp (CTA = false) or by the whole block (CTA = true); every thread runs
// it redundantly on uniform values.  Returns the length drawn for attempt 0.
template <bool REPLAY, bool CTA>
__device__ __forceinline__ uint32_t uread_one(const UreadArgs& a, uint2 key, uint32_t slot, uint64_t pool_base, uint64_t pool_size,
                                              UCtaShared& sh) {
    const DevModel& m = a.m;
    const DevCfg& cfg = a.cfg;
    const int lane = threadIdx.x & 31;
    const bool leader = CTA ? threadIdx.x == 0 : lane == 0;
    const uint64_t rid = a.first_id + slot;
    const uint32_t id_lo = (uint32_t)rid, id_hi = (uint32_t)(rid >> 32);
    uint32_t attempt = REPLAY ? a.reads[slot].attempts : 0u;
    uint64_t op_off = a.pieces[slot].op_off;
    uint32_t* ops = a.ops + op_off;
    // first pass: the slot ends where the next piece's begins; replay: exact slot
    uint32_t cap = REPLAY ? 0xffffffffu : (uint32_t)(a.pieces[slot + 1].op_off - op_off);
    uint32_t first_len = 0;
    for (;;) {
        const uint32_t sw = stream_word(ST_ATT, NS_KIND_UNALIGNED, attempt);
        Rng r0;
        r0.init(cfg.seed, rid, sw);
        // block 0 of the attempt's stream; -med/-sd: np.random.lognormal(log(median), sd) (:1494-1495)
        const double x = cfg.median_len > 0.0 ? lognormal_draw(log(cfg.median_len), cfg.sd_len, r0)
                                              : kde_draw(m.unaligned, r0);
        const int64_t mr = (int64_t)x;
        if (attempt == 0) first_len = mr > 0 ? (uint32_t)mr : 0u;
        if (mr <= 0) {                                       // middle_ref < min_l (:1503)
            ++attempt;
            continue;
        }
        const uint32_t m_ref = (uint32_t)mr;
        if (!REPLAY && attempt > 0) {                        // the slot was sized for attempt 0: take a new one
            const uint32_t need = m_ref + (m_ref >> 1) + 64u;
            unsigned long long off = 0;
            if (leader) off = atomicAdd(a.pool_cursor, (unsigned long long)need);
            if (CTA) {
                if (leader) sh.bc64 = off;
                __syncthreads();
                off = sh.bc64;
                __syncthreads();
            } else {
                off = __shfl_sync(0xffffffffu, off, 0);
            }
            if (off + need <= pool_size) {
                op_off = pool_base + off;
                cap = need;
            } else {
                cap = 0;                                     // pool exhausted: count only, replay later
            }
            ops = a.ops + op_off;
        }
        const UChain ch = CTA ? unaligned_chain_cta(m, key, id_lo, id_hi, sw, m_ref, ops, cap, sh)
                              : unaligned_chain_warp(m, key, id_lo, id_hi, sw, m_ref, ops, cap, lane);
        const uint32_t middle_ref = ch.middle_ref, n_draws = ch.n_draws, n_ops = ch.n_ops;
        const int64_t l_new = ch.l_new;
        if (REPLAY) break;
        const bool ok = middle_ref >= cfg.min_len && middle_ref <= cfg.max_len && l_new >= (int64_t)cfg.min_len &&
                        l_new <= (int64_t)cfg.max_len;
        if (!ok) {
            ++attempt;
            continue;
        }
        // accepted: strand from the next block of the attempt stream (:1526-1527), position (extract_read)
        const uint4 rs = philox4x32_10(make_uint4(id_lo, id_hi, sw, n_draws + 1u), key);
        const uint32_t reversed = u01_double(((uint64_t)rs.x << 32) | rs.y) > (double)m.strandness;
        Rng pr;
        pr.init(cfg.seed, rid, stream_word(ST_POS, NS_KIND_UNALIGNED, attempt));
        uint32_t chrom = 0, ppos = 0;
        if (cfg.metagenome) draw_position_meta(a.ref, pr, -1, middle_ref, chrom, ppos);
        else if (cfg.transcriptome) draw_position_trx(a.ref, cfg.trx_records ? cfg.trx_records : a.ref.n_chrom, pr, middle_ref, chrom, ppos);
        else draw_position(a.ref, cfg, pr, middle_ref, chrom, ppos);
        if (leader) {
            const bool overflow = n_ops > cap;
            NsPieceMeta p;
            p.op_off = op_off;
            p.n_ops = n_ops;
            p.kind = NS_PIECE_UNALIGNED;
            p.chrom = chrom;
            p.pos = ppos;
            p.ref_len = middle_ref;
            p.out_len = (uint32_t)l_new;
            p.out_rel = 0;
            p.l_new = (uint32_t)l_new;
            p.ref_req = m_ref;
            p.read_slot = slot;
            p.ev_off = op_off;
            p.ev_n_ops = n_ops;
            p.polya_len = 0;
            a.pieces[slot] = p;
            NsReadMeta q;
            q.seq_off = 0;
            q.seq_len = (uint32_t)l_new;
            q.head = 0;
            q.tail = 0;
            q.piece_first = slot;
            q.n_pieces = 1;
            q.reversed = (uint8_t)reversed;
            q.flags = overflow ? 1 : 0;
            q.attempts = attempt;
            a.reads[slot] = q;
            if (overflow) atomicAdd(a.n_flagged, 1u);
        }
        break;
    }
    return first_len;
}

#ifndef UREAD_MIN_BLOCKS
#define UREAD_MIN_BLOCKS 3          // 80 registers: 24 warps per SM to hide the shuffle chains (not re-measured on H100)
#endif
template <bool REPLAY>
__global__ void __launch_bounds__(UREAD_WARPS * 32, UREAD_MIN_BLOCKS) uread_kernel(const __grid_constant__ UreadArgs a) {
    const int lane = threadIdx.x & 31;
    const uint2 key = make_uint2((uint32_t)a.cfg.seed, (uint32_t)(a.cfg.seed >> 32));
    if (a.abort && *a.abort) return;
    const uint64_t pool_base = a.pool[0], pool_size = a.pool[1];
    __shared__ UCtaShared sh;

    // ---- the long reads come first in `order`: the whole block walks them, one at a time, until it meets a short one
    if (!REPLAY && a.order && a.cta_min_len) {
        for (;;) {
            if (threadIdx.x == 0) sh.bc32 = atomicAdd(a.counter, 1u);
            __syncthreads();
            const uint32_t idx = sh.bc32;
            __syncthreads();
            if (idx >= a.n_reads) return;
            const uint32_t first_len = uread_one<REPLAY, true>(a, key, a.order[idx], pool_base, pool_size, sh);
            if (first_len <= a.cta_min_len) break;
        }
    }
    // ---- one warp per read
    for (;;) {
        uint32_t idx = 0;
        if (lane == 0) idx = atomicAdd(a.counter, 1u);
        idx = __shfl_sync(0xffffffffu, idx, 0);
        if (idx >= a.n_reads) break;
        const uint32_t slot = a.order ? a.order[idx] : idx;
        if (REPLAY && !(a.reads[slot].flags & 1u)) continue;
        uread_one<REPLAY, false>(a, key, slot, pool_base, pool_size, sh);
    }
}

// Chimeric gaps (simulation_gap :1552-1568: "an unaligned read of gap_len") of the first attempt of every read, one WARP per
// read, before the plan kernel: the same 32-draws-at-a-time evaluation, so that a 50 kb gap is not 50 000 iterations of ONE
// lane of the plan kernel's state machine.  Stream ST_GAP keyed by (attempt 0, piece): the plan kernel's own sequential gap
// walk (later attempts, replays) draws from the same stream, block k + 1 for draw k, and gets the same lengths.
// Results travel in the gap's piece record: n_ops, ref_len (middle_ref), out_len = l_new, polya_len = 1 as "precomputed" mark.
struct GapArgs {
    DevModel m;
    DevCfg cfg;
    uint32_t kind;
    uint64_t first_id;
    uint32_t n_reads;
    const uint32_t* n_seg;
    const uint32_t* piece_first;
    NsPieceMeta* pieces;
    uint32_t* ops;
    uint32_t* counter;
    const uint32_t* abort;
};
__device__ __forceinline__ uint32_t gap_stream_word(uint32_t kind, uint32_t attempt, uint32_t piece_in_read) {
    return stream_word(ST_GAP, kind, (attempt << 5) | (piece_in_read & 31u));
}
__global__ void __launch_bounds__(UREAD_WARPS * 32) gap_kernel(const __grid_constant__ GapArgs a) {
    const int lane = threadIdx.x & 31;
    const uint2 key = make_uint2((uint32_t)a.cfg.seed, (uint32_t)(a.cfg.seed >> 32));
    if (a.abort && *a.abort) return;
    for (;;) {
        uint32_t slot = 0;
        if (lane == 0) slot = atomicAdd(a.counter, 1u);
        slot = __shfl_sync(0xffffffffu, slot, 0);
        if (slot >= a.n_reads) break;
        const uint32_t ns = a.n_seg[slot];
        if (ns < 2) continue;
        const uint32_t pf = a.piece_first[slot];
        const uint64_t rid = a.first_id + slot;
        for (uint32_t q = 1; q < 2 * ns - 1; q += 2) {
            NsPieceMeta& pm = a.pieces[pf + q];
            const uint32_t m_ref = pm.ref_req;
            if (m_ref == 0) continue;                                  // nothing to walk (plan handles it)
            const uint64_t op_off = pm.op_off;
            const uint32_t cap = (uint32_t)(a.pieces[pf + q + 1].op_off - op_off);
            const UChain ch = unaligned_chain_warp(a.m, key, (uint32_t)rid, (uint32_t)(rid >> 32), gap_stream_word(a.kind, 0, q), m_ref,
                                                   a.ops + op_off, cap, lane);
            if (lane == 0) {
                pm.n_ops = ch.n_ops;
                pm.ref_len = ch.middle_ref;
                pm.out_len = (uint32_t)(ch.l_new < 0 ? 0 : ch.l_new);
                pm.l_new = pm.out_len;
                pm.polya_len = 1;
            }
        }
    }
}
