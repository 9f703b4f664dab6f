// Homopolymer pass (-hp -k K): the K-dependent half of mutate_read (/root/reference/src/simulator.py:1920-1947)
// and mutate_homo (:618-705) with its length model (model_homopolymer_lengths.py:167-186, 204-209, 246-260),
// as a rewrite of each aligned segment's edit script.  One LANE walks one segment:
//
//  1. error filter: an error event whose interval touches a homopolymer run (>= K equal bases) of the UNMUTATED,
//     case-converted segment is dropped -- [pos, pos+n) for mis/del, (pos-0.5, pos-0.5+n) for ins, i.e. reference
//     positions pos-1 .. pos+n-1 (:1929-1947).  Dropped events turn into copies in the EVENT script (what the reference
//     logs in <out>_aligned_error_profile is the filtered list).
//  2. mutate_homo: the walker streams the mutated segment base by base (copied reference bases, substituted and
//     inserted bases -- whose values are fixed here and carried to the emit kernel as literal ops), finds runs >= K,
//     draws the new run length round(max(0, N(mu(L), sigma(L)))) and emits the run as literals: a contraction keeps
//     the qualities of the LAST bases of the run (:688-690), an expansion appends "ins"-state qualities (:692-695),
//     each new base is substituted with probability hp_mis_rate and only the first substitution gets a "mis" quality
//     (:671-682, :697-700).
//
// The rewritten script uses COPY / DEL (reference skip) / LIT / HT ops only; the emit kernel needs no random draws for
// its bases.  COUNT pass: new op count and output length per piece; WRITE pass: the scripts.
//
// Reads are taken longest first (the plan kernel's order), so the lanes of a warp walk segments of similar length.
// A segment whose reference span holds plain a/c/g/t only (DevRef::exc_pre) is walked on the 2-bit copy of the reference:
//   * copied stretches 16 bases per step: equal-neighbour bits of the packed word tell whether any run of >= K equal bases
//     can start, end or continue inside it; if not -- the usual case -- the word is accounted for with a handful of integer
//     operations (leading bases join the pending run, the middle becomes a COPY, the trailing run becomes the pending run);
//     otherwise its 16 bases go through the base-by-base path;
//   * the error filter reads the 32 reference bases around a position as one 64-bit word and counts the equal neighbours
//     of the centre base with two count-leading/trailing-zeros.
// NS_FLAG_EMIT_EXACT switches both shortcuts off (tests: identical scripts either way).
//
// CHAIN = true (ns_reemit on a -hp context, intron retention): a read laid out on the genome is a chain of pieces -- a
// segment and the NS_PIECE_CONT pieces that continue it, two apart (zero-op gap pieces in between) -- that the reference
// mutates as ONE sequence (simulator.py:1156-1183).  A lane walks the whole chain as one segment:
//   * chain offset x lies in piece j at offset x'; on a forward piece the base is converted_ref_base(byte[pos + x'], piece j,
//     x'), on an NS_PIECE_REF_REV piece the complement of converted_ref_base(byte[pos + ref_len-1-x'], piece j,
//     ref_len-1-x') -- the keys the emit kernel resolves IUPAC bytes with;
//   * the pending run and the filter window (in_hp) cross piece boundaries; runs of a chain draw ST_HP with the chain's
//     FIRST piece and a run counter over the whole chain, substituted / inserted bases ST_EMIT_B with (piece, op index in
//     that piece's event script) as everywhere else (the error-profile formatters recompute them that way);
//   * output stays per piece: ops that consume reference stay with the piece whose reference they consume.  A boundary
//     crossed while a run is pending becomes a marker (kind 4) in the run's part list; when the run is closed, a marker
//     closes the current piece's script and opens the next one's.  A rewritten run puts its literals into the piece where
//     it starts and splits its reference skip at the markers (LIT consumes no reference, DEL no output: every piece
//     stays consistent with its ref_len and out_len).
// Chains always take the byte-exact route.  The chain code is compiled into the CHAIN instantiations only: the ones
// ns_simulate launches keep their registers (DESIGN.md §3: this kernel is bound by its instruction cache).
#pragma once
#include "device_common.cuh"

struct HpArgs {
    DevRef ref;
    DevCfg cfg;
    uint64_t first_id;
    const NsReadMeta* reads;
    NsPieceMeta* pieces;
    uint32_t n_pieces;
    uint32_t* ops;              // event scripts (in place: dropped events) and rewritten scripts
    uint64_t* out_n_ops;        // COUNT: per piece
    const uint64_t* out_off;    // WRITE: per piece offsets of the rewritten scripts (already includes the base)
    double hp[2][6];            // rows AT, CG: const, alpha1, beta1, breakpoint1, intercept, slope
    double hp_mis_rate;
    uint32_t* counter;
    const uint32_t* order;      // pieces, longest reference span first (nullptr: identity); CHAIN: the chains' first pieces
    uint32_t force_exact;       // NS_FLAG_EMIT_EXACT: no packed-word shortcuts
    uint32_t piece_base;        // CHAIN: out_n_ops / out_off are indexed by piece - piece_base
};

#define HP_MAX_SEG 12

template <bool WRITE>
struct ScriptOut {
    uint32_t* base;
    uint32_t n, pend, out_len;      // pend = pending op word (0xffffffff = none); same-kind ops are merged
    __device__ __forceinline__ void begin(uint32_t* b) {
        base = b;
        n = 0;
        pend = 0xffffffffu;
        out_len = 0;
    }
    __device__ __forceinline__ void flush() {
        if (pend != 0xffffffffu) {
            if (WRITE) base[n] = pend;
            ++n;
        }
        pend = 0xffffffffu;
    }
    // kind word: type<<28 (| base<<26 | state<<24 for LIT); len added to the pending op when the kind matches
    __device__ __forceinline__ void add(uint32_t kind, uint32_t len) {
        if (len == 0) return;
        if ((kind >> 28) != NS_OP_DEL) out_len += len;
        const uint32_t mask = (kind >> 28) == NS_OP_LIT ? 0xff000000u : 0xf0000000u;
        if (pend != 0xffffffffu && (pend & mask) == kind) {
            pend += len;
            return;
        }
        flush();
        pend = kind | len;
    }
};

template <bool CHAIN>
struct HpWalker {
    const uint8_t* cb;
    uint64_t clen, seed, rid;
    uint32_t pos, piece_in_read, ref_len, K;
    // ---- CHAIN: the pieces chain[2j]; the cursor stands on piece c_j, which holds chain offsets [c_lo, c_lo + c_len)
    const NsPieceMeta* chain;
    const uint8_t* bases;
    const uint64_t* chrom_off;
    const uint8_t* c_cb;
    uint32_t head_pir, c_j, c_lo, c_len, c_pos, c_rev;
    __device__ __forceinline__ void load_piece() {
        const NsPieceMeta& p = chain[2u * c_j];
        c_len = p.ref_len;
        c_pos = p.pos;
        c_rev = (p.kind & NS_PIECE_REF_REV) != 0;
        c_cb = bases + chrom_off[p.chrom];
    }
    __device__ __forceinline__ uint32_t chain_base_at(uint32_t x) {
        while (x < c_lo) {
            --c_j;
            load_piece();
            c_lo -= c_len;
        }
        while (x >= c_lo + c_len) {
            c_lo += c_len;
            ++c_j;
            load_piece();
        }
        const uint32_t f = c_rev ? c_lo + c_len - 1u - x : x - c_lo;      // forward offset in the piece (emit_kernel's key)
        const uint32_t c = converted_ref_base(__ldg(&c_cb[c_pos + f]), seed, rid, head_pir + 2u * c_j, f);
        return acgt_fast(c) ? (base_idx(c) ^ (c_rev ? 2u : 0u)) : (4u + (c & 3u));
    }
    __device__ __forceinline__ uint32_t base_at(uint32_t x) {           // case-converted reference base index at offset x
        if (CHAIN) return chain_base_at(x);
        uint64_t ab = (uint64_t)pos + x;
        if (ab >= clen) ab -= clen;
        uint32_t c = converted_ref_base(__ldg(&cb[ab]), seed, rid, piece_in_read, x);
        return acgt_fast(c) ? base_idx(c) : (4u + (c & 3u));            // non-ACGT leftovers never form ACGT runs
    }
    // ---- 2-bit copy of the reference (only used when the segment's packed words hold no exception and it does not wrap)
    const uint32_t* pk;       // first packed word of the chromosome
    bool packed;
    // 16 bases from segment offset x: base x + j in bits [2j+1:2j]
    __device__ __forceinline__ uint32_t bases16(uint32_t x) const {
        const uint32_t l = pos + x;
        const uint32_t* q = pk + (l >> 4);
        return __funnelshift_r(__ldg(q), __ldg(q + 1), (l + l) & 30u);
    }
    // in_hp on the packed copy (K <= 16): the 32 bases x-15 .. x+16 as 64 bits, fields outside [0, ref_len) and fields that
    // differ from the centre base marked; the run through x = 1 + equal neighbours on either side
    __device__ __forceinline__ bool in_hp_packed(int64_t x) const {
        if (x < 0 || x >= (int64_t)ref_len) return false;
        const uint32_t L = pos + (uint32_t)x + 1u;                         // window starts at base L - 16 (>= -15: guard word)
        const uint32_t* q = pk + (L >> 4) - 1;
        const uint32_t w0 = __ldg(q), w1 = __ldg(q + 1), w2 = __ldg(q + 2), sh = (L + L) & 30u;
        const uint64_t W = ((uint64_t)__funnelshift_r(w1, w2, sh) << 32) | __funnelshift_r(w0, w1, sh);
        const uint64_t c = (W >> 30) & 3u;                                 // centre = field 15
        const uint64_t d = W ^ (c * 0x5555555555555555ull);
        uint64_t ne = (d | (d >> 1)) & 0x5555555555555555ull;             // bit 2j: field j differs from the centre
        const uint32_t jlo = x < 15 ? 15u - (uint32_t)x : 0u;              // fields below jlo lie before the segment
        const uint64_t room = (uint64_t)ref_len - (uint64_t)x + 15u;       // fields from here on lie behind it
        if (jlo) ne |= (1ull << (2u * jlo)) - 1ull;
        if (room < 32u) ne |= ~((1ull << (2u * (uint32_t)room)) - 1ull);
        const uint32_t below = (uint32_t)ne & 0x3fffffffu, above = (uint32_t)(ne >> 32);     // fields 0..14 / 16..31
        const uint32_t right = above ? ((uint32_t)__ffs((int)above) - 1u) >> 1 : 16u;        // equal fields directly above 15
        return 1u + left_count(below) + right >= K;
    }
    __device__ __forceinline__ static uint32_t left_count(uint32_t below) {     // equal fields directly below field 15
        if (!below) return 15u;
        const uint32_t top = 31u - (uint32_t)__clz((int)below);               // bit 2j of the nearest differing field j
        return 14u - (top >> 1);
    }
    // is offset x inside a run of >= K equal bases of the unmutated segment?
    __device__ __forceinline__ bool in_hp(int64_t x) {
        if (packed) return in_hp_packed(x);
        if (x < 0 || x >= (int64_t)ref_len) return false;
        const uint32_t b = base_at((uint32_t)x);
        if (b > 3u) return false;
        uint32_t run = 1;
        for (int64_t y = x - 1; y >= 0 && run < K && base_at((uint32_t)y) == b; --y) ++run;
        for (int64_t y = x + 1; y < (int64_t)ref_len && run < K && base_at((uint32_t)y) == b; ++y) ++run;
        return run >= K;
    }
};

#ifndef HP_MIN_BLOCKS
#define HP_MIN_BLOCKS 4
#endif
template <bool WRITE, bool CHAIN = false>
__global__ void __launch_bounds__(128, HP_MIN_BLOCKS) hp_kernel(const __grid_constant__ HpArgs a) {
    const uint2 key = make_uint2((uint32_t)a.cfg.seed, (uint32_t)(a.cfg.seed >> 32));
    const uint32_t K = a.cfg.kmer_bias;
    // A lane walks one segment at a time, as a FLAT state machine.  One loop iteration = one micro-step of every lane: a
    // 16-base word of a copied stretch (ST_WORD, the common case), one base of a stretch that has to be looked at base by
    // base (ST_BASE: a word in which a run reaches K, substituted / inserted bases, the byte-exact route), one op of the
    // script (ST_OP), or the hand-over to the next segment (ST_FETCH).  Every micro-step is split into a part that looks at
    // its input (A), ONE shared place where the pending run is closed if the step asks for it (B: the only copy of
    // flush_run in the kernel -- it is by far the largest piece of code), and a part that applies the step (C).  Nested
    // per-lane loops left 2-5 of 32 lanes active and a kernel that mostly waited for its instruction cache.
    enum : int { ST_FETCH = 0, ST_OP = 1, ST_WORD = 2, ST_BASE = 3 };
    enum : int { SRC_WORD = 0, SRC_EXACT = 1, SRC_MIS = 2, SRC_INS = 3 };
    enum : int { P_NONE = 0, P_END, P_HT, P_LIT, P_COPY, P_DEL, P_BASES, P_SLOW, P_ALL, P_MID, P_NEXT };
    int st = ST_FETCH, bsrc = SRC_WORD;
    uint32_t this_piece = 0;
    NsReadMeta rm;
    NsPieceMeta* pmp = nullptr;
    uint64_t rid = 0;
    HpWalker<CHAIN> w = {};
    uint32_t out_piece = 0, chain_left = 0;                 // CHAIN: piece whose script is being written; pieces still to walk
    uint32_t* ev = nullptr;
    uint32_t n_ev = 0, k = 0, kk = 0, rpos = 0;
    uint32_t len = 0, t = 0, w16 = 0, cur = 0, n = 0;      // the stretch being walked: t of len done; cur / n = rest of its current word
    uint4 rblk = make_uint4(0, 0, 0, 0);                    // random block of the substituted / inserted bases being walked
    ScriptOut<WRITE> out;
    out.begin(nullptr);
    // ---- current run of equal bases in the mutated stream
    uint32_t run_base = 0xffu, run_len = 0, run_ref = 0, nseg = 0, n_runs = 0;
    uint32_t seg_kind[HP_MAX_SEG], seg_cnt[HP_MAX_SEG];     // in order: 0 copy, 1 mis, 2 ins, 3 deleted reference bases
                                                            // (CHAIN: 4 = piece boundary)
    // CHAIN: the script of piece out_piece is complete; the next piece's begins
    auto close_out = [&]() {
        out.flush();
        NsPieceMeta& pm = a.pieces[out_piece];
        if (!WRITE) {
            a.out_n_ops[out_piece - a.piece_base] = out.n;
            pm.out_len = out.out_len;
        } else {
            pm.op_off = a.out_off[out_piece - a.piece_base];
            pm.n_ops = out.n;
        }
    };
    auto next_out = [&]() {
        close_out();
        out_piece += 2;
        out.begin(WRITE ? a.ops + a.out_off[out_piece - a.piece_base] : nullptr);
    };

    auto flush_run = [&]() {
        if (run_len == 0) return;
        if (run_len >= K && run_base < 4u) {
            // new length ~ N(mu(L), sigma(L)), clipped at 0, Python round()
            const uint4 r = philox4x32_10(make_uint4((uint32_t)rid, (uint32_t)(rid >> 32), stream_word(ST_HP, 0, CHAIN ? w.head_pir : w.piece_in_read), n_runs), key);
            const uint32_t cls = (run_base == 0u || run_base == 2u) ? 0u : 1u;      // A,T -> "AT" ; C,G -> "CG"
            const double* p = a.hp[cls];
            const double L = (double)run_len;
            const double mu = p[0] + p[1] * L + p[2] * fmax(L - p[3], 0.0);
            const double sigma = p[4] + p[5] * L;
            const float z = sqrtf(-2.0f * logf(u01_open_low(r.x))) * cospif(2.0f * ((float)(r.y >> 8) * (1.0f / 16777216.0f)));
            double x = mu + sigma * (double)z;
            if (x < 0.0) x = 0.0;
            const uint32_t nn = (uint32_t)rint(x);
            // states of the new bases: last nn members (contraction) / all members + ins (expansion)
            uint32_t skip = run_len > nn ? run_len - nn : 0u;
            bool mis_q_used = false;
            Rng mr;
            if (a.hp_mis_rate > 0.0) mr.init(a.cfg.seed, rid, stream_word(ST_HP, 1, CHAIN ? w.head_pir : w.piece_in_read) ^ (n_runs << 4));
            uint32_t produced = 0;
            for (uint32_t s = 0; s <= nseg && produced < nn; ++s) {
                uint32_t cnt, state;
                if (s < nseg) {
                    if (seg_kind[s] == 3 || (CHAIN && seg_kind[s] == 4)) continue;     // deleted reference bases carry no quality
                    cnt = seg_cnt[s];
                    state = seg_kind[s] == 0 ? 2u : (seg_kind[s] == 1 ? 0u : 1u);
                    if (skip >= cnt) {
                        skip -= cnt;
                        continue;
                    }
                    cnt -= skip;
                    skip = 0;
                } else {
                    cnt = nn - produced;                  // expansion: inserted-base qualities (:692-695)
                    state = 1u;
                }
                if (cnt > nn - produced) cnt = nn - produced;
                if (a.hp_mis_rate > 0.0) {
                    for (uint32_t q = 0; q < cnt; ++q) {
                        const double pr = u01_double(mr.next64());
                        uint32_t b = run_base, sq = state;
                        if (pr > 0.0 && pr <= a.hp_mis_rate) {
                            b = (run_base + 1u + (mr.next() % 3u)) & 3u;
                            if (!mis_q_used) {
                                sq = 0u;
                                mis_q_used = true;
                            }
                        }
                        out.add((NS_OP_LIT << 28) | (b << 26) | (sq << 24), 1);
                    }
                } else {
                    out.add((NS_OP_LIT << 28) | (run_base << 26) | (state << 24), cnt);
                }
                produced += cnt;
            }
            if (!CHAIN) {
                out.add(NS_OP_DEL << 28, run_ref);        // the reference bases the run stood on
            } else {
                uint32_t skip_ref = 0;                    // ... each piece's share of them
                for (uint32_t s = 0; s < nseg; ++s) {
                    if (seg_kind[s] == 4) {
                        out.add(NS_OP_DEL << 28, skip_ref);
                        next_out();
                        skip_ref = 0;
                    } else if (seg_kind[s] != 2) {
                        skip_ref += seg_cnt[s];
                    }
                }
                out.add(NS_OP_DEL << 28, skip_ref);
            }
            ++n_runs;
        } else {
            for (uint32_t s = 0; s < nseg; ++s) {
                if (seg_kind[s] == 0) {
                    out.add(NS_OP_COPY << 28, seg_cnt[s]);
                } else if (seg_kind[s] == 3) {
                    out.add(NS_OP_DEL << 28, seg_cnt[s]);
                } else if (CHAIN && seg_kind[s] == 4) {
                    next_out();
                } else {
                    out.add((NS_OP_LIT << 28) | ((run_base & 3u) << 26) | ((seg_kind[s] == 1 ? 0u : 1u) << 24), seg_cnt[s]);
                    if (seg_kind[s] == 1) out.add(NS_OP_DEL << 28, seg_cnt[s]);
                }
            }
        }
        run_len = 0;
        run_ref = 0;
        nseg = 0;
        run_base = 0xffu;
    };
    auto add_seg = [&](uint32_t kind, uint32_t cnt) {     // cnt more bases of `kind` in the pending run
        if (nseg > 0 && seg_kind[nseg - 1] == kind) {
            seg_cnt[nseg - 1] += cnt;
        } else if (nseg < HP_MAX_SEG) {
            seg_kind[nseg] = kind;
            seg_cnt[nseg] = cnt;
            ++nseg;
        } else {
            seg_cnt[nseg - 1] += cnt;                          // pathological run: lump into the last segment
            if (kind != 2 && seg_kind[nseg - 1] == 2) seg_kind[nseg - 1] = kind;
        }
    };

    for (;;) {
        // ================= A: look at the micro-step's input; does the pending run have to be closed before it?
        int path = P_NONE;
        bool need_flush = false;
        uint32_t b = 0, bkind = 0;                          // ST_BASE: the base and its kind (0 copy, 1 mis, 2 ins)
        uint32_t ne = 0, lead = 0;                          // ST_WORD
        uint32_t op = 0, ty = 0;                            // ST_OP
        if (st == ST_WORD) {
            if (n == 0) {                                   // next word of the stretch (the one after it is requested now)
                n = len - t < 16u ? len - t : 16u;
                cur = w16;
                if (t + n < len) w16 = w.bases16(rpos + t + n);
            }
            // ne: bit 2j set iff base j differs from base j-1 (1 <= j < n)
            const uint32_t fields = (n == 16u ? 0xffffffffu : (1u << (2u * n)) - 1u) & 0x55555554u;   // fields 1 .. n-1
            const uint32_t d = cur ^ (cur << 2);
            ne = (d | (d >> 1)) & fields;
            // a run of >= K equal bases inside the word <=> K-1 consecutive "equal to the previous base" fields
            const uint32_t eq = ~ne & fields;
            uint32_t runs = eq;
            for (uint32_t j = 1; j + 1 < K; ++j) runs &= eq << (2u * j);
            // leading bases that continue the pending run
            lead = (run_len && (cur & 3u) == run_base) ? (ne ? ((uint32_t)__ffs((int)ne) - 1u) >> 1 : n) : 0u;
            if (runs || run_len + lead >= K) {
                path = P_SLOW;                              // a run reaches K here: base by base
            } else {
                if (lead) {
                    add_seg(0u, lead);
                    run_len += lead;
                    run_ref += lead;
                }
                path = lead == n ? P_ALL : P_MID;           // P_MID: the pending run ends inside this word, shorter than K
                need_flush = path == P_MID;
            }
        } else if (st == ST_BASE) {
            if (bsrc == SRC_WORD) {
                b = cur & 3u;
            } else if (bsrc == SRC_EXACT) {
                b = w.base_at(rpos + t);
            } else {
                if ((t & 15u) == 0) rblk = event_base_block(key, rid, w.piece_in_read, kk, t);
                const uint32_t r8 = event_byte(rblk, t);
                if (bsrc == SRC_MIS) {
                    b = event_base(r8, true, w.packed ? (w.bases16(rpos + t) & 3u) : w.base_at(rpos + t));
                    bkind = 1;
                } else {
                    b = event_base(r8, false, 0u);
                    bkind = 2;
                }
            }
            need_flush = b != run_base || b > 3u;
        } else if (st == ST_OP) {
            if (CHAIN && k >= n_ev && chain_left > 0) {     // end of a piece's script inside a chain
                path = P_NEXT;                              // no room for a boundary marker (pathological run): closed here
                need_flush = run_len != 0 && nseg >= HP_MAX_SEG - 1u;
            } else if (k >= n_ev) {                         // end of the segment's script
                path = P_END;
                need_flush = true;
            } else {
                op = ev[k];
                ty = op >> 28;
                len = op & 0x0fffffffu;
                kk = k++;
                if (ty == NS_OP_HT) {
                    path = P_HT;
                    need_flush = true;
                } else if (ty == NS_OP_LIT) {               // polyA tail (appended after mutate_homo, :1229-1230)
                    path = P_LIT;
                    need_flush = true;
                } else {
                    if (ty >= NS_OP_MIS && ty <= NS_OP_DEL && len > 0) {
                        // ---- error filter (:1929-1947)
                        const int64_t lo = ty == NS_OP_INS ? (int64_t)rpos - 1 : (int64_t)rpos;
                        const int64_t hi = (int64_t)rpos + (int64_t)len - 1;
                        bool drop = false;
                        for (int64_t x = lo; x <= hi && !drop; ++x) drop = w.in_hp(x);
                        if (drop) {
                            if (ty == NS_OP_INS) len = 0;
                            if (WRITE) ev[kk] = (NS_OP_COPY << 28) | len;
                            ty = NS_OP_COPY;
                        }
                    }
                    if (len == 0) {
                        path = P_NONE;
                    } else if (ty == NS_OP_COPY) {
                        path = P_COPY;
                    } else if (ty == NS_OP_DEL) {
                        path = P_DEL;                       // pathological run (no room for another part): closed here
                        need_flush = run_len != 0 && !(nseg > 0 && seg_kind[nseg - 1] == 3) && nseg >= HP_MAX_SEG;
                    } else {
                        path = P_BASES;
                    }
                }
            }
        }
        // ================= B
        if (need_flush) flush_run();
        // ================= C: apply the micro-step
        if (st == ST_WORD) {
            if (path == P_SLOW) {
                bsrc = SRC_WORD;
                st = ST_BASE;
            } else {
                if (path == P_MID) {
                    // the trailing run (bases equal to the last one) becomes the pending run, what lies between is copied
                    const uint32_t bound = ne | 1u;        // field 0 bounds the trailing run inside the word
                    const uint32_t trail = n - ((31u - (uint32_t)__clz((int)bound)) >> 1);
                    out.add(NS_OP_COPY << 28, n - lead - trail);
                    run_base = (cur >> (2u * (n - 1u))) & 3u;
                    run_len = run_ref = trail;
                    nseg = 1;
                    seg_kind[0] = 0;
                    seg_cnt[0] = trail;
                }
                t += n;
                n = 0;
                if (t >= len) {
                    rpos += len;
                    st = ST_OP;
                }
            }
        } else if (st == ST_BASE) {
            if (need_flush) run_base = b;
            ++run_len;
            if (bkind != 2) ++run_ref;
            add_seg(bkind, 1u);
            ++t;
            if (bsrc == SRC_WORD) {
                cur >>= 2;
                if (--n == 0) {
                    if (t >= len) {
                        rpos += len;
                        st = ST_OP;
                    } else {
                        st = ST_WORD;
                    }
                }
            } else if (t >= len) {
                if (bsrc != SRC_INS) rpos += len;
                st = ST_OP;
            }
        } else if (st == ST_OP) {
            if (path == P_END) {
                if (CHAIN) {
                    close_out();
                } else {
                    NsPieceMeta& pm = *pmp;
                    out.flush();
                    if (!WRITE) {
                        a.out_n_ops[this_piece] = out.n;
                        pm.out_len = out.out_len;
                    } else {
                        pm.op_off = a.out_off[this_piece];
                        pm.n_ops = out.n;
                    }
                }
                st = ST_FETCH;
            } else if (CHAIN && path == P_NEXT) {
                if (run_len == 0) {
                    next_out();
                } else {                                    // the pending run carries over: mark where the piece ends
                    seg_kind[nseg] = 4;
                    seg_cnt[nseg] = 0;
                    ++nseg;
                }
                this_piece += 2;
                --chain_left;
                const NsPieceMeta& pm = a.pieces[this_piece];
                w.piece_in_read = this_piece - rm.piece_first;
                ev = a.ops + pm.ev_off;
                n_ev = pm.ev_n_ops;
                k = 0;
            } else if (path == P_HT) {
                out.add(NS_OP_HT << 28, len);
            } else if (path == P_LIT) {
                out.add(op & 0xff000000u, op & 0x00ffffffu);
            } else if (path == P_COPY) {
                t = 0;
                if (w.packed) {
                    n = 0;
                    w16 = w.bases16(rpos);
                    st = ST_WORD;
                } else {
                    bsrc = SRC_EXACT;
                    st = ST_BASE;
                }
            } else if (path == P_DEL) {
                // deleted bases vanish from the read: their neighbours become adjacent and may join one run
                if (run_len == 0) {
                    out.add(NS_OP_DEL << 28, len);
                } else {
                    run_ref += len;
                    if (nseg > 0 && seg_kind[nseg - 1] == 3) {
                        seg_cnt[nseg - 1] += len;
                    } else {
                        seg_kind[nseg] = 3;
                        seg_cnt[nseg] = len;
                        ++nseg;
                    }
                }
                rpos += len;
            } else if (path == P_BASES) {
                t = 0;
                bsrc = ty == NS_OP_MIS ? SRC_MIS : SRC_INS;
                st = ST_BASE;
            }
        } else {
            // ---- next segment, longest first (a read's segments go to different lanes: a chimeric read of five 100 kb segments
            //      would otherwise keep one lane busy five times as long as any other)
            const uint32_t wi = atomicAdd(a.counter, 1u);
            if (wi >= a.n_pieces) break;
            if (CHAIN) {
                // ---- a chain: its first piece, then every NS_PIECE_CONT piece two further on
                this_piece = a.order[wi];
                const NsPieceMeta& pm = a.pieces[this_piece];
                rm = a.reads[pm.read_slot];
                rid = a.first_id + pm.read_slot;
                w.seed = a.cfg.seed;
                w.rid = rid;
                w.K = K;
                w.packed = false;
                w.piece_in_read = w.head_pir = this_piece - rm.piece_first;
                w.chain = &pm;
                w.bases = a.ref.bases;
                w.chrom_off = a.ref.chrom_off;
                w.c_j = 0;
                w.c_lo = 0;
                w.load_piece();
                uint32_t total = pm.ref_len;
                chain_left = 0;
                for (uint32_t q = w.head_pir + 2u; q < rm.n_pieces && (a.pieces[rm.piece_first + q].kind & NS_PIECE_CONT); q += 2u) {
                    total += a.pieces[rm.piece_first + q].ref_len;
                    ++chain_left;
                }
                w.ref_len = total;
                ev = a.ops + pm.ev_off;
                n_ev = pm.ev_n_ops;
                k = 0;
                rpos = 0;
                out_piece = this_piece;
                out.begin(WRITE ? a.ops + a.out_off[this_piece - a.piece_base] : nullptr);
                run_base = 0xffu;
                run_len = run_ref = nseg = n_runs = 0;
                st = ST_OP;
                continue;
            }
            this_piece = a.order ? a.order[wi] : wi;
            pmp = &a.pieces[this_piece];
            NsPieceMeta& pm = *pmp;
            if (NS_PIECE_KIND(pm.kind) != NS_PIECE_SEGMENT) {
                if (!WRITE) a.out_n_ops[this_piece] = 0;   // untouched pieces keep their script
                continue;
            }
            rm = a.reads[pm.read_slot];
            rid = a.first_id + pm.read_slot;
            const uint64_t cstart = a.ref.chrom_off[pm.chrom];
            w.cb = a.ref.bases + cstart;
            w.clen = a.ref.chrom_off[pm.chrom + 1] - cstart;
            w.seed = a.cfg.seed;
            w.rid = rid;
            w.pos = pm.pos;
            w.piece_in_read = this_piece - rm.piece_first;
            w.ref_len = pm.ref_len;
            w.K = K;
            {   // packed-word shortcuts: plain a/c/g/t span that stays inside the chromosome, K small enough for the 32-base window
                const uint64_t pk0 = a.ref.pk_off[pm.chrom];
                w.pk = a.ref.packed + pk0;
                bool ok = !a.force_exact && K <= 16u && pm.ref_len > 0 && (uint64_t)pm.pos + pm.ref_len <= w.clen;
                if (ok) {
                    const uint64_t w_lo = pk0 + (pm.pos >> 4), w_hi = pk0 + ((pm.pos + pm.ref_len - 1u) >> 4);
                    ok = __ldg(&a.ref.exc_pre[(w_hi >> REF_EXC_BLOCK_SHIFT) + 1]) == __ldg(&a.ref.exc_pre[w_lo >> REF_EXC_BLOCK_SHIFT]);
                }
                w.packed = ok;
            }
            ev = a.ops + pm.ev_off;
            n_ev = pm.ev_n_ops;
            k = 0;
            rpos = 0;
            out.begin(WRITE ? a.ops + a.out_off[this_piece] : nullptr);
            run_base = 0xffu;
            run_len = run_ref = nseg = n_runs = 0;
            st = ST_OP;
        }
    }
}

// after the COUNT pass: out_rel of every piece and the read length from the new piece lengths
__global__ void hp_fix_reads(NsReadMeta* reads, NsPieceMeta* pieces, uint32_t n) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    NsReadMeta& r = reads[i];
    uint32_t cur = 0;
    for (uint32_t q = 0; q < r.n_pieces; ++q) {
        NsPieceMeta& p = pieces[r.piece_first + q];
        p.out_rel = cur;
        cur += p.out_len;
    }
    r.seq_len = cur;
}
