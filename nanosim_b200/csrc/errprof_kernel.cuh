// Error-profile rows on the device (ns_compress_error_profile): the bytes host_io.cu:format_error_profile_impl writes for
// the last aligned batch (after ns_reemit as well), without the header line, laid out in HBM for
// bgzf_deflate_rows_kernel.  One warp per read.  A read's rows go per mutate_read call -- a segment plus the
// NS_PIECE_CONT pieces that continue it -- and within a call right to left, with Seq_pos counted across the call's
// pieces.  The rows come from the event scripts (ev_off / ev_n_ops), 32 ops at a time: warp scans give every op its
// reference and read offsets and every event its row's size and place; the lane of an event writes its row.
//   pass 1 (errprof_size_kernel): bytes of every read's rows; a scan of them gives the reads' offsets in the text
//   pass 2 (errprof_write_kernel): per call, its size (one walk over its ops), then its rows at their offsets
#pragma once

struct EpArgs {
    const NsReadMeta* reads;
    const NsPieceMeta* pieces;
    const uint32_t* ops;
    const uint8_t* seq;
    const uint8_t* ref;             // reference bytes as stored (case and IUPAC codes kept)
    const uint64_t* chrom_off;
    const char* names;              // NUL-terminated, at name_off[i]
    const uint64_t* name_off;
    uint32_t* name_len;             // pass 1 writes, pass 2 reads
    uint32_t n_reads;
    uint2 key;                      // the context's seed: bases of events the homopolymer pass rewrote
    uint64_t first_id;              // id of the batch's first read
    uint64_t* size;                 // pass 1: bytes of every read's rows
    const uint64_t* off;            // pass 2: their exclusive prefix sum
    uint8_t* text;
};

// one error event of a call, as a lane sees it
struct EpEvent {
    uint32_t k, j;                  // piece index in the read, op index in the piece's event script
    uint32_t ty, len;
    uint32_t rf, o;                 // offset in the piece's reference (direction of the read), offset in the forward read
    uint64_t shown;                 // Seq_pos
    uint64_t x, size;               // bytes of the call's earlier events (in script order), bytes of this row
};

__device__ __forceinline__ uint32_t ep_dec_len(uint64_t v) {
    uint32_t n = 1;
    while (v >= 10) {
        v /= 10;
        ++n;
    }
    return n;
}
__device__ __forceinline__ uint8_t ep_comp(uint8_t c) {
    return c == 'A' ? 'T' : c == 'T' ? 'A' : c == 'C' ? 'G' : c == 'G' ? 'C' : c;
}
template <class T>
__device__ __forceinline__ T ep_warp_incl(T v, uint32_t lane) {
#pragma unroll
    for (uint32_t d = 1; d < 32; d <<= 1) {
        const T u = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += u;
    }
    return v;
}

// The events of one call, pieces kb, kb + 2, ... < ke of read r: fn(event) on the lane that holds it.  Returns the bytes of
// the call's rows (the same on every lane).
template <class Fn>
__device__ uint64_t ep_walk_call(const EpArgs& a, const NsReadMeta& r, uint32_t nl, uint32_t kb, uint32_t ke, uint32_t lane, Fn fn) {
    uint64_t total = 0;
    uint32_t ref_base = 0;
    for (uint32_t k = kb; k < ke; k += 2) {
        const NsPieceMeta& pc = a.pieces[r.piece_first + k];
        if (NS_PIECE_KIND(pc.kind) != NS_PIECE_SEGMENT) continue;
        const uint32_t* sc = a.ops + pc.ev_off;
        const uint32_t n_ops = pc.ev_n_ops;
        uint32_t o = pc.out_rel, rf = 0;
        for (uint32_t j0 = 0; j0 < n_ops; j0 += 32) {
            const uint32_t j = j0 + lane;
            uint32_t ty = NS_OP_COPY, ln = 0;
            if (j < n_ops) {
                const uint32_t op = sc[j];
                ty = NS_OP_TYPE(op);
                ln = NS_OP_LEN(op);
            }
            const bool ev = ty >= NS_OP_MIS && ty <= NS_OP_DEL && ln;
            const uint32_t oa = ty != NS_OP_DEL ? ln : 0u;
            const uint32_t ra = (ty == NS_OP_COPY || ty == NS_OP_MIS || ty == NS_OP_DEL) ? ln : 0u;
            const uint32_t oi = ep_warp_incl(oa, lane), ri = ep_warp_incl(ra, lane);
            EpEvent e;
            e.k = k;
            e.j = j;
            e.ty = ty;
            e.len = ln;
            e.rf = rf + ri - ra;
            e.o = o + oi - oa;
            e.shown = (uint64_t)ref_base + e.rf;
            e.size = ev ? nl + 1 + ep_dec_len(e.shown) + 1 + 3 + 1 + ep_dec_len(ln) + 1 + (uint64_t)ln + 1 + ln + 1 : 0;
            const uint64_t si = ep_warp_incl(e.size, lane);
            e.x = total + si - e.size;
            if (ev) fn(e, pc);
            o += __shfl_sync(0xffffffffu, oi, 31);
            rf += __shfl_sync(0xffffffffu, ri, 31);
            total += __shfl_sync(0xffffffffu, si, 31);
        }
        ref_base += pc.ref_len;
    }
    return total;
}

// fn(kb, ke) for every call of read r, in order (a segment that does not continue the one before starts a call)
template <class Fn>
__device__ void ep_for_each_call(const EpArgs& a, const NsReadMeta& r, Fn fn) {
    uint32_t kb = 0xffffffffu;
    for (uint32_t k = 0; k < r.n_pieces; k += 2) {
        const uint32_t kind = a.pieces[r.piece_first + k].kind;
        if (NS_PIECE_KIND(kind) != NS_PIECE_SEGMENT) continue;
        if (!(kind & NS_PIECE_CONT)) {
            if (kb != 0xffffffffu) fn(kb, k);
            kb = k;
        } else if (kb == 0xffffffffu) {
            kb = k;
        }
    }
    if (kb != 0xffffffffu) fn(kb, (uint32_t)r.n_pieces);
}

__global__ void errprof_size_kernel(EpArgs a) {
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= a.n_reads) return;
    const NsReadMeta r = a.reads[w];
    uint32_t nl = 0;
    if (lane == 0) {
        const char* nm = a.names + a.name_off[w];
        while (nm[nl]) ++nl;
    }
    nl = __shfl_sync(0xffffffffu, nl, 0);
    uint64_t total = 0;
    ep_for_each_call(a, r, [&](uint32_t kb, uint32_t ke) {
        total += ep_walk_call(a, r, nl, kb, ke, lane, [](const EpEvent&, const NsPieceMeta&) {});
    });
    if (lane == 0) {
        a.name_len[w] = nl;
        a.size[w] = total;
    }
}

__device__ __forceinline__ uint8_t* ep_put_dec(uint8_t* p, uint64_t v) {
    const uint32_t n = ep_dec_len(v);
    for (uint32_t k = n; k-- > 0;) {
        p[k] = (uint8_t)('0' + v % 10);
        v /= 10;
    }
    return p + n;
}

// one row: name, Seq_pos, type, length, reference bases, read bases
__device__ void ep_write_row(const EpArgs& a, const NsReadMeta& r, uint32_t i, const char* nm, uint32_t nl, const EpEvent& e,
                             const NsPieceMeta& pc, uint8_t* p) {
    for (uint32_t t = 0; t < nl; ++t) *p++ = (uint8_t)nm[t];
    *p++ = '\t';
    p = ep_put_dec(p, e.shown);
    *p++ = '\t';
    const char* tn = e.ty == NS_OP_MIS ? "mis" : e.ty == NS_OP_INS ? "ins" : "del";
    *p++ = tn[0];
    *p++ = tn[1];
    *p++ = tn[2];
    *p++ = '\t';
    p = ep_put_dec(p, e.len);
    *p++ = '\t';
    const uint64_t cstart = a.chrom_off[pc.chrom], clen = a.chrom_off[pc.chrom + 1] - cstart;
    const bool back = (pc.kind & NS_PIECE_REF_REV) != 0;
    // reference base t of the event: upper case, complemented on a minus-strand piece, wrapping around the chromosome
    auto ref_char = [&](uint32_t t) -> uint8_t {
        const uint32_t f = e.rf + t;
        uint64_t ab = (uint64_t)pc.pos + (back ? pc.ref_len - 1 - f : f);
        if (ab >= clen) ab -= clen;
        uint8_t c = a.ref[cstart + ab];
        if (c >= 'a' && c <= 'z') c = (uint8_t)(c - 32);
        return back ? ep_comp(c) : c;
    };
    for (uint32_t t = 0; t < e.len; ++t) p[t] = e.ty == NS_OP_INS ? (uint8_t)'-' : ref_char(t);
    p += e.len;
    *p++ = '\t';
    if (e.ty == NS_OP_DEL) {
        for (uint32_t t = 0; t < e.len; ++t) p[t] = '-';
    } else if (pc.ev_off != pc.op_off) {                        // the homopolymer pass fixed this event's bases
        uint4 blk;
        const uint64_t rid = a.first_id + i;
        for (uint32_t t = 0; t < e.len; ++t) {
            if ((t & 15u) == 0) blk = event_base_block(a.key, rid, e.k, e.j, t);
            const uint8_t rc = e.ty == NS_OP_MIS ? ref_char(t) : (uint8_t)'-';
            const uint32_t orig = rc == 'C' ? 1u : (rc == 'T' ? 2u : (rc == 'G' ? 3u : 0u));
            p[t] = (uint8_t)"ACTG"[event_base(event_byte(blk, t), e.ty == NS_OP_MIS, orig)];
        }
    } else {
        const uint8_t* rs = a.seq + r.seq_off;
        const uint32_t L = r.seq_len;
        for (uint32_t t = 0; t < e.len; ++t) {
            const uint32_t x = e.o + t;
            p[t] = r.reversed ? ep_comp(rs[L - 1 - x]) : rs[x];
        }
    }
    p += e.len;
    *p = '\n';
}

__global__ void errprof_write_kernel(EpArgs a) {
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= a.n_reads) return;
    const NsReadMeta r = a.reads[w];
    const uint32_t nl = a.name_len[w];
    const char* nm = a.names + a.name_off[w];
    uint8_t* base = a.text + a.off[w];
    ep_for_each_call(a, r, [&](uint32_t kb, uint32_t ke) {
        const uint64_t call = ep_walk_call(a, r, nl, kb, ke, lane, [](const EpEvent&, const NsPieceMeta&) {});
        // right to left: the rows of the events after this one come first
        ep_walk_call(a, r, nl, kb, ke, lane, [&](const EpEvent& e, const NsPieceMeta& pc) {
            ep_write_row(a, r, w, nm, nl, e, pc, base + call - e.x - e.size);
        });
        base += call;
    });
}
