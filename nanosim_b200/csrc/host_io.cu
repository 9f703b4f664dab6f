// Host side of libnanosim_b200.so that needs no context and no stream: expansion of the 2-bit bases, the record,
// error-profile and read-name formatters, and the FASTA/FASTQ reader.  Plain multi-threaded C++; no kernels.
#include <algorithm>
#if defined(__x86_64__)
#include <immintrin.h>
#endif
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fcntl.h>
#include <sched.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "nanosim_b200.h"
#include "device_common.cuh"      // event_base_block / event_byte / event_base: bases of events the homopolymer pass rewrote
#include "host_io.h"

namespace {

constexpr int kMaxThreads = 64;

// Runs fn(lo, hi, part) over the items [0, n) cut into `parts` contiguous ranges (at most kMaxThreads), every non-empty
// range on a thread of its own; a single range, and range 0 when `caller_too`, on the calling thread (the formatters
// measured slower with range 0 on the calling thread).  With `off` (n + 1 ascending prefix offsets) the cuts balance the
// offsets -- bytes -- instead of the item count.
template <class Fn>
void fan_out(uint64_t n, int parts, const uint64_t* off, bool caller_too, Fn fn) {
    const int np = std::max(1, std::min(parts, kMaxThreads));
    std::vector<uint64_t> cut((size_t)np + 1, 0);
    for (int t = 1; t <= np; ++t) {
        if (t == np) {
            cut[t] = n;
        } else if (off) {
            const uint64_t hi = (uint64_t)(std::upper_bound(off, off + n + 1, off[n] * (uint64_t)t / np) - off);
            cut[t] = std::min(std::max(hi, cut[t - 1]), n);
        } else {
            cut[t] = n * (uint64_t)t / np;
        }
    }
    const int first = (np == 1 || caller_too) ? 1 : 0;
    std::vector<std::thread> th;
    for (int t = first; t < np; ++t)
        if (cut[t + 1] > cut[t]) th.emplace_back(fn, cut[t], cut[t + 1], t);
    if (first && cut[1] > 0) fn(uint64_t(0), cut[1], 0);
    for (auto& x : th) x.join();
}

// ---------------------------------------------------------------------------------------------------------
// expansion of the 2-bit bases (pack_bases_kernel) into ASCII
// ---------------------------------------------------------------------------------------------------------
#if defined(__x86_64__)
// 32 characters from 8 packed bytes per step: every output byte gets its source byte (vpshufb), the three shifted copies
// bring the byte's other 2-bit fields down, constant masks keep field j & 3 at output byte j, a second vpshufb turns the
// indices into letters.  ~14 instructions per 32 bases instead of four table lookups: the expansion then runs at memory
// speed, which is what 8 GPU processes sharing one host need.
__attribute__((target("avx2"))) void unpack_range_avx2(const uint8_t* packed, uint8_t* seq, uint64_t lo, uint64_t hi, const char* abc) {
    const __m256i spread = _mm256_setr_epi8(0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 6, 6, 6, 6, 7, 7, 7, 7);
    const __m256i m0 = _mm256_set1_epi32(0x00000003), m1 = _mm256_set1_epi32(0x00000300), m2 = _mm256_set1_epi32(0x00030000),
                  m3 = _mm256_set1_epi32(0x03000000);
    const __m256i letters = _mm256_setr_epi8(abc[0], abc[1], abc[2], abc[3], 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, abc[0], abc[1], abc[2], abc[3], 0,
                                             0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0);
    const bool aligned32 = (reinterpret_cast<uintptr_t>(seq) & 31u) == 0;
    for (uint64_t i = lo; i < hi; ++i) {              // unit: 32 characters
        const __m128i x = _mm_loadl_epi64(reinterpret_cast<const __m128i*>(packed + 8 * i));
        const __m256i src = _mm256_shuffle_epi8(_mm256_broadcastsi128_si256(x), spread);
        const __m256i idx = _mm256_or_si256(_mm256_or_si256(_mm256_and_si256(src, m0), _mm256_and_si256(_mm256_srli_epi16(src, 2), m1)),
                                            _mm256_or_si256(_mm256_and_si256(_mm256_srli_epi16(src, 4), m2), _mm256_and_si256(_mm256_srli_epi16(src, 6), m3)));
        const __m256i out = _mm256_shuffle_epi8(letters, idx);
        if (aligned32) _mm256_stream_si256(reinterpret_cast<__m256i*>(seq + 32 * i), out);     // written once, read much later
        else _mm256_storeu_si256(reinterpret_cast<__m256i*>(seq + 32 * i), out);
    }
    _mm_sfence();
}
#endif

// CPUs this process can really use: the affinity mask, capped by the container's cgroup CPU quota (cpu.max) -- a container
// can show many more logical CPUs than its quota grants
unsigned effective_cpus() {
    unsigned n = std::thread::hardware_concurrency();
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof set, &set) == 0) n = (unsigned)CPU_COUNT(&set);
    if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
        char q[64] = {0};
        unsigned long long period = 0;
        if (fscanf(f, "%63s %llu", q, &period) == 2 && strcmp(q, "max") != 0 && period > 0) {
            const unsigned long long quota = strtoull(q, nullptr, 10);
            const unsigned cores = (unsigned)((quota + period / 2) / period);
            if (cores >= 1 && cores < n) n = cores;
        }
        fclose(f);
    }
    return n ? n : 4u;
}
}  // namespace

void unpack_bases(const uint8_t* packed, uint8_t* seq, uint64_t seq_bytes, bool uracil, int nt) {
#if defined(__x86_64__)
    static const bool have_avx2 = __builtin_cpu_supports("avx2") && !getenv("NANOSIM_B200_NO_AVX2");
    if (have_avx2) {
        const char* abc2 = uracil ? "ACUG" : "ACTG";
        const uint64_t whole32 = seq_bytes / 32;
        fan_out(whole32, whole32 < (1u << 14) ? 1 : nt, nullptr, false,
                [&](uint64_t lo, uint64_t hi, int) { unpack_range_avx2(packed, seq, lo, hi, abc2); });
        for (uint64_t k = whole32 * 32; k < seq_bytes; ++k) seq[k] = (uint8_t)abc2[(packed[k >> 2] >> (2 * (k & 3))) & 3u];
        return;
    }
#endif
    // two packed bytes -> eight characters per table lookup (512 KB table per alphabet, built once)
    static std::vector<uint64_t> tables[2];
    static std::once_flag once[2];
    const char* abc = uracil ? "ACUG" : "ACTG";
    std::call_once(once[uracil ? 1 : 0], [&] {
        std::vector<uint64_t>& t = tables[uracil ? 1 : 0];
        t.resize(65536);
        for (uint32_t b = 0; b < 65536; ++b) {
            uint64_t w = 0;
            for (int j = 0; j < 8; ++j) w |= (uint64_t)(uint8_t)abc[(b >> (2 * j)) & 3u] << (8 * j);
            t[b] = w;
        }
    });
    const uint64_t* lut = tables[uracil ? 1 : 0].data();
    const uint64_t whole = seq_bytes / 8;             // 16-bit groups that expand to 8 in-range characters
    fan_out(whole, whole < (1u << 16) ? 1 : nt, nullptr, false, [&](uint64_t lo, uint64_t hi, int) {
        const bool aligned8 = (reinterpret_cast<uintptr_t>(seq) & 7u) == 0;
        for (uint64_t i = lo; i < hi; ++i) {
            uint16_t b;
            memcpy(&b, packed + 2 * i, 2);
            const uint64_t w = lut[b];
#if defined(__x86_64__)
            // streaming store: the destination is written once and read much later (no read-for-ownership traffic)
            if (aligned8) _mm_stream_si64(reinterpret_cast<long long*>(seq + 8 * i), (long long)w);
            else memcpy(seq + 8 * i, &w, 8);
#else
            memcpy(seq + 8 * i, &w, 8);
#endif
        }
#if defined(__x86_64__)
        _mm_sfence();
#endif
    });
    for (uint64_t k = whole * 8; k < seq_bytes; ++k) seq[k] = (uint8_t)abc[(packed[k >> 2] >> (2 * (k & 3))) & 3u];
}

int unpack_threads() {
    static const int n = [] {
        const char* e = getenv("NANOSIM_B200_UNPACK_THREADS");     // 0: copy the bases as ASCII (no packing)
        if (e && *e) return std::max(0, atoi(e));
        // packing only pays when the host can expand faster than PCIe delivers: one expanding thread per core this GPU
        // process can count on (torchrun exports LOCAL_WORLD_SIZE), at most 16; with fewer than 6 the bases travel as ASCII
        const char* lw = getenv("LOCAL_WORLD_SIZE");
        const unsigned ranks = (lw && *lw) ? (unsigned)std::max(1, atoi(lw)) : 1u;
        const unsigned per_rank = effective_cpus() / ranks;
        return per_rank >= 6u ? (int)std::min(per_rank, 16u) : 0;
    }();
    return n;
}

// ---------------------------------------------------------------------------------------------------------
// formatters: items (records, error-profile rows of a read) laid out back to back at prefix offsets
// ---------------------------------------------------------------------------------------------------------
namespace {
// Sink of a formatter thread: either the caller's buffer, or a private chunk that is written with pwrite() at the right
// file position whenever it fills up (the records of one thread are contiguous in the output).
struct ChunkSink {
    char* out;                // buffer mode: start of the whole output
    int fd;                   // file mode: descriptor + offset of the output's first byte in the file
    uint64_t file_off;
    std::vector<char> buf;
    size_t used = 0;
    uint64_t start = 0;       // output position of buf[0]
    bool ok = true;
    ChunkSink(char* o, int f, uint64_t fo) : out(o), fd(f), file_off(fo) {
        if (fd >= 0) buf.resize(size_t(8) << 20);
    }
    char* reserve(uint64_t at, size_t n) {       // n bytes at output position `at` (positions only grow within a thread)
        if (fd < 0) return out + at;
        if (used + n > buf.size()) {
            flush();
            if (n > buf.size()) buf.resize(n);
        }
        if (used == 0) start = at;
        char* p = buf.data() + used;
        used += n;
        return p;
    }
    void flush() {
        size_t done = 0;
        while (fd >= 0 && done < used) {
            const ssize_t w = pwrite(fd, buf.data() + done, used - done, (off_t)(file_off + start + done));
            if (w <= 0) {
                ok = false;
                break;
            }
            done += (size_t)w;
        }
        used = 0;
    }
};

// Items [0, n) back to back: item i takes size(i) bytes, which put(i, p) writes at p.  They go into `out` (out_cap bytes)
// or, with fd >= 0, into the file at file_off, from up to n_threads threads that each take a byte-balanced stretch.
// Two-call protocol: without out and fd only the total size is returned.  NS_ENOMEM: the total exceeds out_cap;
// NS_EINVAL: a pwrite() failed.
template <class Size, class Put>
int64_t format_items(uint32_t n, int n_threads, char* out, uint64_t out_cap, int fd, uint64_t file_off, Size size, Put put) {
    const int parts = n < 64 ? 1 : n_threads;
    std::vector<uint64_t> off((size_t)n + 1, 0);
    fan_out(n, parts, nullptr, false, [&](uint64_t lo, uint64_t hi, int) {
        for (uint64_t i = lo; i < hi; ++i) off[i + 1] = size((uint32_t)i);
    });
    for (uint32_t i = 0; i < n; ++i) off[i + 1] += off[i];
    if (fd < 0) {
        if (!out) return (int64_t)off[n];
        if (off[n] > out_cap) return NS_ENOMEM;
    }
    std::vector<char> failed(kMaxThreads, 0);
    fan_out(n, parts, off.data(), false, [&](uint64_t lo, uint64_t hi, int part) {
        ChunkSink sink(out, fd, file_off);
        for (uint64_t i = lo; i < hi; ++i)
            if (off[i + 1] > off[i]) put((uint32_t)i, sink.reserve(off[i], (size_t)(off[i + 1] - off[i])));
        sink.flush();
        if (!sink.ok) failed[part] = 1;
    });
    for (char f : failed)
        if (f) return NS_EINVAL;
    return (int64_t)off[n];
}

// host-side FASTA/FASTQ record formatting (simulator.py:1437-1443), multi-threaded memcpy-style assembly
int64_t format_records_impl(const uint8_t* seq, const uint8_t* qual, const NsReadMeta* reads, uint32_t n_reads,
                            const char* names, const uint64_t* name_off, int fastq, char* out, uint64_t out_cap,
                            int n_threads, int fd, uint64_t file_off) {
    if (!seq || !reads || !names || !name_off || (fastq && !qual)) return NS_EINVAL;
    auto size = [&](uint32_t i) -> uint64_t {
        const uint64_t rec = 1 + strlen(names + name_off[i]) + 1 + reads[i].seq_len + 1;
        return fastq ? rec + 2 + reads[i].seq_len + 1 : rec;
    };
    auto put = [&](uint32_t i, char* p) {
        const char* nm = names + name_off[i];
        size_t nl = strlen(nm);
        *p++ = fastq ? '@' : '>';
        memcpy(p, nm, nl);
        p += nl;
        *p++ = '\n';
        memcpy(p, seq + reads[i].seq_off, reads[i].seq_len);
        p += reads[i].seq_len;
        *p++ = '\n';
        if (fastq) {
            *p++ = '+';
            *p++ = '\n';
            memcpy(p, qual + reads[i].seq_off, reads[i].seq_len);
            p += reads[i].seq_len;
            *p++ = '\n';
        }
    };
    return format_items(n_reads, n_threads, out, out_cap, fd, file_off, size, put);
}

inline int dec_len(uint64_t v) {
    int n = 1;
    while (v >= 10) {
        v /= 10;
        ++n;
    }
    return n;
}
inline char* put_dec(char* p, uint64_t v) {
    char tmp[24];
    int n = 0;
    do {
        tmp[n++] = (char)('0' + v % 10);
        v /= 10;
    } while (v);
    while (n) *p++ = tmp[--n];
    return p;
}
struct EvRow {
    uint32_t type, len, ref_start, out_start, index, piece, ref_base;
    bool rewritten;
};

// host-side <out>_aligned_error_profile rows (mutate_read's log, simulator.py:2006-2008; header written by the caller):
// for every aligned segment, its error events right to left: name, position in the segment's reference, type, length,
// reference bases, read bases.  Events come from the segment's EVENT script (after the -k filter); when the
// homopolymer pass rewrote the emitted script, the bases of an event are the ones that pass fixed (event_base_block,
// device_common.cuh), otherwise they are read back from the sequence.  Two-call protocol like ns_format_records.
int64_t format_error_profile_impl(const uint8_t* seq, const NsReadMeta* reads, const NsPieceMeta* pieces, const uint32_t* ops,
                                  uint32_t n_reads, const uint8_t* ref_bases, const uint64_t* chrom_off, const char* names,
                                  const uint64_t* name_off, uint64_t seed, uint64_t first_id, char* out, uint64_t out_cap,
                                  int n_threads, int fd, uint64_t file_off) {
    if (!seq || !reads || !pieces || !ops || !ref_bases || !chrom_off || !names || !name_off) return NS_EINVAL;
    static const char kTypes[3][4] = {"mis", "ins", "del"};
    uint8_t comp[256];
    for (int c = 0; c < 256; ++c) comp[c] = (uint8_t)c;
    comp['A'] = 'T'; comp['T'] = 'A'; comp['C'] = 'G'; comp['G'] = 'C';
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    // one read: returns the bytes its rows take; writes them when p != nullptr
    auto do_read = [&](uint32_t i, char* p) -> uint64_t {
        const NsReadMeta& r = reads[i];
        const char* nm = names + name_off[i];
        const size_t nl = strlen(nm);
        const uint64_t rid = first_id + i;
        const uint32_t L = r.seq_len;
        const uint8_t* rs = seq + r.seq_off;
        const bool rev = r.reversed != 0;
        uint64_t bytes = 0;
        std::vector<EvRow> ev;
        // the pieces of one mutate_read call: a segment plus the pieces that continue it (NS_PIECE_CONT, intron retention)
        auto flush = [&]() {
            for (size_t e = ev.size(); e-- > 0;) {
                const EvRow& w = ev[e];
                const NsPieceMeta& pc = pieces[r.piece_first + w.piece];
                const uint64_t shown = (uint64_t)w.ref_base + w.ref_start;
                const uint64_t row = nl + 1 + dec_len(shown) + 1 + 3 + 1 + dec_len(w.len) + 1 + (uint64_t)w.len + 1 + w.len + 1;
                bytes += row;
                if (!p) continue;
                const uint64_t cstart = chrom_off[pc.chrom], clen = chrom_off[pc.chrom + 1] - cstart;
                const bool back = (pc.kind & NS_PIECE_REF_REV) != 0;
                memcpy(p, nm, nl);
                p += nl;
                *p++ = '\t';
                p = put_dec(p, shown);
                *p++ = '\t';
                memcpy(p, kTypes[w.type - 1], 3);
                p += 3;
                *p++ = '\t';
                p = put_dec(p, w.len);
                *p++ = '\t';
                char* refp = p;
                if (w.type == NS_OP_INS) {
                    memset(p, '-', w.len);
                } else {
                    for (uint32_t t = 0; t < w.len; ++t) {
                        const uint32_t f = w.ref_start + t;             // offset in the piece, in the direction of the read
                        uint64_t ab = (uint64_t)pc.pos + (back ? pc.ref_len - 1 - f : f);
                        if (ab >= clen) ab -= clen;
                        uint8_t c = ref_bases[cstart + ab];
                        if (c >= 'a' && c <= 'z') c = (uint8_t)(c - 32);
                        p[t] = (char)(back ? comp[c] : c);
                    }
                }
                p += w.len;
                *p++ = '\t';
                if (w.type == NS_OP_DEL) {
                    memset(p, '-', w.len);
                } else if (w.rewritten) {
                    uint4 blk;
                    for (uint32_t t = 0; t < w.len; ++t) {
                        if ((t & 15u) == 0) blk = event_base_block(key, rid, w.piece, w.index, t);
                        const char rc = refp[t];
                        const uint32_t orig = rc == 'C' ? 1u : (rc == 'T' ? 2u : (rc == 'G' ? 3u : 0u));
                        p[t] = "ACTG"[event_base(event_byte(blk, t), w.type == NS_OP_MIS, orig)];
                    }
                } else {
                    for (uint32_t t = 0; t < w.len; ++t) {
                        const uint32_t x = w.out_start + t;
                        p[t] = (char)(rev ? comp[rs[L - 1 - x]] : rs[x]);
                    }
                }
                p += w.len;
                *p++ = '\n';
            }
            ev.clear();
        };
        uint32_t ref_base = 0;
        for (uint32_t k = 0; k < r.n_pieces; k += 2) {
            const NsPieceMeta& pc = pieces[r.piece_first + k];
            if (NS_PIECE_KIND(pc.kind) != NS_PIECE_SEGMENT) continue;
            if (!(pc.kind & NS_PIECE_CONT)) {
                flush();
                ref_base = 0;
            }
            const uint32_t* sc = ops + pc.ev_off;
            const bool rewritten = pc.ev_off != pc.op_off;
            uint32_t o = pc.out_rel, rf = 0;
            for (uint32_t j = 0; j < pc.ev_n_ops; ++j) {
                const uint32_t op = sc[j], ty = NS_OP_TYPE(op), ln = NS_OP_LEN(op);
                if (ty >= NS_OP_MIS && ty <= NS_OP_DEL && ln) ev.push_back(EvRow{ty, ln, rf, o, j, k, ref_base, rewritten});
                if (ty != NS_OP_DEL) o += ln;
                if (ty == NS_OP_COPY || ty == NS_OP_MIS || ty == NS_OP_DEL) rf += ln;
            }
            ref_base += pc.ref_len;
        }
        flush();
        return bytes;
    };
    return format_items(n_reads, n_threads, out, out_cap, fd, file_off, [&](uint32_t i) { return do_read(i, nullptr); },
                        [&](uint32_t i, char* p) { do_read(i, p); });
}
}  // namespace

extern "C" {

int ns_unpack_bases(const uint8_t* packed, uint8_t* seq, uint64_t n_bases, int uracil, int threads) {
    if (!packed || !seq) return NS_EINVAL;
    unpack_bases(packed, seq, n_bases, uracil != 0, threads);
    return NS_OK;
}

int64_t ns_format_records(const uint8_t* seq, const uint8_t* qual, const NsReadMeta* reads, uint32_t n_reads,
                          const char* names, const uint64_t* name_off, int fastq, char* out, uint64_t out_cap,
                          int n_threads) {
    return format_records_impl(seq, qual, reads, n_reads, names, name_off, fastq, out, out_cap, n_threads, -1, 0);
}

int64_t ns_write_records(int fd, uint64_t file_off, const uint8_t* seq, const uint8_t* qual, const NsReadMeta* reads,
                         uint32_t n_reads, const char* names, const uint64_t* name_off, int fastq, int n_threads) {
    if (fd < 0) return NS_EINVAL;
    return format_records_impl(seq, qual, reads, n_reads, names, name_off, fastq, nullptr, 0, n_threads, fd, file_off);
}

int64_t ns_format_error_profile(const uint8_t* seq, const NsReadMeta* reads, const NsPieceMeta* pieces, const uint32_t* ops,
                                uint32_t n_reads, const uint8_t* ref_bases, const uint64_t* chrom_off, const char* names,
                                const uint64_t* name_off, uint64_t seed, uint64_t first_id, char* out, uint64_t out_cap,
                                int n_threads) {
    return format_error_profile_impl(seq, reads, pieces, ops, n_reads, ref_bases, chrom_off, names, name_off, seed, first_id, out,
                                     out_cap, n_threads, -1, 0);
}

int64_t ns_write_error_profile(int fd, uint64_t file_off, const uint8_t* seq, const NsReadMeta* reads, const NsPieceMeta* pieces,
                               const uint32_t* ops, uint32_t n_reads, const uint8_t* ref_bases, const uint64_t* chrom_off,
                               const char* names, const uint64_t* name_off, uint64_t seed, uint64_t first_id, int n_threads) {
    if (fd < 0) return NS_EINVAL;
    return format_error_profile_impl(seq, reads, pieces, ops, n_reads, ref_bases, chrom_off, names, name_off, seed, first_id, nullptr,
                                     0, n_threads, fd, file_off);
}

// ---------------------------------------------------------------------------------------------------------
// host-side read names (simulator.py:1390-1402 genome, :965-969 metagenome, :1188-1219 transcriptome, :1332-1343 perfect,
// :1511/:1529-1534 unaligned), written as NUL-terminated strings back to back -- the layout ns_format_records and
// ns_format_error_profile take.  flags: bit 0 perfect, bit 1 metagenome (gap lengths in the name), bit 2 transcriptome.
// ---------------------------------------------------------------------------------------------------------
int64_t ns_format_names(const NsReadMeta* reads, const NsPieceMeta* pieces, uint32_t n_reads, int kind, uint32_t flags,
                        uint64_t index_base, const char* chrom_names, const uint64_t* chrom_name_off, char* out,
                        uint64_t out_cap, uint64_t* name_off) {
    if (!reads || !pieces || !chrom_names || !chrom_name_off) return NS_EINVAL;
    const bool perfect = flags & 1u, meta = flags & 2u, trx = flags & 4u;
    // the reads are cut into ranges, one per thread; every thread builds the names of its range back to back in its own blob
    const int nt = n_reads < 4096 ? 1 : 8;
    std::vector<std::string> blobs((size_t)nt);
    std::vector<std::vector<uint32_t>> lens((size_t)nt);
    fan_out(n_reads, nt, nullptr, true, [&](uint64_t lo, uint64_t hi, int tid) {
        std::string& blob = blobs[tid];
        std::vector<uint32_t>& ln = lens[tid];
        blob.reserve((size_t)(hi - lo) * 64);
        ln.reserve(hi - lo);
        std::string nm;
        char num[32];
        auto add_num = [&](uint64_t v) {
            char* e = put_dec(num, v);
            nm.append(num, (size_t)(e - num));
        };
        for (uint32_t i = (uint32_t)lo; i < hi; ++i) {
            const NsReadMeta& r = reads[i];
            const NsPieceMeta* pc = pieces + r.piece_first;
            const char strand = r.reversed ? 'R' : 'F';
            nm.clear();
            if (kind == NS_KIND_UNALIGNED) {
                nm += chrom_names + chrom_name_off[pc[0].chrom];
                nm += '_';
                add_num(pc[0].pos);
                nm += "_unaligned_";
                add_num(index_base + i);
                nm += '_';
                nm += strand;
                nm += "_0_";
                add_num(pc[0].ref_len);
                nm += "_0";
            } else if (trx && (pc[0].kind & NS_PIECE_GENOME)) {
                // intron-retention layout (:1188-1192, :1217-1219): transcript, genomic start of the first interval, the
                // retained-intron intervals the read covers in genomic order
                uint64_t first_pos = pc[0].pos, mid = 0;
                for (uint32_t k = 0; k < r.n_pieces; k += 2) {
                    first_pos = std::min<uint64_t>(first_pos, pc[k].pos);
                    mid += pc[k].ref_len;
                }
                nm += chrom_names + chrom_name_off[pc[0].ref_req];
                nm += '_';
                add_num(first_pos);
                nm += "_aligned_";
                add_num(index_base + i);
                bool any = false;
                for (uint32_t k = 0; k < r.n_pieces; k += 2) any = any || (pc[k].kind & NS_PIECE_RETAINED);
                if (any) {
                    nm += "_RetainedIntron_";
                    std::vector<std::pair<uint64_t, uint64_t>> ivs;              // in genomic order, whatever the strand
                    for (uint32_t k = 0; k < r.n_pieces; k += 2)
                        if (pc[k].kind & NS_PIECE_RETAINED) ivs.emplace_back(pc[k].pos, (uint64_t)pc[k].pos + pc[k].ref_len);
                    std::stable_sort(ivs.begin(), ivs.end());
                    for (const auto& iv : ivs) {
                        add_num(iv.first);
                        nm += '-';
                        add_num(iv.second);
                        nm += ';';
                    }
                }
                nm += '_';
                nm += strand;
                nm += '_';
                add_num(r.head);
                nm += '_';
                add_num(mid);
                nm += '_';
                add_num((uint64_t)r.tail + pc[0].polya_len);
            } else if (trx) {
                nm += chrom_names + chrom_name_off[pc[0].chrom];
                nm += '_';
                add_num(pc[0].pos);
                nm += perfect ? "_perfect_" : "_aligned_";
                add_num(index_base + i);
                nm += '_';
                nm += strand;
                nm += '_';
                add_num(r.head);
                nm += '_';
                add_num(pc[0].ref_len);
                nm += '_';
                add_num((uint64_t)r.tail + pc[0].polya_len);
            } else if (perfect) {
                uint64_t sum = 0;
                for (uint32_t k = 0; k < r.n_pieces; k += 2) {
                    nm += chrom_names + chrom_name_off[pc[k].chrom];
                    nm += '_';
                    add_num(pc[k].pos);
                    sum += pc[k].ref_len;
                }
                nm += "_perfect_";
                add_num(index_base + i);
                nm += '_';
                nm += strand;
                nm += "_0_";
                add_num(sum);
                nm += "_0";
            } else {
                for (uint32_t k = 0; k < r.n_pieces; ++k) {
                    if (k & 1u) {
                        if (!meta) continue;
                        nm += ";gap_";
                        add_num(pc[k].out_len);
                        continue;
                    }
                    if (k) nm += ';';
                    nm += chrom_names + chrom_name_off[pc[k].chrom];
                    nm += '_';
                    add_num(pc[k].pos);
                }
                nm += "_aligned_";
                add_num(index_base + i);
                if (r.n_pieces > 1) nm += "_chimeric";
                nm += '_';
                nm += strand;
                nm += '_';
                add_num(r.head);
                nm += '_';
                for (uint32_t k = 0; k < r.n_pieces; k += 2) {
                    if (k) nm += ';';
                    add_num(pc[k].ref_len);
                }
                nm += '_';
                add_num(r.tail);
            }
            blob.append(nm.c_str(), nm.size() + 1);
            ln.push_back((uint32_t)nm.size() + 1);
        }
    });
    uint64_t total = 0;
    for (const std::string& bl : blobs) total += bl.size();
    if (!out) return (int64_t)total;
    if (total > out_cap) return NS_ENOMEM;
    uint64_t pos = 0;
    uint32_t i = 0;
    for (int t = 0; t < nt; ++t) {
        memcpy(out + pos, blobs[t].data(), blobs[t].size());
        if (name_off)
            for (uint32_t l : lens[t]) {
                name_off[i++] = pos;
                pos += l;
            }
        else
            pos += blobs[t].size();
    }
    return (int64_t)total;
}

// ---------------------------------------------------------------------------------------------------------
// FASTA / FASTQ reader of read_profile (simulator.py:341-349 with readfq :709-740): the file is mmap()ed and cut into
// line-aligned chunks; every thread finds the record headers of its chunk and counts its sequence bytes (pass 1), a prefix
// sum places the chunks, and the threads copy their sequence lines behind one another (pass 2).  Bytes are kept as they are
// (case, IUPAC codes); line ends (\n, \r\n) are dropped.  A FASTQ file (first byte '@') is read by one thread: its
// quality lines can begin with '>' or '@'.
// Two-call protocol: with bases == NULL only *n_records, *n_bases and *header_bytes are set.  rec_off gets n_records + 1
// offsets into bases; headers gets the header lines (without the marker) NUL-terminated back to back, header_off their starts.
// ---------------------------------------------------------------------------------------------------------
namespace {
struct FaChunk {
    const char* lo;
    const char* hi;
    uint64_t n_bases = 0;
    std::vector<std::pair<const char*, uint64_t>> heads;      // header line start (at the marker), sequence bytes of the chunk before it
};
inline const char* line_end(const char* p, const char* end) {
    const char* nl = (const char*)memchr(p, '\n', (size_t)(end - p));
    return nl ? nl : end;
}
inline size_t trimmed(const char* p, const char* e) {         // line length without a trailing \r
    return (e > p && e[-1] == '\r') ? (size_t)(e - p - 1) : (size_t)(e - p);
}
}  // namespace

int64_t ns_read_fasta(const char* path, uint8_t* bases, uint64_t bases_cap, uint64_t* rec_off, char* headers, uint64_t headers_cap,
                      uint64_t* header_off, uint32_t* n_records, uint64_t* n_bases, uint64_t* header_bytes, int n_threads) {
    if (!path || !n_records || !n_bases || !header_bytes) return NS_EINVAL;
    const int fd = open(path, O_RDONLY);
    if (fd < 0) return NS_EINVAL;
    struct stat sb;
    if (fstat(fd, &sb) != 0) {
        close(fd);
        return NS_EINVAL;
    }
    const size_t size = (size_t)sb.st_size;
    *n_records = 0;
    *n_bases = *header_bytes = 0;
    if (size == 0) {
        close(fd);
        return 0;
    }
    const char* base = (const char*)mmap(nullptr, size, PROT_READ, MAP_PRIVATE, fd, 0);
    close(fd);
    if (base == MAP_FAILED) return NS_ENOMEM;
    madvise((void*)base, size, MADV_SEQUENTIAL);
    const char* end = base + size;
    const bool fastq = base[0] == '@';
    const int nt = (fastq || size < (size_t(1) << 22)) ? 1 : std::max(1, std::min(n_threads, kMaxThreads));
    std::vector<FaChunk> ch((size_t)nt);
    for (int t = 0; t < nt; ++t) {                             // line-aligned chunk boundaries
        const char* p = base + size * (size_t)t / (size_t)nt;
        if (t > 0) {
            p = line_end(p - 1, end);
            if (p < end) ++p;
        }
        ch[t].lo = p;
        if (t > 0) ch[t - 1].hi = p;
    }
    ch[nt - 1].hi = end;
    const bool fill = bases != nullptr;
    // pass 1 / pass 2 over one chunk; FASTQ: sequence lines run to the '+' line, then as many quality bytes are skipped
    auto walk = [&](FaChunk& c, uint8_t* dst) {
        const char* p = c.lo;
        uint64_t count = 0;
        bool in_qual = false;
        uint64_t qual_left = 0, rec_bases = 0;
        while (p < c.hi) {
            const char* e = line_end(p, c.hi);
            const size_t len = trimmed(p, e);
            if (fastq && in_qual) {
                if (qual_left <= len) in_qual = false; else qual_left -= len;
            } else if (len && (p[0] == '>' || (fastq && p[0] == '@'))) {
                if (!dst) c.heads.emplace_back(p, count);
                rec_bases = 0;
            } else if (fastq && len && p[0] == '+') {
                in_qual = rec_bases > 0;
                qual_left = rec_bases;
            } else if (len) {
                if (dst) memcpy(dst + count, p, len);
                count += len;
                rec_bases += len;
            }
            p = e < c.hi ? e + 1 : c.hi;
        }
        if (!dst) c.n_bases = count;
    };
    // one chunk per thread
    fan_out(nt, nt, nullptr, true, [&](uint64_t, uint64_t, int t) { walk(ch[t], nullptr); });
    uint64_t total = 0, n_rec = 0, hbytes = 0;
    std::vector<uint64_t> chunk_off((size_t)nt);
    for (int t = 0; t < nt; ++t) {
        chunk_off[t] = total;
        total += ch[t].n_bases;
        n_rec += ch[t].heads.size();
        for (auto& h : ch[t].heads) hbytes += trimmed(h.first, line_end(h.first, end));       // marker dropped, NUL added
    }
    *n_records = (uint32_t)n_rec;
    *n_bases = total;
    *header_bytes = hbytes;
    int64_t rc = (int64_t)total;
    if (fill) {
        if (total > bases_cap || hbytes > headers_cap || !rec_off || !headers || !header_off) {
            rc = NS_ENOMEM;
        } else {
            uint64_t r = 0, hpos = 0;
            for (int t = 0; t < nt; ++t)
                for (auto& h : ch[t].heads) {
                    rec_off[r] = chunk_off[t] + h.second;
                    const size_t hl = trimmed(h.first, line_end(h.first, end)) - 1;
                    header_off[r] = hpos;
                    memcpy(headers + hpos, h.first + 1, hl);
                    headers[hpos + hl] = 0;
                    hpos += hl + 1;
                    ++r;
                }
            rec_off[n_rec] = total;
            fan_out(nt, nt, nullptr, true, [&](uint64_t, uint64_t, int t) { walk(ch[t], bases + chunk_off[t]); });
        }
    }
    munmap((void*)base, size);
    return rc;
}

}  // extern "C"
