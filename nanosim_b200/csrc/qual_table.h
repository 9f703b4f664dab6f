// Host construction of the base-quality sampler tables that emit_kernel.cuh:qual_pick reads.  Included by the library
// (nanosim_api.cu) and by tests/draw_harness.cu, which holds every table it builds against the 24-bit pmf.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "nanosim_b200.h"
#include "device_common.cuh"      // QLUT_BITS, QLUT_SIZE

// Base-quality sampler tables (emit_kernel.cuh:qual_pick).  The truncated log-normal of a state, floored to integers
// (model_base_qualities.py:9-20, 120-130), arrives as a 32-bit cdf; it is rounded to a 24-bit pmf (masses sum to 2^24) and
// laid out as a Walker alias table with QLUT_SIZE = 2048 slots of capacity 2^13: slot j holds a primary and an alias
// quality and the primary's share t of the slot, so a 24-bit draw (11 bits slot, 13 bits u) returns the primary iff u < t.
// All arithmetic is in integers: the table realises the 24-bit pmf exactly.  Entry: t << 19 | alias char << 8 | primary
// char (ASCII = q + 33); a slot that holds one quality only stores it twice (t is then irrelevant).
inline void build_qlut(const uint32_t cdf32[NS_N_QUAL_STATES][NS_QUAL_SLOTS], std::vector<uint32_t>& lut) {
    lut.assign((size_t)NS_N_QUAL_STATES * QLUT_SIZE, 0);
    const uint32_t cap = 1u << (24 - QLUT_BITS);
    for (int s = 0; s < NS_N_QUAL_STATES; ++s) {
        uint32_t c24[NS_QUAL_SLOTS];
        for (int q = 0; q < NS_QUAL_SLOTS; ++q) {
            uint64_t v = ((uint64_t)cdf32[s][q] + 128u) >> 8;
            c24[q] = (uint32_t)std::min<uint64_t>(v, 1u << 24);
            if (q && c24[q] < c24[q - 1]) c24[q] = c24[q - 1];
        }
        c24[NS_QUAL_SLOTS - 1] = 1u << 24;
        std::vector<uint32_t> mass(QLUT_SIZE, 0u), thr(QLUT_SIZE, 0u), prim(QLUT_SIZE), ali(QLUT_SIZE);
        for (int q = 0; q < NS_QUAL_SLOTS; ++q) mass[q] = c24[q] - (q ? c24[q - 1] : 0u);
        std::vector<uint32_t> small, large;
        for (uint32_t j = 0; j < QLUT_SIZE; ++j) {
            prim[j] = ali[j] = j;
            (mass[j] < cap ? small : large).push_back(j);
        }
        while (!small.empty() && !large.empty()) {
            const uint32_t a = small.back(), g = large.back();
            small.pop_back();
            large.pop_back();
            thr[a] = mass[a];                   // the rest of slot a, cap - mass[a], is taken from g
            ali[a] = g;
            mass[g] -= cap - mass[a];
            (mass[g] < cap ? small : large).push_back(g);
        }
        // what is left holds exactly `cap` (the masses are integers that sum to QLUT_SIZE * cap): pure slots
        for (uint32_t j : small) { thr[j] = 0; ali[j] = prim[j]; }
        for (uint32_t j : large) { thr[j] = 0; ali[j] = prim[j]; }
        // a slot index >= 94 is not a quality: such slots had no mass and are aliased entirely (thr 0)
        for (uint32_t j = 0; j < QLUT_SIZE; ++j) {
            uint32_t pq = prim[j], aq = ali[j];
            if (pq >= (uint32_t)NS_QUAL_SLOTS) pq = aq;
            if (aq >= (uint32_t)NS_QUAL_SLOTS) aq = pq;           // cannot happen: only slots with mass are aliases
            lut[(size_t)s * QLUT_SIZE + j] = (thr[j] << 19) | ((aq + 33u) << 8) | (pq + 33u);
        }
    }
}
