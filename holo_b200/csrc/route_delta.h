// Route-delta classification: how one (job, prefix) cell differs from its base cell (include/holo_lsdb.h,
// HL_DELTA_*).  Host and device: the fused route-delta stage (route_stage.cuh) and the CPU test harness compile
// this same function.  Every cell layout is three 8-byte words with the next-hop atom set in word 0; they differ
// in where the HL_CELL_* flags and the metric sit:
//   OSPF  (hl_route_cell)      w1 lasthop_mask,               w2 winner | metric:16 << 32 | flags << 48
//   IS-IS (hl_isis_route_cell) w1 winner | metric:32 << 32,   w2 flags
//   OSPF routing table (hl_ospf_rib_cell)
//                              w1 aux,                        w2 winner | metric:26 << 32 | path:2 << 58 | flags:4 << 60
// Everything outside word 0 and the metric field (winner, flags, OSPF lasthop_mask, routing-table path type and aux)
// counts as HL_DELTA_OTHER.
#pragma once
#include <cstdint>

#include "holo_lsdb.h"

#if !defined(HSPF_HD)
#if defined(__CUDACC__)
#define HSPF_HD __host__ __device__ __forceinline__
#else
#define HSPF_HD inline
#endif
#endif

namespace hspf {

struct CellWords { uint64_t w0, w1, w2; };  // one cell, as its three 8-byte words in memory order

// Where a cell layout keeps its flags byte ((word >> flags_shift) & 0xFF) and its metric
// ((word & metric_mask) >> metric_shift); words are numbered 0..2 in memory order.
struct OspfCellLayout {
    static constexpr uint32_t flags_word = 2, flags_shift = 48, metric_word = 2, metric_shift = 32;
    static constexpr uint64_t metric_mask = 0xFFFFull << 32;
};
struct IsisCellLayout {
    static constexpr uint32_t flags_word = 2, flags_shift = 0, metric_word = 1, metric_shift = 32;
    static constexpr uint64_t metric_mask = 0xFFFFFFFFull << 32;
};
// flags are 4 bits here: the shifted word holds nothing above them
struct OspfRibCellLayout {
    static constexpr uint32_t flags_word = 2, flags_shift = 60, metric_word = 2, metric_shift = 32;
    static constexpr uint64_t metric_mask = 0x3FFFFFFull << 32;
};

HSPF_HD uint64_t cell_word(const CellWords &c, uint32_t i) { return i == 0 ? c.w0 : (i == 1 ? c.w1 : c.w2); }

template <class L>
HSPF_HD bool cell_present(const CellWords &c) {
    return ((cell_word(c, L::flags_word) >> L::flags_shift) & HL_CELL_PRESENT) != 0;
}

template <class L>
HSPF_HD uint32_t cell_metric(const CellWords &c) {
    return (uint32_t)((cell_word(c, L::metric_word) & L::metric_mask) >> L::metric_shift);
}

// HL_DELTA_* bits of job cell `j` against base cell `b`; 0 = no change (also when neither is present).
template <class L>
HSPF_HD uint32_t route_delta_kind(const CellWords &j, const CellWords &b) {
    const bool jp = cell_present<L>(j), bp = cell_present<L>(b);
    if (jp != bp) return jp ? HL_DELTA_GAINED : HL_DELTA_LOST;
    if (!jp) return 0;
    uint32_t k = 0;
    if (j.w0 != b.w0) k |= HL_DELTA_NEXTHOPS;
    const uint64_t d1 = j.w1 ^ b.w1, d2 = j.w2 ^ b.w2;
    const uint64_t dm = L::metric_word == 1 ? d1 : d2;
    if (dm & L::metric_mask) k |= HL_DELTA_METRIC;
    const uint64_t rest = L::metric_word == 1 ? ((d1 & ~L::metric_mask) | d2) : (d1 | (d2 & ~L::metric_mask));
    if (rest) k |= HL_DELTA_OTHER;
    return k;
}

// the metric a record carries: the job's, or the base's when the prefix was lost
template <class L>
HSPF_HD uint32_t route_delta_metric(const CellWords &j, const CellWords &b, uint32_t kind) {
    return cell_metric<L>(kind == HL_DELTA_LOST ? b : j);
}

}  // namespace hspf
