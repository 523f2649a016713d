// Routing table of an IS-IS backbone router R for a batch of L1 what-if jobs, one cell per (job, affected prefix)
// (include/holo_spf_lsdb.h, hspf_isis_backbone_table_create).
//
// An L1 job changes costs inside one area only.  Each L1/L2 router ("border") of the area re-originates its L2 LSP
// with the same IS reachability and new IP reachability (isis_l1_to_l2_cells.h), so R's L2 SPT is its unperturbed
// one in every job, and only the prefixes that are keys of some border's L1 -> L2 table can route differently.  Per
// such prefix the walk is compute_routes' (isis_route_cells.h, isis_route_add) over R's contributors in the LSDB
// where each border's derived entries are replaced by what it propagates in the job, appended to its zeroth
// fragment:
//   * a static contributor reads R's planes (row 0) as in isis_route_cell_eval;
//   * a slot stands for one (border, key) at the border's vertex, in the place for_each_contribution meets the
//     appended entry: it contributes when the border's L1 -> L2 cell of the job is present, at the cell's metric (a
//     TLV 135 key only up to kIsisMaxWide, as compute_routes reads extended IPv4 reachability).
// The winner of a slot names the border's winning record: n_contribs + base + the border cell's winner, one index
// per (slot, record), so a change of record at an equal metric (another Prefix-SID) shows in the delta; sr[] says
// whether that record's Prefix-SID is SR-relevant at R.
#pragma once
#include <cstdint>
#include <vector>

#include "isis_l1_to_l2_cells.h"

namespace hspf {

constexpr uint32_t kIsisBackboneMaxBorders = 8;
constexpr uint8_t kIsisBackboneStatic = 0xFF;        // IsisBackboneContrib::border of a static contributor
constexpr uint32_t kIsisMaxWide = 0xFE000000u;       // the largest extended IPv4 metric compute_routes reads

// One contribution to an affected prefix, in walk order.
struct alignas(16) IsisBackboneContrib {
    uint32_t vertex;      // R's L2 vertex of `topology`
    uint32_t metric;      // static: the entry metric; slot: its key in the border's cells
    uint32_t base;        // slot: the winner of record w is n_contribs + base + w (mod 2^32)
    uint8_t  topology;    // 0 standard, 1 MT-IPv6
    uint8_t  border;      // kIsisBackboneStatic, or the slot's border
    uint8_t  sr;          // static: its Prefix-SID is SR-relevant
    uint8_t  wide;        // slot: a TLV 135 key
};
static_assert(sizeof(IsisBackboneContrib) == 16, "IsisBackboneContrib layout");

HSPF_HD IsisBackboneContrib load_backbone_contrib(const IsisBackboneContrib *p) {
#if defined(__CUDA_ARCH__)
    const uint4 r = __ldg(reinterpret_cast<const uint4 *>(p));
    IsisBackboneContrib k;
    k.vertex = r.x; k.metric = r.y; k.base = r.z;
    k.topology = (uint8_t)(r.w & 0xFFu); k.border = (uint8_t)((r.w >> 8) & 0xFFu);
    k.sr = (uint8_t)((r.w >> 16) & 0xFFu); k.wide = (uint8_t)(r.w >> 24);
    return k;
#else
    return *p;
#endif
}

// What the walk reads of a table.
struct IsisBackboneView {
    const uint32_t *off;          // [P + 1] into contribs
    const uint32_t *sr;           // [n_slot_records]: the record's Prefix-SID is SR-relevant at R
    const IsisBackboneContrib *contribs;
    uint32_t P, n_contribs;
};

// One job's row of every border's L1 -> L2 cells.
struct IsisBorderRows {
    const hl_isis_route_cell *row[kIsisBackboneMaxBorders];
};

// a border cell: present or not, its winner and metric
HSPF_HD bool border_cell(const hl_isis_route_cell *c, uint32_t &winner, uint32_t &metric) {
#if defined(__CUDA_ARCH__)
    const unsigned long long *w = reinterpret_cast<const unsigned long long *>(c);
    const uint64_t wm = __ldg(w + 1);
    winner = (uint32_t)wm; metric = (uint32_t)(wm >> 32);
    return (__ldg(w + 2) & HL_CELL_PRESENT) != 0;
#else
    winner = c->winner; metric = c->metric;
    return (c->flags & HL_CELL_PRESENT) != 0;
#endif
}

// The cell of prefix p; std_pl / mt6_pl are R's unperturbed planes.
template <class Planes>
HSPF_HD hl_isis_route_cell isis_backbone_cell_eval(const Planes &std_pl, const Planes &mt6_pl, const IsisBackboneView &t,
                                                   uint32_t p, const IsisBorderRows &rows) {
    hl_isis_route_cell c;
    c.nh_mask = 0; c.winner = 0xFFFFFFFFu; c.metric = 0; c.flags = 0;
    for (int i = 0; i < 7; ++i) c._pad[i] = 0;
    uint32_t cur_vertex = 0;
    bool cur_sr = false;
    for (uint32_t i = t.off[p]; i < t.off[p + 1]; ++i) {
        const IsisBackboneContrib k = load_backbone_contrib(t.contribs + i);
        const Planes pl = k.topology ? mt6_pl : std_pl;     // a copy: selecting a reference puts both on the stack
        if (!pl.reached(k.vertex)) continue;
        uint32_t metric = k.metric, winner = i;
        bool sr = k.sr != 0;
        if (k.border != kIsisBackboneStatic) {
            uint32_t w;
            if (!border_cell(rows.row[k.border] + k.metric, w, metric) || (k.wide && metric > kIsisMaxWide)) continue;
            const uint32_t g = k.base + w;
            winner = t.n_contribs + g;
            sr = t.sr[g] != 0;
        }
        isis_route_add(c, cur_vertex, cur_sr, pl, k.vertex, pl.d(k.vertex) + metric, winner, sr);
    }
    return c;
}

}  // namespace hspf

// Host + device image of a backbone router's affected prefixes (include/holo_spf_lsdb.h).
struct hspf_isis_backbone_table {
    std::vector<hl_ip_addr> prefix;          // [P] hl_isis_rib order
    std::vector<uint8_t> len;                // [P]
    std::vector<uint32_t> words;             // the view's u32 arrays: off [P + 1], sr [n_slot_records]
    std::vector<hspf::IsisBackboneContrib> contribs;
    // host decode, per contributor: a static one's IsisContrib and lvl.ipreaches index; a slot's border and key
    std::vector<hspf::IsisContrib> stat;
    std::vector<int32_t> src;
    std::vector<uint32_t> slot_of;           // [n_slot_records] the slot's contributor
    uint32_t P = 0, n_slot_records = 0, n_borders = 0, n_ipreaches = 0;
    uint32_t n_vertices[2] = {0, 0};
    uint32_t root[2] = {0xFFFFFFFFu, 0xFFFFFFFFu};
    const hspf_isis_l1_to_l2_table *borders[hspf::kIsisBackboneMaxBorders] = {};
    hspf::DeviceRouteTable dev;              // hspf_isis_backbone_table_upload

    hspf::IsisBackboneView view(const uint32_t *w, const hspf::IsisBackboneContrib *c) const {
        hspf::IsisBackboneView v;
        v.off = w;
        v.sr = w + P + 1;
        v.contribs = c;
        v.P = P;
        v.n_contribs = (uint32_t)contribs.size();
        return v;
    }
};
