// IS-IS route table of a batch of SPTs, one cell per (job, prefix).
//
// compute_routes (holo-isis/src/spf.rs:838-941) walks each topology's SPT in vertex order and, per
// vertex with a valid zeroth LSP, feeds the IP reachability of its valid fragments through `add`
// (isis_host.cc: topology_routes).  Which contributions a prefix gets, and in which order, is a
// property of the LSDB and the instance configuration; a what-if cost override changes none of it.
// Each prefix is fed by one topology (IPv4: standard; IPv6: standard, or MT-IPv6 only when that
// topology is enabled).  The contributor lists are built once per instance (hspf_isis_rtable_create);
// the walk over one prefix's list is isis_route_cell_eval, one thread per (job, prefix) on the device
// (isis_routes.cu).
//
// What a cell does not hold is decided on the host per job by hspf_isis_routes_from_cells: atoms to
// adjacency next hops (the stateful first-hop replay around the root), max_paths truncation in address
// order, SR labels.
#pragma once
#include <cstdint>
#include <vector>

#include "holo_lsdb.h"
#include "route_cells.h"

namespace hspf {

// One contribution of compute_routes to a prefix, in the order the walk meets them.
struct alignas(16) IsisContrib {
    uint32_t vertex;      // SPT vertex of `topology` (flattener order)
    uint32_t metric;      // entry metric (0 for the ATT-bit default route)
    uint8_t  topology;    // 0 standard, 1 MT-IPv6
    uint8_t  external;    // route type L1/L2 external
    uint8_t  has_psid;    // the entry carries a Prefix-SID
    uint8_t  sr;          // has_psid and SR enabled: the winner's labels depend on the contributing vertex
    uint32_t _pad;
};
static_assert(sizeof(IsisContrib) == 16, "IsisContrib layout");

HSPF_HD IsisContrib load_isis_contrib(const IsisContrib *p) {
#if defined(__CUDA_ARCH__)
    const uint4 r = __ldg(reinterpret_cast<const uint4 *>(p));
    IsisContrib k;
    k.vertex = r.x; k.metric = r.y;
    k.topology = (uint8_t)(r.z & 0xFFu); k.external = (uint8_t)((r.z >> 8) & 0xFFu);
    k.has_psid = (uint8_t)((r.z >> 16) & 0xFFu); k.sr = (uint8_t)(r.z >> 24); k._pad = 0;
    return k;
#else
    return *p;
#endif
}

// The walk of one prefix's contributors = the sequence of `add` calls compute_routes makes for it:
//   * a contributor off its topology's SPT adds nothing;
//   * metric = distance + entry metric in u32 arithmetic;
//   * no route yet or a lower metric replaces (type, CONNECTED and Prefix-SID come from the contributor);
//   * an equal metric merges the next hops; a higher one is dropped.
// Truncating to max_paths after every merge equals truncating the union once, so the atom union is all
// the host needs, except for SR labels: every SrView::update relabels with the latest contributor's
// context.  When the route has an SR-relevant Prefix-SID and its best-metric contributions come from two
// or more vertices the cell is flagged: the host redoes that job from its planes.
//
// One `add` of the walk (isis_backbone_cell_eval): the contribution of `vertex` (reached in `pl`) at total metric m,
// recorded as `winner`; `sr`: its Prefix-SID is SR-relevant.  cur_vertex / cur_sr: the current winner's.
template <class Planes>
HSPF_HD void isis_route_add(hl_isis_route_cell &c, uint32_t &cur_vertex, bool &cur_sr, const Planes &pl,
                            uint32_t vertex, uint32_t m, uint32_t winner, bool sr) {
    if (!(c.flags & HL_CELL_PRESENT) || m < c.metric) {
        c.metric = m;
        c.winner = winner;
        c.flags = (uint8_t)(HL_CELL_PRESENT | (pl.h(vertex) == 0 ? HL_CELL_CONNECTED : 0));
        c.nh_mask = pl.n(vertex);
        cur_vertex = vertex;
        cur_sr = sr;
    } else if (m == c.metric) {
        if (cur_sr && vertex != cur_vertex) c.flags |= HL_CELL_MIXED_SID;
        c.nh_mask |= pl.n(vertex);
    }
}

template <class Planes>
HSPF_HD hl_isis_route_cell isis_route_cell_eval(const Planes &std_pl, const Planes &mt6_pl, const IsisContrib *contribs,
                                                uint32_t begin, uint32_t end) {
    hl_isis_route_cell c;
    c.nh_mask = 0; c.winner = 0xFFFFFFFFu; c.metric = 0; c.flags = 0;
    for (int i = 0; i < 7; ++i) c._pad[i] = 0;
    uint32_t cur_vertex = 0;
    bool cur_sr = false;
    for (uint32_t i = begin; i < end; ++i) {
        const IsisContrib k = load_isis_contrib(contribs + i);
        const Planes pl = k.topology ? mt6_pl : std_pl;     // a copy: selecting a reference puts both on the stack
        if (!pl.reached(k.vertex)) continue;
        // isis_route_add written out: calling it gives the IS-IS route stage's kernels other SASS (delta passes 44 / 46
        // registers instead of 45 / 47), untimed; written out, all three IS-IS stages keep their SASS.  Both copies are
        // held to hspf_isis_routes_from_planes by the route-cell and backbone tests.
        const uint32_t m = pl.d(k.vertex) + k.metric;
        if (!(c.flags & HL_CELL_PRESENT) || m < c.metric) {
            c.metric = m;
            c.winner = i;
            c.flags = (uint8_t)(HL_CELL_PRESENT | (pl.h(k.vertex) == 0 ? HL_CELL_CONNECTED : 0));
            c.nh_mask = pl.n(k.vertex);
            cur_vertex = k.vertex;
            cur_sr = k.sr != 0;
        } else if (m == c.metric) {
            if (cur_sr && k.vertex != cur_vertex) c.flags |= HL_CELL_MIXED_SID;
            c.nh_mask |= pl.n(k.vertex);
        }
    }
    return c;
}

}  // namespace hspf

// Host + device image of an instance's IS-IS route table (include/holo_spf_lsdb.h).
struct hspf_isis_rtable {
    std::vector<hl_ip_addr> prefix;          // [P] NetKey order
    std::vector<uint32_t> len;               // [P]
    std::vector<uint32_t> off;               // [P+1] into contribs
    std::vector<hspf::IsisContrib> contribs;
    std::vector<int32_t> src;                // per contributor: index into lvl.ipreaches, -1 for an ATT default route
    uint32_t n_vertices[2] = {0, 0};         // per topology (0 standard, 1 MT-IPv6)
    uint32_t root[2] = {0xFFFFFFFFu, 0xFFFFFFFFu};
    hspf::DeviceRouteTable dev;              // hspf_isis_rtable_upload
};
