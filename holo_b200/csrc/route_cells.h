// Intra-area route table of a batch of SPTs, one cell per (job, prefix).
//
// update_rib_intra_area (holo-ospf/src/route.rs:343-446) walks the SPT in VertexId order and, per
// vertex, adds one route per stub link / the transit network's own prefix through route_update
// (route.rs:895-971).  The outcome for one prefix depends only on the prefix's own contributors
// (the vertices that advertise it), visited in that same order, and on three values of each
// contributor's SPT vertex: distance, hops, next-hop atom set.  The contributor lists are a property
// of the LSDB (built once per flattened area, RouteTable below); the walk over a prefix's list is
// route_cell_eval, one thread per (job, prefix) on the device (ospfv2_routes.cu).
//
// What a cell does not hold is decided on the host per job by hspf_ospfv2_routes_from_cells: atoms
// to interface next hops (needs the root's interface / neighbour state), SR labels per next hop
// (needs the neighbour's SRGB), max_paths truncation in next-hop order.
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>

#include "holo_lsdb.h"

struct hspf_ctx;

#if defined(__CUDACC__)
#define HSPF_HD __host__ __device__ __forceinline__
#else
#define HSPF_HD inline
#endif

namespace hspf {

// One (vertex, prefix) advertisement, in the order update_rib_intra_area meets them.
struct alignas(16) RouteContrib {
    uint32_t vertex;      // SPT vertex (flattener order)
    uint32_t origin_id;   // LSA id of the vertex's LSA (route.origin, route.rs:356-360)
    uint16_t metric;      // stub link metric; 0 for a transit network's own prefix
    uint16_t sid_class;   // 0: no usable Prefix-SID; else index of the SID descriptor (RouteTable::sids)
    uint8_t  is_network;  // the vertex is a transit network (route.rs:371-384: replaces instead of merging)
    uint8_t  _pad[3];
};
static_assert(sizeof(RouteContrib) == 16, "RouteContrib layout");

// Prefix-SID of an Extended-Prefix entry that update_rib_intra_area would attach (sr.rs:29-77)
struct SidDesc { uint32_t value; uint8_t flags; uint8_t is_label; };

struct RouteTable {
    // prefixes in route-table (Ipv4Network) order
    std::vector<uint32_t> prefix, plen;
    std::vector<uint32_t> off;               // [P+1] into contribs
    std::vector<RouteContrib> contribs;
    // static attributes of a contributor (what the winner gives the route)
    std::vector<uint8_t> origin_type;        // 1 router, 2 network
    std::vector<uint32_t> origin_adv;
    std::vector<SidDesc> sids;               // [0] unused
    uint32_t n_vertices = 0;
    // OSPFv3 tables (hspf_ospfv3_rtable_create): the prefixes proper; `prefix` is then zero-filled and `plen`
    // repeats len6, so that every consumer of the common part (kernel launch, harness) sees P entries
    std::vector<hl_ip_addr> prefix6;
    std::vector<uint8_t> options6;           // per contributor: prefix options of its advertisement
    bool v3 = false;
};

// Normalised view of one job's planes (32/64-bit or 16-bit planes).
struct PlanesWide {
    const uint32_t *dist; const uint16_t *hops; const uint64_t *nh;
    HSPF_HD bool reached(uint32_t v) const { return dist[v] != 0xFFFFFFFFu; }
    HSPF_HD uint32_t d(uint32_t v) const { return dist[v]; }
    HSPF_HD uint32_t h(uint32_t v) const { return hops[v]; }
    HSPF_HD uint64_t n(uint32_t v) const { return nh[v]; }
};
struct PlanesNarrow {
    const uint16_t *dist; const uint16_t *hops; const uint16_t *nh;
    HSPF_HD bool reached(uint32_t v) const { return dist[v] != 0xFFFFu; }
    HSPF_HD uint32_t d(uint32_t v) const { return dist[v]; }
    HSPF_HD uint32_t h(uint32_t v) const { return hops[v]; }
    HSPF_HD uint64_t n(uint32_t v) const { return nh[v]; }
};

// one 16-byte record, one load
HSPF_HD RouteContrib load_contrib(const RouteContrib *p) {
#if defined(__CUDA_ARCH__)
    const uint4 r = __ldg(reinterpret_cast<const uint4 *>(p));
    RouteContrib k;
    k.vertex = r.x; k.origin_id = r.y; k.metric = (uint16_t)(r.z & 0xFFFFu); k.sid_class = (uint16_t)(r.z >> 16);
    k.is_network = (uint8_t)(r.w & 0xFFu); k._pad[0] = k._pad[1] = k._pad[2] = 0;
    return k;
#else
    return *p;
#endif
}

// The walk of one prefix's contributors = the sequence of route_update calls update_rib_intra_area
// makes for that prefix (route.rs:362-443):
//   * a contributor off the SPT adds nothing;
//   * metric = distance + stub metric, clamped to u16 (route.rs:392);
//   * a worse metric than the current route's is dropped (route.rs:403-405 / 371-375);
//   * a transit network meeting an existing route replaces it unless its LSA id is lower
//     (route.rs:371-384, the RFC 2328 16.1 (4) tie-break), never merges;
//   * a stub with a better metric replaces, with an equal metric adds its next hops (route.rs:916-932).
// lasthop marks the atoms whose (last) contributor sits one hop from the root: their SR label is
// the penultimate-hop rule's (sr.rs:158-181).  A merge of contributors with different Prefix-SIDs
// is flagged: the host redoes that job's routes from the planes.
template <class Planes>
HSPF_HD hl_route_cell route_cell_eval(const Planes &pl, const RouteContrib *contribs, uint32_t begin, uint32_t end) {
    hl_route_cell c;
    c.nh_mask = 0; c.lasthop_mask = 0; c.winner = 0xFFFFFFFFu; c.metric = 0; c.flags = 0; c._pad = 0;
    uint32_t cur_origin = 0, cur_class = 0;
    for (uint32_t i = begin; i < end; ++i) {
        const RouteContrib k = load_contrib(contribs + i);
        if (!pl.reached(k.vertex)) continue;
        uint32_t m = pl.d(k.vertex) + k.metric;
        if (m > 0xFFFFu) m = 0xFFFFu;
        bool live = (c.flags & HL_CELL_PRESENT) != 0;
        if (live && m > c.metric) continue;
        if (k.is_network && live) {
            if (k.origin_id < cur_origin) continue;
            live = false;                                  // the old route is removed, not merged
        }
        const uint32_t h = pl.h(k.vertex);
        const uint64_t nh = pl.n(k.vertex);
        if (!live || m < c.metric) {
            c.metric = (uint16_t)m;
            c.winner = i;
            c.flags = (uint8_t)(HL_CELL_PRESENT | (h == 0 ? HL_CELL_CONNECTED : 0));
            c.nh_mask = nh;
            c.lasthop_mask = h == 1 ? nh : 0;
            cur_origin = k.origin_id;
            cur_class = k.sid_class;
        } else {
            if (k.sid_class != cur_class) c.flags |= HL_CELL_MIXED_SID;
            c.lasthop_mask = (c.lasthop_mask & ~nh) | (h == 1 ? nh : 0);
            c.nh_mask |= nh;
        }
    }
    return c;
}

// Device copy of a route table's `off` and contributor records, one allocation (route_stage.cu).  The
// functions are defined in the CUDA library only: the CPU test harnesses include this header without linking it.
struct DeviceRouteTable {
    void *blob = nullptr;
    const uint32_t *off = nullptr;
    const void *contribs = nullptr;
    int device = -1;
};
int upload_route_table(hspf_ctx *ctx, DeviceRouteTable &d, const std::vector<uint32_t> &off, const void *contribs,
                       size_t contrib_bytes);
void release_route_table(DeviceRouteTable &d);

}  // namespace hspf

// Host + device image of a flattened area's route table (include/holo_spf_lsdb.h).
struct hspf_ospfv2_rtable {
    hspf::RouteTable t;
    std::vector<int32_t> ext_of;       // per contributor: index of its Extended-Prefix entry, -1 if none usable
    hspf::DeviceRouteTable dev;        // hspf_ospfv2_rtable_upload
};
