// Routing table of a batch of OSPFv2 SPTs, one cell per (job, prefix), for roots attached to one area.
//
// With one active area, update_rib_full (holo-ospf/src/route.rs:146-193; ospf_rib_host.cc: rib_full) is one walk
// per prefix over what the LSDB says about it, in three steps that never mix (route_compare ranks the path type
// first):
//   1. intra-area: route_cell_eval over the prefix's advertisers (route_cells.h); a route found here wins;
//   2. inter-area (rib_full step 2): the area's usable type-3 LSAs for the prefix, in LSDB order, through an ABR
//      (Router-LSA B flag) the job reaches: dist[abr] + metric; the lowest wins, equal metrics OR their atoms;
//   3. AS-external (rib_full step 4): the type-5 LSAs for the prefix, in LSDB order, through the ASBR's entry as
//      rib_full leaves it after step 2 — the last usable type-4 LSA for the ASBR whose ABR the job reaches
//      (dist[abr] + metric, the ABR's atoms), else the ASBR's own vertex when it is reached and has the E flag;
//      ranked by path type, then type-2 metric, then metric; equal candidates OR their atoms, the first stays.
// Static filters (maxage, infinity, an ABR that is not a router vertex with the B flag) are applied when the
// table is built (hspf_ospfv2_ribtable_create); what depends on the job (reached, the root) is checked here.
// max_paths truncation is left to the decode: the first max_paths of the union in next-hop order are what
// truncating after every merge leaves.
#pragma once
#include <cstdint>
#include <vector>

#include "holo_spf.h"
#include "route_cells.h"
#include "route_delta.h"

namespace hspf {

// Every record of the table is 16 bytes: the intra-area RouteContribs of the area's rtable first, then the
// type-3, type-5, ASBR-slot and type-4 records, each one region of the record array (record index = winner).
struct alignas(16) RibRec { uint32_t x, y, z, w; };
static_assert(sizeof(RibRec) == sizeof(RouteContrib), "one record size");
//   type-3:  x ABR vertex, y LSA metric
//   type-5:  x record index of the ASBR's slot, y LSA metric, z E bit (type-2 metric)
//   slot:    x the ASBR's router vertex (0xFFFFFFFF: none), y 1 if that vertex has the E flag, [z, w) its type-4s
//   type-4:  x ABR vertex, y LSA metric

constexpr uint32_t kNoRecord = 0xFFFFFFFFu;

// What the walk reads of a table: off[3 (P + 1)] = intra, type-3 and type-5 ranges per prefix; the records;
// per vertex its Router-LSA flags (HL_RTR_FLAG_*).
struct RibView {
    const uint32_t *off;
    const RibRec *recs;
    const uint8_t *vflags;
    uint32_t P, V;
};

HSPF_HD RibRec load_rib_rec(const RibRec *p) {
#if defined(__CUDA_ARCH__)
    const uint4 r = __ldg(reinterpret_cast<const uint4 *>(p));
    return RibRec{r.x, r.y, r.z, r.w};
#else
    return *p;
#endif
}

HSPF_HD uint32_t rib_mpf(uint32_t metric, uint32_t path, uint32_t flags) { return HL_RIB_CELL_MPF(metric, path, flags); }

// The jobs the stage refuses (HSPF_JS_* bits added to the planes' status word): root out of range, or an ABR.
HSPF_HD uint32_t rib_job_refusal(const RibView &t, uint32_t root) {
    if (root >= t.V) return HSPF_JS_INVALID;
    return (t.vflags[root] & HL_RTR_FLAG_B) ? HSPF_JS_NOT_INTERNAL : 0u;
}

// The three words of the cell of prefix `p` for a job rooted at vertex `root` (< V) over that job's planes.
template <class Planes>
HSPF_HD CellWords ospf_rib_cell_eval(const Planes &pl, uint32_t root, const RibView &t, uint32_t p) {
    const RouteContrib *contribs = reinterpret_cast<const RouteContrib *>(t.recs);
    const hl_route_cell c = route_cell_eval(pl, contribs, t.off[p], t.off[p + 1]);
    if (c.flags & HL_CELL_PRESENT)
        return {c.nh_mask, c.lasthop_mask, (uint64_t)c.winner | ((uint64_t)rib_mpf(c.metric, HL_PATH_INTRA_AREA, c.flags) << 32)};
    const uint32_t *o3 = t.off + t.P + 1, *o5 = o3 + t.P + 1;
    uint64_t mask = 0;
    uint32_t win = kNoRecord, metric = 0;
    for (uint32_t i = o3[p]; i < o3[p + 1]; ++i) {                      // 2. inter-area
        const RibRec r = load_rib_rec(t.recs + i);
        if (r.x == root || !pl.reached(r.x)) continue;
        const uint32_t m = pl.d(r.x) + r.y;
        if (win == kNoRecord || m < metric) { win = i; metric = m; mask = pl.n(r.x); }
        else if (m == metric) mask |= pl.n(r.x);
    }
    if (win != kNoRecord)
        return {mask, 0, (uint64_t)win | ((uint64_t)rib_mpf(metric, HL_PATH_INTER_AREA, HL_CELL_PRESENT) << 32)};
    uint32_t path = 0, type2 = 0;
    for (uint32_t i = o5[p]; i < o5[p + 1]; ++i) {                      // 3. AS-external
        const RibRec r = load_rib_rec(t.recs + i);
        const RibRec s = load_rib_rec(t.recs + r.x);
        if (s.x == root) continue;                                      // self-originated
        uint32_t em = 0;
        uint64_t en = 0;
        bool have = false;
        for (uint32_t k = s.w; k > s.z; --k) {                          // the last type-4 whose ABR is reached
            const RibRec q = load_rib_rec(t.recs + k - 1);
            if (q.x == root || !pl.reached(q.x)) continue;
            em = pl.d(q.x) + q.y; en = pl.n(q.x); have = true;
            break;
        }
        if (!have) {
            if (!s.y || !pl.reached(s.x)) continue;                     // s.y: s.x is a vertex with the E flag
            em = pl.d(s.x); en = pl.n(s.x);
        }
        const uint32_t cp = r.z ? HL_PATH_TYPE2_EXTERNAL : HL_PATH_TYPE1_EXTERNAL;
        const uint32_t cm = r.z ? em : em + r.y, c2 = r.z ? r.y : 0;
        int cmp = -1;                                                   // route_compare of the candidate and the winner
        if (win != kNoRecord) {
            if (cp != path) cmp = cp < path ? -1 : 1;
            else if (cp == HL_PATH_TYPE2_EXTERNAL && c2 != type2) cmp = c2 < type2 ? -1 : 1;
            else cmp = cm < metric ? -1 : (cm == metric ? 0 : 1);
        }
        if (cmp < 0) { win = i; path = cp; metric = cm; type2 = c2; mask = en; }
        else if (cmp == 0) mask |= en;
    }
    if (win == kNoRecord) return {0, 0, (uint64_t)kNoRecord};
    return {mask, type2, (uint64_t)win | ((uint64_t)rib_mpf(metric, path, HL_CELL_PRESENT) << 32)};
}

}  // namespace hspf

// Host image of an area's routing-table records (include/holo_spf_lsdb.h, hspf_ospfv2_ribtable_create).
struct hspf_ospfv2_ribtable {
    hspf_ospfv2_rtable *intra = nullptr;     // the area's intra-area table: records [0, n_intra) are its contribs
    uint32_t area_id = 0;
    std::vector<uint32_t> prefix, plen;      // prefix order; type-3 / type-5 prefixes keep their host bits
    std::vector<uint32_t> intra_of;          // per prefix: its index in `intra`, 0xFFFFFFFF if none
    std::vector<uint32_t> off;               // [3 (P + 1)]: intra, type-3, type-5 record ranges per prefix
    std::vector<hspf::RibRec> recs;
    std::vector<uint8_t> vflags;             // [V] Router-LSA flags of router vertices
    uint32_t n_intra = 0, ext_base = 0, ext_end = 0;
    std::vector<uint32_t> ext_tag;           // per type-5 record (index - ext_base): the LSA's tag
    std::vector<uint32_t> asbr_id;           // per ASBR record (index - ext_end): the ASBR's router id
    // OSPFv3 tables (hspf_ospfv3_ribtable_create): `intra` is an OSPFv3 rtable, `prefix` is zero-filled (the prefixes
    // are intra->t.prefix6 merged with the LSAs' in prefix6), and options6 holds the prefix options per type-3 /
    // type-5 record (index - n_intra)
    bool v3 = false;
    std::vector<hl_ip_addr> prefix6;
    std::vector<uint8_t> options6;
    hspf::DeviceRouteTable dev;             // hspf_ospfv2_ribtable_upload: off, then records + vflags
    hspf::RibView host_view() const {
        return hspf::RibView{off.data(), recs.data(), vflags.data(), (uint32_t)prefix.size(), (uint32_t)vflags.size()};
    }
};
