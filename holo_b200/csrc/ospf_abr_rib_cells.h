// Routing table of a batch of OSPFv2 SPTs for one area border router, one cell per (job, prefix), over every area
// the router is attached to (include/holo_spf_lsdb.h, hspf_ospfv2_abr_ribtable_create).
//
// update_rib_full (ospf_rib_host.cc: rib_full) over several areas is still one walk per prefix; what a prefix
// becomes depends only on its own records and on the plane values of the vertices they name, each in its own area:
//   1. intra-area: route_cell_eval over each area's advertisers, in area order, folded as rib_full folds the areas'
//      routes: a worse metric is dropped; a route whose LS origin is a transit network replaces the entry unless its
//      LSA id is lower; otherwise the lower metric replaces and an equal one ORs the atoms (the first winner stays);
//   2. inter-area: the type-3 records of the areas step 2 reads (only the backbone when more than one area is
//      active), through an ABR reached in that area; the lowest metric wins, equal metrics OR their atoms;
//   3. transit areas: an area some V-flag router of which the job reaches (the root counts) offers its type-3
//      records again, in area order; each may lower or tie the route only while it is intra- or inter-area and
//      belongs to area 0, which is checked again after every record;
//   4. AS-external: each type-5 record through the best ASBR entry over the areas in area-id order (an intra-area
//      entry through a non-backbone area first, then the lower metric, then the higher area id); an entry is the
//      last usable type-4 whose ABR is reached (areas step 2 reads), else the ASBR's own vertex with the E flag.
// Atom a of area i is bit base_i + a of the cell's masks.  A merge of intra-area routes of two areas, or of a
// transit-area route into an intra-area one, is flagged HL_CELL_MIXED_SID when a Prefix-SID is involved: the
// per-hop labels of the other area's hops are not in the cell.  Static filters (maxage, infinity, an ABR that is
// not a B-flag router vertex, self-originated LSAs) are applied when the table is built.
#pragma once
#include <cstdint>
#include <unordered_map>

#include "ospf_rib_cells.h"

namespace hspf {

constexpr uint32_t kAbrMaxAreas = 8;     // attached areas of one table (the kernel parameter holds them all)

// What the walk reads of a table.  off[(2 A + 1) (P + 1)]: per area its intra-area ranges, then per area its
// type-3 ranges, then the type-5 ranges.  Records as in ospf_rib_cells.h, except that a type-5 record's x is the
// first of A slot records (one per area, in area order) and type-3 / type-4 x is a vertex of that record's area.
// v_flagged[vl_off[i], vl_off[i + 1]) are the router vertices of area i with the V flag.
struct AbrRibView {
    const uint32_t *off;
    const RibRec *recs;
    const uint32_t *v_flagged;
    uint32_t P, n_areas;
    uint32_t step2;                      // bit i: step 2 reads area i's summaries
    uint32_t base[kAbrMaxAreas];         // atom base of area i
    uint32_t area_id[kAbrMaxAreas];
    uint32_t by_id[kAbrMaxAreas];        // area indices in area-id order (stable)
    uint32_t vl_off[kAbrMaxAreas + 1];
};

// Each area's planes: rows of V[i] vertices, n_rows[i] of them, and their status words (may be NULL).
template <class D, class N>
struct AbrPlaneSet {
    const D *dist[kAbrMaxAreas];
    const uint16_t *hops[kAbrMaxAreas];
    const N *nh[kAbrMaxAreas];
    const uint32_t *status[kAbrMaxAreas];
    uint32_t V[kAbrMaxAreas], n_rows[kAbrMaxAreas];
};

// The planes of one job, whose row of area i is row[i] (< n_rows[i]).
template <class Planes, class D, class N>
struct AbrJobPlanes {
    const AbrPlaneSet<D, N> &s;
    const uint32_t *row;
    HSPF_HD Planes operator()(uint32_t i) const {
        const size_t b = (size_t)row[i] * s.V[i];
        return Planes{s.dist[i] + b, s.hops[i] + b, s.nh[i] + b};
    }
};

// The job's status word: the OR of its rows' words, HSPF_JS_INVALID for a row out of range.
template <class D, class N>
HSPF_HD uint32_t abr_job_status(const AbrPlaneSet<D, N> &s, uint32_t n_areas, const uint32_t *row) {
    uint32_t st = 0;
    for (uint32_t i = 0; i < n_areas; ++i) {
        if (row[i] >= s.n_rows[i]) st |= HSPF_JS_INVALID;
        else if (s.status[i]) st |= s.status[i][row[i]];
    }
    return st;
}

// `plane(i)` gives the job's Planes of area i.
template <class Planes, class PF>
HSPF_HD bool abr_transit(const PF &plane, const AbrRibView &t, uint32_t i) {
    const Planes pl = plane(i);
    for (uint32_t k = t.vl_off[i]; k < t.vl_off[i + 1]; ++k)
        if (pl.reached(t.v_flagged[k])) return true;
    return false;
}

// The slots of a walk without them (kSlots off).
struct AbrNoSlots {};

// kSlots (hspf_ospfv2_abr_backbone_table_create, ospf_backbone_cells.h: AbrBorderSlots): a type-3 record that step 2
// reads may be a slot, which `slots.offer` turns into the border's advertisement (or drops), and a type-4 record
// with Slots::kAsbrSlot in w is a type-4 slot, skipped unless plane.asbr says its border originates.
template <class Planes, bool kSlots = false, class PF, class Slots = AbrNoSlots>
HSPF_HD CellWords abr_rib_cell_eval(const PF &plane, const AbrRibView &t, uint32_t p, const Slots &slots = Slots{}) {
    const uint32_t A = t.n_areas, S = t.P + 1;
    const RouteContrib *contribs = reinterpret_cast<const RouteContrib *>(t.recs);
    const uint32_t *o3 = t.off + (size_t)A * S, *o5 = o3 + (size_t)A * S;
    uint64_t mask = 0, aux = 0;
    uint32_t win = kNoRecord, metric = 0, flags = 0, origin = 0, area = 0, path = HL_PATH_INTRA_AREA;
    for (uint32_t i = 0; i < A; ++i) {                                  // 1. intra-area, area by area
        const uint32_t b = t.off[i * S + p], e = t.off[i * S + p + 1];
        if (b == e) continue;
        const hl_route_cell c = route_cell_eval(plane(i), contribs, b, e);
        if (!(c.flags & HL_CELL_PRESENT)) continue;
        const RouteContrib w = load_contrib(contribs + c.winner);
        const uint64_t n = c.nh_mask << t.base[i], l = c.lasthop_mask << t.base[i];
        if (win != kNoRecord) {
            if (c.metric > metric) continue;
            if (w.is_network) {
                if (w.origin_id < origin) continue;
            } else if (c.metric == metric) {
                if (w.sid_class || load_contrib(contribs + win).sid_class) flags |= HL_CELL_MIXED_SID;
                flags |= c.flags & HL_CELL_MIXED_SID;
                mask |= n; aux |= l;
                continue;
            }
        }
        win = c.winner; metric = c.metric; flags = c.flags; mask = n; aux = l; origin = w.origin_id; area = i;
    }
    if (win == kNoRecord) {                                             // 2. inter-area
        for (uint32_t i = 0; i < A; ++i) {
            if (!((t.step2 >> i) & 1u) || o3[i * S + p] == o3[i * S + p + 1]) continue;
            const Planes pl = plane(i);
            for (uint32_t k = o3[i * S + p]; k < o3[i * S + p + 1]; ++k) {
                const RibRec r = load_rib_rec(t.recs + k);
                if (!pl.reached(r.x)) continue;
                uint32_t y = r.y, w = k;
                if constexpr (kSlots) {
                    if (!slots.offer(r, y, w)) continue;
                }
                const uint32_t m = pl.d(r.x) + y;
                const uint64_t n = pl.n(r.x) << t.base[i];
                if (win == kNoRecord || m < metric) { win = w; metric = m; mask = n; area = i; }
                else if (m == metric) mask |= n;
            }
        }
        if (win != kNoRecord) { path = HL_PATH_INTER_AREA; flags = HL_CELL_PRESENT; aux = 0; }
    }
    if (win != kNoRecord) {                                             // 3. transit areas
        for (uint32_t i = 0; i < A && t.area_id[area] == 0; ++i) {
            if (o3[i * S + p] == o3[i * S + p + 1] || !abr_transit<Planes>(plane, t, i)) continue;
            const Planes pl = plane(i);
            for (uint32_t k = o3[i * S + p]; k < o3[i * S + p + 1] && t.area_id[area] == 0; ++k) {
                const RibRec r = load_rib_rec(t.recs + k);
                if (!pl.reached(r.x)) continue;
                const uint32_t m = pl.d(r.x) + r.y;
                const uint64_t n = pl.n(r.x) << t.base[i];
                if (m < metric) {
                    win = k; metric = m; mask = n; aux = 0; area = i;
                    path = HL_PATH_INTER_AREA; flags = HL_CELL_PRESENT;
                } else if (m == metric) {
                    if (path == HL_PATH_INTRA_AREA && load_contrib(contribs + win).sid_class) flags |= HL_CELL_MIXED_SID;
                    mask |= n;
                }
            }
        }
        return {mask, aux, (uint64_t)win | ((uint64_t)rib_mpf(metric, path, flags) << 32)};
    }
    uint32_t type2 = 0;                                                 // 4. AS-external
    for (uint32_t k = o5[p]; k < o5[p + 1]; ++k) {
        const RibRec r = load_rib_rec(t.recs + k);
        bool have = false, best_pref = false;
        uint32_t em = 0, best_id = 0;
        uint64_t en = 0;
        for (uint32_t q = 0; q < A; ++q) {
            const uint32_t i = t.by_id[q];
            const RibRec s = load_rib_rec(t.recs + r.x + i);
            const Planes pl = plane(i);
            uint32_t m = 0;
            uint64_t n = 0;
            bool found = false, intra = false;
            for (uint32_t j = s.w; j > s.z; --j) {                      // the last type-4 whose ABR is reached
                const RibRec f = load_rib_rec(t.recs + j - 1);
                if (!pl.reached(f.x)) continue;
                uint32_t fm = f.y;                                      // a border that does not originate: go on
                if constexpr (kSlots) {
                    if ((f.w & Slots::kAsbrSlot) && !plane.asbr.originates(f.w & ~Slots::kAsbrSlot, f.y, fm)) continue;
                }
                m = pl.d(f.x) + fm; n = pl.n(f.x); found = true;
                break;
            }
            if (!found) {
                if (!s.y || !pl.reached(s.x)) continue;                 // s.y: s.x is a vertex with the E flag
                m = pl.d(s.x); n = pl.n(s.x); intra = true;
            }
            const bool pref = intra && t.area_id[i] != 0;
            if (have && !(pref && !best_pref)) {
                if (pref != best_pref) continue;
                if (!(m < em || (m == em && t.area_id[i] > best_id))) continue;
            }
            have = true; best_pref = pref; em = m; en = n << t.base[i]; best_id = t.area_id[i];
        }
        if (!have) continue;
        const uint32_t cp = r.z ? HL_PATH_TYPE2_EXTERNAL : HL_PATH_TYPE1_EXTERNAL;
        const uint32_t cm = r.z ? em : em + r.y, c2 = r.z ? r.y : 0;
        int cmp = -1;                                                   // route_compare of the candidate and the winner
        if (win != kNoRecord) {
            if (cp != path) cmp = cp < path ? -1 : 1;
            else if (cp == HL_PATH_TYPE2_EXTERNAL && c2 != type2) cmp = c2 < type2 ? -1 : 1;
            else cmp = cm < metric ? -1 : (cm == metric ? 0 : 1);
        }
        if (cmp < 0) { win = k; path = cp; metric = cm; type2 = c2; mask = en; }
        else if (cmp == 0) mask |= en;
    }
    if (win == kNoRecord) return {0, 0, (uint64_t)kNoRecord};
    return {mask, type2, (uint64_t)win | ((uint64_t)rib_mpf(metric, path, HL_CELL_PRESENT) << 32)};
}

}  // namespace hspf

// Host image of an ABR's routing-table records (include/holo_spf_lsdb.h, hspf_ospfv2_abr_ribtable_create).
struct hspf_ospfv2_abr_ribtable {
    uint32_t router_id = 0, n_areas = 0, max_paths = 0, step2 = 0;
    std::vector<hspf_ospfv2_ribtable *> area;     // per area: its one-area table (intra-area records, per-area maps)
    std::vector<uint32_t> area_id, root, n_vertices, base, n_atoms;
    std::vector<uint32_t> intra_base, t3_base;    // per area: first record of its intra-area / type-3 records, and
    uint32_t t3_end = 0, ext_base = 0, ext_end = 0;
    std::vector<std::vector<uint32_t>> area_prefix;   // per area, per prefix: the prefix's index in area[i], or kNoRecord
    std::vector<uint32_t> prefix, plen;
    std::vector<uint32_t> off;                     // [(2 A + 1)(P + 1)]
    std::vector<hspf::RibRec> recs;
    std::vector<uint32_t> v_flagged, vl_off;
    std::vector<uint32_t> ext_tag;                 // per type-5 record (index - ext_base)
    std::vector<uint32_t> group_asbr;              // per ASBR entry group (records ext_end + A g ..): the ASBR's id
    std::vector<std::unordered_map<uint32_t, uint32_t>> rtr_vertex;   // per area: router id -> router vertex
    // OSPFv3 tables (hspf_ospfv3_abr_ribtable_create): each area's table is an OSPFv3 one-area table, `prefix` is
    // zero-filled (the prefixes are prefix6), and options6 holds the prefix options per type-3 / type-5 record
    // (index - t3_base[0], the first type-3 record)
    bool v3 = false;
    std::vector<hl_ip_addr> prefix6;
    std::vector<uint8_t> options6;
    hspf::DeviceRouteTable dev;                    // off, then records + v_flagged
    hspf::AbrRibView view(const uint32_t *o, const hspf::RibRec *r, const uint32_t *vf) const {
        hspf::AbrRibView t{};
        t.off = o; t.recs = r; t.v_flagged = vf;
        t.P = (uint32_t)prefix.size(); t.n_areas = n_areas; t.step2 = step2;
        for (uint32_t i = 0; i < n_areas; ++i) { t.base[i] = base[i]; t.area_id[i] = area_id[i]; t.by_id[i] = i; }
        for (uint32_t i = 1; i < n_areas; ++i)                                      // stable insertion sort by area id
            for (uint32_t k = i; k > 0 && area_id[t.by_id[k - 1]] > area_id[t.by_id[k]]; --k) {
                const uint32_t x = t.by_id[k]; t.by_id[k] = t.by_id[k - 1]; t.by_id[k - 1] = x;
            }
        for (uint32_t i = 0; i <= n_areas; ++i) t.vl_off[i] = vl_off[i];
        return t;
    }
    hspf::AbrRibView host_view() const { return view(off.data(), recs.data(), v_flagged.data()); }
};
