// The two host halves of the OSPF routing-table stage, each written once over a small version trait, as rib_full is
// in ospf_rib_host.cc.  Host only.
//   build_rib_records  the record-building half of hspf_ospfv2_ribtable_create / hspf_ospfv3_ribtable_create
//                      (include/holo_spf_lsdb.h).  The versions differ only in the prefix key, in which field of an
//                      inter-area-router LSA names the ASBR, and in the NU-bit LSAs OSPFv3 skips; the records the walk
//                      reads (ospf_rib_cells.h) are the same.
//   build_abr_ribtable hspf_ospfv2_abr_ribtable_create / hspf_ospfv3_abr_ribtable_create: an area border router's
//                      records over the one-area tables of its areas (ospf_abr_rib_cells.h)
//   build_backbone_table  hspf_ospfv2_backbone_table_create / hspf_ospfv3_backbone_table_create: a backbone router's
//                      affected prefixes over its one-area table and its borders' ABR tables (ospf_backbone_cells.h);
//                      hspf_ospfv{2,3}_nonbackbone_table_create: the same for an internal router of a non-backbone
//                      area
//   build_abr_backbone_table  hspf_ospfv2_abr_backbone_table_create / hspf_ospfv3_abr_backbone_table_create: an area
//                      border router's affected prefixes over its ABR table and the borders' (build_abr_ribtable, and
//                      the slot and border-word helpers build_backbone_table shares)
//   decode_rib         one job's cells -> its routing table, for hspf_ospfv2_rib_from_cells,
//                      hspf_ospfv3_rib_from_cells, hspf_ospfv{2,3}_abr_rib_from_cells (decode_abr_rib),
//                      hspf_ospfv{2,3}_backbone_from_cells (decode_backbone_rib) and
//                      hspf_ospfv{2,3}_abr_backbone_from_cells (decode_abr_backbone_rib).  A one-area table decodes as an area
//                      border router's table with a single area.
//
// For build_rib_records a version trait T provides:
//   Key                        prefix key; its order is the table's prefix order (update_rib_full's IpNetwork order)
//   Sum, Ext                   the summary / inter-area LSA and the AS-external LSA
//   key(Sum), key(Ext)         the LSA's prefix key (host bits kept, as update_rib_full keeps them)
//   intra_key(RouteTable, k)   the key of prefix k of the area's intra-area table
//   skip(Sum), skip(Ext)       LSAs update_rib_full never uses whatever the job (OSPFv3: NU bit)
//   asbr_id(Sum)               the ASBR a type-4 LSA names
//   options(Sum), options(Ext) prefix options a route through the LSA carries
//   set_prefix(rt, u, Key)     writes prefix u of the table (a one-area or an ABR table)
//   kV3                        the table carries OSPFv3 prefixes and per-record prefix options
//
// For build_abr_ribtable it also provides:
//   Flat                       the version's flattened area; its `area` is the area's image
//   root_vertex(f, id)         the router vertex of router `id` in f, or 0xFFFFFFFF
//   n_vertices(f)              f's vertex count
//   atom_count(f, root, &n)    hspf_atom_count over f's CSR
//   area_table(f, id, sums, n_sums, ext, n_ext, transit_walk, &rt)  the area's one-area table (build_rib_records'
//                              transit_walk)
//   table_key(rt, u)           the key of prefix u of a one-area or an ABR table
//
// For build_backbone_table it also provides:
//   router_flags(f, v)         the Router-LSA flags of router vertex v of f (its first fragment's)
//   default_key()              the key of the default route (0.0.0.0/0, ::/0)
//
// For decode_rib it also provides:
//   Area, Rib                  the area image and the caller's output
//   Route, Hop                 a route and a next hop of that output
//   Result, Net                intra_from_cells' output and one route of it
//   Nh, JobDecode              a resolved next hop; one job's decode state over one area (flattened area, root,
//                              Resolver `rs`)
//   intra_from_cells           the intra-area decode of one area's cells (hspf_ospfv{2,3}_routes_from_cells' body)
//   nh_less, nh_same           next-hop order (NexthopKey) and same key
//   nh_conflict(a, b)          a and b have one key, but attributes the cell cannot choose between
//   route_prefix(o, d, u)      writes prefix u of the decode into the route (v2 prefix / mask, v3 prefix6 / len)
//   from_intra(o, net)         what a route takes from its intra-area route (v2 SR label, v3 prefix options)
//   from_record(o, d, rec)     what it takes from type-3 / type-5 record `rec` of the decoded table (v3: d.options)
//   to_nh(hop, sort), to_hop   a next hop into the merged set, naming its interface's sort key, and back out
#pragma once
#include <algorithm>
#include <array>
#include <cstdint>
#include <cstring>
#include <map>
#include <memory>
#include <new>
#include <numeric>
#include <unordered_map>
#include <vector>

#include "holo_spf_lsdb.h"
#include "ospf_abr_rib_cells.h"
#include "ospf_backbone_cells.h"
#include "ospf_rib_cells.h"

namespace hspf {

// rt arrives with vflags filled and rt.intra built; `router_vertex(id)` is the vertex of router `id`, or
// 0xFFFFFFFF.  Fills everything else; HSPF_E_UNSUPPORTED for the tables the walk cannot answer.  `transit_walk`:
// the table is one area of an ABR's table (ospf_abr_rib_cells.h), whose walk has the transit-area step.
template <class T, class RouterVertex>
int build_rib_records(hspf_ospfv2_ribtable &rt, uint32_t area_id, RouterVertex router_vertex, const typename T::Sum *sums,
                      uint32_t n_sums, const typename T::Ext *ext, uint32_t n_ext, bool transit_walk = false) {
    using Key = typename T::Key;
    constexpr uint32_t kNone = 0xFFFFFFFFu;
    // the largest metric a cell holds: a type-1 external behind a type-4 entry, over a distance below saturation
    static_assert(0xFFFEull + 2ull * (HL_LSA_INFINITY - 1) <= HL_RIB_CELL_METRIC_MAX, "cell metric field");
    rt.area_id = area_id;
    rt.v3 = T::kV3;
    const uint32_t V = (uint32_t)rt.vflags.size();
    // rib_full step 3 (transit areas) can rewrite the backbone's intra-area routes when it has virtual links
    if (area_id == 0 && !transit_walk)
        for (uint32_t v = 0; v < V; ++v)
            if (rt.vflags[v] & HL_RTR_FLAG_V) return HSPF_E_UNSUPPORTED;
    auto has_flag = [&](uint32_t v, uint8_t flag) { return v != kNone && (rt.vflags[v] & flag) != 0; };
    auto live = [](uint8_t maxage, uint32_t metric) { return !maxage && metric < HL_LSA_INFINITY; };
    const RouteTable &it = rt.intra->t;

    struct Keyed { Key key; RibRec r; uint32_t tag; uint8_t options; };
    std::vector<Keyed> t3, t5;
    std::unordered_map<uint32_t, uint32_t> slot_of;        // ASBR router id -> slot
    std::vector<uint32_t> slot_id;
    std::vector<std::vector<RibRec>> t4;                    // per slot, LSDB order
    auto slot = [&](uint32_t id) {
        auto ins = slot_of.emplace(id, (uint32_t)slot_id.size());
        if (ins.second) { slot_id.push_back(id); t4.emplace_back(); }
        return ins.first->second;
    };
    for (uint32_t i = 0; i < n_sums; ++i) {
        const auto &l = sums[i];
        if (!live(l.maxage, l.metric) || T::skip(l)) continue;
        const uint32_t abr = router_vertex(l.adv_rtr);
        if (!has_flag(abr, HL_RTR_FLAG_B)) continue;                 // abr(): a router entry with the B flag
        if (l.lsa_type == 3) {
            t3.push_back({T::key(l), RibRec{abr, l.metric, 0, 0}, 0, T::options(l)});
        } else if (l.lsa_type == 4) {
            // the entry a type-4 LSA writes replaces the named router's: were that an ABR, later type-4 LSAs
            // would see abr() change under them
            if (has_flag(router_vertex(T::asbr_id(l)), HL_RTR_FLAG_B)) return HSPF_E_UNSUPPORTED;
            t4[slot(T::asbr_id(l))].push_back(RibRec{abr, l.metric, 0, 0});
        }
    }
    for (uint32_t i = 0; i < n_ext; ++i) {
        const auto &l = ext[i];
        if (!live(l.maxage, l.metric) || T::skip(l)) continue;
        t5.push_back({T::key(l), RibRec{slot(l.adv_rtr), l.metric, l.e_bit ? 1u : 0u, 0}, l.tag, T::options(l)});
    }
    auto by_key = [](const Keyed &x, const Keyed &y) { return x.key < y.key; };
    std::stable_sort(t3.begin(), t3.end(), by_key);        // LSDB order within a prefix
    std::stable_sort(t5.begin(), t5.end(), by_key);
    const uint32_t PI = (uint32_t)it.plen.size();
    std::vector<Key> keys;
    keys.reserve(PI + t3.size() + t5.size());
    for (uint32_t k = 0; k < PI; ++k) {
        keys.push_back(T::intra_key(it, k));
        // the intra-area table is in the same order: merging below walks it once
        if (k && !(keys[k - 1] < keys[k])) return HSPF_E_UNSUPPORTED;
    }
    for (const Keyed &x : t3) keys.push_back(x.key);
    for (const Keyed &x : t5) keys.push_back(x.key);
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    const uint32_t P = (uint32_t)keys.size();
    rt.n_intra = (uint32_t)it.contribs.size();
    const uint64_t n_slots = slot_id.size(), slot_base = (uint64_t)rt.n_intra + t3.size() + t5.size();
    uint64_t n_t4 = 0;
    for (const auto &l : t4) n_t4 += l.size();
    if (slot_base + n_slots + n_t4 >= kNone) return HSPF_E_UNSUPPORTED;      // record indices are u32
    rt.recs.resize(rt.n_intra);
    if (rt.n_intra) std::memcpy(rt.recs.data(), it.contribs.data(), rt.n_intra * sizeof(RibRec));
    rt.prefix.resize(P); rt.plen.resize(P); rt.intra_of.assign(P, kNone);
    if (T::kV3) rt.prefix6.resize(P);
    rt.off.assign(3 * ((size_t)P + 1), 0);
    uint32_t *oi = rt.off.data(), *o3 = oi + P + 1, *o5 = o3 + P + 1;
    uint32_t k = 0;
    for (uint32_t u = 0; u < P; ++u) {
        T::set_prefix(rt, u, keys[u]);
        oi[u] = it.off[k];                                  // an empty range where the prefix has no intra record
        if (k < PI && T::intra_key(it, k) == keys[u]) rt.intra_of[u] = k++;
    }
    oi[P] = rt.n_intra;
    size_t q = 0;
    for (uint32_t u = 0; u < P; ++u) {
        o3[u] = (uint32_t)rt.recs.size();
        for (; q < t3.size() && t3[q].key == keys[u]; ++q) {
            rt.recs.push_back(t3[q].r);
            if (T::kV3) rt.options6.push_back(t3[q].options);
        }
    }
    o3[P] = (uint32_t)rt.recs.size();
    rt.ext_base = o3[P];
    q = 0;
    for (uint32_t u = 0; u < P; ++u) {
        o5[u] = (uint32_t)rt.recs.size();
        for (; q < t5.size() && t5[q].key == keys[u]; ++q) {
            RibRec r = t5[q].r;
            r.x += (uint32_t)slot_base;
            rt.recs.push_back(r);
            rt.ext_tag.push_back(t5[q].tag);
            if (T::kV3) rt.options6.push_back(t5[q].options);
        }
    }
    o5[P] = (uint32_t)rt.recs.size();
    rt.ext_end = o5[P];
    uint32_t t4_at = (uint32_t)(slot_base + n_slots);
    for (uint32_t s = 0; s < n_slots; ++s) {
        const uint32_t v = router_vertex(slot_id[s]);
        rt.recs.push_back(RibRec{v, has_flag(v, HL_RTR_FLAG_E) ? 1u : 0u, t4_at, t4_at + (uint32_t)t4[s].size()});
        t4_at += (uint32_t)t4[s].size();
    }
    for (const auto &l : t4) rt.recs.insert(rt.recs.end(), l.begin(), l.end());
    rt.asbr_id = slot_id;
    return HSPF_OK;
}

// hspf_ospfv2_abr_ribtable_create / hspf_ospfv3_abr_ribtable_create, argument checks included: each area's one-area
// table with the transit-area walk, then the router's records over all of them (ospf_abr_rib_cells.h).
template <class T>
int build_abr_ribtable(uint32_t router_id, uint32_t n_areas, const typename T::Flat *const *flats,
                       const uint32_t *area_ids, const typename T::Sum *const *summaries, const uint32_t *n_summaries,
                       const uint8_t *active, const typename T::Ext *ext, uint32_t n_ext,
                       hspf_ospfv2_abr_ribtable **out) {
    using Key = typename T::Key;
    if (!out || !flats || !area_ids || n_areas == 0 || (n_ext && !ext)) return HSPF_E_INVAL;
    *out = nullptr;
    if (n_areas > kAbrMaxAreas) return HSPF_E_UNSUPPORTED;
    for (uint32_t i = 0; i < n_areas; ++i) {
        if (!flats[i] || !flats[i]->area) return HSPF_E_INVAL;
        if (n_summaries && n_summaries[i] && (!summaries || !summaries[i])) return HSPF_E_INVAL;
    }
    try {
        std::unique_ptr<hspf_ospfv2_abr_ribtable, void (*)(hspf_ospfv2_abr_ribtable *)> t(
            new hspf_ospfv2_abr_ribtable(), hspf_ospfv2_abr_ribtable_free);
        const uint32_t A = n_areas;
        t->router_id = router_id;
        t->n_areas = A;
        t->v3 = T::kV3;
        uint32_t n_active = 0;
        for (uint32_t i = 0; i < A; ++i) n_active += (!active || active[i]) ? 1u : 0u;
        uint32_t atoms = 0;
        for (uint32_t i = 0; i < A; ++i) {
            const typename T::Flat &f = *flats[i];
            if (i == 0) t->max_paths = f.area->max_paths;
            else if (f.area->max_paths != t->max_paths) return HSPF_E_INVAL;   // one instance, one max_paths
            const uint32_t root = T::root_vertex(f, router_id);
            if (root == kNoRecord) return HSPF_E_INVAL;                        // the caller leaves that area out
            uint32_t na = 0;
            int rc = T::atom_count(f, root, &na);
            if (rc) return rc;
            t->base.push_back(na ? atoms : 0);
            t->n_atoms.push_back(na);
            atoms += na;
            if (atoms > 64) return HSPF_E_UNSUPPORTED;                         // the cell's masks are 64 bits
            // rib_full step 2 reads every area's summaries with one active area, else only the backbone's; the
            // other areas' type-3 LSAs are still offered by the transit-area step
            const bool step2 = n_active <= 1 || area_ids[i] == 0;
            if (step2) t->step2 |= 1u << i;
            const uint32_t ns = n_summaries ? n_summaries[i] : 0;
            std::vector<typename T::Sum> sums;
            for (uint32_t k = 0; k < ns; ++k)
                if (step2 || summaries[i][k].lsa_type == 3) sums.push_back(summaries[i][k]);
            hspf_ospfv2_ribtable *rt = nullptr;
            rc = T::area_table(flats[i], area_ids[i], sums.data(), (uint32_t)sums.size(), ext, n_ext, true, &rt);
            if (rc) return rc;
            t->area.push_back(rt);
            t->rtr_vertex.push_back(f.rtr_vertex);
            t->area_id.push_back(area_ids[i]);
            t->root.push_back(root);
            t->n_vertices.push_back(T::n_vertices(f));
        }
        // the prefixes: the union of the areas' in prefix order
        std::vector<Key> keys;
        for (const hspf_ospfv2_ribtable *rt : t->area)
            for (uint32_t u = 0; u < (uint32_t)rt->plen.size(); ++u) keys.push_back(T::table_key(*rt, u));
        std::sort(keys.begin(), keys.end());
        keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
        const uint32_t P = (uint32_t)keys.size(), S = P + 1;
        t->prefix.resize(P); t->plen.resize(P);
        if (T::kV3) t->prefix6.resize(P);
        for (uint32_t u = 0; u < P; ++u) T::set_prefix(*t, u, keys[u]);
        t->area_prefix.assign(A, std::vector<uint32_t>(P, kNoRecord));
        std::vector<std::vector<uint32_t>> first_at(A, std::vector<uint32_t>(P));   // first area prefix >= keys[u]
        for (uint32_t i = 0; i < A; ++i) {
            const hspf_ospfv2_ribtable &rt = *t->area[i];
            uint32_t q = 0;
            for (uint32_t u = 0; u < P; ++u) {
                first_at[i][u] = q;
                if (q < rt.plen.size() && T::table_key(rt, q) == keys[u]) t->area_prefix[i][u] = q++;
            }
        }
        t->off.assign((2 * (size_t)A + 1) * S, 0);
        uint32_t *o3 = t->off.data() + (size_t)A * S, *o5 = o3 + (size_t)A * S;
        auto &recs = t->recs;
        for (uint32_t i = 0; i < A; ++i) {                                  // intra-area records, area by area
            const hspf_ospfv2_ribtable &rt = *t->area[i];
            const uint32_t b = (uint32_t)recs.size();
            t->intra_base.push_back(b);
            recs.insert(recs.end(), rt.recs.begin(), rt.recs.begin() + rt.n_intra);
            for (uint32_t u = 0; u < P; ++u) t->off[i * S + u] = b + rt.off[first_at[i][u]];
            t->off[i * S + P] = b + rt.n_intra;
        }
        for (uint32_t i = 0; i < A; ++i) {                                  // type-3, without the root's own
            const hspf_ospfv2_ribtable &rt = *t->area[i];
            const uint32_t *a3 = rt.off.data() + rt.plen.size() + 1;
            t->t3_base.push_back((uint32_t)recs.size());
            for (uint32_t u = 0; u < P; ++u) {
                o3[i * S + u] = (uint32_t)recs.size();
                const uint32_t q = t->area_prefix[i][u];
                if (q == kNoRecord) continue;
                for (uint32_t k = a3[q]; k < a3[q + 1]; ++k)
                    if (rt.recs[k].x != t->root[i]) {
                        recs.push_back(rt.recs[k]);
                        if (T::kV3) t->options6.push_back(rt.options6[k - rt.n_intra]);
                    }
            }
            o3[i * S + P] = (uint32_t)recs.size();
        }
        t->t3_end = (uint32_t)recs.size();
        // type-5: every area's table holds the same type-5 records in the same order (one external list, one filter);
        // area 0's slot of a record names its ASBR, and each area's slot of that record gives that area's entry
        const hspf_ospfv2_ribtable &r0 = *t->area[0];
        const uint32_t N5 = r0.ext_end - r0.ext_base;
        for (const hspf_ospfv2_ribtable *rt : t->area)
            if (rt->ext_end - rt->ext_base != N5) return HSPF_E_INVAL;
        std::unordered_map<uint32_t, uint32_t> group_of;                    // area 0's slot record -> group
        std::vector<uint32_t> group_rep, rec_group;                         // a type-5 record of each group; group per record
        t->ext_base = (uint32_t)recs.size();
        const uint32_t *a5 = r0.off.data() + 2 * (r0.plen.size() + 1);
        for (uint32_t u = 0; u < P; ++u) {
            o5[u] = (uint32_t)recs.size();
            const uint32_t q = t->area_prefix[0][u];
            if (q == kNoRecord) continue;
            for (uint32_t k = a5[q]; k < a5[q + 1]; ++k) {
                const RibRec r = r0.recs[k];
                if (r0.recs[r.x].x == t->root[0]) continue;                 // self-originated
                auto ins = group_of.emplace(r.x, (uint32_t)group_rep.size());
                if (ins.second) group_rep.push_back(k - r0.ext_base);
                rec_group.push_back(ins.first->second);
                recs.push_back(RibRec{0, r.y, r.z, 0});
                t->ext_tag.push_back(r0.ext_tag[k - r0.ext_base]);
                if (T::kV3) t->options6.push_back(r0.options6[k - r0.n_intra]);
            }
        }
        o5[P] = (uint32_t)recs.size();
        t->ext_end = o5[P];
        const uint32_t group_base = (uint32_t)recs.size(), G = (uint32_t)group_rep.size();
        for (uint32_t k = 0; k < rec_group.size(); ++k) recs[t->ext_base + k].x = group_base + rec_group[k] * A;
        recs.resize((size_t)group_base + (size_t)G * A);
        for (uint32_t g = 0; g < G; ++g)
            t->group_asbr.push_back(r0.asbr_id[r0.recs[r0.ext_base + group_rep[g]].x - r0.ext_end]);
        for (uint32_t g = 0; g < G; ++g)
            for (uint32_t i = 0; i < A; ++i) {
                const hspf_ospfv2_ribtable &rt = *t->area[i];
                const RibRec s = rt.recs[rt.recs[rt.ext_base + group_rep[g]].x];
                const uint32_t z = (uint32_t)recs.size();
                if ((t->step2 >> i) & 1u)
                    for (uint32_t k = s.z; k < s.w; ++k)
                        if (rt.recs[k].x != t->root[i]) recs.push_back(rt.recs[k]);
                recs[group_base + g * A + i] = RibRec{s.x, s.y, z, (uint32_t)recs.size()};
            }
        if (recs.size() >= kNoRecord) return HSPF_E_UNSUPPORTED;           // record indices are u32
        t->vl_off.push_back(0);
        for (uint32_t i = 0; i < A; ++i) {
            const hspf_ospfv2_ribtable &rt = *t->area[i];
            for (uint32_t v = 0; v < rt.vflags.size(); ++v)
                if (rt.vflags[v] & HL_RTR_FLAG_V) t->v_flagged.push_back(v);
            t->vl_off.push_back((uint32_t)t->v_flagged.size());
        }
        *out = t.release();
        return HSPF_OK;
    } catch (const std::bad_alloc &) {
        return HSPF_E_NOMEM;
    } catch (...) {
        return HSPF_E_UNSUPPORTED;
    }
}

// ---- the borders' slots, shared by build_backbone_table and build_abr_backbone_table ----------------------------
using BorderSlots = std::vector<std::pair<uint32_t, uint32_t>>;     // (border, index), in the borders' LsaKey order

inline void sort_by_router_id(BorderSlots &sl, const hspf_ospfv2_abr_ribtable *const *borders) {
    std::stable_sort(sl.begin(), sl.end(), [&](const std::pair<uint32_t, uint32_t> &x, const std::pair<uint32_t, uint32_t> &y) {
        return borders[x.first]->router_id < borders[y.first]->router_id;
    });
}

template <class K>
bool has_border(const std::map<K, BorderSlots> &m, const K &key, uint32_t b) {
    auto it = m.find(key);
    if (it != m.end())
        for (const auto &s : it->second)
            if (s.first == b) return true;
    return false;
}

// Type-4 slots: per ASBR id, the (border, area index) pairs of the borders' areas other than the target area ta where
// it is a router with the E flag, in LsaKey order.  HSPF_E_UNSUPPORTED for such a router with the B flag (its entry
// would replace an ABR's, as hspf_ospfv2_ribtable_create refuses).
inline int border_asbr_origins(const hspf_ospfv2_abr_ribtable *const *borders, uint32_t n_borders, uint32_t ta,
                               std::map<uint32_t, BorderSlots> &orig) {
    for (uint32_t b = 0; b < n_borders; ++b) {
        const hspf_ospfv2_abr_ribtable &bt = *borders[b];
        for (uint32_t i = 0; i < bt.n_areas; ++i) {
            if (bt.area_id[i] == ta) continue;
            for (const auto &e : bt.rtr_vertex[i]) {
                const uint8_t fl = bt.area[i]->vflags[e.second];
                if (!(fl & HL_RTR_FLAG_E)) continue;
                if (fl & HL_RTR_FLAG_B) return HSPF_E_UNSUPPORTED;
                orig[e.first].emplace_back(b, i);
            }
        }
    }
    for (auto &e : orig) sort_by_router_id(e.second, borders);
    return HSPF_OK;
}

// Type-3 slots: per prefix key, the (border, prefix index) pairs of the borders that can advertise it into the target
// area ta: an intra-area record in one of the border's areas other than ta, or, into a non-backbone area (nb), a
// type-3 record in its area 0 (index a0[b]); `skip(key)` drops a key.  Sorted into LsaKey order.
template <class T, class Skip>
void border_prefix_slots(const hspf_ospfv2_abr_ribtable *const *borders, uint32_t n_borders, const uint32_t *a0,
                         uint32_t ta, bool nb, Skip skip, std::map<typename T::Key, BorderSlots> &slots) {
    for (uint32_t b = 0; b < n_borders; ++b) {
        const hspf_ospfv2_abr_ribtable &bt = *borders[b];
        const uint32_t P = (uint32_t)bt.prefix.size(), S = P + 1, A = bt.n_areas;
        for (uint32_t u = 0; u < P; ++u) {
            bool adv = nb && bt.off[(A + a0[b]) * S + u] != bt.off[(A + a0[b]) * S + u + 1];
            for (uint32_t i = 0; i < A && !adv; ++i)
                adv = bt.area_id[i] != ta && bt.off[i * S + u] != bt.off[i * S + u + 1];
            if (adv && !skip(T::table_key(bt, u))) slots[T::table_key(bt, u)].emplace_back(b, u);
        }
    }
    for (auto &e : slots) sort_by_router_id(e.second, borders);
}

// A range of static records (in LsaKey order, `adv_rtr(s)` each) with every slot of `sl` at its border's LsaKey place.
template <class S, class AdvRtr, class PutStatic, class PutSlot>
void merge_lsakey(const std::vector<S> &statics, AdvRtr adv_rtr, const BorderSlots &sl,
                  const hspf_ospfv2_abr_ribtable *const *borders, PutStatic put_static, PutSlot put_slot) {
    size_t k = 0;
    for (const S &s : statics) {
        while (k < sl.size() && borders[sl[k].first]->router_id < adv_rtr(s)) put_slot(sl[k++]);
        put_static(s);
    }
    while (k < sl.size()) put_slot(sl[k++]);
}

// The type-4 slot of (border, area index) o for ASBR `id`, whose border is vertex bv of the table's area; its plane set
// is added to `sets` when new.
inline RibRec asbr_slot(const hspf_ospfv2_abr_ribtable *const *borders, uint32_t bv, const std::pair<uint32_t, uint32_t> &o,
                        uint32_t id, std::map<std::pair<uint32_t, uint32_t>, uint32_t> &set_of,
                        std::vector<std::pair<uint32_t, uint32_t>> &sets) {
    auto ins = set_of.emplace(o, (uint32_t)sets.size());
    if (ins.second) sets.push_back(o);
    return RibRec{bv, borders[o.first]->rtr_vertex[o.second].at(id), o.first, kOspfBackboneAsbrSlot | ins.first->second};
}

// Border b's words (OspfBackboneView::border): its intra-area records of area index i, and i's atom bits.
inline std::array<uint32_t, 4> border_words(const hspf_ospfv2_abr_ribtable &bt, uint32_t i) {
    const uint32_t lo = bt.intra_base[i], na = bt.n_atoms[i];
    const uint64_t atoms = na == 0 ? 0 : ((na == 64 ? ~0ull : ((1ull << na) - 1)) << bt.base[i]);
    return {lo, lo + bt.area[i]->n_intra, (uint32_t)atoms, (uint32_t)(atoms >> 32)};
}

// Border C's words over a third-area table (build_backbone_table with `third`): the walk's intra-area records of
// area index i of C's restricted table (an intra-area winner of C's cells is one of those), and i's atom bits.
inline std::array<uint32_t, 4> walk_border_words(const hspf_ospfv2_abr_backbone_table &c, uint32_t i) {
    const hspf_ospfv2_abr_ribtable &a = *c.abr;
    const size_t S = a.prefix.size() + 1;
    std::array<uint32_t, 4> w = border_words(a, i);
    w[0] = a.off[i * S];
    w[1] = a.off[i * S + S - 1];
    return w;
}

// Every C's walk_border_words over its target-area index at[b], appended to `words` (which ends on a 16-byte
// boundary).  OSPFv3 (kV3): 8 words per C, the fifth the byte offset from the first border word of C's options bytes
// and the sixth C's record count (border_summary with kSlotWinners), then every C's options bytes, each padded to a
// word: one per record index below that count, the prefix options of a walk intra-area record (its decode record's
// entry in its area's intra-area table) and of a type-3 record (C's options6), 0 for any other.  HSPF_E_INVAL when a
// C's table does not hold those options.
template <bool kV3>
int append_walk_border_words(std::vector<uint32_t> &words, const hspf_ospfv2_abr_backbone_table *const *cs,
                             uint32_t n_borders, const uint32_t *at) {
    uint32_t opt_words = (kV3 ? 8 : 4) * n_borders;
    for (uint32_t b = 0; b < n_borders; ++b) {
        const std::array<uint32_t, 4> bw = walk_border_words(*cs[b], at[b]);
        words.insert(words.end(), bw.begin(), bw.end());
        if (kV3) {
            const uint32_t n = cs[b]->n_recs();
            words.insert(words.end(), {4 * opt_words, n, 0u, 0u});
            opt_words += (n + 3) / 4;
        }
    }
    if (kV3) {
        for (uint32_t b = 0; b < n_borders; ++b) {
            const hspf_ospfv2_abr_backbone_table &c = *cs[b];
            const hspf_ospfv2_abr_ribtable &a = *c.abr;
            const uint32_t n = c.n_recs();
            std::vector<uint8_t> opt(((size_t)n + 3) & ~(size_t)3, 0);
            if (a.t3_base.empty() || a.options6.size() < a.t3_end - a.t3_base[0] ||
                c.intra_src.size() != n - c.walk_intra)
                return HSPF_E_INVAL;
            for (uint32_t k = a.t3_base[0]; k < a.t3_end; ++k) opt[k] = a.options6[k - a.t3_base[0]];
            for (uint32_t k = c.walk_intra; k < n; ++k) {
                const uint32_t src = c.intra_src[k - c.walk_intra];
                uint32_t i = 0;
                while (i < a.n_areas && !(src >= a.intra_base[i] && src < a.intra_base[i] + a.area[i]->n_intra)) ++i;
                if (i == a.n_areas) return HSPF_E_INVAL;
                const std::vector<uint8_t> &o = a.area[i]->intra->t.options6;
                if (o.size() != a.area[i]->n_intra) return HSPF_E_INVAL;
                opt[k] = o[src - a.intra_base[i]];
            }
            const size_t w = words.size();
            words.resize(w + opt.size() / 4);
            if (!opt.empty()) std::memcpy(words.data() + w, opt.data(), opt.size());
        }
    }
    return HSPF_OK;
}

// Every border's words over its target-area index at[b], appended to `words` (which ends on a 16-byte boundary).
// OSPFv3 (kV3): 8 words per border, the fifth the byte offset from the first border word of the border's options
// bytes, which follow all the border words, each border's padded to a word: one per record an advertised cell's
// winner can be, its intra-area records and, into a non-backbone area (nb), its type-3 records too.  HSPF_E_INVAL when
// a border's table does not hold those options.
template <bool kV3>
int append_border_words(std::vector<uint32_t> &words, const hspf_ospfv2_abr_ribtable *const *borders,
                        uint32_t n_borders, const uint32_t *at, bool nb) {
    uint32_t opt_words = (kV3 ? 8 : 4) * n_borders;
    auto opt_end = [&](const hspf_ospfv2_abr_ribtable &bt) { return nb ? bt.t3_end : bt.t3_base[0]; };
    for (uint32_t b = 0; b < n_borders; ++b) {
        const hspf_ospfv2_abr_ribtable &bt = *borders[b];
        const std::array<uint32_t, 4> bw = border_words(bt, at[b]);
        words.insert(words.end(), bw.begin(), bw.end());
        if (kV3) {
            words.insert(words.end(), {4 * opt_words, 0u, 0u, 0u});
            opt_words += (opt_end(bt) + 3) / 4;
        }
    }
    if (kV3) {
        // per border, the prefix options of each intra-area record of its table, as the OSPFv3 intra-area decode
        // reads them for that winner: the record's entry in its area's intra-area table; into a non-backbone area
        // also those of each type-3 record (an inter-area cell's winner), the options of its LSA
        for (uint32_t b = 0; b < n_borders; ++b) {
            const hspf_ospfv2_abr_ribtable &bt = *borders[b];
            std::vector<uint8_t> opt;
            for (uint32_t i = 0; i < bt.n_areas; ++i) {
                const std::vector<uint8_t> &o = bt.area[i]->intra->t.options6;
                if (o.size() != bt.area[i]->n_intra || opt.size() != bt.intra_base[i]) return HSPF_E_INVAL;
                opt.insert(opt.end(), o.begin(), o.end());
            }
            if (nb) {
                const size_t n3 = bt.t3_end - bt.t3_base[0];
                if (opt.size() != bt.t3_base[0] || bt.options6.size() < n3) return HSPF_E_INVAL;
                opt.insert(opt.end(), bt.options6.begin(), bt.options6.begin() + n3);
            }
            opt.resize(((size_t)opt_end(bt) + 3) & ~(size_t)3, 0);
            const size_t w = words.size();
            words.resize(w + opt.size() / 4);
            if (!opt.empty()) std::memcpy(words.data() + w, opt.data(), opt.size());
        }
    }
    return HSPF_OK;
}

// hspf_ospfv2_backbone_table_create / hspf_ospfv3_backbone_table_create, argument checks included: R's one-area table
// over area 0 without the borders' type-3 LSAs, and per affected prefix R's intra-area records, its static type-3
// records with one slot per (border, prefix) at the border's place in LsaKey order, and its type-5 records
// (ospf_backbone_cells.h).  Border tables of the other version are refused (HSPF_E_INVAL).  `asbr`
// (hspf_ospfv{2,3}_backbone_asbr_table_create): the borders' type-4 / Inter-Area-Router LSAs are re-originated per job
// too, as type-4 slots, and the prefixes of the type-5 LSAs they lead to are affected; else a usable one is
// HSPF_E_UNSUPPORTED.  The table keeps the flag (hspf_ospfv2_backbone_table::asbr).
// `config` (hspf_ospfv{2,3}_nonbackbone_table_create): R is an internal router of the non-backbone area of `flat` with
// that configuration, the target area A.  The borders re-originate into A their intra-area routes of their other
// areas and their inter-area routes, and type-4 / Inter-Area-Router LSAs for the ASBRs they reach intra-area outside A
// (plane sets of any of those areas, area 0 included); in a stub area the default route stays static and no type-4
// LSA is originated, and a totally stubby area has no slot.  OSPFv3: a border's options bytes also cover its type-3
// records, so that an inter-area cell's winner gives the options of the LSA the border copies them from.
// `third` (with `config`, build_third_area_table): borders[b] is third[b]->abr, C's table restricted to its affected
// prefixes.  A C LSA for a key outside C's prefixes, or a type-4 / Inter-Area-Router LSA for an ASBR without type-4
// slots in C's table, stays a static record; the type-4 slots are chain slots (ospf_backbone_cells.h: OspfChainJob),
// one per (C, group of C with type-4 slots), and the border words name C's walk intra-area records
// (append_walk_border_words; OSPFv3: with C's record count and options bytes, which its slot winners need).
template <class T>
int build_backbone_table(const typename T::Flat *flat, uint32_t router_id, const typename T::Sum *sums, uint32_t n_sums,
                         const typename T::Ext *ext, uint32_t n_ext, const hspf_ospfv2_abr_ribtable *const *borders,
                         uint32_t n_borders, hspf_ospfv2_backbone_table **out, bool asbr = false,
                         const hl_ospf_area_config *config = nullptr,
                         const hspf_ospfv2_abr_backbone_table *const *third = nullptr) {
    using Key = typename T::Key;
    using Sum = typename T::Sum;
    constexpr uint32_t kNone = 0xFFFFFFFFu;
    if (!flat || !flat->area || !out || (n_sums && !sums) || (n_ext && !ext) || !borders) return HSPF_E_INVAL;
    *out = nullptr;
    if (third && !config) return HSPF_E_INVAL;
    const bool nb = config != nullptr;                            // a non-backbone target area
    const uint32_t ta = nb ? flat->area->area_id : 0;
    if (nb) {
        if (ta == 0) return HSPF_E_INVAL;
        if (config->area_type == HL_AREA_NSSA || n_borders == 0 || n_borders > kOspfBackboneMaxBorders)
            return HSPF_E_UNSUPPORTED;
        asbr = true;
    }
    if (n_borders == 0 || n_borders > kOspfBackboneMaxBorders) return HSPF_E_INVAL;
    const bool normal = !nb || config->area_type == HL_AREA_NORMAL;
    try {
        std::unique_ptr<hspf_ospfv2_backbone_table, void (*)(hspf_ospfv2_backbone_table *)> t(
            new hspf_ospfv2_backbone_table(), hspf_ospfv2_backbone_table_free);
        const typename T::Flat &f = *flat;
        auto vertex = [&](uint32_t id) { return T::root_vertex(f, id); };
        auto flags = [&](uint32_t v) { return v == kNone ? (uint8_t)0 : T::router_flags(f, v); };
        const uint32_t root = vertex(router_id);
        if (root == kNone || (flags(root) & HL_RTR_FLAG_B)) return HSPF_E_INVAL;
        t->router_id = router_id; t->root = root; t->n_vertices = T::n_vertices(f);
        t->max_paths = f.area->max_paths; t->n_borders = n_borders; t->v3 = T::kV3; t->area_id = ta; t->asbr = asbr;
        t->third_area = third != nullptr;
        // per border: its area-0 index, its target-area index, its vertex
        std::vector<uint32_t> a0(n_borders), at(n_borders), bv(n_borders);
        std::unordered_map<uint32_t, uint32_t> border_of;           // router id -> border
        for (uint32_t b = 0; b < n_borders; ++b) {
            const hspf_ospfv2_abr_ribtable *bt = borders[b];
            if (!bt || bt->v3 != T::kV3 || bt->router_id == router_id || !border_of.emplace(bt->router_id, b).second)
                return HSPF_E_INVAL;
            a0[b] = at[b] = kNone;
            for (uint32_t i = 0; i < bt->n_areas; ++i) {
                if (bt->area_id[i] == 0 && a0[b] == kNone) a0[b] = i;
                if (bt->area_id[i] == ta && at[b] == kNone) at[b] = i;
            }
            bv[b] = vertex(bt->router_id);
            if (a0[b] == kNone || at[b] == kNone || !(flags(bv[b]) & HL_RTR_FLAG_B)) return HSPF_E_INVAL;
            t->borders[b] = bt;
            if (third) {
                t->third[b] = third[b];
                // a border of C's that is a router of R's area is an ABR of both areas
                for (uint32_t k = 0; k < third[b]->n_borders; ++k)
                    if (vertex(third[b]->borders[k]->router_id) != kNone) return HSPF_E_UNSUPPORTED;
            }
            if (nb) {
                // an inter-area router entry at the border (from another ABR's type-4 LSA in area 0) would be
                // re-originated into A at a distance the job moves
                const hspf_ospfv2_ribtable &r0 = *bt->area[a0[b]];
                for (uint32_t a = 0; a < (uint32_t)r0.asbr_id.size(); ++a) {
                    const RibRec &s = r0.recs[r0.ext_end + a];
                    for (uint32_t k = s.z; k < s.w; ++k)
                        if (r0.recs[k].x != bt->root[a0[b]]) return HSPF_E_UNSUPPORTED;
                }
            }
        }
        // the default route a border originates into a stub area, at default_cost whatever the job
        const Key dflt = T::default_key();
        auto stub_default = [&](const Sum &l) { return nb && !normal && l.lsa_type == 3 && T::key(l) == dflt; };
        // R's area without the borders' type-3 LSAs: R's one-area table over the rest
        auto live = [](const Sum &l) { return !l.maxage && l.metric < HL_LSA_INFINITY && !T::skip(l); };
        std::vector<Sum> rest;
        std::vector<std::pair<uint32_t, Key>> border_t3;            // (border, prefix key) of the borders' LSAs
        std::vector<std::pair<uint32_t, uint32_t>> border_t4;       // (border, ASBR id)
        // third: per C, the keys of its prefixes and the ASBRs of its groups with type-4 slots (chain ids)
        std::vector<std::map<Key, uint32_t>> c_keys(third ? n_borders : 0);
        std::vector<std::map<uint32_t, uint32_t>> c_ids(third ? n_borders : 0);
        for (uint32_t b = 0; third && b < n_borders; ++b) {
            const hspf_ospfv2_abr_ribtable &ca = *borders[b];
            for (uint32_t u = 0; u < (uint32_t)ca.prefix.size(); ++u) c_keys[b].emplace(T::table_key(ca, u), u);
            for (uint32_t g = 0; g < (uint32_t)third[b]->asbr_group.size(); ++g)
                c_ids[b].emplace(ca.group_asbr[third[b]->asbr_group[g]], g);
        }
        auto stays = [&](uint32_t b, const Sum &l) {                 // a C LSA the job cannot move
            if (!third) return false;
            return l.lsa_type == 3 ? !c_keys[b].count(T::key(l)) : !c_ids[b].count(T::asbr_id(l));
        };
        for (uint32_t i = 0; i < n_sums; ++i) {
            const Sum &l = sums[i];
            auto it = border_of.find(l.adv_rtr);
            if (it == border_of.end() || stub_default(l) || stays(it->second, l)) { rest.push_back(l); continue; }
            if (!live(l)) continue;
            if (l.lsa_type == 4) {                                   // re-originated per job too
                if (!asbr) return HSPF_E_UNSUPPORTED;
                border_t4.emplace_back(it->second, T::asbr_id(l));
            }
            if (l.lsa_type == 3) border_t3.emplace_back(it->second, T::key(l));
        }
        int rc = T::area_table(flat, ta, rest.data(), (uint32_t)rest.size(), ext, n_ext, false, &t->r);
        if (rc) return rc;
        const hspf_ospfv2_ribtable &r = *t->r;
        if (nb)                                                      // A is a transit area
            for (uint8_t fl : r.vflags)
                if (fl & HL_RTR_FLAG_V) return HSPF_E_UNSUPPORTED;
        // type-4 slots: per ASBR id, the (border, area index) pairs of the borders' areas other than the target where
        // it is a router with the E flag, each border's in area order (none into a stub area)
        std::map<uint32_t, BorderSlots> orig;
        if (asbr && normal) {
            if (third) {                                             // chain slots: C's groups with type-4 slots
                for (uint32_t b = 0; b < n_borders; ++b)
                    for (const auto &e : c_ids[b]) orig[e.first].emplace_back(b, e.second);
                for (auto &e : orig) sort_by_router_id(e.second, borders);
            } else if (const int rc2 = border_asbr_origins(borders, n_borders, ta, orig)) {
                return rc2;
            }
            for (const auto &x : border_t4)
                if (!has_border(orig, x.second, x.first)) return HSPF_E_INVAL;   // the LSDB disagrees with the border's table
        }
        // the affected prefixes: each border's prefixes with an intra-area record in one of its areas other than the
        // target (into a non-backbone area also those with a type-3 record in its area 0; none into a totally stubby
        // area, and not a stub area's default route)
        std::map<Key, BorderSlots> slots;                            // key -> (border, its prefix index)
        if (!nb || config->summary)
            border_prefix_slots<T>(borders, n_borders, a0.data(), ta, nb,
                                   [&](const Key &k) { return nb && !normal && k == dflt; }, slots);
        for (const auto &x : border_t3)
            if (!has_border(slots, x.second, x.first)) return HSPF_E_INVAL;      // the LSDB disagrees with the border's table
        // ... and the prefixes of the type-5 LSAs of an ASBR some border can originate a type-4 LSA for
        const uint32_t *rx = r.off.data() + 2 * (r.prefix.size() + 1);
        if (!orig.empty())
            for (uint32_t u = 0; u < (uint32_t)r.prefix.size(); ++u)
                for (uint32_t k = rx[u]; k < rx[u + 1]; ++k)
                    if (orig.count(r.asbr_id[r.recs[k].x - r.ext_end])) {
                        slots[T::table_key(r, u)];
                        break;
                    }
        // R's static type-3 records per prefix, in LsaKey order: (adv_rtr, ABR vertex, metric, prefix options)
        std::map<Key, std::vector<std::array<uint32_t, 4>>> statics;
        for (const Sum &l : rest) {
            if (l.lsa_type != 3 || !live(l)) continue;
            const uint32_t v = vertex(l.adv_rtr);
            if (!(flags(v) & HL_RTR_FLAG_B)) continue;
            statics[T::key(l)].push_back({l.adv_rtr, v, l.metric, T::options(l)});
        }
        std::map<Key, uint32_t> q_of;
        const uint32_t PR = (uint32_t)r.prefix.size();
        for (uint32_t u = 0; u < PR; ++u) q_of.emplace(T::table_key(r, u), u);
        const uint32_t P = (uint32_t)slots.size();
        std::vector<uint32_t> q(P), o3(P + 1), o5(P + 1);
        t->recs = r.recs;
        t->prefix.resize(P); t->plen.resize(P);
        if (T::kV3) t->prefix6.resize(P);
        uint32_t u = 0;
        const std::vector<std::array<uint32_t, 4>> none;
        for (auto &e : slots) {
            T::set_prefix(*t, u, e.first);
            auto qi = q_of.find(e.first);
            q[u] = qi == q_of.end() ? kNoRecord : qi->second;
            o3[u] = (uint32_t)t->recs.size();
            auto st = statics.find(e.first);
            merge_lsakey(
                st != statics.end() ? st->second : none, [](const std::array<uint32_t, 4> &s) { return s[0]; },
                e.second, borders,
                [&](const std::array<uint32_t, 4> &s) {
                    t->recs.push_back(RibRec{s[1], s[2], kOspfBackboneStatic, 0});
                    if (T::kV3) t->options6.push_back((uint8_t)s[3]);
                },
                [&](const std::pair<uint32_t, uint32_t> &s) {
                    t->slot_rec.push_back((uint32_t)t->recs.size());
                    t->recs.push_back(RibRec{bv[s.first], s.second, s.first, (uint32_t)t->slot_rec.size() - 1});
                    if (T::kV3) t->options6.push_back(0);
                });
            ++u;
        }
        o3[P] = (uint32_t)t->recs.size();
        const uint32_t *r5 = r.off.data() + 2 * ((size_t)PR + 1);
        t->ext_base = (uint32_t)t->recs.size();
        for (u = 0; u < P; ++u) {
            o5[u] = (uint32_t)t->recs.size();
            if (q[u] == kNoRecord) continue;
            for (uint32_t k = r5[q[u]]; k < r5[q[u] + 1]; ++k) {
                t->recs.push_back(r.recs[k]);
                t->ext_tag.push_back(r.ext_tag[k - r.ext_base]);
                if (T::kV3) t->options6.push_back(r.options6[k - r.n_intra]);
            }
        }
        o5[P] = (uint32_t)t->recs.size();
        if (!orig.empty()) {
            // each such ASBR's type-4 range again, at the end: its static records (R's one-area table has them in
            // LSDB order) with the borders' slots at their LsaKey places (by advertising router)
            std::map<uint32_t, std::vector<std::pair<uint32_t, RibRec>>> t4;   // ASBR id -> (adv_rtr, static record)
            for (const Sum &l : rest) {
                if (l.lsa_type != 4 || !live(l)) continue;
                const uint32_t v = vertex(l.adv_rtr);
                if (flags(v) & HL_RTR_FLAG_B) t4[T::asbr_id(l)].push_back({l.adv_rtr, RibRec{v, l.metric, 0, 0}});
            }
            std::map<std::pair<uint32_t, uint32_t>, uint32_t> set_of;
            for (uint32_t a = 0; a < (uint32_t)r.asbr_id.size(); ++a) {
                const uint32_t id = r.asbr_id[a];
                auto o = orig.find(id);
                if (o == orig.end()) continue;
                const auto st = t4.find(id);
                const uint32_t z = (uint32_t)t->recs.size();
                const std::vector<std::pair<uint32_t, RibRec>> none;
                merge_lsakey(
                    st != t4.end() ? st->second : none, [](const std::pair<uint32_t, RibRec> &x) { return x.first; },
                    o->second, borders, [&](const std::pair<uint32_t, RibRec> &x) { t->recs.push_back(x.second); },
                    [&](const std::pair<uint32_t, uint32_t> &x) {
                        t->recs.push_back(third ? RibRec{bv[x.first], x.second, x.first, kOspfBackboneAsbrSlot | x.first}
                                                : asbr_slot(borders, bv[x.first], x, id, set_of, t->asbr_set));
                        ++t->n_asbr_slots;
                    });
                RibRec &s = t->recs[r.ext_end + a];
                s.z = z;
                s.w = (uint32_t)t->recs.size();
            }
            if (t->asbr_set.size() > kOspfBackboneMaxAsbrSets) return HSPF_E_UNSUPPORTED;   // the kernel parameter's
        }
        if (!backbone_winners_fit(t->recs.size(), t->slot_rec.size(), T::kV3)) return HSPF_E_UNSUPPORTED;
        t->words.assign(r.off.begin(), r.off.begin() + PR + 1);
        t->words.insert(t->words.end(), q.begin(), q.end());
        t->words.insert(t->words.end(), o3.begin(), o3.end());
        t->words.insert(t->words.end(), o5.begin(), o5.end());
        t->words.resize(t->border_at(), 0);
        if (const int rc2 = third ? append_walk_border_words<T::kV3>(t->words, third, n_borders, at.data())
                                  : append_border_words<T::kV3>(t->words, borders, n_borders, at.data(), nb))
            return rc2;
        *out = t.release();
        return HSPF_OK;
    } catch (const std::bad_alloc &) {
        return HSPF_E_NOMEM;
    } catch (...) {
        return HSPF_E_UNSUPPORTED;
    }
}

// hspf_ospfv2_third_area_table_create / hspf_ospfv3_third_area_table_create, argument checks included: an internal
// router R of a non-backbone area over jobs inside another non-backbone area.  The borders are R's area's ABRs attached
// to area 0 (C), each an abr_backbone table of R's version over the perturbed area's ABRs (another version's is
// HSPF_E_INVAL); the table is build_backbone_table's `config` path over the C's restricted tables, with `third` (chain
// slots, the walk's border words).
template <class T>
int build_third_area_table(const typename T::Flat *flat, uint32_t router_id, const hl_ospf_area_config *config,
                           const typename T::Sum *sums, uint32_t n_sums, const typename T::Ext *ext, uint32_t n_ext,
                           const hspf_ospfv2_abr_backbone_table *const *borders, uint32_t n_borders,
                           hspf_ospfv2_backbone_table **out) {
    if (out) *out = nullptr;
    if (!config || !borders || n_borders == 0 || n_borders > kOspfBackboneMaxBorders) return HSPF_E_INVAL;
    const hspf_ospfv2_abr_ribtable *abr[kOspfBackboneMaxBorders];
    for (uint32_t b = 0; b < n_borders; ++b) {
        if (!borders[b] || !borders[b]->abr || borders[b]->abr->v3 != T::kV3) return HSPF_E_INVAL;
        abr[b] = borders[b]->abr;
    }
    return build_backbone_table<T>(flat, router_id, sums, n_sums, ext, n_ext, abr, n_borders, out, true, config,
                                   borders);
}

// hspf_ospfv2_abr_backbone_table_create, argument checks included: an area border router R of area 0 and other areas
// over jobs inside an area it is not attached to.  R's ABR table (build_abr_ribtable) over its areas, with area 0's
// summaries without the borders' type-3 / type-4 LSAs, restricted to the affected prefixes: those some border can
// advertise into area 0, and those of the type-5 LSAs of an ASBR some border can originate a type-4 LSA for.  Area
// 0's type-3 ranges get the borders' slots and its type-4 ranges their type-4 slots, at the borders' LsaKey places,
// as build_backbone_table places them (ospf_backbone_cells.h: AbrBorderSlots).  OSPFv3
// (hspf_ospfv3_abr_backbone_table_create): the restricted table carries its IPv6 prefixes and the options of its
// type-3 / type-5 records, and the border words carry each border's options bytes, as build_backbone_table's do.
template <class T>
int build_abr_backbone_table(uint32_t router_id, uint32_t n_areas, const typename T::Flat *const *flats,
                             const uint32_t *area_ids, const typename T::Sum *const *summaries,
                             const uint32_t *n_summaries, const uint8_t *active, const typename T::Ext *ext,
                             uint32_t n_ext, const hspf_ospfv2_abr_ribtable *const *borders, uint32_t n_borders,
                             hspf_ospfv2_abr_backbone_table **out) {
    using Key = typename T::Key;
    using Sum = typename T::Sum;
    constexpr uint32_t kNone = 0xFFFFFFFFu;
    if (!out || !flats || !area_ids || n_areas == 0 || !borders || (n_ext && !ext)) return HSPF_E_INVAL;
    *out = nullptr;
    if (n_borders == 0 || n_borders > kOspfBackboneMaxBorders) return HSPF_E_INVAL;
    if (n_areas > kAbrMaxAreas) return HSPF_E_UNSUPPORTED;
    uint32_t i0 = kNone, n_active = 0;
    for (uint32_t i = 0; i < n_areas; ++i) {
        if (!flats[i] || !flats[i]->area) return HSPF_E_INVAL;
        if (n_summaries && n_summaries[i] && (!summaries || !summaries[i])) return HSPF_E_INVAL;
        if (area_ids[i] == 0 && i0 == kNone) i0 = i;
        n_active += (!active || active[i]) ? 1u : 0u;
    }
    if (i0 == kNone || (active && !active[i0]) || n_active < 2) return HSPF_E_INVAL;
    try {
        std::unique_ptr<hspf_ospfv2_abr_backbone_table, void (*)(hspf_ospfv2_abr_backbone_table *)> t(
            new hspf_ospfv2_abr_backbone_table(), hspf_ospfv2_abr_backbone_table_free);
        const typename T::Flat &f = *flats[i0];
        auto vertex = [&](uint32_t id) { return T::root_vertex(f, id); };
        auto flags = [&](uint32_t v) { return v == kNone ? (uint8_t)0 : T::router_flags(f, v); };
        if (!(flags(vertex(router_id)) & HL_RTR_FLAG_B)) return HSPF_E_INVAL;
        // the borders: their area-0 index and their vertex in R's area 0
        std::vector<uint32_t> a0(n_borders), bv(n_borders);
        std::unordered_map<uint32_t, uint32_t> border_of;
        for (uint32_t b = 0; b < n_borders; ++b) {
            const hspf_ospfv2_abr_ribtable *bt = borders[b];
            if (!bt || bt->v3 != T::kV3 || bt->router_id == router_id || !border_of.emplace(bt->router_id, b).second)
                return HSPF_E_INVAL;
            a0[b] = kNone;
            for (uint32_t i = 0; i < bt->n_areas && a0[b] == kNone; ++i)
                if (bt->area_id[i] == 0) a0[b] = i;
            bv[b] = vertex(bt->router_id);
            if (a0[b] == kNone || !(flags(bv[b]) & HL_RTR_FLAG_B)) return HSPF_E_INVAL;
            t->borders[b] = bt;
        }
        t->n_borders = n_borders;
        t->area0 = i0;
        // area 0's summaries without the borders' LSAs, which the slots stand for
        const uint32_t n0 = n_summaries ? n_summaries[i0] : 0;
        auto live = [](const Sum &l) { return !l.maxage && l.metric < HL_LSA_INFINITY && !T::skip(l); };
        std::vector<Sum> rest;
        std::vector<std::pair<uint32_t, Key>> border_t3;
        std::vector<std::pair<uint32_t, uint32_t>> border_t4;
        for (uint32_t k = 0; k < n0; ++k) {
            const Sum &l = summaries[i0][k];
            auto it = border_of.find(l.adv_rtr);
            if (it == border_of.end()) { rest.push_back(l); continue; }
            if (!live(l)) continue;
            if (l.lsa_type == 3) border_t3.emplace_back(it->second, T::key(l));
            if (l.lsa_type == 4) border_t4.emplace_back(it->second, T::asbr_id(l));
        }
        std::map<uint32_t, BorderSlots> orig;
        if (const int rc = border_asbr_origins(borders, n_borders, 0, orig)) return rc;
        for (const auto &x : border_t4)
            if (!has_border(orig, x.second, x.first)) return HSPF_E_INVAL;
        std::map<Key, BorderSlots> slots;
        border_prefix_slots<T>(borders, n_borders, a0.data(), 0, false, [](const Key &) { return false; }, slots);
        for (const auto &x : border_t3)
            if (!has_border(slots, x.second, x.first)) return HSPF_E_INVAL;
        // R's whole table over those summaries
        std::vector<const Sum *> sp(n_areas);
        std::vector<uint32_t> ns(n_areas);
        for (uint32_t i = 0; i < n_areas; ++i) {
            sp[i] = i == i0 ? rest.data() : (summaries ? summaries[i] : nullptr);
            ns[i] = i == i0 ? (uint32_t)rest.size() : (n_summaries ? n_summaries[i] : 0);
        }
        hspf_ospfv2_abr_ribtable *full_raw = nullptr;
        int rc = build_abr_ribtable<T>(router_id, n_areas, flats, area_ids, sp.data(), ns.data(), active, ext, n_ext,
                                       &full_raw);
        if (rc) return rc;
        std::unique_ptr<hspf_ospfv2_abr_ribtable, void (*)(hspf_ospfv2_abr_ribtable *)> full(full_raw,
                                                                                            hspf_ospfv2_abr_ribtable_free);
        const hspf_ospfv2_abr_ribtable &F = *full;
        if (!F.v_flagged.empty()) return HSPF_E_UNSUPPORTED;          // the transit-area step
        const uint32_t A = n_areas, PF = (uint32_t)F.prefix.size(), SF = PF + 1;
        const uint32_t G = (uint32_t)F.group_asbr.size();
        // ... and the prefixes of the type-5 LSAs of an ASBR with type-4 slots
        std::map<Key, uint32_t> uf;                                  // R's prefix index of a key
        for (uint32_t u = 0; u < PF; ++u) uf.emplace(T::table_key(F, u), u);
        const uint32_t *f5 = F.off.data() + 2 * (size_t)A * SF;
        for (uint32_t u = 0; u < PF; ++u)
            for (uint32_t k = f5[u]; k < f5[u + 1]; ++k)
                if (orig.count(F.group_asbr[(F.recs[k].x - F.ext_end) / A])) {
                    slots[T::table_key(F, u)];
                    break;
                }
        // the table over the affected prefixes
        std::unique_ptr<hspf_ospfv2_abr_ribtable, void (*)(hspf_ospfv2_abr_ribtable *)> r(new hspf_ospfv2_abr_ribtable(),
                                                                                         hspf_ospfv2_abr_ribtable_free);
        r->router_id = F.router_id; r->n_areas = A; r->max_paths = F.max_paths; r->step2 = F.step2; r->v3 = F.v3;
        r->area = F.area; full->area.clear();                        // the area tables move over
        r->area_id = F.area_id; r->root = F.root; r->n_vertices = F.n_vertices; r->base = F.base;
        r->n_atoms = F.n_atoms; r->intra_base = F.intra_base; r->rtr_vertex = F.rtr_vertex;
        r->group_asbr = F.group_asbr;
        const uint32_t P = (uint32_t)slots.size(), S = P + 1;
        std::vector<uint32_t> from(P);                               // R's prefix index of each, or kNone
        r->prefix.resize(P); r->plen.resize(P);
        if (T::kV3) r->prefix6.resize(P);
        r->area_prefix.assign(A, std::vector<uint32_t>(P, kNoRecord));
        uint32_t u = 0;
        for (const auto &e : slots) {
            T::set_prefix(*r, u, e.first);
            auto it = uf.find(e.first);
            from[u] = it == uf.end() ? kNone : it->second;
            for (uint32_t i = 0; i < A && from[u] != kNone; ++i) r->area_prefix[i][u] = F.area_prefix[i][from[u]];
            ++u;
        }
        r->off.assign((2 * (size_t)A + 1) * S, 0);
        uint32_t *o3 = r->off.data() + (size_t)A * S, *o5 = o3 + (size_t)A * S;
        auto &recs = r->recs;
        recs.assign(F.recs.begin(), F.recs.begin() + F.t3_base[0]);  // every intra-area record, for the decode
        // R's router id of each area-0 vertex, for the LsaKey order of the static records
        std::unordered_map<uint32_t, uint32_t> id_of;
        for (const auto &e : F.rtr_vertex[i0]) id_of.emplace(e.second, e.first);
        auto adv_rtr = [&](const RibRec &x) { return id_of.at(x.x); };
        // OSPFv3: options6 holds each type-3 / type-5 record's prefix options (index - t3_base[0]), R's for a static
        // one and a placeholder for a slot, whose options come from its winner
        auto put = [&](const RibRec &x, uint32_t k) {
            recs.push_back(x);
            if (T::kV3) r->options6.push_back(F.options6[k - F.t3_base[0]]);
        };
        for (uint32_t i = 0; i < A; ++i) {                           // type-3, area 0's with the slots
            r->t3_base.push_back((uint32_t)recs.size());
            const uint32_t *g3 = F.off.data() + (A + i) * (size_t)SF;
            u = 0;
            for (const auto &e : slots) {
                o3[i * S + u] = (uint32_t)recs.size();
                std::vector<uint32_t> st;                            // R's records of the prefix
                if (from[u] != kNone)
                    for (uint32_t k = g3[from[u]]; k < g3[from[u] + 1]; ++k) st.push_back(k);
                if (i != i0) {
                    for (uint32_t k : st) put(F.recs[k], k);
                } else {
                    merge_lsakey(st, [&](uint32_t k) { return adv_rtr(F.recs[k]); }, e.second, borders,
                                 [&](uint32_t k) { put(RibRec{F.recs[k].x, F.recs[k].y, kOspfBackboneStatic, 0}, k); },
                                 [&](const std::pair<uint32_t, uint32_t> &s) {
                                     t->slot_rec.push_back((uint32_t)recs.size());
                                     recs.push_back(RibRec{bv[s.first], s.second, s.first, (uint32_t)t->slot_rec.size() - 1});
                                     if (T::kV3) r->options6.push_back(0);
                                 });
                }
                ++u;
            }
            o3[i * S + P] = (uint32_t)recs.size();
        }
        r->t3_end = (uint32_t)recs.size();
        // type-5, then the ASBR entries and their type-4 ranges, moved by `shift`
        r->ext_base = (uint32_t)recs.size();
        size_t n5 = 0;
        for (u = 0; u < P; ++u)
            if (from[u] != kNone) n5 += f5[from[u] + 1] - f5[from[u]];
        const uint32_t shift = (uint32_t)(recs.size() + n5) - F.ext_end;
        for (u = 0; u < P; ++u) {
            o5[u] = (uint32_t)recs.size();
            if (from[u] == kNone) continue;
            for (uint32_t k = f5[from[u]]; k < f5[from[u] + 1]; ++k) {
                put(RibRec{F.recs[k].x + shift, F.recs[k].y, F.recs[k].z, F.recs[k].w}, k);
                r->ext_tag.push_back(F.ext_tag[k - F.ext_base]);
            }
        }
        o5[P] = (uint32_t)recs.size();
        r->ext_end = o5[P];
        recs.insert(recs.end(), F.recs.begin() + F.ext_end, F.recs.end());
        for (uint32_t k = 0; k < G * A; ++k) {
            recs[r->ext_end + k].z += shift;
            recs[r->ext_end + k].w += shift;
        }
        std::map<std::pair<uint32_t, uint32_t>, uint32_t> set_of;
        for (uint32_t g = 0; g < G; ++g) {                           // area 0's entry of an ASBR with type-4 slots
            auto o = orig.find(F.group_asbr[g]);
            if (o == orig.end()) continue;
            const RibRec s = recs[r->ext_end + g * A + i0];
            const std::vector<RibRec> st(recs.begin() + s.z, recs.begin() + s.w);
            const uint32_t z = (uint32_t)recs.size();
            merge_lsakey(st, adv_rtr, o->second, borders, [&](const RibRec &x) { recs.push_back(x); },
                         [&](const std::pair<uint32_t, uint32_t> &x) {
                             recs.push_back(asbr_slot(borders, bv[x.first], x, o->first, set_of, t->asbr_set));
                             ++t->n_asbr_slots;
                         });
            recs[r->ext_end + g * A + i0] = RibRec{s.x, s.y, z, (uint32_t)recs.size()};
            t->asbr_group.push_back(g);
            t->asbr_group_id.push_back(o->first);
        }
        if (t->asbr_set.size() > kOspfBackboneMaxAsbrSets) return HSPF_E_UNSUPPORTED;   // the kernel parameter's
        // the walk's intra-area ranges: the affected prefixes' records again, each naming its decode record
        t->walk_intra = (uint32_t)recs.size();
        for (uint32_t i = 0; i < A; ++i) {
            for (u = 0; u < P; ++u) {
                r->off[i * S + u] = (uint32_t)recs.size();
                if (from[u] == kNone) continue;
                for (uint32_t k = F.off[i * SF + from[u]]; k < F.off[i * SF + from[u] + 1]; ++k) {
                    recs.push_back(F.recs[k]);
                    t->intra_src.push_back(k);
                }
            }
            r->off[i * S + P] = (uint32_t)recs.size();
        }
        r->vl_off.assign(A + 1, 0);
        if (recs.size() >= kNoRecord || !backbone_winners_fit(recs.size(), t->slot_rec.size(), T::kV3))
            return HSPF_E_UNSUPPORTED;
        t->words = r->off;
        t->words.resize(((t->words.size() + 3) & ~(size_t)3), 0);
        if (const int rc2 = append_border_words<T::kV3>(t->words, borders, n_borders, a0.data(), false)) return rc2;
        t->abr = r.release();
        *out = t.release();
        return HSPF_OK;
    } catch (const std::bad_alloc &) {
        return HSPF_E_NOMEM;
    } catch (...) {
        return HSPF_E_UNSUPPORTED;
    }
}

// One area of a decode: record and prefix indices are the decoded table's unless said otherwise.
template <class T>
struct RibDecodeArea {
    const typename T::Area *a;
    const hspf_ospfv2_ribtable *rt;      // the area's one-area table
    const uint32_t *prefix_of;           // per prefix: its index in rt, 0xFFFFFFFF if none
    uint32_t intra_first;                // the first of the area's intra-area records, which are rt's in rt's order
    uint64_t intra_end;                  // one past the last record an intra-area cell of the area may name
    const uint32_t *o3;                  // [P + 1] the area's type-3 record ranges
    uint32_t base;                       // atom a of the area is bit base + a of the cell's masks ...
    uint64_t mask;                       // ... and these are its bits
    uint32_t area_id;
    typename T::JobDecode *jd;           // the job's decode state over the area
};

template <class T>
struct RibDecode {
    std::vector<RibDecodeArea<T>> area;
    uint32_t P;
    const uint32_t *prefix, *plen;       // [P] (OSPFv3: prefix6)
    const hl_ip_addr *prefix6;
    const uint32_t *o5;                  // [P + 1] type-5 record ranges
    const uint32_t *ext_tag;             // per type-5 record (index - ext_base): the LSA's tag
    uint32_t ext_base;
    uint32_t max_paths;
    const uint8_t *options;              // OSPFv3: per type-3 / type-5 record (index - options_base), its prefix options
    uint32_t options_base;
};

// One job's cells -> its routing table, in prefix order, into `out` (HSPF_E_NOMEM with the counts when it does not
// fit).  1. Each area's intra-area winners go through that area's intra-area decode, every area before step 2, so
// that its refusals come before step 2's.  2. A route is the intra-area route, or the type-3 / type-5 winner checked
// against its record range; every other atom of the cell resolves through its own area's resolver; the union of the
// next hops in next-hop order, cut to max_paths, is what rib_full's merge-then-clip leaves.  Two atoms that give one
// next hop with different attributes refuse the job (HSPF_E_UNSUPPORTED): the reference keeps whichever came last.
template <class T>
int decode_rib(const RibDecode<T> &d, const hl_ospf_rib_cell *cells, typename T::Rib *out) {
    using Nh = typename T::Nh;
    constexpr uint32_t kNone = 0xFFFFFFFFu;
    const uint32_t A = (uint32_t)d.area.size(), P = d.P;
    auto intra_area = [&](uint32_t w) {
        for (uint32_t i = 0; i < A; ++i)
            if (w >= d.area[i].intra_first && w < d.area[i].intra_end) return i;
        return kNone;
    };
    // 1. per area, the intra-area cells its records won, through the intra-area decode
    std::vector<std::vector<typename T::Net>> nets(A);
    std::vector<std::vector<typename T::Hop>> nh(A);
    std::vector<typename T::Result> res(A);
    for (uint32_t i = 0; i < A; ++i) {
        const RibDecodeArea<T> &ar = d.area[i];
        const hspf_ospfv2_ribtable &rt = *ar.rt;
        const uint32_t PI = (uint32_t)rt.intra->t.plen.size();
        std::vector<hl_route_cell> ic(PI, hl_route_cell{0, 0, kNone, 0, 0, 0});
        for (uint32_t u = 0; u < P; ++u) {
            const hl_ospf_rib_cell &c = cells[u];
            if (!(HL_RIB_CELL_FLAGS(c) & HL_CELL_PRESENT) || HL_RIB_CELL_PATH(c) != HL_PATH_INTRA_AREA) continue;
            if (intra_area(c.winner) != i) continue;
            const uint32_t q = ar.prefix_of[u];
            if (q == kNone || rt.intra_of[q] == kNone || HL_RIB_CELL_METRIC(c) > 0xFFFFu) return HSPF_E_INVAL;
            ic[rt.intra_of[q]] = hl_route_cell{(c.nh_mask & ar.mask) >> ar.base, (c.aux & ar.mask) >> ar.base,
                                               c.winner - ar.intra_first, (uint16_t)HL_RIB_CELL_METRIC(c),
                                               (uint8_t)HL_RIB_CELL_FLAGS(c), 0};
        }
        nets[i].resize(PI);
        nh[i].resize(std::max<size_t>(64, (size_t)PI * 2));
        int rc = HSPF_OK;
        for (int attempt = 0; attempt < 2; ++attempt) {
            res[i] = typename T::Result{};
            res[i].routes_cap = PI; res[i].routes = nets[i].data();
            res[i].nexthops_cap = (uint32_t)nh[i].size(); res[i].nexthops = nh[i].data();
            rc = T::intra_from_cells(*ar.jd, ar.a, rt.intra, ic.data(), &res[i]);
            if (rc != HSPF_E_NOMEM) break;
            nh[i].resize(res[i].n_nexthops);
        }
        if (rc) return rc;
    }
    // 2. every route in prefix order; the atoms no intra-area route gave through their own area's resolver
    std::vector<typename T::Route> routes;
    std::vector<typename T::Hop> hops;
    std::vector<Nh> set;
    std::vector<uint32_t> ri(A, 0);
    auto sort_key = [&](uint32_t i, uint32_t iface) {
        const typename T::Area &a = *d.area[i].a;
        return iface < a.n_ifaces ? a.ifaces[iface].sort_key : 0xFFFFFFFFu;
    };
    auto add_atoms = [&](uint64_t m) {
        for (; m; m &= m - 1) {
            const uint32_t b = (uint32_t)__builtin_ctzll(m);
            uint32_t i = 0;
            while (i < A && !((d.area[i].mask >> b) & 1u)) ++i;
            if (i == A) return HSPF_E_INVAL;                       // an atom no area has
            for (const Nh &x : d.area[i].jd->rs->resolve(b - d.area[i].base)) {
                auto at = std::lower_bound(set.begin(), set.end(), x, T::nh_less);
                if (at == set.end() || !T::nh_same(*at, x)) { set.insert(at, x); continue; }
                if (T::nh_conflict(*at, x)) return HSPF_E_UNSUPPORTED;
            }
        }
        return HSPF_OK;
    };
    for (uint32_t u = 0; u < P; ++u) {
        const hl_ospf_rib_cell &c = cells[u];
        if (!(HL_RIB_CELL_FLAGS(c) & HL_CELL_PRESENT)) continue;
        const uint32_t path = HL_RIB_CELL_PATH(c);
        typename T::Route o;
        std::memset(&o, 0, sizeof(o));
        T::route_prefix(o, d, u);
        o.path_type = (uint8_t)path;
        o.nh_off = (uint32_t)hops.size();
        set.clear();
        uint64_t rest = c.nh_mask;
        if (path == HL_PATH_INTRA_AREA) {
            const uint32_t w = intra_area(c.winner);
            if (w == kNone || ri[w] >= res[w].n_routes) return HSPF_E_INVAL;
            const typename T::Net &r = nets[w][ri[w]++];
            o.metric = r.metric; o.area_id = d.area[w].area_id; o.has_area = 1; o.flags = r.flags;
            T::from_intra(o, r);
            rest &= ~d.area[w].mask;
            for (uint32_t k = 0; k < r.n_nh; ++k) {
                typename T::Hop h = nh[w][r.nh_off + k];
                const uint32_t sort = sort_key(w, h.iface);
                // with no other area's atoms the area's decode has merged and cut them: straight to the output
                if (rest) set.push_back(T::to_nh(h, sort));
                else { h.iface = sort; hops.push_back(h); }
            }
        } else {
            if (path == HL_PATH_INTER_AREA) {
                uint32_t w = 0;
                while (w < A && !(c.winner >= d.area[w].o3[u] && c.winner < d.area[w].o3[u + 1])) ++w;
                if (w == A) return HSPF_E_INVAL;
                o.metric = HL_RIB_CELL_METRIC(c); o.area_id = d.area[w].area_id; o.has_area = 1;
            } else {
                if (c.winner < d.o5[u] || c.winner >= d.o5[u + 1]) return HSPF_E_INVAL;
                o.metric = HL_RIB_CELL_METRIC(c);
                o.tag = d.ext_tag[c.winner - d.ext_base];
                if (path == HL_PATH_TYPE2_EXTERNAL) { o.has_type2 = 1; o.type2_metric = (uint32_t)c.aux; }
            }
            T::from_record(o, d, c.winner);
        }
        const int rc = add_atoms(rest);
        if (rc) return rc;
        if (set.size() > d.max_paths) set.resize(d.max_paths);
        for (const Nh &x : set) hops.push_back(T::to_hop(x));
        o.n_nh = (uint32_t)hops.size() - o.nh_off;
        routes.push_back(o);
    }
    out->n_routes = (uint32_t)routes.size();
    out->n_nexthops = (uint32_t)hops.size();
    if (out->n_routes > out->routes_cap || out->n_nexthops > out->nexthops_cap) return HSPF_E_NOMEM;
    if ((out->n_routes && !out->routes) || (out->n_nexthops && !out->nexthops)) return HSPF_E_INVAL;
    std::copy(routes.begin(), routes.end(), out->routes);
    std::copy(hops.begin(), hops.end(), out->nexthops);
    return HSPF_OK;
}

// hspf_ospfv2_rib_from_cells / hspf_ospfv3_rib_from_cells after their argument checks: the decode of a table with
// one area whose prefixes, records and atoms are all the table's own.  Every intra-area cell is the area's, so that
// the intra-area decode refuses a winner outside the intra-area records, as it does for the area's own cells.
template <class T>
int decode_one_area_rib(const typename T::Area *a, const hspf_ospfv2_ribtable &rt, const hl_ospf_rib_cell *cells,
                        const uint32_t *gather_v, const uint64_t *gather_nh, uint32_t n_gather, typename T::Rib *out) {
    typename T::JobDecode jd;
    const int rc = jd.init(a, (uint32_t)rt.vflags.size(), gather_v, gather_nh, n_gather);
    if (rc) return rc;
    if (jd.root == 0xFFFFFFFFu) return HSPF_E_INVAL;               // not the root of any job over this table
    const uint32_t P = (uint32_t)rt.plen.size();
    const uint32_t *o3 = rt.off.data() + P + 1;
    std::vector<uint32_t> same(P);
    std::iota(same.begin(), same.end(), 0u);
    RibDecode<T> d{{RibDecodeArea<T>{a, &rt, same.data(), 0, ~0ull, o3, 0, ~0ull, rt.area_id, &jd}},
                   P, rt.prefix.data(), rt.plen.data(), rt.prefix6.data(), o3 + P + 1, rt.ext_tag.data(), rt.ext_base,
                   a->max_paths, rt.options6.data(), rt.n_intra};
    return decode_rib(d, cells, out);
}

// hspf_ospfv2_abr_rib_from_cells / hspf_ospfv3_abr_rib_from_cells, argument checks included: each area's job
// decode over its own gathers, and the decode of the router's table over them.  A table of the other version is
// refused (HSPF_E_INVAL).  `options` (OSPFv3): the prefix options of each type-3 / type-5 record (index -
// t3_base[0]) the routes take, the table's own when NULL.
template <class T>
int decode_abr_rib(const hspf_ospfv2_abr_ribtable *t, const typename T::Area *areas, uint32_t n_areas,
                   const hl_ospf_rib_cell *cells, const uint32_t *gather_area, const uint32_t *gather_v,
                   const uint64_t *gather_nh, uint32_t n_gather, typename T::Rib *out,
                   const uint8_t *options = nullptr) {
    if (!t || t->v3 != T::kV3 || !areas || !cells || !out || n_areas != t->n_areas ||
        (n_gather && (!gather_area || !gather_v || !gather_nh)))
        return HSPF_E_INVAL;
    try {
        out->n_routes = out->n_nexthops = 0;
        const uint32_t A = n_areas, P = (uint32_t)t->plen.size(), S = P + 1;
        std::vector<typename T::JobDecode> jd(A);
        RibDecode<T> d{{}, P, t->prefix.data(), t->plen.data(), t->prefix6.data(), t->off.data() + 2 * (size_t)A * S,
                       t->ext_tag.data(), t->ext_base, t->max_paths, options ? options : t->options6.data(),
                       t->t3_base[0]};
        for (uint32_t i = 0; i < A; ++i) {
            const typename T::Area &a = areas[i];
            if (a.router_id != t->router_id || a.area_id != t->area_id[i] || a.max_paths != t->max_paths) return HSPF_E_INVAL;
            std::vector<uint32_t> gv;
            std::vector<uint64_t> gn;
            for (uint32_t g = 0; g < n_gather; ++g) {
                if (gather_area[g] >= A) return HSPF_E_INVAL;
                if (gather_area[g] == i) { gv.push_back(gather_v[g]); gn.push_back(gather_nh[g]); }
            }
            const int rc = jd[i].init(&a, t->n_vertices[i], gv.data(), gn.data(), (uint32_t)gv.size());
            if (rc) return rc;
            if (jd[i].root != t->root[i]) return HSPF_E_INVAL;
            const uint32_t na = t->n_atoms[i];
            const uint64_t mask = na == 0 ? 0 : ((na == 64 ? ~0ull : ((1ull << na) - 1)) << t->base[i]);
            d.area.push_back({&a, t->area[i], t->area_prefix[i].data(), t->intra_base[i],
                              (uint64_t)t->intra_base[i] + t->area[i]->n_intra, t->off.data() + (A + i) * (size_t)S,
                              t->base[i], mask, t->area_id[i], &jd[i]});
        }
        return decode_rib(d, cells, out);
    } catch (const std::bad_alloc &) {
        return HSPF_E_NOMEM;
    } catch (...) {
        return HSPF_E_INVAL;
    }
}

// hspf_ospfv2_abr_backbone_from_cells / hspf_ospfv3_abr_backbone_from_cells, argument checks included: a slot winner
// names its type-3 record (OSPFv3: and carries the options the route takes, written into this job's copy of the
// table's options) and a walk intra-area record the decode's, then decode_abr_rib over the table's prefixes.  A table
// of the other version is refused (HSPF_E_INVAL).
template <class T>
int decode_abr_backbone_rib(const hspf_ospfv2_abr_backbone_table *t, const typename T::Area *areas, uint32_t n_areas,
                            const hl_ospf_rib_cell *cells, const uint32_t *gather_area, const uint32_t *gather_v,
                            const uint64_t *gather_nh, uint32_t n_gather, typename T::Rib *out) {
    if (!t || !t->abr || t->abr->v3 != T::kV3 || !cells || !out) return HSPF_E_INVAL;
    try {
        const uint32_t n_recs = t->n_recs();
        std::vector<hl_ospf_rib_cell> c(cells, cells + t->P());
        std::vector<uint8_t> options(t->abr->options6);
        for (hl_ospf_rib_cell &x : c) {
            if (!(HL_RIB_CELL_FLAGS(x) & HL_CELL_PRESENT)) continue;
            if (x.winner >= n_recs) {
                uint32_t s = x.winner - n_recs, opt = 0;
                if (T::kV3) { opt = s & 0xFFu; s >>= 8; }
                if (HL_RIB_CELL_PATH(x) != HL_PATH_INTER_AREA || s >= t->slot_rec.size()) return HSPF_E_INVAL;
                x.winner = t->slot_rec[s];
                if (T::kV3) options[x.winner - t->abr->t3_base[0]] = (uint8_t)opt;
            } else if (HL_RIB_CELL_PATH(x) == HL_PATH_INTRA_AREA) {
                if (x.winner < t->walk_intra || x.winner - t->walk_intra >= t->intra_src.size()) return HSPF_E_INVAL;
                x.winner = t->intra_src[x.winner - t->walk_intra];
            }
        }
        return decode_abr_rib<T>(t->abr, areas, n_areas, c.data(), gather_area, gather_v, gather_nh, n_gather, out,
                                 T::kV3 ? options.data() : nullptr);
    } catch (const std::bad_alloc &) {
        return HSPF_E_NOMEM;
    } catch (...) {
        return HSPF_E_INVAL;
    }
}

// hspf_ospfv2_backbone_from_cells / hspf_ospfv3_backbone_from_cells, argument checks included: the decode of R's
// one-area table (over the table's target area) over the affected prefixes, a slot winner naming its type-3 record (and, OSPFv3, carrying the
// options the route takes).  A table of the other version is refused (HSPF_E_INVAL).
template <class T>
int decode_backbone_rib(const hspf_ospfv2_backbone_table *t, const typename T::Area *a, const hl_ospf_rib_cell *cells,
                        const uint32_t *gather_v, const uint64_t *gather_nh, uint32_t n_gather, typename T::Rib *out) {
    if (!t || t->v3 != T::kV3 || !a || !cells || !out || (n_gather && (!gather_v || !gather_nh))) return HSPF_E_INVAL;
    if (a->router_id != t->router_id || a->area_id != t->area_id || a->max_paths != t->max_paths) return HSPF_E_INVAL;
    try {
        out->n_routes = out->n_nexthops = 0;
        typename T::JobDecode jd;
        const int rc = jd.init(a, t->n_vertices, gather_v, gather_nh, n_gather);
        if (rc) return rc;
        if (jd.root != t->root) return HSPF_E_INVAL;
        const uint32_t P = t->P(), n_recs = (uint32_t)t->recs.size();
        const OspfBackboneView v = t->host_view();
        std::vector<hl_ospf_rib_cell> c(cells, cells + P);
        std::vector<uint8_t> options(t->options6);                 // OSPFv3: this job's, a slot's from its winner
        for (hl_ospf_rib_cell &x : c) {
            if (!(HL_RIB_CELL_FLAGS(x) & HL_CELL_PRESENT) || HL_RIB_CELL_PATH(x) != HL_PATH_INTER_AREA || x.winner < n_recs)
                continue;
            uint32_t s = x.winner - n_recs, opt = 0;
            if (T::kV3) { opt = s & 0xFFu; s >>= 8; }
            if (s >= t->slot_rec.size()) return HSPF_E_INVAL;
            x.winner = t->slot_rec[s];
            if (T::kV3) options[x.winner - v.o3[0]] = (uint8_t)opt;
        }
        RibDecode<T> d{{RibDecodeArea<T>{a, t->r, v.q, 0, ~0ull, v.o3, 0, ~0ull, t->area_id, &jd}},
                       P, t->prefix.data(), t->plen.data(), T::kV3 ? t->prefix6.data() : nullptr, v.o5,
                       t->ext_tag.data(), t->ext_base, t->max_paths, T::kV3 ? options.data() : nullptr,
                       T::kV3 ? v.o3[0] : 0};
        return decode_rib(d, c.data(), out);
    } catch (const std::bad_alloc &) {
        return HSPF_E_NOMEM;
    } catch (...) {
        return HSPF_E_INVAL;
    }
}

}  // namespace hspf
