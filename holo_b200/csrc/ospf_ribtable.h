// The record-building half of hspf_ospfv2_ribtable_create / hspf_ospfv3_ribtable_create (include/holo_spf_lsdb.h),
// written once over a small version trait, as rib_full is in ospf_rib_host.cc.  The versions differ only in the prefix
// key, in which field of an inter-area-router LSA names the ASBR, and in the NU-bit LSAs OSPFv3 skips; the records the
// walk reads (ospf_rib_cells.h) are the same.  Host only.
//
// A version trait T provides:
//   Key                        prefix key; its order is the table's prefix order (update_rib_full's IpNetwork order)
//   Sum, Ext                   the summary / inter-area LSA and the AS-external LSA
//   key(Sum), key(Ext)         the LSA's prefix key (host bits kept, as update_rib_full keeps them)
//   intra_key(RouteTable, k)   the key of prefix k of the area's intra-area table
//   skip(Sum), skip(Ext)       LSAs update_rib_full never uses whatever the job (OSPFv3: NU bit)
//   asbr_id(Sum)               the ASBR a type-4 LSA names
//   options(Sum), options(Ext) prefix options a route through the LSA carries
//   set_prefix(rt, u, Key)     writes prefix u of the table
//   kV3                        the table carries OSPFv3 prefixes and per-record prefix options
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <unordered_map>
#include <vector>

#include "holo_spf_lsdb.h"
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
    return HSPF_OK;
}

}  // namespace hspf
