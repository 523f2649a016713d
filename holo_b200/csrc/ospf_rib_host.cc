// OSPF routing table after the per-area SPFs: hspf_ospfv2_update_rib_full /
// hspf_ospfv3_update_rib_full (include/holo_spf_lsdb.h).  Host-side table joins over the
// results of hspf_ospfv{2,3}_run_area; replaces, for the stages after the SPT,
//   update_rib_full                  holo-ospf/src/route.rs:146-193
//   update_rib_inter_area_networks   route.rs:449-533   (type-3 Summary / Inter-Area-Prefix LSAs)
//   update_rib_inter_area_routers    route.rs:653-714   (type-4 Summary / Inter-Area-Router LSAs)
//   update_rib_transit_area          route.rs:535-650   (RFC 2328 16.3, virtual links)
//   update_rib_external              route.rs:717-827   (AS-external LSAs)
//   route_update / route_compare     route.rs:895-971
// The reference is generic over the OSPF version; so is this file: one template, two small
// trait structs for the address / record types.  Routes live in one flat vector with a hash
// index on (address bytes, prefix length); next-hop sets are small vectors kept sorted by
// NexthopKey (interface sort key, then address with None first), merged like
// BTreeMap::extend (a later entry with the same key replaces the earlier one).
#include <algorithm>
#include <array>
#include <cstdint>
#include <cstring>
#include <map>
#include <new>
#include <unordered_map>
#include <vector>

#include "../../include/holo_lsdb.h"
#include "../../include/holo_spf.h"
#include "../../include/holo_spf_lsdb.h"

namespace {

// ---- prefix key: 16 address bytes (IPv4 in the first four, network byte order) + length ----
struct PKey {
    std::array<uint8_t, 17> b{};
    bool operator==(const PKey &o) const { return b == o.b; }
    bool operator<(const PKey &o) const { return b < o.b; }   // address, then prefix length
};
struct PKeyHash {
    size_t operator()(const PKey &k) const {
        uint64_t h = 1469598103934665603ull;
        for (uint8_t x : k.b) { h ^= x; h *= 1099511628211ull; }
        return (size_t)h;
    }
};

template <class Nh>
struct HopT {
    uint64_t ka;                      // NexthopKey, major: sort_key << 1 | has_addr (None first)
    std::array<uint8_t, 16> kb;       // minor: the address
    Nh nh;
};
template <class Nh> bool key_less(const HopT<Nh> &p, const HopT<Nh> &q) { return p.ka != q.ka ? p.ka < q.ka : p.kb < q.kb; }
template <class Nh> bool key_same(const HopT<Nh> &p, const HopT<Nh> &q) { return p.ka == q.ka && p.kb == q.kb; }

// dst <- dst extended with src (same key: src wins)
template <class Nh>
void merge_hops(std::vector<HopT<Nh>> &dst, const std::vector<HopT<Nh>> &src) {
    std::vector<HopT<Nh>> out;
    out.reserve(dst.size() + src.size());
    size_t i = 0, j = 0;
    while (i < dst.size() || j < src.size()) {
        if (j == src.size() || (i < dst.size() && key_less(dst[i], src[j]))) out.push_back(dst[i++]);
        else if (i == dst.size() || key_less(src[j], dst[i])) out.push_back(src[j++]);
        else { out.push_back(src[j++]); ++i; }
    }
    dst.swap(out);
}

// ---- version traits --------------------------------------------------------------------------
struct V2 {
    using Area = hl_ospfv2_rib_area;
    using Sum = hl_ospfv2_summary_lsa;
    using Ext = hl_ospfv2_external_lsa;
    using Rib = hl_ospfv2_rib;
    using NetIn = hl_route_net;
    using Nh = hl_nexthop;
    using Out = hl_rib_route;
    static void put4(PKey &k, uint32_t a, uint32_t mask) {
        k.b[0] = (uint8_t)(a >> 24); k.b[1] = (uint8_t)(a >> 16); k.b[2] = (uint8_t)(a >> 8); k.b[3] = (uint8_t)a;
        k.b[16] = (uint8_t)__builtin_popcount(mask);
    }
    static PKey key(const NetIn &r) { PKey k; put4(k, r.prefix, r.mask); return k; }
    // with_netmask(lsa_id, mask) without apply_mask (ospfv2/spf.rs:552,602): host bits are kept
    static PKey key(const Sum &l) { PKey k; put4(k, l.lsa_id, l.mask); return k; }
    static PKey key(const Ext &l) { PKey k; put4(k, l.lsa_id, l.mask); return k; }
    static bool skip(const Sum &) { return false; }
    static bool skip(const Ext &) { return false; }
    static uint32_t asbr_id(const Sum &l) { return l.lsa_id; }
    static uint8_t options(const NetIn &) { return 0; }
    static uint8_t options(const Out &) { return 0; }
    static uint8_t options(const Sum &) { return 0; }
    static uint8_t options(const Ext &) { return 0; }
    static void label_in(bool &has, uint32_t &label, const NetIn &r) { has = r.has_sr_label != 0; label = r.sr_label; }
    static void label_out(Out &o, bool has, uint32_t label) { o.has_sr_label = has ? 1 : 0; o.sr_label = has ? label : 0; }
    static bool same_label(const Out &a, const Out &b) {
        return a.has_sr_label == b.has_sr_label && (!a.has_sr_label || a.sr_label == b.sr_label);
    }
    static void old_label(hl_rib_action &act, const Out &o) { act.has_old_sr_label = o.has_sr_label; act.old_sr_label = o.has_sr_label ? o.sr_label : 0; }
    static bool same_prefix(const Out &a, const Out &b) { return a.prefix == b.prefix && a.mask == b.mask; }
    static bool prefix_less(const Out &a, const Out &b) { return a.prefix != b.prefix ? a.prefix < b.prefix : a.mask < b.mask; }
    static bool same_hop(const Nh &a, const Nh &b) {
        return a.iface == b.iface && a.has_addr == b.has_addr && (!a.has_addr || a.addr == b.addr) && a.has_nbr == b.has_nbr &&
               (!a.has_nbr || a.nbr_router_id == b.nbr_router_id) && a.has_label == b.has_label &&
               (!a.has_label || a.sr_label == b.sr_label);
    }
    static void addr_key(const Nh &n, std::array<uint8_t, 16> &kb) {
        kb.fill(0);
        if (n.has_addr) { kb[0] = (uint8_t)(n.addr >> 24); kb[1] = (uint8_t)(n.addr >> 16); kb[2] = (uint8_t)(n.addr >> 8); kb[3] = (uint8_t)n.addr; }
    }
    // the key of a route in net_summaries' table: (prefix, mask), as the summary LSA names it
    using SumKey = std::pair<uint32_t, uint32_t>;
    static SumKey sum_key(const Out &r) { return {r.prefix, r.mask}; }
    static void emit(Out &o, const PKey &k, uint8_t /*options*/) {
        o.prefix = ((uint32_t)k.b[0] << 24) | ((uint32_t)k.b[1] << 16) | ((uint32_t)k.b[2] << 8) | k.b[3];
        o.mask = k.b[16] ? 0xFFFFFFFFu << (32 - k.b[16]) : 0u;
    }
};

struct V3 {
    using Area = hl_ospfv3_rib_area;
    using Sum = hl_ospfv3_inter_area_lsa;
    using Ext = hl_ospfv3_external_lsa;
    using Rib = hl_ospfv3_rib;
    using NetIn = hl_route_net6;
    using Nh = hl_nexthop6;
    using Out = hl_rib_route6;
    static PKey mk(const hl_ip_addr &a, uint8_t len) { PKey k; std::memcpy(k.b.data(), a.bytes, 16); k.b[16] = len; return k; }
    static PKey key(const NetIn &r) { return mk(r.prefix, r.len); }
    static PKey key(const Sum &l) { return mk(l.prefix, l.len); }
    static PKey key(const Ext &l) { return mk(l.prefix, l.len); }
    static bool skip(const Sum &l) { return l.lsa_type == 3 && (l.prefix_options & HL_PFX_OPT_NU); }   // ospfv3/spf.rs:494
    static bool skip(const Ext &l) { return (l.prefix_options & HL_PFX_OPT_NU) != 0; }                   // ospfv3/spf.rs:538
    static uint32_t asbr_id(const Sum &l) { return l.router_id; }
    static uint8_t options(const NetIn &r) { return r.prefix_options; }
    static uint8_t options(const Out &r) { return r.prefix_options; }
    static uint8_t options(const Sum &l) { return l.prefix_options; }
    static uint8_t options(const Ext &l) { return l.prefix_options; }
    static void label_in(bool &, uint32_t &, const NetIn &) {}
    static void label_out(Out &, bool, uint32_t) {}
    static bool same_label(const Out &, const Out &) { return true; }
    static void old_label(hl_rib_action &, const Out &) {}
    static bool same_prefix(const Out &a, const Out &b) { return a.len == b.len && std::memcmp(a.prefix.bytes, b.prefix.bytes, 16) == 0; }
    static bool prefix_less(const Out &a, const Out &b) {
        const int c = std::memcmp(a.prefix.bytes, b.prefix.bytes, 16);
        return c != 0 ? c < 0 : a.len < b.len;
    }
    static bool same_hop(const Nh &a, const Nh &b) {
        return a.iface == b.iface && a.has_addr == b.has_addr && (!a.has_addr || std::memcmp(a.addr.bytes, b.addr.bytes, 16) == 0) &&
               a.has_nbr == b.has_nbr && (!a.has_nbr || a.nbr_router_id == b.nbr_router_id);
    }
    static void addr_key(const Nh &n, std::array<uint8_t, 16> &kb) {
        kb.fill(0);
        if (n.has_addr) std::memcpy(kb.data(), n.addr.bytes, 16);
    }
    using SumKey = PKey;
    static SumKey sum_key(const Out &r) { return mk(r.prefix, r.len); }
    static void emit(Out &o, const PKey &k, uint8_t options) {
        std::memcpy(o.prefix.bytes, k.b.data(), 16);
        o.prefix.is_v6 = 1;
        o.len = k.b[16];
        o.prefix_options = options;
    }
};

// ---- router entries (area.state.routers), shared by rib_full and rtr_summaries -------------------
template <class T> using HopsT = std::vector<HopT<typename T::Nh>>;
template <class T>
struct RtrT {
    uint32_t area, metric;
    uint8_t path, flags;
    HopsT<T> hops;
};
template <class T> using RtrTable = std::unordered_map<uint32_t, RtrT<T>>;

// the areas' SPF results are consistent with their next-hop arrays
template <class T>
bool areas_ok(const typename T::Area *areas, uint32_t n_areas) {
    if (!areas && n_areas) return false;
    for (uint32_t ai = 0; ai < n_areas; ++ai) {
        const auto &a = areas[ai];
        if (!a.spf || (a.n_ifaces && !a.ifaces) || (a.n_summaries && !a.summaries)) return false;
        const auto &r = *a.spf;
        if ((r.n_routers && !r.routers) || (r.n_routes && !r.routes) || (r.n_nexthops && !r.nexthops)) return false;
        for (uint32_t i = 0; i < r.n_routers; ++i)
            if ((uint64_t)r.routers[i].nh_off + r.routers[i].n_nh > r.n_nexthops) return false;
        for (uint32_t i = 0; i < r.n_routes; ++i)
            if ((uint64_t)r.routes[i].nh_off + r.routes[i].n_nh > r.n_nexthops) return false;
    }
    return true;
}

// an SPF entry's next hops, interfaces named by sort key, in NexthopKey order (same key twice: the later one stays)
template <class T>
HopsT<T> hops_of(const typename T::Area &a, uint32_t off, uint32_t n) {
    HopsT<T> h;
    h.reserve(n);
    for (uint32_t i = 0; i < n; ++i) {
        HopT<typename T::Nh> x;
        x.nh = a.spf->nexthops[off + i];
        const uint32_t sk = x.nh.iface < a.n_ifaces ? a.ifaces[x.nh.iface].sort_key : 0xFFFFFFFFu;
        x.nh.iface = sk;                   // the merged table names interfaces by sort key
        x.ka = ((uint64_t)sk << 1) | (x.nh.has_addr ? 1u : 0u);
        T::addr_key(x.nh, x.kb);
        h.push_back(x);
    }
    std::stable_sort(h.begin(), h.end(), key_less<typename T::Nh>);
    HopsT<T> u;
    for (const auto &x : h) {
        if (!u.empty() && key_same(u.back(), x)) u.back() = x;
        else u.push_back(x);
    }
    return u;
}

template <class T>
bool summary_usable(uint32_t router_id, const typename T::Sum &l) {
    return !l.maxage && l.metric < HL_LSA_INFINITY && l.adv_rtr != router_id && !T::skip(l);
}

// abr(): the area's entry for `adv` when it has the B flag
template <class T>
const RtrT<T> *abr_entry(const RtrTable<T> &rtrs, uint32_t adv) {
    auto it = rtrs.find(adv);
    return (it != rtrs.end() && (it->second.flags & HL_RTR_FLAG_B)) ? &it->second : nullptr;
}

// rib_full step 1, routers: the area's intra-area router entries
template <class T>
void intra_area_routers(const typename T::Area &a, RtrTable<T> &rtrs) {
    for (uint32_t i = 0; i < a.spf->n_routers; ++i) {
        const hl_route_rtr &r = a.spf->routers[i];
        rtrs[r.router_id] = RtrT<T>{a.area_id, r.metric, HL_PATH_INTRA_AREA, r.flags, hops_of<T>(a, r.nh_off, r.n_nh)};
    }
}

// rib_full step 2, ASBRs (update_rib_inter_area_routers): each usable type-4 / Inter-Area-Router LSA of the area
// whose ABR has an entry writes an inter-area entry for the ASBR it names, replacing any earlier one
template <class T>
void inter_area_routers(uint32_t router_id, const typename T::Area &a, RtrTable<T> &rtrs) {
    for (uint32_t i = 0; i < a.n_summaries; ++i) {
        const auto &l = a.summaries[i];
        if (l.lsa_type != 4 || !summary_usable<T>(router_id, l)) continue;
        const RtrT<T> *br = abr_entry<T>(rtrs, l.adv_rtr);
        if (!br) continue;
        RtrT<T> e{a.area_id, br->metric + l.metric, HL_PATH_INTER_AREA, HL_RTR_FLAG_E, br->hops};
        rtrs[T::asbr_id(l)] = std::move(e);
    }
}

// rib_full step 2 reads every area's summaries with one active area, else only the backbone's
template <class T>
bool reads_summaries(const typename T::Area *areas, uint32_t n_areas, uint32_t ai) {
    uint32_t n_active = 0;
    for (uint32_t i = 0; i < n_areas; ++i) n_active += areas[i].active ? 1u : 0u;
    return n_active <= 1 || areas[ai].area_id == 0;
}

// ---- the stages ------------------------------------------------------------------------------
template <class T>
int rib_full(uint32_t router_id, uint32_t max_paths, const typename T::Area *areas, uint32_t n_areas,
             const typename T::Ext *ext, uint32_t n_ext, typename T::Rib *out) {
    using Hop = HopT<typename T::Nh>;
    using Hops = HopsT<T>;
    using Rtr = RtrT<T>;
    struct Net {
        PKey key;
        uint32_t metric, type2, tag, area;
        uint8_t path, flags, options;
        bool has_area, has_type2;
        Hops hops;
        bool has_label = false;
        uint32_t label = 0;
        uint32_t origin_id = 0;            // LS origin of an intra-area route
    };
    if (!areas_ok<T>(areas, n_areas) || (!ext && n_ext) || !out) return HSPF_E_INVAL;
    auto clip = [&](Hops &h) { if (h.size() > max_paths) h.resize(max_paths); };
    auto prefer = [](const Net &a, const Net &b) -> int {      // route_compare; negative: a wins
        if (a.path != b.path) return a.path < b.path ? -1 : 1;
        if (a.path == HL_PATH_TYPE2_EXTERNAL) {
            if (a.has_type2 != b.has_type2) return a.has_type2 ? 1 : -1;     // None < Some
            if (a.type2 != b.type2) return a.type2 < b.type2 ? -1 : 1;
        }
        if (a.metric != b.metric) return a.metric < b.metric ? -1 : 1;
        return 0;
    };
    std::vector<Net> nets;
    std::unordered_map<PKey, uint32_t, PKeyHash> index;
    auto find = [&](const PKey &k) -> Net * {
        auto it = index.find(k);
        return it == index.end() ? nullptr : &nets[it->second];
    };
    auto offer = [&](Net &&n) {                                 // route_update
        Net *cur = find(n.key);
        if (!cur) {
            index.emplace(n.key, (uint32_t)nets.size());
            nets.push_back(std::move(n));
            cur = &nets.back();
        } else {
            const int c = prefer(n, *cur);
            if (c < 0) *cur = std::move(n);
            else if (c == 0) merge_hops(cur->hops, n.hops);
        }
        clip(cur->hops);
    };
    auto usable = [&](const typename T::Sum &l) { return summary_usable<T>(router_id, l); };
    std::vector<RtrTable<T>> rtrs(n_areas);

    // 1. per-area router tables; intra-area routes of all areas into one table
    for (uint32_t ai = 0; ai < n_areas; ++ai) {
        const auto &a = areas[ai];
        intra_area_routers<T>(a, rtrs[ai]);
        for (uint32_t i = 0; i < a.spf->n_routes; ++i) {
            const auto &r = a.spf->routes[i];
            const PKey k = T::key(r);
            Net *cur = find(k);
            if (cur && r.metric > cur->metric) continue;
            Net n{k, r.metric, 0, 0, a.area_id, HL_PATH_INTRA_AREA, r.flags, T::options(r), true, false,
                  hops_of<T>(a, r.nh_off, r.n_nh)};
            T::label_in(n.has_label, n.label, r);
            n.origin_id = r.origin_lsa_id;
            if (cur && r.origin_type == 2) {
                // the areas share one table in the reference: a transit network that maps to a prefix
                // another area already gave takes the entry over unless its LSA id is lower, and
                // never merges into it (route.rs:387-397)
                if (r.origin_lsa_id < cur->origin_id) continue;
                *cur = std::move(n);
                clip(cur->hops);
                continue;
            }
            offer(std::move(n));
        }
    }

    // 2. summaries: only the backbone's when more than one area is active
    auto abr = [&](uint32_t ai, uint32_t adv) { return abr_entry<T>(rtrs[ai], adv); };
    for (uint32_t ai = 0; ai < n_areas; ++ai) {
        const auto &a = areas[ai];
        if (!reads_summaries<T>(areas, n_areas, ai)) continue;
        for (uint32_t i = 0; i < a.n_summaries; ++i) {            // networks
            const auto &l = a.summaries[i];
            if (l.lsa_type != 3 || !usable(l)) continue;
            const Rtr *br = abr(ai, l.adv_rtr);
            if (!br) continue;
            offer(Net{T::key(l), br->metric + l.metric, 0, 0, a.area_id, HL_PATH_INTER_AREA, 0, T::options(l), true,
                      false, br->hops});
        }
        inter_area_routers<T>(router_id, a, rtrs[ai]);            // ASBRs
    }

    // 3. transit areas
    for (uint32_t ai = 0; ai < n_areas; ++ai) {
        const auto &a = areas[ai];
        if (!a.spf->transit_capability) continue;
        for (uint32_t i = 0; i < a.n_summaries; ++i) {
            const auto &l = a.summaries[i];
            if (l.lsa_type != 3 || !usable(l)) continue;
            Net *cur = find(T::key(l));
            if (!cur || cur->path > HL_PATH_INTER_AREA || !cur->has_area || cur->area != 0) continue;
            const Rtr *br = abr(ai, l.adv_rtr);
            if (!br) continue;
            const uint32_t metric = br->metric + l.metric;
            if (metric < cur->metric) {
                const PKey k = cur->key;
                *cur = Net{k, metric, 0, 0, a.area_id, HL_PATH_INTER_AREA, 0, T::options(l), true, false, br->hops};
            } else if (metric == cur->metric) {
                merge_hops(cur->hops, br->hops);
            }
            clip(cur->hops);
        }
    }

    // 4. AS-external LSAs through the best ASBR entry (areas in area-id order)
    std::vector<uint32_t> order(n_areas);
    for (uint32_t i = 0; i < n_areas; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return areas[x].area_id < areas[y].area_id; });
    for (uint32_t i = 0; i < n_ext; ++i) {
        const auto &l = ext[i];
        if (l.maxage || !(l.metric < HL_LSA_INFINITY) || l.adv_rtr == router_id || T::skip(l)) continue;
        const Rtr *best = nullptr;
        bool best_pref = false;          // intra-area through a non-backbone area
        for (uint32_t ai : order) {
            auto it = rtrs[ai].find(l.adv_rtr);
            if (it == rtrs[ai].end() || !(it->second.flags & HL_RTR_FLAG_E)) continue;
            const Rtr *r = &it->second;
            const bool pref = r->path == HL_PATH_INTRA_AREA && r->area != 0;
            if (!best || (pref && !best_pref)) { best = r; best_pref = pref; continue; }
            if (pref != best_pref) continue;
            if (r->metric < best->metric || (r->metric == best->metric && r->area > best->area)) best = r;
        }
        if (!best) continue;
        Net n{T::key(l), 0, 0, l.tag, 0, 0, 0, T::options(l), false, false, best->hops};
        if (l.e_bit) { n.path = HL_PATH_TYPE2_EXTERNAL; n.metric = best->metric; n.has_type2 = true; n.type2 = l.metric; }
        else { n.path = HL_PATH_TYPE1_EXTERNAL; n.metric = best->metric + l.metric; }
        offer(std::move(n));
    }

    // emit in IpNetwork order (address, then prefix length)
    std::vector<uint32_t> idx(nets.size());
    for (uint32_t i = 0; i < idx.size(); ++i) idx[i] = i;
    std::sort(idx.begin(), idx.end(), [&](uint32_t x, uint32_t y) { return nets[x].key < nets[y].key; });
    uint32_t n_h = 0;
    for (const Net &n : nets) n_h += (uint32_t)n.hops.size();
    out->n_routes = (uint32_t)nets.size();
    out->n_nexthops = n_h;
    if (out->n_routes > out->routes_cap || n_h > out->nexthops_cap) return HSPF_E_NOMEM;
    if ((out->n_routes && !out->routes) || (n_h && !out->nexthops)) return HSPF_E_INVAL;
    uint32_t h = 0;
    for (uint32_t r = 0; r < idx.size(); ++r) {
        const Net &n = nets[idx[r]];
        typename T::Out o;
        std::memset(&o, 0, sizeof(o));
        T::emit(o, n.key, n.options);
        o.metric = n.metric; o.type2_metric = n.type2; o.tag = n.tag; o.area_id = n.area; o.path_type = n.path;
        o.flags = n.flags; o.has_area = n.has_area ? 1 : 0; o.has_type2 = n.has_type2 ? 1 : 0;
        o.nh_off = h; o.n_nh = (uint32_t)n.hops.size();
        T::label_out(o, n.has_label, n.label);
        for (const Hop &x : n.hops) out->nexthops[h++] = x.nh;
        out->routes[r] = o;
    }
    return HSPF_OK;
}

// update_global_rib (route.rs:833-893): both tables are in prefix order, so one merge walk
template <class T>
int rib_diff(const typename T::Rib *old_rib, typename T::Rib *new_rib, hl_rib_action *out, uint32_t cap, uint32_t *n_out) {
    if (!new_rib || !n_out || (cap && !out)) return HSPF_E_INVAL;
    if ((new_rib->n_routes && !new_rib->routes) || (new_rib->n_nexthops && !new_rib->nexthops)) return HSPF_E_INVAL;
    const uint32_t n_old = old_rib ? old_rib->n_routes : 0;
    if (old_rib && ((n_old && !old_rib->routes) || (old_rib->n_nexthops && !old_rib->nexthops))) return HSPF_E_INVAL;
    for (uint32_t i = 0; i < new_rib->n_routes; ++i)
        if ((uint64_t)new_rib->routes[i].nh_off + new_rib->routes[i].n_nh > new_rib->n_nexthops) return HSPF_E_INVAL;
    for (uint32_t i = 0; i < n_old; ++i)
        if ((uint64_t)old_rib->routes[i].nh_off + old_rib->routes[i].n_nh > old_rib->n_nexthops) return HSPF_E_INVAL;
    auto metric_of = [](const typename T::Out &r) { return r.path_type == HL_PATH_TYPE2_EXTERNAL ? r.type2_metric : r.metric; };
    std::vector<hl_rib_action> acts;
    auto push = [&](uint8_t kind, uint32_t route, const typename T::Out *replaced) {
        hl_rib_action a;
        std::memset(&a, 0, sizeof(a));
        a.kind = kind; a.route = route;
        if (replaced) T::old_label(a, *replaced);
        acts.push_back(a);
    };
    std::vector<uint32_t> gone;       // old routes without a successor, installed
    uint32_t io = 0;
    for (uint32_t in = 0; in < new_rib->n_routes; ++in) {
        typename T::Out &r = new_rib->routes[in];
        while (io < n_old && T::prefix_less(old_rib->routes[io], r)) {
            if (old_rib->routes[io].flags & HL_ROUTE_INSTALLED) gone.push_back(io);
            ++io;
        }
        const typename T::Out *o = (io < n_old && T::same_prefix(old_rib->routes[io], r)) ? &old_rib->routes[io++] : nullptr;
        if (o) {
            bool same = metric_of(*o) == metric_of(r) && o->tag == r.tag && T::same_label(*o, r) && o->n_nh == r.n_nh;
            for (uint32_t k = 0; same && k < r.n_nh; ++k)
                same = T::same_hop(old_rib->nexthops[o->nh_off + k], new_rib->nexthops[r.nh_off + k]);
            if (same) {
                if (o->flags & HL_ROUTE_INSTALLED) r.flags |= HL_ROUTE_INSTALLED;
                continue;
            }
        }
        if (!(r.flags & HL_ROUTE_CONNECTED) && r.n_nh != 0) {
            push(HL_RIB_INSTALL, in, o);
            r.flags |= HL_ROUTE_INSTALLED;
        } else if (r.flags & HL_ROUTE_INSTALLED) {
            // only for tables a caller carries over: update_rib_full builds every route with
            // empty or CONNECTED flags, so after a full run this branch is not taken
            push(HL_RIB_UNINSTALL, in, nullptr);
            r.flags &= (uint8_t)~HL_ROUTE_INSTALLED;
        }
    }
    for (; io < n_old; ++io)
        if (old_rib->routes[io].flags & HL_ROUTE_INSTALLED) gone.push_back(io);
    for (uint32_t i : gone) push(HL_RIB_UNINSTALL_OLD, i, nullptr);
    *n_out = (uint32_t)acts.size();
    if (acts.size() > cap) return HSPF_E_NOMEM;
    for (size_t i = 0; i < acts.size(); ++i) out[i] = acts[i];
    return HSPF_OK;
}

template <class T, class... A>
int guarded(A... args) {
    try {
        return rib_full<T>(args...);
    } catch (const std::bad_alloc &) {
        return HSPF_E_NOMEM;
    } catch (...) {
        return HSPF_E_INVAL;
    }
}

}  // namespace

extern "C" int hspf_ospfv2_update_rib_full(uint32_t router_id, uint32_t max_paths, const hl_ospfv2_rib_area *areas,
                                           uint32_t n_areas, const hl_ospfv2_external_lsa *ext, uint32_t n_ext,
                                           hl_ospfv2_rib *out) {
    return guarded<V2>(router_id, max_paths, areas, n_areas, ext, n_ext, out);
}

extern "C" int hspf_ospfv3_update_rib_full(uint32_t router_id, uint32_t max_paths, const hl_ospfv3_rib_area *areas,
                                           uint32_t n_areas, const hl_ospfv3_external_lsa *ext, uint32_t n_ext,
                                           hl_ospfv3_rib *out) {
    return guarded<V3>(router_id, max_paths, areas, n_areas, ext, n_ext, out);
}

namespace {

// nexthops_area_check (holo-ospf area.rs:742): a next hop on one of area `ta`'s interfaces (next hops name them by
// sort key)
template <class Area, class Nh>
bool nexthops_on_area(const Area &ta, const Nh *h, uint32_t n) {
    for (uint32_t k = 0; k < n; ++k)
        for (uint32_t i = 0; i < ta.n_ifaces; ++i)
            if (h[k].iface == ta.ifaces[i].sort_key) return true;
    return false;
}

// The checks both versions' net_summaries make of a routing table and the areas
template <class Rib, class Area>
bool net_summaries_args(const Rib *rib, const Area *areas, const hl_ospf_area_config *config, uint32_t n_areas,
                        uint32_t target) {
    if (!rib || !areas || !config || target >= n_areas) return false;
    if ((rib->n_routes && !rib->routes) || (rib->n_nexthops && !rib->nexthops)) return false;
    for (uint32_t i = 0; i < rib->n_routes; ++i)
        if ((uint64_t)rib->routes[i].nh_off + rib->routes[i].n_nh > rib->n_nexthops) return false;
    for (uint32_t i = 0; i < n_areas; ++i)
        if (areas[i].n_ifaces && !areas[i].ifaces) return false;
    return true;
}

// compute_net_summaries (holo-ospf area.rs:561-659) of an ABR for one target area, without area ranges and without
// LSA ids: the type-3 / Inter-Area-Prefix contents keyed as the reference's summary table (T::sum_key; `dflt` is
// the default route's key), each (metric, prefix options), a later entry replacing an earlier one.  Empty when at
// most one area is active (not an ABR).
template <class T>
std::map<typename T::SumKey, std::pair<uint32_t, uint8_t>> net_summaries(const typename T::Rib &rib,
                                                                        const typename T::Area *areas, uint32_t n_areas,
                                                                        uint32_t target, const hl_ospf_area_config &cfg,
                                                                        const typename T::SumKey &dflt) {
    std::map<typename T::SumKey, std::pair<uint32_t, uint8_t>> net;
    uint32_t n_active = 0;
    for (uint32_t i = 0; i < n_areas; ++i) n_active += areas[i].active ? 1u : 0u;
    if (n_active <= 1) return net;
    const typename T::Area &ta = areas[target];
    const bool backbone = ta.area_id == 0;
    if (cfg.summary)
        for (uint32_t i = 0; i < rib.n_routes; ++i) {
            const typename T::Out &r = rib.routes[i];
            if (r.path_type >= HL_PATH_TYPE1_EXTERNAL || r.metric >= HL_LSA_INFINITY) continue;
            if (r.has_area && r.area_id == ta.area_id) continue;
            if (backbone && r.path_type != HL_PATH_INTRA_AREA) continue;
            if (nexthops_on_area(ta, rib.nexthops + r.nh_off, r.n_nh)) continue;
            net[T::sum_key(r)] = {r.metric, T::options(r)};
        }
    if (cfg.area_type != HL_AREA_NORMAL) net[dflt] = {cfg.default_cost, 0};
    return net;
}

// compute_rtr_summaries (holo-ospf area.rs:699-740) of an ABR for one target area: ASBR id -> metric.  `each(f)` calls
// f(area_id, router_id, metric, path_type, flags, next hops, n_nh) for every router entry, in the call's area order
// (an id in two areas keeps the later area's).  Only into a normal area, and only when more than one area is active.
template <class Area, class Each>
std::map<uint32_t, uint32_t> rtr_summaries(const Area *areas, uint32_t n_areas, uint32_t target,
                                           const hl_ospf_area_config &cfg, Each each) {
    std::map<uint32_t, uint32_t> rtr;
    uint32_t n_active = 0;
    for (uint32_t i = 0; i < n_areas; ++i) n_active += areas[i].active ? 1u : 0u;
    if (n_active <= 1 || cfg.area_type != HL_AREA_NORMAL) return rtr;
    const Area &ta = areas[target];
    const bool backbone = ta.area_id == 0;
    each([&](uint32_t area_id, uint32_t id, uint32_t metric, uint8_t path, uint8_t flags, const auto *nh, uint32_t n_nh) {
        if (area_id == ta.area_id || !(flags & HL_RTR_FLAG_E) || metric >= HL_LSA_INFINITY) return;
        if (backbone && path != HL_PATH_INTRA_AREA) return;
        if (nexthops_on_area(ta, nh, n_nh)) return;
        rtr[id] = metric;
    });
    return rtr;
}

}  // namespace

// compute_net_summaries / compute_rtr_summaries (holo-ospf area.rs:561-740) of an ABR for one target area, without
// area ranges and without LSA ids: each map keyed as the reference's summary tables, a later entry replacing
// an earlier one
extern "C" int hspf_ospfv2_net_summaries(uint32_t router_id, const hl_ospfv2_rib *rib, const hl_ospfv2_rtr_tables *rtrs,
                                         const hl_ospfv2_rib_area *areas, const hl_ospf_area_config *config,
                                         uint32_t n_areas, uint32_t target, hl_ospfv2_summary_lsa *out, uint32_t cap,
                                         uint32_t *n_out) {
    if (!rtrs || !n_out || (cap && !out) || !net_summaries_args(rib, areas, config, n_areas, target)) return HSPF_E_INVAL;
    if ((rtrs->n_rtrs && !rtrs->rtrs) || (rtrs->n_nexthops && !rtrs->nexthops)) return HSPF_E_INVAL;
    for (uint32_t i = 0; i < rtrs->n_rtrs; ++i)
        if ((uint64_t)rtrs->rtrs[i].nh_off + rtrs->rtrs[i].n_nh > rtrs->n_nexthops) return HSPF_E_INVAL;
    try {
        *n_out = 0;
        const auto net = net_summaries<V2>(*rib, areas, n_areas, target, config[target], {0u, 0u});
        const auto rtr = rtr_summaries(areas, n_areas, target, config[target], [&](auto f) {
            for (uint32_t i = 0; i < rtrs->n_rtrs; ++i) {
                const hl_rib_rtr &r = rtrs->rtrs[i];
                f(r.area_id, r.router_id, r.metric, r.path_type, r.flags, rtrs->nexthops + r.nh_off, r.n_nh);
            }
        });
        *n_out = (uint32_t)(net.size() + rtr.size());
        if (*n_out > cap) return HSPF_E_NOMEM;
        uint32_t k = 0;
        auto put = [&](uint8_t type, uint32_t id, uint32_t mask, uint32_t metric) {
            hl_ospfv2_summary_lsa l;
            std::memset(&l, 0, sizeof(l));
            l.adv_rtr = router_id; l.lsa_id = id; l.mask = mask; l.metric = metric; l.lsa_type = type;
            out[k++] = l;
        };
        for (const auto &e : net) put(3, e.first.first, e.first.second, e.second.first);
        for (const auto &e : rtr) put(4, e.first, 0, e.second);
        return HSPF_OK;
    } catch (const std::bad_alloc &) {
        return HSPF_E_NOMEM;
    } catch (...) {
        return HSPF_E_INVAL;
    }
}

// compute_net_summaries for OSPFv3 (Inter-Area-Prefix contents, lsa_orig_inter_area_network, ospfv3/lsdb.rs:341-386):
// each route's prefix options go into the LSA it originates
extern "C" int hspf_ospfv3_net_summaries(uint32_t router_id, const hl_ospfv3_rib *rib, const hl_ospfv3_rib_area *areas,
                                         const hl_ospf_area_config *config, uint32_t n_areas, uint32_t target,
                                         hl_ospfv3_inter_area_lsa *out, uint32_t cap, uint32_t *n_out) {
    if (!n_out || (cap && !out) || !net_summaries_args(rib, areas, config, n_areas, target)) return HSPF_E_INVAL;
    try {
        *n_out = 0;
        const auto net = net_summaries<V3>(*rib, areas, n_areas, target, config[target], PKey{});
        *n_out = (uint32_t)net.size();
        if (*n_out > cap) return HSPF_E_NOMEM;
        uint32_t k = 0;
        for (const auto &e : net) {
            hl_ospfv3_inter_area_lsa l;
            std::memset(&l, 0, sizeof(l));
            l.adv_rtr = router_id; l.metric = e.second.first; l.lsa_type = 3;
            std::memcpy(l.prefix.bytes, e.first.b.data(), 16);
            l.prefix.is_v6 = 1;
            l.len = e.first.b[16]; l.prefix_options = e.second.second;
            out[k++] = l;
        }
        return HSPF_OK;
    } catch (const std::bad_alloc &) {
        return HSPF_E_NOMEM;
    } catch (...) {
        return HSPF_E_INVAL;
    }
}

extern "C" int hspf_ospfv2_rib_diff(const hl_ospfv2_rib *old_rib, hl_ospfv2_rib *new_rib, hl_rib_action *out, uint32_t cap,
                                    uint32_t *n_out) {
    try { return rib_diff<V2>(old_rib, new_rib, out, cap, n_out); }
    catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

extern "C" int hspf_ospfv3_rib_diff(const hl_ospfv3_rib *old_rib, hl_ospfv3_rib *new_rib, hl_rib_action *out, uint32_t cap,
                                    uint32_t *n_out) {
    try { return rib_diff<V3>(old_rib, new_rib, out, cap, n_out); }
    catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

// compute_rtr_summaries for OSPFv3 (Inter-Area-Router contents): the type-4 rule of hspf_ospfv2_net_summaries over
// the router entries update_rib_full leaves (hspf_ospfv2_rib_router_tables' for OSPFv2), rebuilt from the same areas
extern "C" int hspf_ospfv3_rtr_summaries(uint32_t router_id, const hl_ospfv3_rib_area *areas,
                                         const hl_ospf_area_config *config, uint32_t n_areas, uint32_t target,
                                         hl_ospfv3_inter_area_lsa *out, uint32_t cap, uint32_t *n_out) {
    if (!n_out || (cap && !out) || !areas || !config || target >= n_areas || !areas_ok<V3>(areas, n_areas))
        return HSPF_E_INVAL;
    try {
        *n_out = 0;
        std::vector<RtrTable<V3>> rtrs(n_areas);
        for (uint32_t ai = 0; ai < n_areas; ++ai) intra_area_routers<V3>(areas[ai], rtrs[ai]);
        for (uint32_t ai = 0; ai < n_areas; ++ai)
            if (reads_summaries<V3>(areas, n_areas, ai)) inter_area_routers<V3>(router_id, areas[ai], rtrs[ai]);
        const auto rtr = rtr_summaries(areas, n_areas, target, config[target], [&](auto f) {
            std::vector<hl_nexthop6> nh;
            for (const RtrTable<V3> &tab : rtrs) {
                std::map<uint32_t, const RtrT<V3> *> by_id;             // router-id order
                for (const auto &e : tab) by_id.emplace(e.first, &e.second);
                for (const auto &e : by_id) {
                    const RtrT<V3> &r = *e.second;
                    nh.clear();
                    for (const auto &h : r.hops) nh.push_back(h.nh);
                    f(r.area, e.first, r.metric, r.path, r.flags, nh.data(), (uint32_t)nh.size());
                }
            }
        });
        *n_out = (uint32_t)rtr.size();
        if (*n_out > cap) return HSPF_E_NOMEM;
        uint32_t k = 0;
        for (const auto &e : rtr) {
            hl_ospfv3_inter_area_lsa l;
            std::memset(&l, 0, sizeof(l));
            l.adv_rtr = router_id; l.router_id = e.first; l.metric = e.second; l.lsa_type = 4;
            out[k++] = l;
        }
        return HSPF_OK;
    } catch (const std::bad_alloc &) {
        return HSPF_E_NOMEM;
    } catch (...) {
        return HSPF_E_INVAL;
    }
}
