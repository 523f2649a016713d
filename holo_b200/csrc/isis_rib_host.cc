// The end of holo-isis' update_rib: hspf_isis_rib_merge / hspf_isis_rib_diff
// (include/holo_spf_lsdb.h) — merge of the per-level tables with L1 preferred
// (holo-isis/src/route.rs:236-242) and update_global_rib (route.rs:255-314).  Both inputs are in
// prefix order (IPv4 before IPv6, address, then length), so both are single merge walks.
// Also the L1/L2-router pieces that sit between the two SPF levels: active summary routes
// (route.rs:193-229) and lsp_propagate_l1_to_l2 (lsdb.rs:1149-1357).
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <new>
#include <unordered_map>
#include <vector>

#include "../../include/holo_lsdb.h"
#include "../../include/holo_spf.h"
#include "../../include/holo_spf_lsdb.h"
#include "isis_propagation.h"

namespace {

int cmp_prefix(const hl_isis_route &a, const hl_isis_route &b) {
    if (a.prefix.is_v6 != b.prefix.is_v6) return a.prefix.is_v6 < b.prefix.is_v6 ? -1 : 1;
    const int c = std::memcmp(a.prefix.bytes, b.prefix.bytes, 16);
    if (c) return c < 0 ? -1 : 1;
    return a.len == b.len ? 0 : (a.len < b.len ? -1 : 1);
}

bool rib_ok(const hl_isis_rib *r) {
    if (!r) return true;
    if ((r->n_routes && !r->routes) || (r->n_nexthops && !r->nexthops)) return false;
    for (uint32_t i = 0; i < r->n_routes; ++i)
        if ((uint64_t)r->routes[i].nh_off + r->routes[i].n_nh > r->n_nexthops) return false;
    return true;
}

bool same_hop(const hl_isis_nexthop &a, const hl_isis_nexthop &b) {   // Nexthop == (route.rs:50-61)
    return a.system_id == b.system_id && a.iface == b.iface && a.addr.is_v6 == b.addr.is_v6 &&
           std::memcmp(a.addr.bytes, b.addr.bytes, 16) == 0 && a.has_label == b.has_label &&
           (!a.has_label || a.sr_label == b.sr_label);
}

}  // namespace

extern "C" int hspf_isis_rib_merge(const hl_isis_rib *l2, const hl_isis_rib *l1, hl_isis_rib *out) {
    if (!out || !rib_ok(l2) || !rib_ok(l1)) return HSPF_E_INVAL;
    try {
        struct Pick { const hl_isis_rib *src; uint32_t idx; };
        std::vector<Pick> picks;
        const uint32_t n2 = l2 ? l2->n_routes : 0, n1 = l1 ? l1->n_routes : 0;
        uint32_t i = 0, j = 0, n_h = 0;
        while (i < n2 || j < n1) {
            int c = i == n2 ? 1 : (j == n1 ? -1 : cmp_prefix(l2->routes[i], l1->routes[j]));
            if (c < 0) picks.push_back(Pick{l2, i++});
            else { picks.push_back(Pick{l1, j++}); if (c == 0) ++i; }   // same prefix: the L1 route wins
        }
        for (const Pick &p : picks) n_h += p.src->routes[p.idx].n_nh;
        out->n_routes = (uint32_t)picks.size();
        out->n_nexthops = n_h;
        if (out->n_routes > out->routes_cap || n_h > out->nexthops_cap) return HSPF_E_NOMEM;
        if ((out->n_routes && !out->routes) || (n_h && !out->nexthops)) return HSPF_E_INVAL;
        uint32_t h = 0;
        for (uint32_t r = 0; r < picks.size(); ++r) {
            hl_isis_route o = picks[r].src->routes[picks[r].idx];
            const hl_isis_nexthop *from = picks[r].src->nexthops + o.nh_off;
            o.nh_off = h;
            for (uint32_t k = 0; k < o.n_nh; ++k) out->nexthops[h++] = from[k];
            out->routes[r] = o;
        }
        return HSPF_OK;
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

extern "C" int hspf_isis_rib_diff(const hl_isis_rib *old_rib, hl_isis_rib *new_rib, hl_rib_action *out, uint32_t cap,
                                  uint32_t *n_out) {
    if (!new_rib || !n_out || (cap && !out) || !rib_ok(new_rib) || !rib_ok(old_rib)) return HSPF_E_INVAL;
    try {
        const uint32_t n_old = old_rib ? old_rib->n_routes : 0;
        std::vector<hl_rib_action> acts;
        auto push = [&](uint8_t kind, uint32_t route, const hl_isis_route *replaced) {
            hl_rib_action a;
            std::memset(&a, 0, sizeof(a));
            a.kind = kind; a.route = route;
            if (replaced) { a.has_old_sr_label = replaced->has_sr_label; a.old_sr_label = replaced->has_sr_label ? replaced->sr_label : 0; }
            acts.push_back(a);
        };
        std::vector<uint32_t> gone;
        uint32_t io = 0;
        for (uint32_t in = 0; in < new_rib->n_routes; ++in) {
            hl_isis_route &r = new_rib->routes[in];
            while (io < n_old && cmp_prefix(old_rib->routes[io], r) < 0) {
                if (old_rib->routes[io].flags & HL_ROUTE_INSTALLED) gone.push_back(io);
                ++io;
            }
            const hl_isis_route *o = (io < n_old && cmp_prefix(old_rib->routes[io], r) == 0) ? &old_rib->routes[io++] : nullptr;
            if (o) {
                bool same = o->metric == r.metric && o->n_nh == r.n_nh;      // tag: always None here
                for (uint32_t k = 0; same && k < r.n_nh; ++k)
                    same = same_hop(old_rib->nexthops[o->nh_off + k], new_rib->nexthops[r.nh_off + k]);
                if (same) {
                    if (o->flags & HL_ROUTE_INSTALLED) r.flags |= HL_ROUTE_INSTALLED;
                    continue;
                }
            }
            if (!(r.flags & HL_ROUTE_CONNECTED) && ((r.flags & HL_ROUTE_SUMMARY) || r.n_nh != 0)) {
                push(HL_RIB_INSTALL, in, o);
                r.flags |= HL_ROUTE_INSTALLED;
            } else if (r.flags & HL_ROUTE_INSTALLED) {
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
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

// ---- L1/L2 routers: summaries and L1 -> L2 propagation ---------------------------------------
namespace {

struct Pfx { hl_ip_addr a; uint8_t len; };

int cmp_pfx(const hl_ip_addr &a, uint8_t al, const hl_ip_addr &b, uint8_t bl) {
    if (a.is_v6 != b.is_v6) return a.is_v6 < b.is_v6 ? -1 : 1;
    const int c = std::memcmp(a.bytes, b.bytes, 16);
    if (c) return c < 0 ? -1 : 1;
    return al == bl ? 0 : (al < bl ? -1 : 1);
}

bool covers(const hl_ip_addr &net, uint8_t nlen, const hl_ip_addr &a, uint8_t alen) {   // net/nlen contains a/alen
    if (net.is_v6 != a.is_v6 || nlen > alen) return false;
    for (uint32_t bit = 0; bit < nlen; bit += 8) {
        const uint32_t left = nlen - bit;
        const uint8_t mask = left >= 8 ? 0xFF : (uint8_t)(0xFF << (8 - left));
        if ((net.bytes[bit / 8] ^ a.bytes[bit / 8]) & mask) return false;
    }
    return true;
}

// JointPrefixMap::get_spm: the SHORTEST configured prefix that contains the query
int shortest_match(const hl_isis_summary *cfg, uint32_t n, const hl_ip_addr &a, uint8_t len) {
    int best = -1;
    for (uint32_t i = 0; i < n; ++i)
        if (covers(cfg[i].prefix, cfg[i].len, a, len) && (best < 0 || cfg[i].len < cfg[best].len)) best = (int)i;
    return best;
}

uint32_t summary_metric(const hl_isis_summary &s) { return s.has_cfg_metric ? s.cfg_metric : s.metric; }

}  // namespace

namespace hspf {
int isis_summary_match(const hl_isis_summary *cfg, uint32_t n_cfg, const hl_ip_addr &a, uint8_t len) {
    return shortest_match(cfg, n_cfg, a, len);
}
}  // namespace hspf

extern "C" int hspf_isis_summaries(const hl_isis_rib *l1, const hl_isis_summary *cfg, uint32_t n_cfg,
                                   hl_isis_summary *out, uint32_t *n_out) {
    if (!n_out || (n_cfg && (!cfg || !out)) || !rib_ok(l1)) return HSPF_E_INVAL;
    try {
        std::vector<uint32_t> low(n_cfg, 0);
        std::vector<uint8_t> active(n_cfg, 0);
        for (uint32_t i = 0; l1 && i < l1->n_routes; ++i) {
            const hl_isis_route &r = l1->routes[i];
            const int k = shortest_match(cfg, n_cfg, r.prefix, r.len);
            if (k < 0) continue;
            if (!active[k] || r.metric < low[k]) low[k] = r.metric;
            active[k] = 1;
        }
        uint32_t n = 0;
        for (uint32_t k = 0; k < n_cfg; ++k)
            if (active[k]) { out[n] = cfg[k]; out[n].metric = low[k]; ++n; }
        *n_out = n;
        return HSPF_OK;
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

extern "C" int hspf_isis_rib_add_summaries(const hl_isis_rib *l2, const hl_isis_summary *active, uint32_t n_active,
                                           hl_isis_rib *out) {
    if (!out || !rib_ok(l2) || (n_active && !active)) return HSPF_E_INVAL;
    const uint32_t n2 = l2 ? l2->n_routes : 0;
    // both inputs are in prefix order: one merge walk, a summary replaces the L2 route of its prefix
    uint32_t i = 0, j = 0, n_r = 0, n_h = 0;
    while (i < n2 || j < n_active) {
        const int c = i == n2 ? 1 : (j == n_active ? -1 : cmp_pfx(l2->routes[i].prefix, l2->routes[i].len, active[j].prefix, active[j].len));
        if (c < 0) { n_h += l2->routes[i].n_nh; ++i; } else { ++j; if (c == 0) ++i; }
        ++n_r;
    }
    out->n_routes = n_r; out->n_nexthops = n_h;
    if (n_r > out->routes_cap || n_h > out->nexthops_cap) return HSPF_E_NOMEM;
    if ((n_r && !out->routes) || (n_h && !out->nexthops)) return HSPF_E_INVAL;
    i = j = 0;
    uint32_t r = 0, h = 0;
    while (i < n2 || j < n_active) {
        const int c = i == n2 ? 1 : (j == n_active ? -1 : cmp_pfx(l2->routes[i].prefix, l2->routes[i].len, active[j].prefix, active[j].len));
        if (c < 0) {
            hl_isis_route o = l2->routes[i];
            const hl_isis_nexthop *from = l2->nexthops + o.nh_off;
            o.nh_off = h;
            for (uint32_t k = 0; k < o.n_nh; ++k) out->nexthops[h++] = from[k];
            out->routes[r++] = o;
            ++i;
        } else {
            hl_isis_route o;
            std::memset(&o, 0, sizeof(o));
            o.prefix = active[j].prefix; o.len = active[j].len;
            o.metric = summary_metric(active[j]);
            o.route_type = HL_ISIS_RT_L2_INTRA;
            o.flags = HL_ROUTE_SUMMARY;
            o.nh_off = h;
            out->routes[r++] = o;
            ++j;
            if (c == 0) ++i;
        }
    }
    return HSPF_OK;
}

extern "C" int hspf_isis_l1_to_l2(const hl_isis_level *l1, const uint8_t *up_down, uint64_t local_system_id,
                                  const hl_isis_spt *spt_std, const hl_isis_spt *spt_v6, uint8_t l1_metric_type,
                                  uint8_t l2_metric_type, const hl_isis_summary *cfg, uint32_t n_cfg,
                                  const hl_isis_summary *active, uint32_t n_active, hl_isis_ipreach *out, uint32_t cap,
                                  uint32_t *n_out) {
    if (!l1 || !n_out || !spt_std || (cap && !out) || (n_cfg && !cfg) || (n_active && !active)) return HSPF_E_INVAL;
    try {
        // Vertex.distance of a system in an SPT
        auto index_of = [](const hl_isis_spt *spt) {
            std::unordered_map<uint64_t, uint32_t> m;
            if (spt) { m.reserve(spt->n_vertices * 2); for (uint32_t i = 0; i < spt->n_vertices; ++i) m.emplace(spt->vertices[i].lan_id, spt->vertices[i].distance); }
            return m;
        };
        const auto dmap_std = index_of(spt_std), dmap_v6 = index_of(spt_v6);
        auto dist_of = [](const std::unordered_map<uint64_t, uint32_t> &m, uint64_t lan_id) -> uint32_t {
            auto it = m.find(lan_id);
            return it == m.end() ? HSPF_DIST_INF : it->second;
        };
        auto std_on = [](uint8_t t) { return t == HL_ISIS_METRIC_STANDARD || t == HL_ISIS_METRIC_BOTH; };
        auto wide_on = [](uint8_t t) { return t == HL_ISIS_METRIC_WIDE || t == HL_ISIS_METRIC_BOTH; };
        const bool mt6 = spt_v6 != nullptr;           // IPv6 unicast topology enabled
        std::vector<hl_isis_ipreach> best;            // kept sorted by (kind, prefix)
        auto key_cmp = [](const hl_isis_ipreach &a, const hl_isis_ipreach &b) {
            if (a.kind != b.kind) return a.kind < b.kind ? -1 : 1;
            return cmp_pfx(a.prefix, a.len, b.prefix, b.len);
        };
        auto offer = [&](hl_isis_ipreach e) {
            size_t lo = 0, hi = best.size();
            while (lo < hi) { const size_t mid = (lo + hi) / 2; if (key_cmp(best[mid], e) < 0) lo = mid + 1; else hi = mid; }
            if (lo < best.size() && key_cmp(best[lo], e) == 0) { if (e.metric < best[lo].metric) best[lo] = e; }
            else best.insert(best.begin() + (long)lo, e);
        };
        hspf::for_each_propagation(*l1, local_system_id, l1_metric_type, l2_metric_type, mt6, up_down, cfg, n_cfg,
                                   [&](const hl_isis_lsp &lsp, uint32_t k, uint8_t kind, uint32_t topology, bool is_narrow) {
            const uint32_t d = dist_of(topology ? dmap_v6 : dmap_std, lsp.lan_id);
            if (d == HSPF_DIST_INF) return;                             // originator not on the L1 SPT
            hl_isis_ipreach e = l1->ipreaches[k];
            if (e.kind != kind) { e.kind = kind; e.mt_id = 0; }         // MT-IPv6 into the L2 LSP's IPv6 reachability
            const uint64_t sum = (uint64_t)e.metric + d;
            e.metric = is_narrow ? (uint32_t)std::min<uint64_t>(sum, 63) : (uint32_t)std::min<uint64_t>(sum, 0xFFFFFFFFull);
            hspf::isis_propagated_sid(e);
            offer(e);
        });
        for (uint32_t j = 0; j < n_active; ++j) {       // active summaries (inserted: they replace an equal prefix)
            hl_isis_ipreach e;
            std::memset(&e, 0, sizeof(e));
            e.prefix = active[j].prefix; e.len = active[j].len;
            const uint32_t m = summary_metric(active[j]);
            auto put = [&](uint8_t kind, uint32_t metric) {
                e.kind = kind; e.metric = metric;
                size_t lo = 0, hi = best.size();
                while (lo < hi) { const size_t mid = (lo + hi) / 2; if (key_cmp(best[mid], e) < 0) lo = mid + 1; else hi = mid; }
                if (lo < best.size() && key_cmp(best[lo], e) == 0) best[lo] = e; else best.insert(best.begin() + (long)lo, e);
            };
            if (!active[j].prefix.is_v6) {
                if (!l1->ipv4_enabled) continue;
                if (std_on(l2_metric_type)) put(HL_ISIS_IP_V4_INTERNAL, std::min<uint32_t>(m, 63));
                if (wide_on(l2_metric_type)) put(HL_ISIS_IP_V4_EXT, m);
            } else {
                if (!l1->ipv6_enabled) continue;
                put(HL_ISIS_IP_V6, m);
            }
        }
        *n_out = (uint32_t)best.size();
        if (best.size() > cap) return HSPF_E_NOMEM;
        for (size_t i = 0; i < best.size(); ++i) out[i] = best[i];
        return HSPF_OK;
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}
