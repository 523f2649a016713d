// isis_host.cc — IS-IS host side of the engine: level LSDB image -> CSR, and device
// result planes -> the reference's Spt (vertices with ordered ECMP parents, next-hop
// Vecs, first/second hops).
//
// The LSDB walk the reference repeats for every visited edge (vertex_edges over up
// to 256 fragments x 4 TLV kinds, plus the mutual-link re-iteration,
// holo-isis/src/spf.rs:605-625,1005-1120) happens here once; the per-vertex transit
// gates (missing zeroth LSP, overload bit, protocols-supported, spf.rs:556-602)
// become vertex flags.  Distances / hops / first-hop sets come from the CUDA kernel
// (hspf_run_batch); this file only orders what the kernel found the way the
// reference's pop order would have (parents: spf.rs:675, nexthops: spf.rs:678-702).
#include <algorithm>
#include <cstring>
#include <new>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "holo_spf_lsdb.h"

namespace {
constexpr uint32_t kNone = 0xFFFFFFFFu;
constexpr uint32_t kMaxWide = 0xFE000000u;
inline bool is_pn(hl_lan_id id) { return (id & 0xFF) != 0; }
}  // namespace

struct hspf_isis_flat {
    const hl_isis_level *lvl = nullptr;
    std::vector<hl_lan_id> ids;                 // [V] in VertexId order
    std::vector<uint32_t> row, col, cost;
    std::vector<uint8_t> vflags;
    std::vector<uint32_t> irow, isrc, ieid;     // transposed (host copy)
    std::unordered_map<uint64_t, uint32_t> index;
    uint32_t reject_above = 0, gflags = 0;
};

namespace {

int flatten(const hl_isis_level *l, hspf_isis_flat &f) {
    f.lvl = l;
    const bool mt_none = l->mt_id == HL_ISIS_MT_NONE, mt_std = l->mt_id == HL_ISIS_MT_STANDARD;
    const bool std_en = l->metric_type == HL_ISIS_METRIC_STANDARD || l->metric_type == HL_ISIS_METRIC_BOTH;
    const bool wide_en = l->metric_type == HL_ISIS_METRIC_WIDE || l->metric_type == HL_ISIS_METRIC_BOTH;
    const bool hopcount = l->metric_mode == HL_ISIS_MODE_HOPCOUNT;
    auto valid = [&](const hl_isis_lsp &p) { return p.seqno != 0 && p.rem_lifetime != 0; };

    // fragments in LspId order
    std::vector<uint32_t> order(l->n_lsps);
    for (uint32_t i = 0; i < l->n_lsps; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
        const auto &x = l->lsps[a], &y = l->lsps[b];
        return x.lan_id != y.lan_id ? x.lan_id < y.lan_id : x.fragment < y.fragment;
    });
    // vertices: every LAN id owning at least one valid fragment
    std::vector<hl_lan_id> pn, rt;
    for (uint32_t i : order) {
        const auto &p = l->lsps[i];
        if (!valid(p)) continue;
        auto &dst = is_pn(p.lan_id) ? pn : rt;
        if (dst.empty() || dst.back() != p.lan_id) dst.push_back(p.lan_id);
    }
    f.ids = pn;
    f.ids.insert(f.ids.end(), rt.begin(), rt.end());
    const uint32_t V = (uint32_t)f.ids.size();
    for (uint32_t v = 0; v < V; ++v) f.index.emplace(f.ids[v], v);
    f.vflags.assign(V, 0);
    std::vector<uint8_t> has_zeroth(V, 0);
    for (uint32_t v = 0; v < V; ++v) if (!is_pn(f.ids[v])) f.vflags[v] |= HSPF_VF_HOP;

    struct Raw { uint32_t u, v, cost; };
    std::vector<Raw> raw;
    raw.reserve(l->n_reaches);
    auto ecost = [&](hl_lan_id nbr, uint32_t metric) { return hopcount ? (is_pn(nbr) ? 0u : 1u) : metric; };
    for (uint32_t i : order) {
        const auto &p = l->lsps[i];
        if (!valid(p)) continue;
        const uint32_t u = f.index[p.lan_id];
        if (p.fragment == 0) {
            has_zeroth[u] = 1;
            if (!is_pn(p.lan_id)) {
                // overload bit: skipped unless root (spf.rs:566-572), only with an MT id
                if (!mt_none) {
                    const bool ol = mt_std ? (p.flags & HL_LSPF_OL) : (p.flags & HL_LSPF_MT_IPV6_OL);
                    if (ol) f.vflags[u] |= HSPF_VF_LEAF_UNLESS_ROOT;
                }
                // protocols-supported gate (spf.rs:580-602), standard topology only
                if (mt_std) {
                    bool ok = p.flags & HL_LSPF_HAS_PROTOCOLS;
                    if (ok && l->ipv4_enabled && !(p.flags & HL_LSPF_NLPID_IPV4)) ok = false;
                    if (ok && l->ipv6_enabled && !(p.flags & HL_LSPF_NLPID_IPV6)) ok = false;
                    if (!ok) f.vflags[u] |= HSPF_VF_LEAF;
                }
            }
        }
        const hl_isis_reach *re = l->reaches + p.reach_off;
        auto emit = [&](const hl_isis_reach &r) {
            auto it = f.index.find(r.neighbor);
            if (it == f.index.end()) return;       // no LSP: the mutual check can never pass
            raw.push_back({u, it->second, ecost(r.neighbor, r.metric)});
        };
        if ((mt_none || mt_std) && std_en)
            for (uint32_t k = 0; k < p.n_reach; ++k) if (re[k].kind == HL_ISIS_REACH_LEGACY) emit(re[k]);
        if (((mt_none || mt_std) || is_pn(p.lan_id)) && wide_en)
            for (uint32_t k = 0; k < p.n_reach; ++k)
                if (re[k].kind == HL_ISIS_REACH_EXT && re[k].metric < kMaxWide) emit(re[k]);
        if (!mt_none && !mt_std)
            for (uint32_t k = 0; k < p.n_reach; ++k)
                if (re[k].kind == HL_ISIS_REACH_MT && re[k].mt_id == l->mt_id && re[k].metric < kMaxWide) emit(re[k]);
        if (mt_none)
            for (uint32_t k = 0; k < p.n_reach; ++k)
                if (re[k].kind == HL_ISIS_REACH_MT && re[k].metric < kMaxWide) emit(re[k]);
    }
    for (uint32_t v = 0; v < V; ++v) if (!has_zeroth[v]) f.vflags[v] |= HSPF_VF_LEAF;

    // mutual-link filter; raw is grouped by u in iteration order (fragments of one
    // LAN id are contiguous in LspId order)
    std::unordered_set<uint64_t> have;
    have.reserve(raw.size() * 2);
    for (auto &e : raw) have.insert(((uint64_t)e.u << 32) | e.v);
    auto keep = [&](const Raw &e) {
        if (e.u == e.v) return false;
        // a link between two pseudonodes can never be mutual-checked into the SPT in
        // a sane LSDB; the engine's CSR forbids it, so drop it
        if (!(f.vflags[e.u] & HSPF_VF_HOP) && !(f.vflags[e.v] & HSPF_VF_HOP)) return false;
        return have.count(((uint64_t)e.v << 32) | e.u) != 0;
    };
    f.row.assign(V + 1, 0);
    for (auto &e : raw) if (keep(e)) f.row[e.u + 1]++;
    for (uint32_t v = 0; v < V; ++v) f.row[v + 1] += f.row[v];
    const uint32_t E = f.row[V];
    f.col.resize(E); f.cost.resize(E);
    std::vector<uint32_t> fill(f.row.begin(), f.row.end() - 1);
    for (auto &e : raw) if (keep(e)) { const uint32_t k = fill[e.u]++; f.col[k] = e.v; f.cost[k] = e.cost; }
    // transposed copy for the host-side ordering passes
    f.irow.assign(V + 1, 0);
    for (uint32_t e = 0; e < E; ++e) f.irow[f.col[e] + 1]++;
    for (uint32_t v = 0; v < V; ++v) f.irow[v + 1] += f.irow[v];
    f.isrc.resize(E); f.ieid.resize(E);
    std::vector<uint32_t> ifill(f.irow.begin(), f.irow.end() - 1);
    for (uint32_t u = 0; u < V; ++u)
        for (uint32_t e = f.row[u]; e < f.row[u + 1]; ++e) { const uint32_t k = ifill[f.col[e]]++; f.isrc[k] = u; f.ieid[k] = e; }
    f.reject_above = l->metric_type == HL_ISIS_METRIC_STANDARD ? 1023u : kMaxWide;
    f.gflags = HSPF_GF_NOHOP_TARGET_NO_NEXTHOP | (hopcount ? HSPF_GF_HOPCOUNT : 0u);
    return HSPF_OK;
}

void fill_csr(const hspf_isis_flat &f, hspf_csr *c) {
    std::memset(c, 0, sizeof(*c));
    c->n_vertices = (uint32_t)f.ids.size();
    c->n_edges = (uint32_t)f.col.size();
    c->row_ptr = f.row.data(); c->col = f.col.data(); c->cost = f.cost.data(); c->vflags = f.vflags.data();
    c->reject_above = f.reject_above;
    c->saturate_at = 0;
    c->flags = f.gflags;
    c->delta = 0;
}

inline bool expands(uint8_t fl, uint32_t u, uint32_t root) {
    return !((fl & HSPF_VF_LEAF) || ((fl & HSPF_VF_LEAF_UNLESS_ROOT) && u != root));
}

int spt_from_planes(const hspf_isis_flat &f, uint32_t root, const uint32_t *dist, const uint16_t *hops,
                    uint32_t n_ov, const uint32_t *ov_edge, const uint32_t *ov_cost, hl_isis_spt *out) {
    const uint32_t V = (uint32_t)f.ids.size();
    const bool hopcount = f.gflags & HSPF_GF_HOPCOUNT;
    auto ecost = [&](uint32_t e) {
        uint32_t c = f.cost[e];
        for (uint32_t k = 0; k < n_ov; ++k) if (ov_edge[k] == e) c = ov_cost[k];
        return c;
    };
    auto is_dag = [&](uint32_t u, uint32_t e, uint32_t v) {
        if (v == root || dist[u] == HSPF_DIST_INF || dist[v] == HSPF_DIST_INF) return false;
        if (!expands(f.vflags[u], u, root)) return false;
        const uint32_t c = ecost(e);
        if (c == HSPF_COST_DISABLED) return false;
        const uint64_t s = (uint64_t)dist[u] + c;
        return s == dist[v];
    };
    // hop-count mode: a pseudonode's only parent is its lowest-numbered router of the same level
    std::vector<uint32_t> owner;
    if (hopcount) {
        owner.assign(V, kNone);
        for (uint32_t v = 0; v < V; ++v) {
            if ((f.vflags[v] & HSPF_VF_HOP) || dist[v] == HSPF_DIST_INF) continue;
            for (uint32_t i = f.irow[v]; i < f.irow[v + 1]; ++i)
                if (is_dag(f.isrc[i], f.ieid[i], v)) owner[v] = std::min(owner[v], f.isrc[i]);
        }
    }
    // pop order
    std::vector<uint32_t> spt;
    for (uint32_t v = 0; v < V; ++v) if (dist[v] != HSPF_DIST_INF) spt.push_back(v);
    std::vector<uint32_t> pop = spt;
    auto key = [&](uint32_t v) {
        // (distance, tie): plain VertexId order, or the interleaved hop-count order
        uint64_t tie = v;
        if (hopcount) tie = (f.vflags[v] & HSPF_VF_HOP) ? ((uint64_t)v << 33) : (((uint64_t)owner[v] << 33) | (1ull << 32) | v);
        return std::make_pair(dist[v], tie);
    };
    std::sort(pop.begin(), pop.end(), [&](uint32_t a, uint32_t b) { return key(a) < key(b); });
    std::vector<uint32_t> pos(V, kNone), rank(V, kNone);
    for (uint32_t i = 0; i < pop.size(); ++i) pos[pop[i]] = i;
    for (uint32_t i = 0; i < spt.size(); ++i) rank[spt[i]] = i;

    // parents in push order: by (pop position of the tail, edge order of the tail)
    std::vector<std::vector<uint32_t>> parents(V);
    size_t n_par = 0;
    std::vector<std::pair<uint64_t, uint32_t>> tmp;
    for (uint32_t v : spt) {
        tmp.clear();
        for (uint32_t i = f.irow[v]; i < f.irow[v + 1]; ++i) {
            const uint32_t u = f.isrc[i], e = f.ieid[i];
            if (!is_dag(u, e, v)) continue;
            if (hopcount && !(f.vflags[v] & HSPF_VF_HOP) && u != owner[v]) continue;
            tmp.emplace_back(((uint64_t)pos[u] << 32) | e, u);
        }
        std::sort(tmp.begin(), tmp.end());
        for (auto &t : tmp) parents[v].push_back(t.second);
        n_par += tmp.size();
    }
    // next-hop Vecs in pop order
    std::vector<std::vector<uint64_t>> nh(V);
    size_t n_nh = 0;
    const size_t cap = (size_t)1 << 22;
    for (uint32_t v : pop) {
        auto &dst = nh[v];
        for (uint32_t p : parents[v]) {
            if (hops[p] == 0) {
                if (f.vflags[v] & HSPF_VF_HOP) dst.push_back(f.ids[v] >> 8);
            } else {
                if (n_nh + dst.size() + nh[p].size() > cap) return HSPF_E_UNSUPPORTED;
                dst.insert(dst.end(), nh[p].begin(), nh[p].end());
            }
        }
        n_nh += dst.size();
    }
    std::vector<uint32_t> fh, sh;
    for (uint32_t v : pop) {
        if (!(f.vflags[v] & HSPF_VF_HOP)) continue;
        if (hops[v] == 1) fh.push_back(rank[v]);
        if (hops[v] == 2) sh.push_back(rank[v]);
    }
    out->n_vertices = (uint32_t)spt.size();
    out->n_parents = (uint32_t)n_par;
    out->n_nexthops = (uint32_t)n_nh;
    out->n_first_hops = (uint32_t)fh.size();
    out->n_second_hops = (uint32_t)sh.size();
    if (out->n_vertices > out->vertices_cap || out->n_parents > out->parents_cap ||
        out->n_nexthops > out->nexthops_cap || out->n_first_hops > out->first_hops_cap ||
        out->n_second_hops > out->second_hops_cap)
        return HSPF_E_NOMEM;
    uint32_t i = 0, p = 0, n = 0;
    for (uint32_t v : spt) {
        hl_isis_vertex o{};
        o.lan_id = f.ids[v]; o.distance = dist[v]; o.hops = hops[v];
        o.par_off = p; o.n_par = (uint32_t)parents[v].size();
        o.nh_off = n; o.n_nh = (uint32_t)nh[v].size();
        for (uint32_t u : parents[v]) out->parents[p++] = rank[u];
        for (uint64_t x : nh[v]) out->nexthops[n++] = x;
        out->vertices[i++] = o;
    }
    std::copy(fh.begin(), fh.end(), out->first_hops);
    std::copy(sh.begin(), sh.end(), out->second_hops);
    return HSPF_OK;
}

}  // namespace

extern "C" {

int hspf_isis_flatten(const hl_isis_level *lvl, hspf_isis_flat **out) {
    if (!lvl || !out) return HSPF_E_INVAL;
    *out = nullptr;
    try {
        auto *f = new hspf_isis_flat();
        int rc = flatten(lvl, *f);
        if (rc) { delete f; return rc; }
        *out = f;
        return HSPF_OK;
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

void hspf_isis_flat_free(hspf_isis_flat *flat) { delete flat; }

int hspf_isis_flat_csr(const hspf_isis_flat *flat, hspf_csr *out) {
    if (!flat || !out) return HSPF_E_INVAL;
    fill_csr(*flat, out);
    return HSPF_OK;
}

int hspf_isis_spf_type(const hl_isis_level *ol, const hl_isis_level *nl, const hl_isis_lsp_trigger *tr, uint32_t n,
                       uint32_t *spf_type) {
    if (!ol || !nl || !spf_type || (n && !tr)) return HSPF_E_INVAL;
    auto find = [](const hl_isis_level *l, hl_lan_id id, uint8_t frag) -> const hl_isis_lsp * {
        for (uint32_t i = 0; i < l->n_lsps; ++i)
            if (l->lsps[i].lan_id == id && l->lsps[i].fragment == frag) return &l->lsps[i];
        return nullptr;
    };
    // the IS-reachability entries of one TLV kind, in TLV order
    auto same_kind = [](const hl_isis_level *a, const hl_isis_lsp *x, const hl_isis_level *b, const hl_isis_lsp *y, uint8_t kind) {
        uint32_t i = 0, j = 0;
        for (;;) {
            while (i < x->n_reach && a->reaches[x->reach_off + i].kind != kind) ++i;
            while (j < y->n_reach && b->reaches[y->reach_off + j].kind != kind) ++j;
            if (i == x->n_reach || j == y->n_reach) return i == x->n_reach && j == y->n_reach;
            const hl_isis_reach &p = a->reaches[x->reach_off + i], &q = b->reaches[y->reach_off + j];
            if (p.neighbor != q.neighbor || p.metric != q.metric) return false;
            ++i; ++j;
        }
    };
    *spf_type = HL_ISIS_SPF_ROUTE_ONLY;
    for (uint32_t k = 0; k < n; ++k) {
        const hl_isis_lsp *x = find(ol, tr[k].lan_id, tr[k].fragment), *y = find(nl, tr[k].lan_id, tr[k].fragment);
        if (!y) return HSPF_E_INVAL;                         // a trigger is an LSP that was just installed
        bool topology_change = true;
        // lsp.flags (LspFlags: the image carries its OL and ATT bits; the other image flags come from TLVs, which the
        // reference does not compare here)
        const uint8_t hdr_bits = HL_LSPF_OL | HL_LSPF_ATT;
        if (x && (x->rem_lifetime == 0) == (y->rem_lifetime == 0) && (x->flags & hdr_bits) == (y->flags & hdr_bits) &&
            same_kind(ol, x, nl, y, HL_ISIS_REACH_LEGACY) && same_kind(ol, x, nl, y, HL_ISIS_REACH_EXT))
            topology_change = false;
        if (topology_change) { *spf_type = HL_ISIS_SPF_FULL; break; }
    }
    return HSPF_OK;
}

int hspf_isis_flat_update(hspf_isis_flat *flat, const hl_isis_level *nl, uint32_t *kind, uint32_t *edges, uint32_t *costs,
                          uint32_t cap, uint32_t *n_changed) {
    if (!flat || !nl || !kind || !n_changed) return HSPF_E_INVAL;
    try {
        *n_changed = 0;
        hspf_isis_flat fresh;
        const int rc = flatten(nl, fresh);
        if (rc) return rc;
        hspf_isis_flat &f = *flat;
        const bool same_graph = f.ids == fresh.ids && f.row == fresh.row && f.col == fresh.col && f.vflags == fresh.vflags &&
                                f.reject_above == fresh.reject_above && f.gflags == fresh.gflags;
        if (!same_graph) {
            f = std::move(fresh);
            *kind = HSPF_FLAT_REBUILT;
            return HSPF_OK;
        }
        uint32_t changed = 0;
        for (uint32_t e = 0; e < (uint32_t)f.cost.size(); ++e) {
            if (f.cost[e] == fresh.cost[e]) continue;
            if (changed < cap && edges && costs) { edges[changed] = e; costs[changed] = fresh.cost[e]; }
            ++changed;
        }
        f.cost = std::move(fresh.cost);
        f.lvl = nl;
        *n_changed = changed;
        *kind = changed ? HSPF_FLAT_COSTS : HSPF_FLAT_UNCHANGED;
        return changed > cap ? HSPF_E_NOMEM : HSPF_OK;
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

int hspf_isis_flat_vertices(const hspf_isis_flat *flat, const uint64_t **lan_ids, uint32_t *n_vertices) {
    if (!flat) return HSPF_E_INVAL;
    if (lan_ids) *lan_ids = flat->ids.data();
    if (n_vertices) *n_vertices = (uint32_t)flat->ids.size();
    return HSPF_OK;
}

uint32_t hspf_isis_flat_vertex(const hspf_isis_flat *flat, uint64_t lan_id) {
    if (!flat) return kNone;
    auto it = flat->index.find(lan_id);
    return it == flat->index.end() ? kNone : it->second;
}

int hspf_isis_spt_from_planes(const hspf_isis_flat *flat, uint32_t root_vertex, const uint32_t *dist,
                              const uint16_t *hops, uint32_t n_ov, const uint32_t *ov_edge,
                              const uint32_t *ov_cost, hl_isis_spt *out) {
    if (!flat || !dist || !hops || !out || root_vertex >= flat->ids.size()) return HSPF_E_INVAL;
    try {
        return spt_from_planes(*flat, root_vertex, dist, hops, n_ov, ov_edge, ov_cost, out);
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

int hspf_isis_compute_spt(hspf_ctx *ctx, const hl_isis_level *lvl, uint64_t root_system_id, hl_isis_spt *out) {
    if (!ctx || !lvl || !out) return HSPF_E_INVAL;
    try {
        hspf_isis_flat f;
        int rc = flatten(lvl, f);
        if (rc) return rc;
        const hl_lan_id root_id = (hl_lan_id)(root_system_id << 8);
        auto it = f.index.find(root_id);
        if (it == f.index.end()) {
            // the root owns no LSP: the SPT is the root alone (popped, zeroth LSP missing)
            out->n_vertices = 1; out->n_parents = out->n_nexthops = out->n_first_hops = out->n_second_hops = 0;
            if (out->vertices_cap < 1) return HSPF_E_NOMEM;
            hl_isis_vertex o{};
            o.lan_id = root_id;
            out->vertices[0] = o;
            return HSPF_OK;
        }
        const uint32_t root = it->second;
        const uint32_t V = (uint32_t)f.ids.size();
        hspf_csr csr;
        fill_csr(f, &csr);
        hspf_graph *g = nullptr;
        rc = hspf_graph_upload(ctx, &csr, &g);
        if (rc) return rc;
        std::vector<uint32_t> dist(V);
        std::vector<uint16_t> hops(V);
        uint32_t status = 0;
        hspf_jobs jobs{};
        jobs.n_jobs = 1; jobs.roots = &root;
        hspf_result res{};
        res.dist = dist.data(); res.hops = hops.data(); res.nh_words = 4; res.job_status = &status;
        rc = hspf_run_batch(ctx, g, &jobs, &res, 0);
        hspf_graph_free(ctx, g);
        // first-hop atom overflow is irrelevant here: the Vec is rebuilt from parents
        if (rc == HSPF_E_JOB_STATUS && !(status & ~HSPF_JS_TOO_MANY_ATOMS)) rc = HSPF_OK;
        if (rc) return rc;
        return spt_from_planes(f, root, dist.data(), hops.data(), 0, nullptr, nullptr, out);
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

}  // extern "C"

// =====================================================================================
// Route path of compute_spf (holo-isis/src/spf.rs:742-799): per enabled topology one
// SPT with `local = true` next-hop resolution (resolve_nexthop, spf.rs:948-1002), then
// compute_routes (spf.rs:838-941).  Distances/hops come from the device; the host
// replays only the first-hop bookkeeping of the hops==0 vertices (root and the
// pseudonodes attached to it) in pop order, because resolve_nexthop is stateful
// ("the same adjacency shouldn't be used more than once", used_adjs).
// =====================================================================================
#include <array>
#include <map>
#include <set>

namespace {

struct LNh { uint64_t sysid; bool has_iface; uint32_t iface; bool has4; uint32_t ipv4; bool has6; hl_ip_addr ipv6; };

struct IpLess {
    bool operator()(const hl_ip_addr &a, const hl_ip_addr &b) const {
        if (a.is_v6 != b.is_v6) return a.is_v6 < b.is_v6;
        return std::memcmp(a.bytes, b.bytes, 16) < 0;
    }
};
struct NetKey {
    hl_ip_addr a; uint8_t len;
    bool operator<(const NetKey &o) const {
        if (a.is_v6 != o.a.is_v6) return a.is_v6 < o.a.is_v6;
        int c = std::memcmp(a.bytes, o.a.bytes, 16);
        return c ? c < 0 : len < o.len;
    }
};
struct RNh { uint64_t sysid; uint32_t iface; hl_ip_addr addr; bool has_label = false; uint32_t label = 0; };
struct PrefixSid { bool present = false; uint8_t flags = 0; bool is_label = false; uint32_t value = 0; };
struct RouteE {
    uint8_t type, flags; uint32_t metric; std::map<hl_ip_addr, RNh, IpLess> nh;
    PrefixSid psid;                               // Route.prefix_sid (route.rs:100)
    bool has_label = false; uint32_t label = 0;   // Route.sr_label
};

// SR view of one level's LSDB (holo-isis/src/sr.rs): per system the label blocks and address
// family flags of its first valid SR-Capabilities sub-TLV, per LAN id whether a valid fragment
// lists SPF in an SR-Algorithm sub-TLV.  Built once per route computation.
struct SrView {
    struct Cap { const hl_srgb *blocks; uint32_t n; uint8_t flags; };
    std::unordered_map<uint64_t, Cap> cap;          // system id -> capabilities
    std::unordered_map<uint64_t, bool> algo_spf;    // LAN id -> SR-Algorithm contains SPF
    explicit SrView(const hl_isis_level &l) {
        // LspId order: (lan_id, fragment); the first valid LSP with the sub-TLV wins
        std::vector<uint32_t> order(l.n_lsps);
        for (uint32_t i = 0; i < l.n_lsps; ++i) order[i] = i;
        std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
            const auto &x = l.lsps[a], &y = l.lsps[b];
            return x.lan_id != y.lan_id ? x.lan_id < y.lan_id : x.fragment < y.fragment;
        });
        for (uint32_t i : order) {
            const auto &p = l.lsps[i];
            if (!p.seqno || !p.rem_lifetime) continue;
            if (p.sr_flags & HL_LSP_SR_ALGO_SPF) algo_spf[p.lan_id] = true;
            if ((p.sr_flags & HL_LSP_SR_HAS_CAP) && !cap.count(p.lan_id >> 8))
                cap.emplace(p.lan_id >> 8, Cap{l.srgbs + p.srgb_off, p.n_srgb, p.sr_flags});
        }
    }
    // index_to_label (sr.rs:268-300)
    static bool label_of(const Cap &c, uint32_t index, uint32_t &label) {
        for (uint32_t i = 0; i < c.n; ++i) {
            if (c.blocks[i].first_is_index) continue;
            if (index >= c.blocks[i].range) { index -= c.blocks[i].range; continue; }
            label = c.blocks[i].first + index;
            return true;
        }
        return false;
    }
    // prefix_sid_update (sr.rs:33-99) with prefix_sid_input_label / prefix_sid_output_label
    void update(RouteE &r, uint64_t own_system, uint64_t adv_lan_id, bool v6, bool local, bool last_hop) const {
        const PrefixSid &ps = r.psid;
        auto al = algo_spf.find(adv_lan_id);
        if (al == algo_spf.end()) return;                 // remote node does not run SPF for SR
        const bool p_flag = ps.flags & HL_ISIS_PSID_P, e_flag = ps.flags & HL_ISIS_PSID_E;
        if (local && (!p_flag || e_flag)) {
            r.has_label = false;
        } else if (ps.is_label) {
            r.has_label = true; r.label = ps.value;
        } else {
            auto own = cap.find(own_system);
            uint32_t lab;
            if (own != cap.end() && label_of(own->second, ps.value, lab)) { r.has_label = true; r.label = lab; }
        }
        for (auto &kv : r.nh) {
            RNh &nh = kv.second;
            if (last_hop && !p_flag) { nh.has_label = true; nh.label = 3; continue; }                 // implicit null
            auto c = cap.find(nh.sysid);
            if (c == cap.end()) continue;
            if (!(c->second.flags & (v6 ? HL_LSP_SR_CAP_V : HL_LSP_SR_CAP_I))) continue;
            if (last_hop && e_flag) { nh.has_label = true; nh.label = v6 ? 2u : 0u; continue; }      // explicit null
            uint32_t lab;
            if (ps.is_label) { nh.has_label = true; nh.label = last_hop ? ps.value : 3u; }
            else if (label_of(c->second, ps.value, lab)) { nh.has_label = true; nh.label = lab; }
        }
    }
};

// The SPT's pop order (distance, then vertex id) and each vertex's position in it.
void pop_order(uint32_t V, const uint32_t *dist, std::vector<uint32_t> &pop, std::vector<uint32_t> &pos) {
    pop.clear();
    for (uint32_t v = 0; v < V; ++v) if (dist[v] != HSPF_DIST_INF) pop.push_back(v);
    std::sort(pop.begin(), pop.end(), [&](uint32_t a, uint32_t b) { return dist[a] != dist[b] ? dist[a] < dist[b] : a < b; });
    pos.assign(V, kNone);
    for (uint32_t i = 0; i < pop.size(); ++i) pos[pop[i]] = i;
}

// would the reference relax edge e out of u at all?  `cost` is the job's edge cost array
// (HSPF_COST_DISABLED: the edge is gone)
inline bool relax_ok(const hspf_isis_flat &f, uint32_t root, const uint32_t *dist, const uint32_t *cost, uint32_t u,
                     uint32_t e) {
    if (dist[u] == HSPF_DIST_INF || !expands(f.vflags[u], u, root) || cost[e] == HSPF_COST_DISABLED) return false;
    return (uint64_t)dist[u] + cost[e] <= f.reject_above;
}

// The resolved next hop of every final DAG edge out of a hops==0 vertex (the root and the pseudonodes
// attached to it), keyed by forward edge id: resolve_nexthop replayed in pop order.
std::map<uint32_t, LNh> first_hop_replay(const hspf_isis_flat &f, const hl_isis_instance *in, uint8_t mt_id,
                                         uint32_t root, const uint32_t *dist, const uint16_t *hops, const uint32_t *cost,
                                         const std::vector<uint32_t> &pop, const std::vector<uint32_t> &pos) {
    const uint8_t level_bit = in->level == 1 ? 1 : 2;
    std::set<std::array<uint8_t, 6>> used;
    auto resolve = [&](uint32_t P, uint32_t e, uint32_t R) {
        LNh nh{f.ids[R] >> 8, false, 0, false, 0, false, hl_ip_addr{}};
        const bool want_bcast = is_pn(f.ids[P]);
        for (uint32_t i = 0; i < in->n_ifaces; ++i) {
            const auto &iface = in->ifaces[i];
            if ((bool)iface.is_broadcast != want_bcast) continue;
            const hl_isis_adj *adj = nullptr;
            if (iface.is_broadcast) {
                for (uint32_t k = 0; k < iface.n_adj && !adj; ++k)
                    if (in->adjs[iface.adj_off + k].system_id == nh.sysid) adj = &in->adjs[iface.adj_off + k];
                if (adj && (!(mt_id == HL_ISIS_MT_STANDARD ? adj->topo_std : adj->topo_ipv6) || !adj->up)) adj = nullptr;
            } else {
                if (iface.metric != cost[e] || !iface.n_adj) continue;
                const auto &a = in->adjs[iface.adj_off];
                if ((mt_id == HL_ISIS_MT_STANDARD ? a.topo_std : a.topo_ipv6) && (a.level_usage & level_bit) &&
                    a.system_id == nh.sysid && a.up)
                    adj = &a;
            }
            if (!adj) continue;
            std::array<uint8_t, 6> snpa;
            std::memcpy(snpa.data(), adj->snpa, 6);
            if (!used.insert(snpa).second) continue;
            nh.has_iface = true; nh.iface = i;
            nh.has4 = adj->has_ipv4; nh.ipv4 = adj->ipv4;
            nh.has6 = adj->has_ipv6; nh.ipv6 = adj->ipv6;
            break;
        }
        return nh;
    };
    // replay the relaxations out of the hops==0 vertices, in pop order
    std::map<uint32_t, LNh> first_hop;    // forward edge id -> resolved next hop (final DAG edges only)
    for (uint32_t P : pop) {
        if (hops[P] != 0 || !expands(f.vflags[P], P, root)) continue;
        for (uint32_t e = f.row[P]; e < f.row[P + 1]; ++e) {
            const uint32_t R = f.col[e];
            if (pos[R] != kNone && pos[R] < pos[P]) continue;            // already on the SPT
            if (cost[e] == HSPF_COST_DISABLED) continue;
            const uint64_t d = (uint64_t)dist[P] + cost[e];
            if (d > f.reject_above) continue;
            // candidate distance of R at this moment
            uint64_t cb = ~0ull;
            for (uint32_t i = f.irow[R]; i < f.irow[R + 1]; ++i) {
                const uint32_t u = f.isrc[i], e2 = f.ieid[i];
                if (!relax_ok(f, root, dist, cost, u, e2)) continue;
                const bool earlier = (u == P) ? (e2 < e) : (pos[u] < pos[P]);
                if (earlier) cb = std::min<uint64_t>(cb, (uint64_t)dist[u] + cost[e2]);
            }
            if (d > cb) continue;
            if (!(f.vflags[R] & HSPF_VF_HOP)) continue;                  // pseudonode: nothing is pushed
            LNh nh = resolve(P, e, R);
            if (d == dist[R]) first_hop[e] = nh;
        }
    }
    return first_hop;
}

// Next-hop Vecs of a `local = true` SPT for every SPT vertex (indexed by vertex).
int local_nexthops(const hspf_isis_flat &f, const hl_isis_instance *in, uint8_t mt_id, uint32_t root,
                   const uint32_t *dist, const uint16_t *hops, const uint32_t *cost, std::vector<std::vector<LNh>> &out) {
    const uint32_t V = (uint32_t)f.ids.size();
    std::vector<uint32_t> pop, pos;
    pop_order(V, dist, pop, pos);
    const std::map<uint32_t, LNh> first_hop = first_hop_replay(f, in, mt_id, root, dist, hops, cost, pop, pos);
    // final Vecs in pop order: parents in (pop position, edge order)
    out.assign(V, {});
    std::vector<std::pair<uint64_t, uint32_t>> tmp;
    for (uint32_t v : pop) {
        if (v == root) continue;
        tmp.clear();
        for (uint32_t i = f.irow[v]; i < f.irow[v + 1]; ++i) {
            const uint32_t u = f.isrc[i], e = f.ieid[i];
            if (!relax_ok(f, root, dist, cost, u, e) || (uint64_t)dist[u] + cost[e] != dist[v]) continue;
            tmp.emplace_back(((uint64_t)pos[u] << 32) | e, u);
        }
        std::sort(tmp.begin(), tmp.end());
        for (auto &t : tmp) {
            const uint32_t u = t.second, e = (uint32_t)(t.first & 0xFFFFFFFFu);
            if (hops[u] == 0) {
                if (f.vflags[v] & HSPF_VF_HOP) {
                    auto it = first_hop.find(e);
                    if (it != first_hop.end()) out[v].push_back(it->second);
                }
            } else {
                if (out[v].size() + out[u].size() > ((size_t)1 << 22)) return HSPF_E_UNSUPPORTED;
                out[v].insert(out[v].end(), out[u].begin(), out[u].end());
            }
        }
    }
    return HSPF_OK;
}

}  // namespace

namespace {

// One topology of compute_spf's route path: flatten with the topology's edge rules and find
// the root.  Returns HSPF_OK and `have_root`.
int topology_flat(const hl_isis_instance *in, uint8_t mt_id, hspf_isis_flat &f, uint32_t &root, bool &have_root) {
    hl_isis_level l = in->lvl;
    l.mt_id = mt_id;
    l.metric_mode = HL_ISIS_MODE_NORMAL;
    int rc = flatten(&l, f);
    if (rc) return rc;
    const hl_lan_id root_id = (hl_lan_id)(in->system_id << 8);
    auto it = f.index.find(root_id);
    have_root = it != f.index.end();      // root owns no LSP: nothing reachable, no routes
    root = have_root ? it->second : 0;
    return HSPF_OK;
}

// The contributions compute_routes (spf.rs:838-941) makes in one topology, in its order: every
// vertex `visit(v)` accepts, in id_tree (= vertex index) order, with a valid zeroth LSP; its valid
// fragments in LspId order; per fragment the ATT-bit default routes, then TLV 128, 130, 135 and
// 236/237 entries.  emit(v, prefix, len, entry metric, external, entry with its Prefix-SID or NULL, index of the
// entry in lvl.ipreaches or -1 for an ATT-bit default route).  Which contributions there are depends only on the
// LSDB and the instance configuration.
template <class Visit, class Emit>
void for_each_contribution(const hl_isis_instance *in, const hspf_isis_flat &f, uint8_t mt_id, Visit visit, Emit emit) {
    const hl_isis_level &l0 = in->lvl;
    const bool std_en = l0.metric_type == HL_ISIS_METRIC_STANDARD || l0.metric_type == HL_ISIS_METRIC_BOTH;
    const bool wide_en = l0.metric_type == HL_ISIS_METRIC_WIDE || l0.metric_type == HL_ISIS_METRIC_BOTH;
    const uint32_t V = (uint32_t)f.ids.size();
    bool attached = false;
    for (uint32_t i = 0; i < in->n_adjs; ++i) {
        const auto &a = in->adjs[i];
        if ((mt_id == HL_ISIS_MT_STANDARD ? a.topo_std : a.topo_ipv6) && a.up && (a.level_usage & 2) && a.area_disjoint) attached = true;
    }
    const bool ipv4_enabled = l0.ipv4_enabled && mt_id == HL_ISIS_MT_STANDARD;
    const bool ipv6_enabled = l0.ipv6_enabled && (mt_id == HL_ISIS_MT_STANDARD ? !in->mt_ipv6_enabled : true);
    // fragments per LAN id in LspId order
    std::vector<uint32_t> order(l0.n_lsps);
    for (uint32_t i = 0; i < l0.n_lsps; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
        const auto &x = l0.lsps[a], &y = l0.lsps[b];
        return x.lan_id != y.lan_id ? x.lan_id < y.lan_id : x.fragment < y.fragment;
    });
    std::unordered_map<uint64_t, std::vector<uint32_t>> frags;
    for (uint32_t i : order) frags[l0.lsps[i].lan_id].push_back(i);
    for (uint32_t v = 0; v < V; ++v) {
        if (!visit(v)) continue;
        const auto &fr = frags[f.ids[v]];
        const hl_isis_lsp *z = nullptr;
        for (uint32_t i : fr)
            if (l0.lsps[i].fragment == 0) { if (l0.lsps[i].seqno && l0.lsps[i].rem_lifetime) z = &l0.lsps[i]; break; }
        if (!z) continue;
        const bool att_bit = !in->att_ignore &&
                             (mt_id == HL_ISIS_MT_STANDARD ? (z->flags & HL_LSPF_ATT) : (z->flags & HL_LSPF_MT_IPV6_ATT));
        for (uint32_t i : fr) {
            const auto &lsp = l0.lsps[i];
            if (!lsp.seqno || !lsp.rem_lifetime) continue;
            if (att_bit && in->level == 1 && (in->level_type == 1 || !attached)) {
                if (ipv4_enabled) emit(v, hl_ip_addr{}, 0, 0, false, nullptr, -1);
                if (ipv6_enabled) { hl_ip_addr z6{}; z6.is_v6 = 1; emit(v, z6, 0, 0, false, nullptr, -1); }
            }
            const hl_isis_ipreach *ip = l0.ipreaches + lsp.ipreach_off;
            const auto at = [&](uint32_t k) { return (int32_t)(lsp.ipreach_off + k); };
            if (mt_id == HL_ISIS_MT_STANDARD && ipv4_enabled) {
                if (std_en) {
                    for (uint32_t k = 0; k < lsp.n_ipreach; ++k)
                        if (ip[k].kind == HL_ISIS_IP_V4_INTERNAL) emit(v, ip[k].prefix, ip[k].len, ip[k].metric, false, nullptr, at(k));
                    for (uint32_t k = 0; k < lsp.n_ipreach; ++k)
                        if (ip[k].kind == HL_ISIS_IP_V4_EXTERNAL) emit(v, ip[k].prefix, ip[k].len, ip[k].metric, true, nullptr, at(k));
                }
                if (wide_en)
                    for (uint32_t k = 0; k < lsp.n_ipreach; ++k)
                        if (ip[k].kind == HL_ISIS_IP_V4_EXT && ip[k].metric <= kMaxWide)
                            emit(v, ip[k].prefix, ip[k].len, ip[k].metric, ip[k].external != 0, &ip[k], at(k));
            }
            if (ipv6_enabled)
                for (uint32_t k = 0; k < lsp.n_ipreach; ++k) {
                    const bool take = mt_id == HL_ISIS_MT_IPV6 ? (ip[k].kind == HL_ISIS_IP_MT_V6 && ip[k].mt_id == HL_ISIS_MT_IPV6)
                                                               : (ip[k].kind == HL_ISIS_IP_V6);
                    if (take) emit(v, ip[k].prefix, ip[k].len, ip[k].metric, ip[k].external != 0, &ip[k], at(k));
                }
        }
    }
}

// RouteE.type of a contribution
inline uint8_t route_type(const hl_isis_instance *in, bool external) {
    return in->level == 1 ? (external ? HL_ISIS_RT_L1_EXT : HL_ISIS_RT_L1_INTRA)
                          : (external ? HL_ISIS_RT_L2_EXT : HL_ISIS_RT_L2_INTRA);
}

// A next hop's address in the prefix's family; false when the adjacency has none.
inline bool nh_addr(const LNh &nh, bool v6, hl_ip_addr &addr) {
    addr = hl_ip_addr{};
    if (!v6) {
        if (!nh.has4) return false;
        addr.bytes[0] = (uint8_t)(nh.ipv4 >> 24); addr.bytes[1] = (uint8_t)(nh.ipv4 >> 16);
        addr.bytes[2] = (uint8_t)(nh.ipv4 >> 8); addr.bytes[3] = (uint8_t)nh.ipv4;
    } else {
        if (!nh.has6) return false;
        addr = nh.ipv6; addr.is_v6 = 1;
    }
    return true;
}

// compute_routes (spf.rs:838-941) for one topology, over that topology's SPT planes
// (vertex order of `f`).
int topology_routes(const hl_isis_instance *in, const hspf_isis_flat &f, uint8_t mt_id, uint32_t root,
                    const uint32_t *dist, const uint16_t *hops, std::map<NetKey, RouteE> &rib) {
    const SrView sr(in->lvl);
    std::vector<std::vector<LNh>> vnh;
    int rc = local_nexthops(f, in, mt_id, root, dist, hops, f.cost.data(), vnh);
    if (rc) return rc;
    auto add = [&](uint32_t v, const hl_ip_addr &prefix, uint8_t len, uint32_t nmetric, bool external,
                   const hl_isis_ipreach *src, int32_t) {
        auto build = [&](std::map<hl_ip_addr, RNh, IpLess> &m) {
            for (const LNh &nh : vnh[v]) {
                hl_ip_addr addr;
                if (nh_addr(nh, prefix.is_v6 != 0, addr)) m[addr] = RNh{nh.sysid, nh.iface, addr};
            }
        };
        const uint32_t metric = dist[v] + nmetric;
        NetKey key{prefix, len};
        auto rit = rib.find(key);
        RouteE *route;
        if (rit == rib.end() || metric < rit->second.metric) {
            RouteE r{};
            r.flags = hops[v] == 0 ? HL_ROUTE_CONNECTED : 0;
            r.type = route_type(in, external);
            r.metric = metric;
            build(r.nh);
            if (src && src->has_psid) r.psid = PrefixSid{true, src->psid_flags, src->psid_is_label != 0, src->psid_value};
            if (rit == rib.end()) route = &rib.emplace(key, std::move(r)).first->second;
            else { rit->second = std::move(r); route = &rit->second; }
        } else if (metric == rit->second.metric) {
            build(rit->second.nh);
            route = &rit->second;
        } else {
            return;
        }
        while (route->nh.size() > in->max_paths) route->nh.erase(std::prev(route->nh.end()));
        if (in->sr_enabled && route->psid.present)      // spf.rs:923-939
            sr.update(*route, in->system_id, f.ids[v], prefix.is_v6 != 0, hops[v] == 0, hops[v] == 1);
    };
    for_each_contribution(in, f, mt_id, [&](uint32_t v) { return dist[v] != HSPF_DIST_INF; }, add);
    return HSPF_OK;
}

int emit_rib(std::map<NetKey, RouteE> &rib, hl_isis_rib *out) {
    uint32_t need_h = 0;
    for (auto &kv : rib) need_h += (uint32_t)kv.second.nh.size();
    out->n_routes = (uint32_t)rib.size(); out->n_nexthops = need_h;
    if (out->n_routes > out->routes_cap || need_h > out->nexthops_cap) return HSPF_E_NOMEM;
    uint32_t i = 0, h = 0;
    for (auto &kv : rib) {
        hl_isis_route o{};
        o.prefix = kv.first.a; o.len = kv.first.len; o.metric = kv.second.metric; o.route_type = kv.second.type;
        o.flags = kv.second.flags; o.nh_off = h; o.n_nh = (uint32_t)kv.second.nh.size();
        o.has_sr_label = kv.second.has_label ? 1 : 0; o.sr_label = kv.second.has_label ? kv.second.label : 0;
        for (auto &nk : kv.second.nh) {
            hl_isis_nexthop x{};
            x.system_id = nk.second.sysid; x.iface = nk.second.iface; x.addr = nk.second.addr;
            x.has_label = nk.second.has_label ? 1 : 0; x.sr_label = nk.second.has_label ? nk.second.label : 0;
            out->nexthops[h++] = x;
        }
        out->routes[i++] = o;
    }
    return HSPF_OK;
}

}  // namespace

extern "C" int hspf_isis_compute_routes(hspf_ctx *ctx, const hl_isis_instance *in, hl_isis_rib *out) {
    if (!ctx || !in || !out) return HSPF_E_INVAL;
    try {
        std::map<NetKey, RouteE> rib;
        const uint8_t mts[2] = {HL_ISIS_MT_STANDARD, HL_ISIS_MT_IPV6};
        for (uint8_t mt_id : mts) {
            if (mt_id == HL_ISIS_MT_IPV6 && !in->mt_ipv6_enabled) continue;
            hspf_isis_flat f;
            uint32_t root = 0;
            bool have_root = false;
            int rc = topology_flat(in, mt_id, f, root, have_root);
            if (rc) return rc;
            if (!have_root) continue;
            const uint32_t V = (uint32_t)f.ids.size();
            hspf_csr csr;
            fill_csr(f, &csr);
            hspf_graph *g = nullptr;
            rc = hspf_graph_upload(ctx, &csr, &g);
            if (rc) return rc;
            std::vector<uint32_t> dist(V);
            std::vector<uint16_t> hops(V);
            uint32_t status = 0;
            hspf_jobs jobs{};
            jobs.n_jobs = 1; jobs.roots = &root;
            hspf_result res{};
            res.dist = dist.data(); res.hops = hops.data(); res.nh_words = 4; res.job_status = &status;
            rc = hspf_run_batch(ctx, g, &jobs, &res, 0);
            hspf_graph_free(ctx, g);
            if (rc == HSPF_E_JOB_STATUS && !(status & ~HSPF_JS_TOO_MANY_ATOMS)) rc = HSPF_OK;
            if (rc) return rc;
            rc = topology_routes(in, f, mt_id, root, dist.data(), hops.data(), rib);
            if (rc) return rc;
        }
        return emit_rib(rib, out);
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

/* The same route stage over SPT planes the caller already has (e.g. one job of a what-if batch
 * run through hspf_isis_flatten + hspf_run_batch): `dist_*` / `hops_*` are indexed by the vertex
 * order of hspf_isis_flatten for that topology (lvl.mt_id = HL_ISIS_MT_STANDARD / HL_ISIS_MT_IPV6,
 * lvl.metric_mode = HL_ISIS_MODE_NORMAL); the IPv6-topology planes are ignored unless
 * inst->mt_ipv6_enabled.  Host only. */
extern "C" int hspf_isis_routes_from_planes(const hl_isis_instance *in, const uint32_t *dist_std, const uint16_t *hops_std,
                                            const uint32_t *dist_mt6, const uint16_t *hops_mt6, hl_isis_rib *out) {
    if (!in || !out) return HSPF_E_INVAL;
    try {
        std::map<NetKey, RouteE> rib;
        const uint8_t mts[2] = {HL_ISIS_MT_STANDARD, HL_ISIS_MT_IPV6};
        for (uint8_t mt_id : mts) {
            if (mt_id == HL_ISIS_MT_IPV6 && !in->mt_ipv6_enabled) continue;
            const uint32_t *dist = mt_id == HL_ISIS_MT_STANDARD ? dist_std : dist_mt6;
            const uint16_t *hops = mt_id == HL_ISIS_MT_STANDARD ? hops_std : hops_mt6;
            hspf_isis_flat f;
            uint32_t root = 0;
            bool have_root = false;
            int rc = topology_flat(in, mt_id, f, root, have_root);
            if (rc) return rc;
            if (!have_root) continue;
            if (!dist || !hops) return HSPF_E_INVAL;
            rc = topology_routes(in, f, mt_id, root, dist, hops, rib);
            if (rc) return rc;
        }
        return emit_rib(rib, out);
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

/* ---- batched route stage: the table and the per-job decode (isis_route_cells.h) ------------- */
#include <cassert>
#include <memory>

#include "isis_backbone_cells.h"
#include "isis_l1_to_l2_cells.h"
#include "isis_l1l2_rib_cells.h"
#include "isis_propagation.h"
#include "isis_route_cells.h"

namespace {
const uint8_t kTopologies[2] = {HL_ISIS_MT_STANDARD, HL_ISIS_MT_IPV6};    // table topology 0, 1

// src: the lvl.ipreaches index of an entry that can carry a Prefix-SID, else -1; idx: the entry's index, -1 for an
// ATT-bit default route
struct RawContrib { NetKey key; hspf::IsisContrib c; int32_t src, idx; };

// Every contribution compute_routes can make in the instance's enabled topologies, in NetKey order and, within a
// prefix, in walk order; entries whose lvl.ipreaches byte in `drop` is non-zero are left out (drop NULL: none).
// Sets each topology's vertex count and root (kNone: the root owns no LSP there, or the topology is off).
int collect_contributions(const hl_isis_instance *in, const uint8_t *drop, std::vector<RawContrib> &raw,
                          uint32_t n_vertices[2], uint32_t root_out[2]) {
    for (uint32_t t = 0; t < 2; ++t) {
        n_vertices[t] = 0;
        root_out[t] = kNone;
        const uint8_t mt_id = kTopologies[t];
        if (mt_id == HL_ISIS_MT_IPV6 && !in->mt_ipv6_enabled) continue;
        hspf_isis_flat f;
        uint32_t root = 0;
        bool have_root = false;
        const int rc = topology_flat(in, mt_id, f, root, have_root);
        if (rc) return rc;
        n_vertices[t] = (uint32_t)f.ids.size();
        if (!have_root) continue;
        root_out[t] = root;
        // every vertex: whether a contributor is on the SPT is the job's business
        for_each_contribution(in, f, mt_id, [](uint32_t) { return true; },
                              [&](uint32_t v, const hl_ip_addr &prefix, uint8_t len, uint32_t nmetric, bool external,
                                  const hl_isis_ipreach *src, int32_t idx) {
                                  if (drop && idx >= 0 && drop[idx]) return;
                                  RawContrib r{};
                                  r.key = NetKey{prefix, len};
                                  r.c.vertex = v; r.c.metric = nmetric; r.c.topology = (uint8_t)t;
                                  r.c.external = external ? 1 : 0;
                                  r.c.has_psid = (src && src->has_psid) ? 1 : 0;
                                  r.c.sr = (r.c.has_psid && in->sr_enabled) ? 1 : 0;
                                  r.src = src ? (int32_t)(src - in->lvl.ipreaches) : -1;
                                  r.idx = idx;
                                  raw.push_back(r);
                              });
    }
    // NetKey order, walk order within a prefix
    std::stable_sort(raw.begin(), raw.end(), [](const RawContrib &a, const RawContrib &b) { return a.key < b.key; });
    return HSPF_OK;
}

// One job's decode state for one level's topologies: the flat, the job's planes, and what each first-hop atom
// resolves to (hspf_isis_routes_from_cells, hspf_isis_l1l2_rib_from_cells).
struct DecodeTopo {
    hspf_isis_flat f;
    const uint16_t *hops = nullptr;
    bool live = false;
    LNh atom_nh[64];
    bool atom_has[64] = {};
};

// The job's planes of topology t of `in` (pl[t]); the table recorded n_vertices[t] and root[t] for that instance.
int decode_topos(const hl_isis_instance *in, const uint32_t n_vertices[2], const uint32_t table_root[2],
                 const hspf_isis_job_planes pl[2], DecodeTopo tp[2]) {
    for (uint32_t t = 0; t < 2; ++t) {
        const uint8_t mt_id = kTopologies[t];
        if (mt_id == HL_ISIS_MT_IPV6 && !in->mt_ipv6_enabled) continue;
        DecodeTopo &T = tp[t];
        uint32_t root = 0;
        bool have_root = false;
        int rc = topology_flat(in, mt_id, T.f, root, have_root);
        if (rc) return rc;
        // not the instance the table was built from
        if (T.f.ids.size() != n_vertices[t] || (have_root ? root : kNone) != table_root[t]) return HSPF_E_INVAL;
        if (!have_root) continue;
        const uint32_t *dist = pl[t].dist;
        T.hops = pl[t].hops;
        const uint32_t n_ov = pl[t].n_ov;
        if (!dist || !T.hops || (n_ov && (!pl[t].ov_edge || !pl[t].ov_cost))) return HSPF_E_INVAL;
        std::vector<uint32_t> cost(T.f.cost);
        for (uint32_t k = 0; k < n_ov; ++k) {
            if (pl[t].ov_edge[k] >= cost.size()) return HSPF_E_INVAL;
            cost[pl[t].ov_edge[k]] = pl[t].ov_cost[k];
        }
        std::vector<uint32_t> pop, pos;
        pop_order((uint32_t)T.f.ids.size(), dist, pop, pos);
        const std::map<uint32_t, LNh> first_hop = first_hop_replay(T.f, in, mt_id, root, dist, T.hops, cost.data(), pop, pos);
        hspf_csr csr;
        fill_csr(T.f, &csr);
        uint32_t n_atoms = 0;
        if (hspf_atom_count(&csr, root, &n_atoms) != HSPF_OK) return HSPF_E_INVAL;
        for (uint32_t a = 0; a < std::min<uint32_t>(n_atoms, 64); ++a) {
            uint32_t tail = 0, edge = 0;
            if (hspf_atom_decode(&csr, root, a, &tail, &edge) != HSPF_OK) continue;
            auto it = first_hop.find(edge);
            if (it == first_hop.end()) continue;
            T.atom_nh[a] = it->second;
            T.atom_has[a] = true;
        }
        T.live = true;
    }
    return HSPF_OK;
}

// The route of a present cell won by contributor k of `in`; psid: the entry whose Prefix-SID the route takes when
// k.has_psid.
int decode_route(const hl_isis_instance *in, const DecodeTopo tp[2], const SrView &sr, const hspf::IsisContrib &k,
                 const hl_isis_ipreach *psid, const hl_isis_route_cell &c, bool v6, RouteE &r) {
    const DecodeTopo &T = tp[k.topology];
    if (!T.live || k.vertex >= T.f.ids.size()) return HSPF_E_INVAL;
    r = RouteE{};
    r.flags = (c.flags & HL_CELL_CONNECTED) ? HL_ROUTE_CONNECTED : 0;
    r.type = route_type(in, k.external != 0);
    r.metric = c.metric;
    // the union of the best-metric contributors' next hops; an address reached over two different
    // adjacencies keeps whichever `add` wrote last, which the cell cannot tell
    for (uint64_t m = c.nh_mask; m; m &= m - 1) {
        const uint32_t a = (uint32_t)__builtin_ctzll(m);
        hl_ip_addr addr;
        if (!T.atom_has[a] || !nh_addr(T.atom_nh[a], v6, addr)) continue;
        const RNh x{T.atom_nh[a].sysid, T.atom_nh[a].iface, addr};
        auto ins = r.nh.emplace(addr, x);
        if (!ins.second && (ins.first->second.sysid != x.sysid || ins.first->second.iface != x.iface))
            return HSPF_E_UNSUPPORTED;
    }
    while (r.nh.size() > in->max_paths) r.nh.erase(std::prev(r.nh.end()));
    if (k.has_psid) r.psid = PrefixSid{true, psid->psid_flags, psid->psid_is_label != 0, psid->psid_value};
    // all best-metric contributions come from the winner's vertex (else the cell is flagged):
    // one update with its context gives the labels every repeated update would
    if (in->sr_enabled && r.psid.present)
        sr.update(r, in->system_id, T.f.ids[k.vertex], v6, T.hops[k.vertex] == 0, T.hops[k.vertex] == 1);
    return HSPF_OK;
}

// ... won by contributor k whose entry is src (its lvl.ipreaches index)
int decode_route(const hl_isis_instance *in, const DecodeTopo tp[2], const SrView &sr, const hspf::IsisContrib &k,
                 int32_t src, const hl_isis_route_cell &c, bool v6, RouteE &r) {
    const DecodeTopo &T = tp[k.topology];
    if (!T.live || k.vertex >= T.f.ids.size()) return HSPF_E_INVAL;
    if (k.has_psid && (src < 0 || (uint32_t)src >= in->lvl.n_ipreaches)) return HSPF_E_INVAL;
    return decode_route(in, tp, sr, k, k.has_psid ? &in->lvl.ipreaches[src] : nullptr, c, v6, r);
}

}  // namespace

extern "C" {

void hspf_isis_rtable_free(hspf_isis_rtable *rt) {
    if (!rt) return;
    hspf::release_route_table(rt->dev);
    delete rt;
}

int hspf_isis_rtable_create(const hl_isis_instance *in, hspf_isis_rtable **out) {
    if (!in || !out) return HSPF_E_INVAL;
    *out = nullptr;
    try {
        auto rt = std::make_unique<hspf_isis_rtable>();
        std::vector<RawContrib> raw;
        const int rc = collect_contributions(in, nullptr, raw, rt->n_vertices, rt->root);
        if (rc) return rc;
        for (size_t i = 0; i < raw.size(); ++i) {
            if (i == 0 || raw[i - 1].key < raw[i].key) {
                rt->prefix.push_back(raw[i].key.a); rt->len.push_back(raw[i].key.len); rt->off.push_back((uint32_t)i);
            }
            rt->contribs.push_back(raw[i].c);
            rt->src.push_back(raw[i].src);
        }
        rt->off.push_back((uint32_t)raw.size());
        *out = rt.release();
        return HSPF_OK;
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

uint32_t hspf_isis_rtable_prefixes(const hspf_isis_rtable *rt) { return rt ? (uint32_t)rt->prefix.size() : 0; }
uint32_t hspf_isis_rtable_contributors(const hspf_isis_rtable *rt) { return rt ? (uint32_t)rt->contribs.size() : 0; }

int hspf_isis_rtable_topology(const hspf_isis_rtable *rt, uint32_t topology, uint32_t *n_vertices, uint32_t *root) {
    if (!rt || topology > 1) return HSPF_E_INVAL;
    if (n_vertices) *n_vertices = rt->n_vertices[topology];
    if (root) *root = rt->root[topology];
    return HSPF_OK;
}

int hspf_isis_rtable_arrays(const hspf_isis_rtable *rt, const hl_ip_addr **prefix, const uint32_t **len,
                            const uint32_t **off, const void **contribs) {
    if (!rt) return HSPF_E_INVAL;
    if (prefix) *prefix = rt->prefix.data();
    if (len) *len = rt->len.data();
    if (off) *off = rt->off.data();
    if (contribs) *contribs = rt->contribs.data();
    return HSPF_OK;
}

int hspf_isis_routes_from_cells(const hl_isis_instance *in, const hspf_isis_rtable *rt, const hl_isis_route_cell *cells,
                                const uint32_t *dist_std, const uint16_t *hops_std,
                                const uint32_t *dist_mt6, const uint16_t *hops_mt6,
                                uint32_t n_ov_std, const uint32_t *ov_edge_std, const uint32_t *ov_cost_std,
                                uint32_t n_ov_mt6, const uint32_t *ov_edge_mt6, const uint32_t *ov_cost_mt6,
                                hl_isis_rib *out) {
    if (!in || !rt || !out || (!cells && !rt->prefix.empty())) return HSPF_E_INVAL;
    try {
        const hspf_isis_job_planes pl[2] = {{dist_std, hops_std, n_ov_std, ov_edge_std, ov_cost_std},
                                            {dist_mt6, hops_mt6, n_ov_mt6, ov_edge_mt6, ov_cost_mt6}};
        auto tp = std::make_unique<DecodeTopo[]>(2);
        int rc = decode_topos(in, rt->n_vertices, rt->root, pl, tp.get());
        if (rc) return rc;
        const SrView sr(in->lvl);
        std::map<NetKey, RouteE> rib;
        const uint32_t P = (uint32_t)rt->prefix.size();
        for (uint32_t p = 0; p < P; ++p) {
            const hl_isis_route_cell &c = cells[p];
            if (!(c.flags & HL_CELL_PRESENT)) continue;
            if (c.flags & HL_CELL_MIXED_SID) return HSPF_E_UNSUPPORTED;
            if (c.winner < rt->off[p] || c.winner >= rt->off[p + 1]) return HSPF_E_INVAL;
            RouteE r;
            rc = decode_route(in, tp.get(), sr, rt->contribs[c.winner], rt->src[c.winner], c, rt->prefix[p].is_v6 != 0, r);
            if (rc) return rc;
            rib.emplace_hint(rib.end(), NetKey{rt->prefix[p], (uint8_t)rt->len[p]}, std::move(r));
        }
        return emit_rib(rib, out);
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

}  // extern "C"

/* ---- routing table of an L1/L2 router (isis_l1l2_rib_cells.h) -------------------------------- */
namespace {

// The own-LSP argument of hspf_isis_l1l2_ribtable_create needs every L1 entry that lsp_propagate_l1_to_l2 could
// carry into the router's L2 LSP (its static filters, holo-isis lsdb.rs:1163-1258, as hspf_isis_l1_to_l2 applies
// them, up/down bits aside) to be an entry compute_routes feeds into the L1 table (spf.rs:862-882, vertex_networks
// spf.rs:1141, for_each_contribution above) whenever its originator is on the same topology's SPT.  False when
// some entry breaks that.
bool propagation_within_routes(const hl_isis_instance *l1, const hl_isis_instance *l2, const hl_isis_summary *cfg,
                               uint32_t n_cfg) {
    const hl_isis_level &lv = l1->lvl;
    std::unordered_set<uint64_t> zeroth;          // LAN ids with a valid zeroth LSP
    for (uint32_t i = 0; i < lv.n_lsps; ++i)
        if (lv.lsps[i].fragment == 0 && lv.lsps[i].seqno && lv.lsps[i].rem_lifetime) zeroth.insert(lv.lsps[i].lan_id);
    bool within = true;
    hspf::for_each_propagation(lv, l1->system_id, lv.metric_type, l2->lvl.metric_type, l1->mt_ipv6_enabled != 0, nullptr,
                               cfg, n_cfg, [&](const hl_isis_lsp &lsp, uint32_t k, uint8_t, uint32_t, bool) {
        const hl_isis_ipreach &e = lv.ipreaches[k];
        const bool routed = zeroth.count(lsp.lan_id) != 0 && (e.kind != HL_ISIS_IP_V4_EXT || e.metric <= kMaxWide) &&
                            (e.kind != HL_ISIS_IP_MT_V6 || lv.ipv6_enabled);
        if (!routed) within = false;
    });
    return within;
}

// NetKey of a summary
NetKey summary_key(const hl_isis_summary &s) { return NetKey{s.prefix, s.len}; }

}  // namespace

extern "C" {

void hspf_isis_l1l2_ribtable_free(hspf_isis_l1l2_ribtable *t) {
    if (!t) return;
    hspf::release_route_table(t->dev);
    delete t;
}

int hspf_isis_l1l2_ribtable_create(const hl_isis_instance *l1, const hl_isis_instance *l2, const uint8_t *l2_derived,
                                   const hl_isis_summary *cfg, uint32_t n_cfg, hspf_isis_l1l2_ribtable **out) {
    if (!out) return HSPF_E_INVAL;
    *out = nullptr;
    if (!l1 || !l2 || (n_cfg && !cfg)) return HSPF_E_INVAL;
    if (l1->level_type != 3 || l2->level_type != 3 || l1->level != 1 || l2->level != 2 ||
        l1->system_id != l2->system_id || l1->max_paths != l2->max_paths)
        return HSPF_E_INVAL;
    for (uint32_t s = 1; s < n_cfg; ++s)
        if (!(summary_key(cfg[s - 1]) < summary_key(cfg[s]))) return HSPF_E_INVAL;
    try {
        // a derived entry is one of the root's own (non-pseudonode) L2 LSPs
        if (l2_derived) {
            std::vector<uint8_t> own(l2->lvl.n_ipreaches, 0);
            for (uint32_t i = 0; i < l2->lvl.n_lsps; ++i) {
                const hl_isis_lsp &lsp = l2->lvl.lsps[i];
                if (lsp.lan_id != (l2->system_id << 8)) continue;
                for (uint32_t k = lsp.ipreach_off; k < lsp.ipreach_off + lsp.n_ipreach && k < l2->lvl.n_ipreaches; ++k) own[k] = 1;
            }
            for (uint32_t k = 0; k < l2->lvl.n_ipreaches; ++k)
                if (l2_derived[k] && !own[k]) return HSPF_E_INVAL;
        }
        if (!propagation_within_routes(l1, l2, cfg, n_cfg)) return HSPF_E_UNSUPPORTED;
        auto t = std::make_unique<hspf_isis_l1l2_ribtable>();
        std::vector<RawContrib> r1, r2;
        int rc = collect_contributions(l1, nullptr, r1, t->n_vertices[0], t->root[0]);
        if (rc) return rc;
        rc = collect_contributions(l2, l2_derived, r2, t->n_vertices[1], t->root[1]);
        if (rc) return rc;
        t->n1 = (uint32_t)r1.size();
        t->S = n_cfg;
        t->cfg.assign(cfg, cfg + n_cfg);
        for (const auto &x : r1) { t->contribs.push_back(x.c); t->src.push_back(x.src); }
        for (const auto &x : r2) { t->contribs.push_back(x.c); t->src.push_back(x.src); }
        // the union of the L1, L2 and summary prefixes in NetKey (= hl_isis_rib) order
        std::vector<uint32_t> off1, off2, sum_of;
        std::vector<std::vector<uint32_t>> cov(n_cfg);
        size_t i = 0, j = 0, s = 0;
        while (i < r1.size() || j < r2.size() || s < n_cfg) {
            NetKey k{};
            bool have = false;
            auto low = [&](const NetKey &x) { if (!have || x < k) { k = x; have = true; } };
            if (i < r1.size()) low(r1[i].key);
            if (j < r2.size()) low(r2[j].key);
            if (s < n_cfg) low(summary_key(cfg[s]));
            const uint32_t p = (uint32_t)t->prefix.size();
            t->prefix.push_back(k.a);
            t->len.push_back(k.len);
            off1.push_back((uint32_t)i);
            while (i < r1.size() && !(k < r1[i].key)) ++i;
            off2.push_back(t->n1 + (uint32_t)j);
            while (j < r2.size() && !(k < r2[j].key)) ++j;
            const bool is_summary = s < n_cfg && !(k < summary_key(cfg[s]));
            sum_of.push_back(is_summary ? (uint32_t)s : hspf::kIsisNoSummary);
            if (is_summary) ++s;
            if (off1.back() != i) {          // an L1 prefix: the summary that is its shortest configured match
                const int m = hspf::isis_summary_match(cfg, n_cfg, k.a, k.len);
                if (m >= 0) cov[m].push_back(p);
            }
        }
        t->P = (uint32_t)t->prefix.size();
        off1.push_back((uint32_t)r1.size());
        off2.push_back(t->n1 + (uint32_t)r2.size());
        auto &w = t->words;
        w.insert(w.end(), off1.begin(), off1.end());
        w.insert(w.end(), off2.begin(), off2.end());
        w.insert(w.end(), sum_of.begin(), sum_of.end());
        uint32_t n_cov = 0;
        for (uint32_t k = 0; k < n_cfg; ++k) { w.push_back(n_cov); n_cov += (uint32_t)cov[k].size(); }
        w.push_back(n_cov);
        for (const auto &c : cov) w.insert(w.end(), c.begin(), c.end());
        t->n_cov = n_cov;
        for (uint32_t k = 0; k < n_cfg; ++k) { w.push_back(cfg[k].has_cfg_metric ? 1u : 0u); w.push_back(cfg[k].cfg_metric); }
        *out = t.release();
        return HSPF_OK;
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

uint32_t hspf_isis_l1l2_ribtable_prefixes(const hspf_isis_l1l2_ribtable *t) { return t ? t->P : 0; }
uint32_t hspf_isis_l1l2_ribtable_contributors(const hspf_isis_l1l2_ribtable *t) {
    return t ? (uint32_t)t->contribs.size() : 0;
}

int hspf_isis_l1l2_ribtable_topology(const hspf_isis_l1l2_ribtable *t, uint32_t level, uint32_t topology,
                                     uint32_t *n_vertices, uint32_t *root) {
    if (!t || level < 1 || level > 2 || topology > 1) return HSPF_E_INVAL;
    if (n_vertices) *n_vertices = t->n_vertices[level - 1][topology];
    if (root) *root = t->root[level - 1][topology];
    return HSPF_OK;
}

int hspf_isis_l1l2_ribtable_arrays(const hspf_isis_l1l2_ribtable *t, const hl_ip_addr **prefix, const uint32_t **len,
                                   const uint32_t **off, const void **contribs) {
    if (!t) return HSPF_E_INVAL;
    if (prefix) *prefix = t->prefix.data();
    if (len) *len = t->len.data();
    if (off) *off = t->words.data();
    if (contribs) *contribs = t->contribs.data();
    return HSPF_OK;
}

int hspf_isis_l1l2_ribtable_summaries(const hspf_isis_l1l2_ribtable *t, uint32_t *n_l1, uint32_t *n_summaries,
                                      const uint32_t **sum_of, const uint32_t **cov_off, const uint32_t **cov) {
    if (!t) return HSPF_E_INVAL;
    const hspf::IsisL1L2View v = t->view(t->words.data(), t->contribs.data());
    if (n_l1) *n_l1 = t->n1;
    if (n_summaries) *n_summaries = t->S;
    if (sum_of) *sum_of = v.sum_of;
    if (cov_off) *cov_off = v.cov_off;
    if (cov) *cov = v.cov;
    return HSPF_OK;
}

int hspf_isis_l1l2_rib_from_cells(const hl_isis_instance *l1, const hl_isis_instance *l2,
                                  const hspf_isis_l1l2_ribtable *t, const hl_isis_route_cell *cells,
                                  const uint64_t *summary_words, const hspf_isis_job_planes *planes, hl_isis_rib *out) {
    if (!l1 || !l2 || !t || !planes || !out || (!cells && t->P) || (!summary_words && t->S)) return HSPF_E_INVAL;
    if (l1->level != 1 || l2->level != 2) return HSPF_E_INVAL;
    try {
        const hl_isis_instance *in[2] = {l1, l2};
        auto tp = std::make_unique<DecodeTopo[]>(4);
        for (uint32_t l = 0; l < 2; ++l) {
            const int rc = decode_topos(in[l], t->n_vertices[l], t->root[l], planes + 2 * l, tp.get() + 2 * l);
            if (rc) return rc;
        }
        const SrView sr[2] = {SrView(l1->lvl), SrView(l2->lvl)};
        const hspf::IsisL1L2View v = t->view(t->words.data(), t->contribs.data());
        std::map<NetKey, RouteE> rib;
        for (uint32_t p = 0; p < t->P; ++p) {
            const hl_isis_route_cell &c = cells[p];
            if (!(c.flags & HL_CELL_PRESENT)) continue;
            if (c.flags & HL_CELL_MIXED_SID) return HSPF_E_UNSUPPORTED;
            RouteE r{};
            if (c.winner >= v.n_contribs) {            // an active summary: a blackhole route
                const uint32_t s = c.winner - v.n_contribs;
                if (s != v.sum_of[p] || !(summary_words[s] & hspf::kIsisSummaryActive)) return HSPF_E_INVAL;
                r.type = HL_ISIS_RT_L2_INTRA;
                r.flags = HL_ROUTE_SUMMARY;
                r.metric = c.metric;
            } else {
                const uint32_t l = c.winner < t->n1 ? 0 : 1;
                const uint32_t *off = v.off + l * (t->P + 1);
                if (c.winner < off[p] || c.winner >= off[p + 1]) return HSPF_E_INVAL;
                const int rc = decode_route(in[l], tp.get() + 2 * l, sr[l], t->contribs[c.winner], t->src[c.winner], c,
                                            t->prefix[p].is_v6 != 0, r);
                if (rc) return rc;
            }
            rib.emplace_hint(rib.end(), NetKey{t->prefix[p], (uint8_t)t->len[p]}, std::move(r));
        }
        return emit_rib(rib, out);
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

}  // extern "C"

/* ---- what an L1/L2 router propagates into its L2 LSP (isis_l1_to_l2_cells.h) --------------------- */
namespace {

// hspf_isis_l1_to_l2's output order: kind, then prefix
bool key_less(uint8_t ka, const NetKey &a, uint8_t kb, const NetKey &b) { return ka != kb ? ka < kb : a < b; }

}  // namespace

extern "C" {

void hspf_isis_l1_to_l2_table_free(hspf_isis_l1_to_l2_table *t) {
    if (!t) return;
    hspf::release_route_table(t->dev);
    delete t;
}

int hspf_isis_l1_to_l2_table_create(const hl_isis_instance *l1, const hl_isis_instance *l2, const uint8_t *up_down,
                                    const hspf_isis_l1l2_ribtable *rib, hspf_isis_l1_to_l2_table **out) {
    if (!out) return HSPF_E_INVAL;
    *out = nullptr;
    if (!l1 || !l2 || !rib) return HSPF_E_INVAL;
    if (l1->level != 1 || l2->level != 2 || l1->level_type != 3 || l2->level_type != 3 || l1->system_id != l2->system_id)
        return HSPF_E_INVAL;
    try {
        // the L1 flats of the rib table's instance: same vertex counts and roots
        hspf_isis_flat f[2];
        for (uint32_t t = 0; t < 2; ++t) {
            uint32_t root = 0;
            bool have_root = false;
            if (kTopologies[t] == HL_ISIS_MT_STANDARD || l1->mt_ipv6_enabled) {
                const int rc = topology_flat(l1, kTopologies[t], f[t], root, have_root);
                if (rc) return rc;
            }
            if (f[t].ids.size() != rib->n_vertices[0][t] || (have_root ? root : kNone) != rib->root[0][t])
                return HSPF_E_INVAL;
        }
        auto t = std::make_unique<hspf_isis_l1_to_l2_table>();
        struct Raw { uint8_t kind; NetKey key; hspf::IsisPropRecord r; uint32_t src; };
        std::vector<Raw> raw;
        const hl_isis_level &lv = l1->lvl;
        hspf::for_each_propagation(lv, l1->system_id, lv.metric_type, l2->lvl.metric_type, l1->mt_ipv6_enabled != 0,
                                   up_down, rib->cfg.data(), rib->S,
                                   [&](const hl_isis_lsp &lsp, uint32_t k, uint8_t kind, uint32_t topology, bool narrow) {
            if (rib->root[0][topology] == kNone) return;             // no SPT in that topology: never reached
            auto it = f[topology].index.find(lsp.lan_id);
            if (it == f[topology].index.end()) return;               // not a vertex: never on the SPT
            Raw x{};
            x.kind = kind;
            x.key = NetKey{lv.ipreaches[k].prefix, lv.ipreaches[k].len};
            x.r.vertex = it->second; x.r.metric = lv.ipreaches[k].metric;
            x.r.topology = (uint8_t)topology; x.r.narrow = narrow ? 1 : 0;
            x.src = k;
            raw.push_back(x);
        });
        std::stable_sort(raw.begin(), raw.end(), [](const Raw &a, const Raw &b) { return key_less(a.kind, a.key, b.kind, b.key); });
        // the summary keys, as hspf_isis_l1_to_l2 adds an active summary
        struct SumKey { uint8_t kind; NetKey key; uint32_t word; };
        std::vector<SumKey> sk;
        auto std_on = [](uint8_t m) { return m == HL_ISIS_METRIC_STANDARD || m == HL_ISIS_METRIC_BOTH; };
        auto wide_on = [](uint8_t m) { return m == HL_ISIS_METRIC_WIDE || m == HL_ISIS_METRIC_BOTH; };
        for (uint32_t s = 0; s < rib->S; ++s) {
            const NetKey key{rib->cfg[s].prefix, rib->cfg[s].len};
            if (!key.a.is_v6) {
                if (!lv.ipv4_enabled) continue;
                if (std_on(l2->lvl.metric_type)) sk.push_back(SumKey{HL_ISIS_IP_V4_INTERNAL, key, (s << 1) | 1u});
                if (wide_on(l2->lvl.metric_type)) sk.push_back(SumKey{HL_ISIS_IP_V4_EXT, key, s << 1});
            } else if (lv.ipv6_enabled) {
                sk.push_back(SumKey{HL_ISIS_IP_V6, key, s << 1});
            }
        }
        std::stable_sort(sk.begin(), sk.end(), [](const SumKey &a, const SumKey &b) { return key_less(a.kind, a.key, b.kind, b.key); });
        // merge: the keys in output order, each propagated key with its records
        std::vector<uint32_t> off, sum;
        size_t i = 0, j = 0;
        while (i < raw.size() || j < sk.size()) {
            const bool take_sum = i == raw.size() || (j < sk.size() && key_less(sk[j].kind, sk[j].key, raw[i].kind, raw[i].key));
            // a summary covers its own prefix, so no propagated entry shares a summary key
            assert(take_sum || j == sk.size() || key_less(raw[i].kind, raw[i].key, sk[j].kind, sk[j].key));
            const uint8_t kind = take_sum ? sk[j].kind : raw[i].kind;
            const NetKey key = take_sum ? sk[j].key : raw[i].key;
            t->kind.push_back(kind);
            t->prefix.push_back(key.a);
            t->len.push_back(key.len);
            off.push_back((uint32_t)t->recs.size());
            if (take_sum) {
                sum.push_back(sk[j++].word);
                continue;
            }
            sum.push_back(hspf::kIsisNoSummary);
            for (; i < raw.size() && raw[i].kind == kind && !(key < raw[i].key) && !(raw[i].key < key); ++i) {
                t->recs.push_back(raw[i].r);
                t->src.push_back(raw[i].src);
                t->has_psid.push_back(lv.ipreaches[raw[i].src].has_psid);
            }
        }
        off.push_back((uint32_t)t->recs.size());
        t->K = (uint32_t)t->kind.size();
        t->words = off;
        t->words.insert(t->words.end(), sum.begin(), sum.end());
        t->n_ipreaches = lv.n_ipreaches;
        t->system_id = l1->system_id;
        t->rib = rib;
        *out = t.release();
        return HSPF_OK;
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

int hspf_isis_l1_to_l2_table_keys(const hspf_isis_l1_to_l2_table *t, uint32_t *n_keys, uint32_t *n_records,
                                  const uint8_t **kind, const hl_ip_addr **prefix, const uint8_t **len) {
    if (!t) return HSPF_E_INVAL;
    if (n_keys) *n_keys = t->K;
    if (n_records) *n_records = (uint32_t)t->recs.size();
    if (kind) *kind = t->kind.data();
    if (prefix) *prefix = t->prefix.data();
    if (len) *len = t->len.data();
    return HSPF_OK;
}

int hspf_isis_l1_to_l2_from_cells(const hl_isis_instance *l1, const hspf_isis_l1_to_l2_table *t,
                                  const hl_isis_route_cell *cells, const uint64_t *summary_words, hl_isis_ipreach *out,
                                  uint32_t cap, uint32_t *n_out) {
    if (!l1 || !t || !n_out || (!cells && t->K) || (!summary_words && t->rib->S) || (cap && !out)) return HSPF_E_INVAL;
    if (l1->level != 1 || l1->lvl.n_ipreaches != t->n_ipreaches) return HSPF_E_INVAL;    // not the table's instance
    try {
        const hspf::IsisL1ToL2View v = t->view(t->words.data(), t->recs.data());
        std::vector<hl_isis_ipreach> got;
        for (uint32_t k = 0; k < t->K; ++k) {
            const hl_isis_route_cell &c = cells[k];
            if (!(c.flags & HL_CELL_PRESENT)) continue;
            hl_isis_ipreach e;
            if (v.sum[k] != hspf::kIsisNoSummary) {               // an active summary
                const uint32_t s = v.sum[k] >> 1;
                if (c.winner != v.n_records + s || !(summary_words[s] & hspf::kIsisSummaryActive)) return HSPF_E_INVAL;
                std::memset(&e, 0, sizeof(e));
                e.prefix = t->prefix[k];
                e.len = t->len[k];
                e.kind = t->kind[k];
            } else {
                if (c.winner < v.off[k] || c.winner >= v.off[k + 1]) return HSPF_E_INVAL;
                e = l1->lvl.ipreaches[t->src[c.winner]];
                e.kind = t->kind[k];
                if (e.kind != l1->lvl.ipreaches[t->src[c.winner]].kind) e.mt_id = 0;   // MT-IPv6 into IPv6
                hspf::isis_propagated_sid(e);
            }
            e.metric = c.metric;
            got.push_back(e);
        }
        *n_out = (uint32_t)got.size();
        if (got.size() > cap) return HSPF_E_NOMEM;
        std::copy(got.begin(), got.end(), out);
        return HSPF_OK;
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

}  // extern "C"

/* ---- routing table of a backbone router over the L1 jobs of an area (isis_backbone_cells.h) ------------------- */
namespace {

static_assert(hspf::kIsisMaxWide == kMaxWide, "the device walk and compute_routes read TLV 135 up to one limit");

using BorderKey = std::pair<uint8_t, NetKey>;

BorderKey border_key(const hspf_isis_l1_to_l2_table *b, uint32_t k) { return {b->kind[k], NetKey{b->prefix[k], b->len[k]}}; }

// the key's records in the border's cells: its first winner and how many (a summary key: its one summary winner)
void key_records(const hspf_isis_l1_to_l2_table *b, uint32_t k, uint32_t &first, uint32_t &count) {
    const hspf::IsisL1ToL2View v = b->view(b->words.data(), b->recs.data());
    if (v.sum[k] != hspf::kIsisNoSummary) { first = v.n_records + (v.sum[k] >> 1); count = 1; }
    else { first = v.off[k]; count = v.off[k + 1] - v.off[k]; }
}

// How compute_routes takes an entry of kind `kind` as `emit` passes it (for_each_contribution): whether it carries a
// Prefix-SID (TLV 128 / 130 never do) and its external bit.
inline bool kind_has_psid(uint8_t kind) { return kind != HL_ISIS_IP_V4_INTERNAL && kind != HL_ISIS_IP_V4_EXTERNAL; }
inline bool kind_external(uint8_t kind, const hl_isis_ipreach &e) {
    return kind_has_psid(kind) ? e.external != 0 : kind == HL_ISIS_IP_V4_EXTERNAL;
}

}  // namespace

extern "C" {

void hspf_isis_backbone_table_free(hspf_isis_backbone_table *t) {
    if (!t) return;
    hspf::release_route_table(t->dev);
    delete t;
}

int hspf_isis_backbone_table_create(const hl_isis_instance *l2, const uint8_t *derived, uint32_t n_borders,
                                    const hspf_isis_l1_to_l2_table *const *borders, hspf_isis_backbone_table **out) {
    if (!out) return HSPF_E_INVAL;
    *out = nullptr;
    if (!l2 || !borders || n_borders == 0 || n_borders > hspf::kIsisBackboneMaxBorders) return HSPF_E_INVAL;
    if (l2->level != 2 || (l2->level_type != 2 && l2->level_type != 3)) return HSPF_E_INVAL;
    for (uint32_t b = 0; b < n_borders; ++b) {
        if (!borders[b] || borders[b]->system_id == l2->system_id) return HSPF_E_INVAL;
        for (uint32_t c = 0; c < b; ++c)
            if (borders[c]->system_id == borders[b]->system_id) return HSPF_E_INVAL;
    }
    try {
        const hl_isis_level &lv = l2->lvl;
        // each entry's border (-1: none), each border's valid zeroth fragment of its non-pseudonode LSP
        std::vector<int32_t> owner(lv.n_ipreaches, -1), zeroth(n_borders, -1);
        for (uint32_t i = 0; i < lv.n_lsps; ++i) {
            const hl_isis_lsp &lsp = lv.lsps[i];
            if (is_pn(lsp.lan_id)) continue;
            for (uint32_t b = 0; b < n_borders; ++b) {
                if ((lsp.lan_id >> 8) != borders[b]->system_id) continue;
                if (lsp.fragment == 0 && lsp.seqno && lsp.rem_lifetime) zeroth[b] = (int32_t)i;
                for (uint32_t k = lsp.ipreach_off; k < lsp.ipreach_off + lsp.n_ipreach && k < lv.n_ipreaches; ++k)
                    owner[k] = (int32_t)b;
            }
        }
        std::vector<std::map<BorderKey, uint32_t>> keys(n_borders);
        for (uint32_t b = 0; b < n_borders; ++b) {
            if (zeroth[b] < 0) return HSPF_E_INVAL;
            for (uint32_t k = 0; k < borders[b]->K; ++k) keys[b][border_key(borders[b], k)] = k;
        }
        // a derived entry is a key of its border; a summary key overwrites an entry of the border's own, which the
        // splice below cannot express
        for (uint32_t k = 0; k < lv.n_ipreaches; ++k) {
            const int32_t b = owner[k];
            const bool der = derived && derived[k];
            if (der && b < 0) return HSPF_E_INVAL;
            if (b < 0) continue;
            const auto it = keys[b].find(BorderKey{lv.ipreaches[k].kind, NetKey{lv.ipreaches[k].prefix, lv.ipreaches[k].len}});
            if (der && it == keys[b].end()) return HSPF_E_INVAL;
            if (!der && it != keys[b].end()) {
                const hspf::IsisL1ToL2View v = borders[b]->view(borders[b]->words.data(), borders[b]->recs.data());
                if (v.sum[it->second] != hspf::kIsisNoSummary) return HSPF_E_UNSUPPORTED;
            }
        }
        // The spliced image: the derived entries dropped, one placeholder per border key appended to the border's
        // zeroth fragment.  collect_contributions over it meets static entries and slots in walk order.
        std::vector<hl_isis_lsp> lsps(lv.lsps, lv.lsps + lv.n_lsps);
        std::vector<hl_isis_ipreach> ips;
        std::vector<int64_t> origin;              // per spliced entry: its lvl.ipreaches index, or -1 - slot
        std::vector<std::pair<uint32_t, uint32_t>> slot_key;     // (border, key)
        for (uint32_t i = 0; i < lv.n_lsps; ++i) {
            const uint32_t at = (uint32_t)ips.size();
            for (uint32_t k = lsps[i].ipreach_off; k < lsps[i].ipreach_off + lsps[i].n_ipreach && k < lv.n_ipreaches; ++k) {
                if (derived && derived[k]) continue;
                ips.push_back(lv.ipreaches[k]);
                origin.push_back(k);
            }
            for (uint32_t b = 0; b < n_borders; ++b) {
                if (zeroth[b] != (int32_t)i) continue;
                for (uint32_t k = 0; k < borders[b]->K; ++k) {
                    hl_isis_ipreach e{};
                    e.prefix = borders[b]->prefix[k];
                    e.len = borders[b]->len[k];
                    e.kind = borders[b]->kind[k];
                    ips.push_back(e);
                    origin.push_back(-1 - (int64_t)slot_key.size());
                    slot_key.emplace_back(b, k);
                }
            }
            lsps[i].ipreach_off = at;
            lsps[i].n_ipreach = (uint32_t)ips.size() - at;
        }
        hl_isis_instance sp = *l2;
        sp.lvl.lsps = lsps.data();
        sp.lvl.ipreaches = ips.data();
        sp.lvl.n_ipreaches = (uint32_t)ips.size();
        auto t = std::make_unique<hspf_isis_backbone_table>();
        std::vector<RawContrib> raw;
        const int rc = collect_contributions(&sp, nullptr, raw, t->n_vertices, t->root);
        if (rc) return rc;
        // the affected prefixes, each with its contributions
        std::set<NetKey> affected;
        for (uint32_t b = 0; b < n_borders; ++b)
            for (uint32_t k = 0; k < borders[b]->K; ++k) affected.insert(NetKey{borders[b]->prefix[k], borders[b]->len[k]});
        std::vector<uint32_t> off, sr;
        size_t i = 0;
        for (const NetKey &p : affected) {
            t->prefix.push_back(p.a);
            t->len.push_back(p.len);
            off.push_back((uint32_t)t->contribs.size());
            for (; i < raw.size() && raw[i].key < p; ++i) {}
            for (; i < raw.size() && !(p < raw[i].key); ++i) {
                const RawContrib &r = raw[i];
                hspf::IsisBackboneContrib c{};
                c.vertex = r.c.vertex;
                c.topology = r.c.topology;
                const int64_t o = r.idx >= 0 ? origin[r.idx] : -1;
                if (r.idx < 0 || o >= 0) {                 // a static contribution
                    c.metric = r.c.metric;
                    c.border = hspf::kIsisBackboneStatic;
                    c.sr = r.c.sr;
                    t->stat.push_back(r.c);
                    t->src.push_back((int32_t)(r.src >= 0 ? o : -1));
                } else {
                    const uint32_t b = slot_key[-1 - o].first, k = slot_key[-1 - o].second;
                    uint32_t first, count;
                    key_records(borders[b], k, first, count);
                    c.metric = k;
                    c.base = (uint32_t)sr.size() - first;
                    c.border = (uint8_t)b;
                    c.wide = borders[b]->kind[k] == HL_ISIS_IP_V4_EXT;
                    for (uint32_t w = 0; w < count; ++w) {
                        const bool rec = first + w < borders[b]->recs.size();
                        sr.push_back(rec && kind_has_psid(borders[b]->kind[k]) && borders[b]->has_psid[first + w] &&
                                     l2->sr_enabled);
                        t->slot_of.push_back((uint32_t)t->contribs.size());
                    }
                    t->stat.push_back(hspf::IsisContrib{});
                    t->src.push_back(-1);
                }
                t->contribs.push_back(c);
            }
        }
        t->P = (uint32_t)t->prefix.size();
        off.push_back((uint32_t)t->contribs.size());
        t->n_slot_records = (uint32_t)sr.size();
        t->words = off;
        t->words.insert(t->words.end(), sr.begin(), sr.end());
        t->n_borders = n_borders;
        t->n_ipreaches = lv.n_ipreaches;
        std::copy(borders, borders + n_borders, t->borders);
        *out = t.release();
        return HSPF_OK;
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

int hspf_isis_backbone_table_prefixes(const hspf_isis_backbone_table *t, uint32_t *n_prefixes, const hl_ip_addr **prefix,
                                      const uint8_t **len) {
    if (!t) return HSPF_E_INVAL;
    if (n_prefixes) *n_prefixes = t->P;
    if (prefix) *prefix = t->prefix.data();
    if (len) *len = t->len.data();
    return HSPF_OK;
}

int hspf_isis_backbone_from_cells(const hl_isis_instance *l2, const hspf_isis_backbone_table *t,
                                  const hl_isis_route_cell *cells, const hspf_isis_job_planes *planes,
                                  const hl_isis_ipreach *const *entries, const uint32_t *n_entries, hl_isis_rib *out) {
    if (!l2 || !t || !planes || !out || (!cells && t->P) || !entries || !n_entries) return HSPF_E_INVAL;
    if (l2->level != 2 || l2->lvl.n_ipreaches != t->n_ipreaches) return HSPF_E_INVAL;     // not the table's instance
    try {
        auto tp = std::make_unique<DecodeTopo[]>(2);
        int rc = decode_topos(l2, t->n_vertices, t->root, planes, tp.get());
        if (rc) return rc;
        // each border's job entries by key
        std::vector<std::map<BorderKey, const hl_isis_ipreach *>> job(t->n_borders);
        for (uint32_t b = 0; b < t->n_borders; ++b) {
            if (n_entries[b] && !entries[b]) return HSPF_E_INVAL;
            for (uint32_t e = 0; e < n_entries[b]; ++e)
                job[b][BorderKey{entries[b][e].kind, NetKey{entries[b][e].prefix, entries[b][e].len}}] = &entries[b][e];
        }
        const SrView sr(l2->lvl);
        const hspf::IsisBackboneView v = t->view(t->words.data(), t->contribs.data());
        std::map<NetKey, RouteE> rib;
        for (uint32_t p = 0; p < t->P; ++p) {
            const hl_isis_route_cell &c = cells[p];
            if (!(c.flags & HL_CELL_PRESENT)) continue;
            if (c.flags & HL_CELL_MIXED_SID) return HSPF_E_UNSUPPORTED;
            const bool v6 = t->prefix[p].is_v6 != 0;
            RouteE r;
            if (c.winner < v.n_contribs) {             // a static contribution
                if (c.winner < v.off[p] || c.winner >= v.off[p + 1] || t->contribs[c.winner].border != hspf::kIsisBackboneStatic)
                    return HSPF_E_INVAL;
                rc = decode_route(l2, tp.get(), sr, t->stat[c.winner], t->src[c.winner], c, v6, r);
            } else {                                   // a slot: the border's entry of the job
                const uint32_t g = c.winner - v.n_contribs;
                if (g >= t->n_slot_records) return HSPF_E_INVAL;
                const uint32_t i = t->slot_of[g];
                if (i < v.off[p] || i >= v.off[p + 1]) return HSPF_E_INVAL;
                const hspf::IsisBackboneContrib &s = t->contribs[i];
                const auto it = job[s.border].find(border_key(t->borders[s.border], s.metric));
                if (it == job[s.border].end()) return HSPF_E_INVAL;
                const hl_isis_ipreach &e = *it->second;
                hspf::IsisContrib k{};
                k.vertex = s.vertex;
                k.topology = s.topology;
                k.external = kind_external(e.kind, e);
                k.has_psid = kind_has_psid(e.kind) && e.has_psid;
                rc = decode_route(l2, tp.get(), sr, k, &e, c, v6, r);
            }
            if (rc) return rc;
            rib.emplace_hint(rib.end(), NetKey{t->prefix[p], t->len[p]}, std::move(r));
        }
        return emit_rib(rib, out);
    } catch (const std::bad_alloc &) { return HSPF_E_NOMEM; } catch (...) { return HSPF_E_INVAL; }
}

}  // extern "C"
