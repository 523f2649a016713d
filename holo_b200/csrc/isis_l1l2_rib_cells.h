// Routing table of a batch of IS-IS SPT pairs for one L1/L2 router, one cell per (job, prefix)
// (include/holo_spf_lsdb.h, hspf_isis_l1l2_ribtable_create).
//
// update_rib (holo-isis/src/route.rs:182-249) builds the L1 table, derives the active summaries from it (get_spm:
// the shortest configured match of each L1 route, the lowest covered metric), lets each active summary replace the
// L2 route of its prefix with a blackhole route, and merges the two tables with the L1 route preferred.  Per prefix
// that is one walk:
//   1. isis_route_cell_eval over the prefix's L1 contributors with the job's L1 planes: if present, that is the cell;
//   2. else, the prefix is an active summary of the job: a cell without atoms whose winner is the summary's record
//      and whose metric is the configured one, or else the lowest covered L1 metric;
//   3. else isis_route_cell_eval over the prefix's L2 contributors with the job's L2 planes.
// Levels never merge, so the winner says which level's first-hop atoms nh_mask names.  Which summaries are active
// is one reduction per (job, summary) over the L1 prefixes it covers (isis_summary_eval); the device runs it as its
// own pass before the cells, and the cells read its words.
#pragma once
#include <cstdint>
#include <vector>

#include "isis_route_cells.h"

namespace hspf {

constexpr uint32_t kIsisNoSummary = 0xFFFFFFFFu;

// host (isis_rib_host.cc): the configured summary that is the shortest match of a/len (get_spm), -1 when none
int isis_summary_match(const hl_isis_summary *cfg, uint32_t n_cfg, const hl_ip_addr &a, uint8_t len);

// What the walk reads of a table.  Contributor indices share one space: the L1 contributors [0, n1), the L2
// contributors [n1, n_contribs), then one winner index per configured summary (n_contribs + s).
struct IsisL1L2View {
    const uint32_t *off;          // [2 (P + 1)]: the L1 ranges, then the L2 ranges, into contribs
    const uint32_t *sum_of;       // [P] the summary whose prefix this is, kIsisNoSummary when none
    const uint32_t *cov_off;      // [S + 1] into cov
    const uint32_t *cov;          // per summary: the prefixes with L1 contributors it is the shortest match of
    const uint32_t *cfg;          // [S][2]: has a configured metric, the configured metric
    const IsisContrib *contribs;
    uint32_t P, S, n_contribs;
};

// A job's summary word: 0 inactive, (1 << 32) | lowest covered L1 metric when active.
constexpr uint64_t kIsisSummaryActive = 1ull << 32;

// The L1 walk of prefix p; true and its metric when the prefix has an L1 route.
template <class Planes>
HSPF_HD bool isis_l1_metric(const Planes &s1, const Planes &m1, const IsisL1L2View &t, uint32_t p, uint32_t &metric) {
    const hl_isis_route_cell c = isis_route_cell_eval(s1, m1, t.contribs, t.off[p], t.off[p + 1]);
    metric = c.metric;
    return (c.flags & HL_CELL_PRESENT) != 0;
}

// The summary word of summary s for one job (serial; the device splits the covered prefixes over a warp).
template <class Planes>
HSPF_HD uint64_t isis_summary_eval(const Planes &s1, const Planes &m1, const IsisL1L2View &t, uint32_t s) {
    bool any = false;
    uint32_t low = 0xFFFFFFFFu;
    for (uint32_t i = t.cov_off[s]; i < t.cov_off[s + 1]; ++i) {
        uint32_t m;
        if (!isis_l1_metric(s1, m1, t, t.cov[i], m)) continue;
        any = true;
        low = m < low ? m : low;
    }
    return any ? (kIsisSummaryActive | low) : 0;
}

// The cell of prefix p; `words` are the job's S summary words.
template <class Planes>
HSPF_HD hl_isis_route_cell isis_l1l2_cell_eval(const Planes &s1, const Planes &m1, const Planes &s2, const Planes &m2,
                                               const IsisL1L2View &t, uint32_t p, const uint64_t *words) {
    hl_isis_route_cell c = isis_route_cell_eval(s1, m1, t.contribs, t.off[p], t.off[p + 1]);
    if (c.flags & HL_CELL_PRESENT) return c;
    const uint32_t s = t.sum_of[p];
    if (s != kIsisNoSummary) {
        const uint64_t w = words[s];
        if (w & kIsisSummaryActive) {
            c.nh_mask = 0;
            c.winner = t.n_contribs + s;
            c.metric = t.cfg[2 * s] ? t.cfg[2 * s + 1] : (uint32_t)w;
            c.flags = HL_CELL_PRESENT;
            return c;
        }
    }
    const uint32_t *off2 = t.off + t.P + 1;
    return isis_route_cell_eval(s2, m2, t.contribs, off2[p], off2[p + 1]);
}

}  // namespace hspf

// Host + device image of an L1/L2 router's routing table (include/holo_spf_lsdb.h).
struct hspf_isis_l1l2_ribtable {
    std::vector<hl_ip_addr> prefix;          // [P] in hl_isis_rib order
    std::vector<uint32_t> len;               // [P]
    // the view's u32 arrays, in this order: off [2 (P + 1)], sum_of [P], cov_off [S + 1], cov, cfg [S][2]
    std::vector<uint32_t> words;
    std::vector<hspf::IsisContrib> contribs; // the L1 contributors, then the L2 contributors
    std::vector<int32_t> src;                // per contributor: index into its level's ipreaches, -1 for an ATT default
    std::vector<hl_isis_summary> cfg;        // [S] the configured summaries
    uint32_t P = 0, S = 0, n1 = 0, n_cov = 0;
    uint32_t n_vertices[2][2] = {{0, 0}, {0, 0}};     // [level - 1][topology]
    uint32_t root[2][2] = {{0xFFFFFFFFu, 0xFFFFFFFFu}, {0xFFFFFFFFu, 0xFFFFFFFFu}};
    hspf::DeviceRouteTable dev;              // hspf_isis_l1l2_ribtable_upload

    // the view over `w` (words, on the host or the device) and `c` (contribs)
    hspf::IsisL1L2View view(const uint32_t *w, const hspf::IsisContrib *c) const {
        hspf::IsisL1L2View v;
        v.off = w;
        v.sum_of = v.off + 2 * (P + 1);
        v.cov_off = v.sum_of + P;
        v.cov = v.cov_off + S + 1;
        v.cfg = v.cov + n_cov;
        v.contribs = c;
        v.P = P; v.S = S; v.n_contribs = (uint32_t)contribs.size();
        return v;
    }
};
