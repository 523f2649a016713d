// What an IS-IS L1/L2 router propagates into its L2 LSP for a batch of L1 SPTs, one cell per (job, key)
// (include/holo_spf_lsdb.h, hspf_isis_l1_to_l2_table_create).
//
// lsp_propagate_l1_to_l2 (holo-isis lsdb.rs:1149-1357; hspf_isis_l1_to_l2) offers, per (kind, prefix) key, every L1
// entry its static filters let through (isis_propagation.h) whose originator is on the L1 SPT, at metric + the
// originator's distance, and keeps the lowest total; then each active summary adds its keys.  What-if jobs change
// costs only, so the filters, and with them each key's records, hold for every job: per job a record only asks
// whether its originator is reached, and at what distance.  Per key that is one walk:
//   * a summary key (one of the router's summaries; none of the propagated entries, since a summary covers its own
//     prefix): present when the job's summary word is active, at the configured metric or else the word's lowest
//     covered L1 metric, capped at 63 for the narrow IPv4 key;
//   * a propagated key: over its records in LSP order, total = min(entry + distance, 63) for a narrow TLV, else
//     min(entry + distance, 2^32 - 1), in 64 bits; only a strictly lower total replaces the winner, so on a tie the
//     first record in LSP order keeps the key.
// A cell is the 24-byte hl_isis_route_cell: nh_mask 0, winner the record (summary s: n_records + s), metric the
// advertised one, HL_CELL_PRESENT.  The summary words come from the summary pass of the L1/L2 routing-table stage
// (isis_summary.cuh), run over the router's hspf_isis_l1l2_ribtable.
#pragma once
#include <cstdint>
#include <vector>

#include "isis_l1l2_rib_cells.h"

namespace hspf {

// One L1 entry that may be propagated into a key, in the order the host loop meets them.
struct alignas(16) IsisPropRecord {
    uint32_t vertex;      // the originator's vertex in the L1 flat of `topology`
    uint32_t metric;      // the entry metric
    uint8_t  topology;    // 0 standard, 1 MT-IPv6
    uint8_t  narrow;      // a narrow TLV: the total is capped at 63
    uint16_t _pad0;
    uint32_t _pad1;
};
static_assert(sizeof(IsisPropRecord) == 16, "IsisPropRecord layout");

HSPF_HD IsisPropRecord load_prop_record(const IsisPropRecord *p) {
#if defined(__CUDA_ARCH__)
    const uint4 r = __ldg(reinterpret_cast<const uint4 *>(p));
    IsisPropRecord k;
    k.vertex = r.x; k.metric = r.y;
    k.topology = (uint8_t)(r.z & 0xFFu); k.narrow = (uint8_t)((r.z >> 8) & 0xFFu); k._pad0 = 0; k._pad1 = 0;
    return k;
#else
    return *p;
#endif
}

// What the walk reads of a table.
struct IsisL1ToL2View {
    const uint32_t *off;          // [K + 1] into recs
    const uint32_t *sum;          // [K]: kIsisNoSummary, or (s << 1) | 1 when the key is summary s's narrow IPv4 key
    const IsisPropRecord *recs;
    uint32_t K, n_records;
};

// The cell of key k; `rib` gives the configured summary metrics, `words` are the job's S summary words.
template <class Planes>
HSPF_HD hl_isis_route_cell isis_l1_to_l2_cell_eval(const Planes &s1, const Planes &m1, const IsisL1ToL2View &t,
                                                   const IsisL1L2View &rib, uint32_t k, const uint64_t *words) {
    hl_isis_route_cell c;
    c.nh_mask = 0; c.winner = 0xFFFFFFFFu; c.metric = 0; c.flags = 0;
    for (int i = 0; i < 7; ++i) c._pad[i] = 0;
    const uint32_t sm = t.sum[k];
    if (sm != kIsisNoSummary) {
        const uint32_t s = sm >> 1;
        const uint64_t w = words[s];
        if (w & kIsisSummaryActive) {
            uint32_t m = rib.cfg[2 * s] ? rib.cfg[2 * s + 1] : (uint32_t)w;
            if ((sm & 1u) && m > 63u) m = 63u;
            c.winner = t.n_records + s;
            c.metric = m;
            c.flags = HL_CELL_PRESENT;
        }
        return c;
    }
    for (uint32_t i = t.off[k]; i < t.off[k + 1]; ++i) {
        const IsisPropRecord r = load_prop_record(t.recs + i);
        const Planes pl = r.topology ? m1 : s1;             // a copy: selecting a reference puts both on the stack
        if (!pl.reached(r.vertex)) continue;
        const uint64_t sum = (uint64_t)pl.d(r.vertex) + r.metric;
        const uint64_t cap = r.narrow ? 63u : 0xFFFFFFFFu;
        const uint32_t m = (uint32_t)(sum < cap ? sum : cap);
        if (!(c.flags & HL_CELL_PRESENT) || m < c.metric) {
            c.metric = m;
            c.winner = i;
            c.flags = HL_CELL_PRESENT;
        }
    }
    return c;
}

}  // namespace hspf

// Host + device image of what an L1/L2 router propagates into its L2 LSP (include/holo_spf_lsdb.h).
struct hspf_isis_l1_to_l2_table {
    std::vector<uint8_t> kind;               // [K] the keys in hspf_isis_l1_to_l2's output order
    std::vector<hl_ip_addr> prefix;          // [K]
    std::vector<uint8_t> len;                // [K]
    std::vector<uint32_t> words;             // the view's u32 arrays: off [K + 1], sum [K]
    std::vector<hspf::IsisPropRecord> recs;
    std::vector<uint32_t> src;               // per record: index of its entry in the L1 ipreaches
    std::vector<uint8_t> has_psid;           // per record: its entry carries a Prefix-SID
    uint32_t K = 0, n_ipreaches = 0;
    uint64_t system_id = 0;                  // the router's
    const hspf_isis_l1l2_ribtable *rib = nullptr;   // the summaries, their metrics and cover lists
    hspf::DeviceRouteTable dev;              // hspf_isis_l1_to_l2_table_upload

    // the view over `w` (words, on the host or the device) and `r` (records)
    hspf::IsisL1ToL2View view(const uint32_t *w, const hspf::IsisPropRecord *r) const {
        hspf::IsisL1ToL2View v;
        v.off = w;
        v.sum = w + K + 1;
        v.recs = r;
        v.K = K;
        v.n_records = (uint32_t)recs.size();
        return v;
    }
};
