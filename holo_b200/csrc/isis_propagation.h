// The static filters of lsp_propagate_l1_to_l2 (holo-isis lsdb.rs:1163-1258), host only.  Which L1 entries an
// L1/L2 router may carry into its L2 LSP depends on the L1 LSDB and the configuration, never on the L1 SPT: the SPT
// only says whether the originator is reached and at what distance.  One walker serves hspf_isis_l1_to_l2
// (isis_rib_host.cc), the own-LSP check of hspf_isis_l1l2_ribtable_create and the records of
// hspf_isis_l1_to_l2_table_create (isis_host.cc).
#pragma once
#include <cstdint>

#include "holo_lsdb.h"

namespace hspf {

// host (isis_rib_host.cc): the configured summary that is the shortest match of a/len (get_spm), -1 when none
int isis_summary_match(const hl_isis_summary *cfg, uint32_t n_cfg, const hl_ip_addr &a, uint8_t len);

// A propagated entry's Prefix-SID: R (re-advertised) and P (no PHP) set, E (explicit null) cleared.
inline void isis_propagated_sid(hl_isis_ipreach &e) {
    if (e.has_psid) { e.psid_flags |= HL_ISIS_PSID_R | HL_ISIS_PSID_P; e.psid_flags &= (uint8_t)~HL_ISIS_PSID_E; }
}

// Every entry of the other systems' valid non-pseudonode L1 LSPs that propagation lets through, in l1.lsps order
// and entry order: its kind enabled by the address families and by both levels' metric types (`mt6`: the IPv6
// unicast topology is enabled, so plain IPv6 entries stay out and MT-IPv6 ones go in), its up/down byte clear
// (`up_down` NULL: none set), and no configured summary covering it.
//   emit(lsp, k, kind, topology, narrow): k the entry's index in l1.ipreaches; kind the one it gets in the L2 LSP
//   (MT-IPv6 becomes IPv6); topology the L1 SPT whose distance it takes (0 standard, 1 MT-IPv6); narrow: its total
//   is capped at 63.
template <class Emit>
void for_each_propagation(const hl_isis_level &l1, uint64_t local_system_id, uint8_t l1_metric_type,
                          uint8_t l2_metric_type, bool mt6, const uint8_t *up_down, const hl_isis_summary *cfg,
                          uint32_t n_cfg, Emit emit) {
    auto std_on = [](uint8_t t) { return t == HL_ISIS_METRIC_STANDARD || t == HL_ISIS_METRIC_BOTH; };
    auto wide_on = [](uint8_t t) { return t == HL_ISIS_METRIC_WIDE || t == HL_ISIS_METRIC_BOTH; };
    const bool narrow = std_on(l1_metric_type) && std_on(l2_metric_type);
    const bool wide = wide_on(l1_metric_type) && wide_on(l2_metric_type);
    for (uint32_t li = 0; li < l1.n_lsps; ++li) {
        const hl_isis_lsp &lsp = l1.lsps[li];
        if (lsp.seqno == 0 || lsp.rem_lifetime == 0) continue;
        if ((lsp.lan_id & 0xFF) != 0) continue;                     // pseudonode LSP
        if ((lsp.lan_id >> 8) == local_system_id) continue;
        for (uint32_t k = lsp.ipreach_off; k < lsp.ipreach_off + lsp.n_ipreach; ++k) {
            const hl_isis_ipreach &e = l1.ipreaches[k];
            uint8_t kind = e.kind;
            uint32_t topology = 0;
            bool is_narrow = false;
            switch (e.kind) {
            case HL_ISIS_IP_V4_INTERNAL: case HL_ISIS_IP_V4_EXTERNAL:
                if (!l1.ipv4_enabled || !narrow) continue;
                is_narrow = true;
                break;
            case HL_ISIS_IP_V4_EXT:
                if (!l1.ipv4_enabled || !wide) continue;
                break;
            case HL_ISIS_IP_V6:
                if (mt6 || !l1.ipv6_enabled) continue;
                break;
            case HL_ISIS_IP_MT_V6:
                if (!mt6 || e.mt_id != HL_ISIS_MT_IPV6) continue;
                kind = HL_ISIS_IP_V6;                                   // lands in the L2 LSP's IPv6 reachability
                topology = 1;
                break;
            default: continue;
            }
            if (up_down && up_down[k]) continue;
            if (isis_summary_match(cfg, n_cfg, e.prefix, e.len) >= 0) continue;
            emit(lsp, k, kind, topology, is_narrow);
        }
    }
}

}  // namespace hspf
