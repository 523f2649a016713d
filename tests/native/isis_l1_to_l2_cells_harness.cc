// TEST HARNESS (not part of libholo_spf.so): runs the body of the IS-IS L1 -> L2 propagation kernels,
// holo_b200/csrc/isis_l1_to_l2_cells.h — isis_summary_eval over the router's L1/L2 routing table, then
// isis_l1_to_l2_cell_eval — serially on the CPU over planes the test supplies.  Planes per L1 topology k (std,
// MT-IPv6): [rows][V_k] dist, hops, nh, NULL where L1 has no root in the topology; rows [n_jobs]: the job's L1 row.
#include <cstdint>

#include "../../holo_b200/csrc/isis_l1_to_l2_cells.h"

extern "C" int harness_isis_l1_to_l2_cells(const hspf_isis_l1_to_l2_table *t, uint32_t n_jobs,
                                           const uint32_t *const *dist, const uint16_t *const *hops,
                                           const uint64_t *const *nh, const uint32_t *rows, uint64_t *words,
                                           hl_isis_route_cell *cells) {
    const hspf::IsisL1ToL2View v = t->view(t->words.data(), t->recs.data());
    const hspf::IsisL1L2View rib = t->rib->view(t->rib->words.data(), t->rib->contribs.data());
    for (uint32_t j = 0; j < n_jobs; ++j) {
        hspf::PlanesWide pl[2];
        for (uint32_t k = 0; k < 2; ++k) {
            const size_t b = (size_t)rows[j] * t->rib->n_vertices[0][k];
            pl[k] = dist[k] ? hspf::PlanesWide{dist[k] + b, hops[k] + b, nh[k] + b} : hspf::PlanesWide{nullptr, nullptr, nullptr};
        }
        uint64_t *w = words + (size_t)j * rib.S;
        for (uint32_t s = 0; s < rib.S; ++s) w[s] = hspf::isis_summary_eval(pl[0], pl[1], rib, s);
        for (uint32_t k = 0; k < v.K; ++k)
            cells[(size_t)j * v.K + k] = hspf::isis_l1_to_l2_cell_eval(pl[0], pl[1], v, rib, k, w);
    }
    return 0;
}
