// TEST HARNESS (not part of libholo_spf.so): runs the body of the IS-IS L1/L2 routing-table kernels,
// holo_b200/csrc/isis_l1l2_rib_cells.h — isis_summary_eval, then isis_l1l2_cell_eval — serially on the CPU over
// planes the test supplies.  Planes per topology k (L1 std, L1 MT-IPv6, L2 std, L2 MT-IPv6): [rows][V_k] dist, hops,
// nh, NULL where that level has no root in the topology; rows [n_jobs][2]: the job's L1 row and L2 row.
#include <cstdint>

#include "../../holo_b200/csrc/isis_l1l2_rib_cells.h"

extern "C" int harness_isis_l1l2_rib_cells(const hspf_isis_l1l2_ribtable *t, uint32_t n_jobs, const uint32_t *const *dist,
                                           const uint16_t *const *hops, const uint64_t *const *nh, const uint32_t *rows,
                                           uint64_t *words, hl_isis_route_cell *cells) {
    const hspf::IsisL1L2View v = t->view(t->words.data(), t->contribs.data());
    for (uint32_t j = 0; j < n_jobs; ++j) {
        hspf::PlanesWide pl[4];
        for (uint32_t k = 0; k < 4; ++k) {
            const size_t b = (size_t)rows[2 * j + k / 2] * t->n_vertices[k / 2][k % 2];
            pl[k] = dist[k] ? hspf::PlanesWide{dist[k] + b, hops[k] + b, nh[k] + b} : hspf::PlanesWide{nullptr, nullptr, nullptr};
        }
        uint64_t *w = words + (size_t)j * v.S;
        for (uint32_t s = 0; s < v.S; ++s) w[s] = hspf::isis_summary_eval(pl[0], pl[1], v, s);
        for (uint32_t p = 0; p < v.P; ++p)
            cells[(size_t)j * v.P + p] = hspf::isis_l1l2_cell_eval(pl[0], pl[1], pl[2], pl[3], v, p, w);
    }
    return 0;
}
