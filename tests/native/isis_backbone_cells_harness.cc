// TEST HARNESS (not part of libholo_spf.so): runs the body of the IS-IS backbone cell kernel,
// holo_b200/csrc/isis_backbone_cells.h — isis_backbone_cell_eval — serially on the CPU.  Planes per L2 topology k
// (std, MT-IPv6) of the backbone router: one row [V_k] of dist, hops, nh, NULL where it has no root in the topology;
// border_cells[b]: border b's [n_jobs][K_b] L1 -> L2 cells.
#include <cstdint>

#include "../../holo_b200/csrc/isis_backbone_cells.h"

extern "C" int harness_isis_backbone_cells(const hspf_isis_backbone_table *t, uint32_t n_jobs,
                                           const uint32_t *const *dist, const uint16_t *const *hops,
                                           const uint64_t *const *nh, const hl_isis_route_cell *const *border_cells,
                                           hl_isis_route_cell *cells) {
    const hspf::IsisBackboneView v = t->view(t->words.data(), t->contribs.data());
    hspf::PlanesWide pl[2];
    for (uint32_t k = 0; k < 2; ++k)
        pl[k] = dist[k] ? hspf::PlanesWide{dist[k], hops[k], nh[k]} : hspf::PlanesWide{nullptr, nullptr, nullptr};
    for (uint32_t j = 0; j < n_jobs; ++j) {
        hspf::IsisBorderRows rows{};
        for (uint32_t b = 0; b < t->n_borders; ++b) rows.row[b] = border_cells[b] + (size_t)j * t->borders[b]->K;
        for (uint32_t p = 0; p < v.P; ++p) cells[(size_t)j * v.P + p] = hspf::isis_backbone_cell_eval(pl[0], pl[1], v, p, rows);
    }
    return 0;
}
