// TEST HARNESS (not part of libholo_spf.so): runs the body of the backbone cell kernel for OSPFv3 tables,
// holo_b200/csrc/ospf_backbone_cells.h — ospf_backbone_cell_eval<true> — serially on the CPU, with the kernel's job
// status rule.  R's area-0 planes: one row [V] of dist, hops, nh and its status word; border_cells[b]: border b's
// [n_jobs][K_b] routing-table cells; border_status[b]: its [n_jobs] status words (NULL: none).
#include <cstdint>

#include "../../holo_b200/csrc/ospf_backbone_cells.h"

namespace {

template <class Planes, class D, class N>
void cells_of(const hspf_ospfv2_backbone_table *t, uint32_t n_jobs, const void *dist, const uint16_t *hops,
              const void *nh, uint32_t root_status, const hl_ospf_rib_cell *const *border_cells,
              const uint32_t *const *border_status, hl_ospf_rib_cell *cells, uint32_t *status_out) {
    const hspf::OspfBackboneView v = t->host_view();
    const Planes pl{static_cast<const D *>(dist), hops, static_cast<const N *>(nh)};
    for (uint32_t j = 0; j < n_jobs; ++j) {
        uint32_t st = root_status;
        hspf::OspfBorderRows rows{};
        for (uint32_t b = 0; b < t->n_borders; ++b) {
            rows.row[b] = border_cells[b] + (size_t)j * t->borders[b]->prefix.size();
            if (border_status && border_status[b]) st |= border_status[b][j];
        }
        if (status_out) status_out[j] = st;
        for (uint32_t p = 0; p < v.P; ++p) {
            const hspf::CellWords w =
                st ? hspf::CellWords{0, 0, hspf::kNoRecord} : hspf::ospf_backbone_cell_eval<true>(pl, v, p, rows);
            hl_ospf_rib_cell &c = cells[(size_t)j * v.P + p];
            c.nh_mask = w.w0; c.aux = w.w1; c.winner = (uint32_t)w.w2; c.mpf = (uint32_t)(w.w2 >> 32);
        }
    }
}

}  // namespace

extern "C" int harness_ospfv3_backbone_cells(const hspf_ospfv2_backbone_table *t, uint32_t n_jobs, const void *dist,
                                             const uint16_t *hops, const void *nh, uint32_t root_status,
                                             const hl_ospf_rib_cell *const *border_cells,
                                             const uint32_t *const *border_status, hl_ospf_rib_cell *cells,
                                             uint32_t *status_out) {
    if (!t || !t->v3) return -1;
    cells_of<hspf::PlanesWide, uint32_t, uint64_t>(t, n_jobs, dist, hops, nh, root_status, border_cells, border_status,
                                                   cells, status_out);
    return 0;
}

extern "C" int harness_ospfv3_backbone_cells16(const hspf_ospfv2_backbone_table *t, uint32_t n_jobs, const void *dist,
                                               const uint16_t *hops, const void *nh, uint32_t root_status,
                                               const hl_ospf_rib_cell *const *border_cells,
                                               const uint32_t *const *border_status, hl_ospf_rib_cell *cells,
                                               uint32_t *status_out) {
    if (!t || !t->v3) return -1;
    cells_of<hspf::PlanesNarrow, uint16_t, uint16_t>(t, n_jobs, dist, hops, nh, root_status, border_cells,
                                                     border_status, cells, status_out);
    return 0;
}
