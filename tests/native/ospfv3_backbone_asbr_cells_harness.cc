// TEST HARNESS (not part of libholo_spf.so): runs the body of the OSPFv3 backbone cell kernel over a table with
// Inter-Area-Router slots (hspf_ospfv3_backbone_asbr_table_create), holo_b200/csrc/ospf_backbone_cells.h —
// ospf_backbone_cell_eval with kV3 and kAsbr — serially on the CPU, with the kernel's job status rule.  The arguments
// are those of ospf_backbone_asbr_cells_harness.cc: R's planes are one row of R's area 0; a plane set is a border's
// non-backbone area.
#include <cstdint>

#include "../../holo_b200/csrc/ospf_backbone_cells.h"

namespace {

template <class Planes, class D, class N>
void cells_of(const hspf_ospfv2_backbone_table *t, uint32_t n_jobs, const void *dist, const uint16_t *hops,
              const void *nh, uint32_t root_status, const hl_ospf_rib_cell *const *border_cells,
              const uint32_t *const *border_status, const void *const *const *border_dist,
              const uint32_t *const *const *border_pstatus, const uint32_t *const *border_n_rows,
              const uint32_t *const *border_rows, hl_ospf_rib_cell *cells, uint32_t *status_out) {
    const hspf::OspfBackboneView v = t->host_view();
    const Planes pl{static_cast<const D *>(dist), hops, static_cast<const N *>(nh)};
    hspf::OspfAsbrSets<D> s{};
    s.n = (uint32_t)t->asbr_set.size();
    for (uint32_t k = 0; k < s.n; ++k) {
        const uint32_t b = t->asbr_set[k].first, i = t->asbr_set[k].second;
        s.dist[k] = static_cast<const D *>(border_dist[b][i]);
        s.status[k] = border_pstatus && border_pstatus[b] ? border_pstatus[b][i] : nullptr;
        s.rows[k] = border_rows[b];
        s.V[k] = t->borders[b]->n_vertices[i]; s.n_rows[k] = border_n_rows[b][i];
        s.stride[k] = t->borders[b]->n_areas; s.area[k] = i;
    }
    for (uint32_t j = 0; j < n_jobs; ++j) {
        uint32_t st = root_status | hspf::asbr_job_status(s, j);
        hspf::OspfBorderRows rows{};
        const hspf::OspfAsbrPlanes<Planes, D> apl{pl, {s, j}};
        for (uint32_t b = 0; b < t->n_borders; ++b) {
            rows.row[b] = border_cells[b] + (size_t)j * t->borders[b]->prefix.size();
            if (border_status && border_status[b]) st |= border_status[b][j];
        }
        if (status_out) status_out[j] = st;
        for (uint32_t p = 0; p < v.P; ++p) {
            const hspf::CellWords w = st ? hspf::CellWords{0, 0, hspf::kNoRecord}
                                         : hspf::ospf_backbone_cell_eval<true, true, false>(apl, v, p, rows);
            hl_ospf_rib_cell &c = cells[(size_t)j * v.P + p];
            c.nh_mask = w.w0; c.aux = w.w1; c.winner = (uint32_t)w.w2; c.mpf = (uint32_t)(w.w2 >> 32);
        }
    }
}

}  // namespace

extern "C" int harness_ospfv3_backbone_asbr_cells(const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                                  const void *dist, const uint16_t *hops, const void *nh,
                                                  uint32_t root_status, const hl_ospf_rib_cell *const *border_cells,
                                                  const uint32_t *const *border_status,
                                                  const void *const *const *border_dist,
                                                  const uint32_t *const *const *border_pstatus,
                                                  const uint32_t *const *border_n_rows,
                                                  const uint32_t *const *border_rows, hl_ospf_rib_cell *cells,
                                                  uint32_t *status_out) {
    if (!t || !t->v3 || t->area_id || !t->asbr) return -1;
    cells_of<hspf::PlanesWide, uint32_t, uint64_t>(t, n_jobs, dist, hops, nh, root_status, border_cells, border_status,
                                                   border_dist, border_pstatus, border_n_rows, border_rows, cells,
                                                   status_out);
    return 0;
}

extern "C" int harness_ospfv3_backbone_asbr_cells16(const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                                    const void *dist, const uint16_t *hops, const void *nh,
                                                    uint32_t root_status, const hl_ospf_rib_cell *const *border_cells,
                                                    const uint32_t *const *border_status,
                                                    const void *const *const *border_dist,
                                                    const uint32_t *const *const *border_pstatus,
                                                    const uint32_t *const *border_n_rows,
                                                    const uint32_t *const *border_rows, hl_ospf_rib_cell *cells,
                                                    uint32_t *status_out) {
    if (!t || !t->v3 || t->area_id || !t->asbr) return -1;
    cells_of<hspf::PlanesNarrow, uint16_t, uint16_t>(t, n_jobs, dist, hops, nh, root_status, border_cells,
                                                     border_status, border_dist, border_pstatus, border_n_rows,
                                                     border_rows, cells, status_out);
    return 0;
}
