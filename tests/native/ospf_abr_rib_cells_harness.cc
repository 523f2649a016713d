// TEST HARNESS (not part of libholo_spf.so): runs abr_rib_cell_eval — the body of the device routing-table kernel
// for area border routers, holo_b200/csrc/ospf_abr_rib_cells.h — on the CPU over planes the test supplies, with the
// kernel's job status rule, so that the walk and the host decode can be checked against update_rib_full without a GPU.
#include <cstdint>

#include "../../holo_b200/csrc/ospf_abr_rib_cells.h"

namespace {

template <class Planes, class D, class N>
void cells_of(const hspf_ospfv2_abr_ribtable *rt, uint32_t n_jobs, const uint32_t *rows, const void *const *dist,
              const void *const *hops, const void *const *nh, const uint32_t *const *status, const uint32_t *n_rows,
              hl_ospf_rib_cell *cells, uint32_t *status_out) {
    const hspf::AbrRibView t = rt->host_view();
    hspf::AbrPlaneSet<D, N> s{};
    for (uint32_t i = 0; i < t.n_areas; ++i) {
        s.dist[i] = static_cast<const D *>(dist[i]); s.hops[i] = static_cast<const uint16_t *>(hops[i]);
        s.nh[i] = static_cast<const N *>(nh[i]); s.status[i] = status ? status[i] : nullptr;
        s.V[i] = rt->n_vertices[i]; s.n_rows[i] = n_rows[i];
    }
    for (uint32_t j = 0; j < n_jobs; ++j) {
        const uint32_t *row = rows + (size_t)j * t.n_areas;
        const uint32_t st = hspf::abr_job_status(s, t.n_areas, row);
        if (status_out) status_out[j] = st;
        const hspf::AbrJobPlanes<Planes, D, N> plane{s, row};
        for (uint32_t p = 0; p < t.P; ++p) {
            const hspf::CellWords w = st ? hspf::CellWords{0, 0, hspf::kNoRecord} : hspf::abr_rib_cell_eval<Planes>(plane, t, p);
            hl_ospf_rib_cell &c = cells[(size_t)j * t.P + p];
            c.nh_mask = w.w0; c.aux = w.w1; c.winner = (uint32_t)w.w2; c.mpf = (uint32_t)(w.w2 >> 32);
        }
    }
}

}  // namespace

extern "C" int harness_abr_rib_cells(const hspf_ospfv2_abr_ribtable *rt, uint32_t n_jobs, const uint32_t *rows,
                                     const void *const *dist, const void *const *hops, const void *const *nh,
                                     const uint32_t *const *status, const uint32_t *n_rows, hl_ospf_rib_cell *cells,
                                     uint32_t *status_out) {
    cells_of<hspf::PlanesWide, uint32_t, uint64_t>(rt, n_jobs, rows, dist, hops, nh, status, n_rows, cells, status_out);
    return 0;
}

extern "C" int harness_abr_rib_cells16(const hspf_ospfv2_abr_ribtable *rt, uint32_t n_jobs, const uint32_t *rows,
                                       const void *const *dist, const void *const *hops, const void *const *nh,
                                       const uint32_t *const *status, const uint32_t *n_rows, hl_ospf_rib_cell *cells,
                                       uint32_t *status_out) {
    cells_of<hspf::PlanesNarrow, uint16_t, uint16_t>(rt, n_jobs, rows, dist, hops, nh, status, n_rows, cells, status_out);
    return 0;
}
