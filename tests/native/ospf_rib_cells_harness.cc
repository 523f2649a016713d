// TEST HARNESS (not part of libholo_spf.so): runs ospf_rib_cell_eval — the body of the device routing-table
// kernel, holo_b200/csrc/ospf_rib_cells.h — on the CPU over planes the test supplies, with the kernel's refusal
// rule, so that the walk and the host decode can be checked against update_rib_full without a GPU.
#include <cstdint>

#include "../../holo_b200/csrc/ospf_rib_cells.h"

namespace {

template <class Planes, class D, class N>
void cells_of(const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const uint32_t *roots, const uint32_t *status,
              const D *dist, const uint16_t *hops, const N *nh, hl_ospf_rib_cell *cells, uint32_t *status_out) {
    const hspf::RibView t = rt->host_view();
    for (uint32_t j = 0; j < n_jobs; ++j) {
        const uint32_t st = (status ? status[j] : 0u) | hspf::rib_job_refusal(t, roots[j]);
        if (status_out) status_out[j] = st;
        const Planes pl{dist + (size_t)j * t.V, hops + (size_t)j * t.V, nh + (size_t)j * t.V};
        for (uint32_t p = 0; p < t.P; ++p) {
            const hspf::CellWords w = st ? hspf::CellWords{0, 0, hspf::kNoRecord} : hspf::ospf_rib_cell_eval(pl, roots[j], t, p);
            hl_ospf_rib_cell &c = cells[(size_t)j * t.P + p];
            c.nh_mask = w.w0; c.aux = w.w1; c.winner = (uint32_t)w.w2; c.mpf = (uint32_t)(w.w2 >> 32);
        }
    }
}

}  // namespace

extern "C" int harness_rib_cells(const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const uint32_t *roots,
                                 const uint32_t *status, const uint32_t *dist, const uint16_t *hops, const uint64_t *nh,
                                 hl_ospf_rib_cell *cells, uint32_t *status_out) {
    cells_of<hspf::PlanesWide>(rt, n_jobs, roots, status, dist, hops, nh, cells, status_out);
    return 0;
}

extern "C" int harness_rib_cells16(const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const uint32_t *roots,
                                   const uint32_t *status, const uint16_t *dist, const uint16_t *hops, const uint16_t *nh,
                                   hl_ospf_rib_cell *cells, uint32_t *status_out) {
    cells_of<hspf::PlanesNarrow>(rt, n_jobs, roots, status, dist, hops, nh, cells, status_out);
    return 0;
}
