// TEST HARNESS (not part of libholo_spf.so): runs isis_route_cell_eval — the body of the IS-IS device route
// kernel, holo_b200/csrc/isis_route_cells.h — on the CPU over planes the test supplies, so that the cell walk
// and the host decode can be checked against the oracle without a GPU.  Planes per topology: [n_jobs][V_t];
// the MT-IPv6 ones may be NULL when the table has no MT-IPv6 root.
#include <cstdint>

#include "../../holo_b200/csrc/isis_route_cells.h"

extern "C" int harness_isis_route_cells(const hspf_isis_rtable *rt, uint32_t n_jobs, const uint32_t *dist0,
                                        const uint16_t *hops0, const uint64_t *nh0, const uint32_t *dist1,
                                        const uint16_t *hops1, const uint64_t *nh1, hl_isis_route_cell *cells) {
    const uint32_t P = (uint32_t)rt->prefix.size(), V0 = rt->n_vertices[0], V1 = rt->n_vertices[1];
    for (uint32_t j = 0; j < n_jobs; ++j) {
        const hspf::PlanesWide s{dist0 + (size_t)j * V0, hops0 + (size_t)j * V0, nh0 + (size_t)j * V0};
        const hspf::PlanesWide m = dist1 ? hspf::PlanesWide{dist1 + (size_t)j * V1, hops1 + (size_t)j * V1, nh1 + (size_t)j * V1}
                                         : hspf::PlanesWide{nullptr, nullptr, nullptr};
        for (uint32_t p = 0; p < P; ++p)
            cells[(size_t)j * P + p] = hspf::isis_route_cell_eval(s, m, rt->contribs.data(), rt->off[p], rt->off[p + 1]);
    }
    return 0;
}
