// TEST HARNESS (not part of libholo_spf.so): runs the body of the OSPFv3 area-border-router kernel over jobs inside
// another area (hspf_ospfv3_abr_backbone_table_create), holo_b200/csrc/ospf_abr_rib_cells.h — abr_rib_cell_eval with
// kSlots over AbrBorderSlots<true> — serially on the CPU, with the kernel's job status rule.  The arguments are those
// of ospf_abr_backbone_cells_harness.cc.  Returns -1 for a table that is not an OSPFv3 one.
#include <cstdint>

#include "../../holo_b200/csrc/ospf_backbone_cells.h"

namespace {

template <class Planes, class D, class N>
void cells_of(const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs, const void *const *dist,
              const void *const *hops, const void *const *nh, const uint32_t *root_status,
              const hl_ospf_rib_cell *const *border_cells, const uint32_t *const *border_status,
              const void *const *const *border_dist, const uint32_t *const *const *border_pstatus,
              const uint32_t *const *border_n_rows, const uint32_t *const *border_rows, hl_ospf_rib_cell *cells,
              uint32_t *status_out) {
    const hspf::AbrRibView v = t->view(t->words.data(), t->abr->recs.data());
    hspf::AbrPlaneSet<D, N> s{};
    for (uint32_t i = 0; i < v.n_areas; ++i) {
        s.dist[i] = static_cast<const D *>(dist[i]); s.hops[i] = static_cast<const uint16_t *>(hops[i]);
        s.nh[i] = static_cast<const N *>(nh[i]); s.status[i] = root_status ? root_status + i : nullptr;
        s.V[i] = t->abr->n_vertices[i]; s.n_rows[i] = 1;
    }
    hspf::OspfAsbrSets<D> sets{};
    sets.n = (uint32_t)t->asbr_set.size();
    for (uint32_t k = 0; k < sets.n; ++k) {
        const uint32_t b = t->asbr_set[k].first, i = t->asbr_set[k].second;
        sets.dist[k] = static_cast<const D *>(border_dist[b][i]);
        sets.status[k] = border_pstatus && border_pstatus[b] ? border_pstatus[b][i] : nullptr;
        sets.rows[k] = border_rows[b];
        sets.V[k] = t->borders[b]->n_vertices[i]; sets.n_rows[k] = border_n_rows[b][i];
        sets.stride[k] = t->borders[b]->n_areas; sets.area[k] = i;
    }
    for (uint32_t j = 0; j < n_jobs; ++j) {
        uint32_t st = hspf::abr_row0_status(s, v.n_areas) | hspf::asbr_job_status(sets, j);
        hspf::AbrBorderSlots<true> sl{};
        sl.border = t->words.data() + t->border_at();
        sl.n_recs = t->n_recs();
        for (uint32_t b = 0; b < t->n_borders; ++b) {
            sl.rows.row[b] = border_cells[b] + (size_t)j * t->borders[b]->prefix.size();
            if (border_status && border_status[b]) st |= border_status[b][j];
        }
        if (status_out) status_out[j] = st;
        const hspf::AbrRow0Planes<Planes, D, N> plane{s, {sets, j}};
        for (uint32_t p = 0; p < v.P; ++p) {
            const hspf::CellWords w = st ? hspf::CellWords{0, 0, hspf::kNoRecord}
                                         : hspf::abr_rib_cell_eval<Planes, true>(plane, v, p, sl);
            hl_ospf_rib_cell &c = cells[(size_t)j * v.P + p];
            c.nh_mask = w.w0; c.aux = w.w1; c.winner = (uint32_t)w.w2; c.mpf = (uint32_t)(w.w2 >> 32);
        }
    }
}

}  // namespace

// the create's winner rule (ospf_backbone_cells.h), at sizes no test table reaches
extern "C" int harness_abr_backbone_winners_fit(uint64_t n_recs, uint64_t n_slots, int v3) {
    return hspf::backbone_winners_fit(n_recs, n_slots, v3 != 0) ? 1 : 0;
}

extern "C" int harness_ospfv3_abr_backbone_cells(const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                                 const void *const *dist, const void *const *hops,
                                                 const void *const *nh, const uint32_t *root_status,
                                                 const hl_ospf_rib_cell *const *border_cells,
                                                 const uint32_t *const *border_status,
                                                 const void *const *const *border_dist,
                                                 const uint32_t *const *const *border_pstatus,
                                                 const uint32_t *const *border_n_rows,
                                                 const uint32_t *const *border_rows, hl_ospf_rib_cell *cells,
                                                 uint32_t *status_out) {
    if (!t || !t->abr || !t->abr->v3) return -1;
    cells_of<hspf::PlanesWide, uint32_t, uint64_t>(t, n_jobs, dist, hops, nh, root_status, border_cells, border_status,
                                                   border_dist, border_pstatus, border_n_rows, border_rows, cells,
                                                   status_out);
    return 0;
}

extern "C" int harness_ospfv3_abr_backbone_cells16(const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                                   const void *const *dist, const void *const *hops,
                                                   const void *const *nh, const uint32_t *root_status,
                                                   const hl_ospf_rib_cell *const *border_cells,
                                                   const uint32_t *const *border_status,
                                                   const void *const *const *border_dist,
                                                   const uint32_t *const *const *border_pstatus,
                                                   const uint32_t *const *border_n_rows,
                                                   const uint32_t *const *border_rows, hl_ospf_rib_cell *cells,
                                                   uint32_t *status_out) {
    if (!t || !t->abr || !t->abr->v3) return -1;
    cells_of<hspf::PlanesNarrow, uint16_t, uint16_t>(t, n_jobs, dist, hops, nh, root_status, border_cells,
                                                     border_status, border_dist, border_pstatus, border_n_rows,
                                                     border_rows, cells, status_out);
    return 0;
}
