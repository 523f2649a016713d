// TEST HARNESS (not part of libholo_spf.so): runs the bodies of the OSPFv2 third-area kernels serially on the CPU,
// with the kernels' job status rules (holo_b200/csrc/ospf_backbone_cells.h):
//   harness_ospf_third_area_cells[16]  ospf_backbone_cell_eval with kAsbr and kNonBackbone over a third-area table
//       (hspf_ospfv2_third_area_table_create), the chain slots reading each border's entries (OspfChainJob).  R's
//       planes are one row of R's area; border_cells[b] / border_status[b] as ospf_backbone_cells_harness.cc;
//       border_entries[b] u32 [n_jobs][G_b] and border_entry_status[b] (NULL: none).
//   harness_ospf_abr_asbr_entries[16]  abr_asbr_entry per (job, group) of an abr_backbone table: C's planes per area
//       one row (dist[i], hops[i], nh[i], root_status[i]); the B plane sets as ospf_abr_backbone_cells_harness.cc.
//   harness_third_area_winners_fit  backbone_winners_fit with the OSPFv2 encoding.
#include <cstdint>

#include "../../holo_b200/csrc/ospf_backbone_cells.h"

namespace {

template <class Planes, class D, class N>
void cells_of(const hspf_ospfv2_backbone_table *t, uint32_t n_jobs, const void *dist, const uint16_t *hops,
              const void *nh, uint32_t root_status, const hl_ospf_rib_cell *const *border_cells,
              const uint32_t *const *border_status, const uint32_t *const *border_entries,
              const uint32_t *const *border_entry_status, hl_ospf_rib_cell *cells, uint32_t *status_out) {
    const hspf::OspfBackboneView v = t->host_view();
    const Planes pl{static_cast<const D *>(dist), hops, static_cast<const N *>(nh)};
    hspf::OspfChainSet s{};
    for (uint32_t b = 0; b < t->n_borders; ++b) {
        s.entries[b] = border_entries ? border_entries[b] : nullptr;
        s.status[b] = border_entry_status ? border_entry_status[b] : nullptr;
        s.G[b] = (uint32_t)t->third[b]->asbr_group.size();
    }
    for (uint32_t j = 0; j < n_jobs; ++j) {
        uint32_t st = root_status;
        hspf::OspfBorderRows rows{};
        const hspf::OspfThirdAreaPlanes<Planes> tpl{pl, {s, j}};
        for (uint32_t b = 0; b < t->n_borders; ++b) {
            rows.row[b] = border_cells[b] + (size_t)j * t->borders[b]->prefix.size();
            if (border_status && border_status[b]) st |= border_status[b][j];
            if (s.status[b]) st |= s.status[b][j];
        }
        if (status_out) status_out[j] = st;
        for (uint32_t p = 0; p < v.P; ++p) {
            const hspf::CellWords w = st ? hspf::CellWords{0, 0, hspf::kNoRecord}
                                         : hspf::ospf_backbone_cell_eval<false, true, true>(tpl, v, p, rows);
            hl_ospf_rib_cell &c = cells[(size_t)j * v.P + p];
            c.nh_mask = w.w0; c.aux = w.w1; c.winner = (uint32_t)w.w2; c.mpf = (uint32_t)(w.w2 >> 32);
        }
    }
}

template <class Planes, class D, class N>
void entries_of(const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs, const void *const *dist,
                const void *const *hops, const void *const *nh, const uint32_t *root_status,
                const void *const *const *border_dist, const uint32_t *const *const *border_pstatus,
                const uint32_t *const *border_n_rows, const uint32_t *const *border_rows, uint32_t *entries,
                uint32_t *status_out) {
    const hspf_ospfv2_abr_ribtable &a = *t->abr;
    hspf::AbrPlaneSet<D, N> s{};
    for (uint32_t i = 0; i < a.n_areas; ++i) {
        s.dist[i] = static_cast<const D *>(dist[i]); s.hops[i] = static_cast<const uint16_t *>(hops[i]);
        s.nh[i] = static_cast<const N *>(nh[i]); s.status[i] = root_status ? root_status + i : nullptr;
        s.V[i] = a.n_vertices[i]; s.n_rows[i] = 1;
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
    const uint32_t G = (uint32_t)t->asbr_group.size(), i0 = t->area0;
    const Planes pl{s.dist[i0], s.hops[i0], s.nh[i0]};
    for (uint32_t j = 0; j < n_jobs; ++j) {
        const uint32_t st = hspf::abr_row0_status(s, a.n_areas) | hspf::asbr_job_status(sets, j);
        if (status_out) status_out[j] = st;
        const hspf::OspfAsbrJob<Planes, D> asbr{sets, j};
        for (uint32_t k = 0; k < G; ++k)
            entries[(size_t)j * G + k] =
                st ? hspf::kOspfNoEntry
                   : hspf::abr_asbr_entry(pl, asbr, a.recs.data(), a.ext_end + t->asbr_group[k] * a.n_areas + i0);
    }
}

}  // namespace

// the create's check that every slot winner (n_records + slot index) fits below kNoRecord
extern "C" int harness_third_area_winners_fit(uint64_t n_recs, uint64_t n_slots) {
    return hspf::backbone_winners_fit(n_recs, n_slots, false) ? 1 : 0;
}

extern "C" int harness_ospf_third_area_cells(const hspf_ospfv2_backbone_table *t, uint32_t n_jobs, const void *dist,
                                             const uint16_t *hops, const void *nh, uint32_t root_status,
                                             const hl_ospf_rib_cell *const *border_cells,
                                             const uint32_t *const *border_status,
                                             const uint32_t *const *border_entries,
                                             const uint32_t *const *border_entry_status, hl_ospf_rib_cell *cells,
                                             uint32_t *status_out) {
    cells_of<hspf::PlanesWide, uint32_t, uint64_t>(t, n_jobs, dist, hops, nh, root_status, border_cells, border_status,
                                                   border_entries, border_entry_status, cells, status_out);
    return 0;
}

extern "C" int harness_ospf_third_area_cells16(const hspf_ospfv2_backbone_table *t, uint32_t n_jobs, const void *dist,
                                               const uint16_t *hops, const void *nh, uint32_t root_status,
                                               const hl_ospf_rib_cell *const *border_cells,
                                               const uint32_t *const *border_status,
                                               const uint32_t *const *border_entries,
                                               const uint32_t *const *border_entry_status, hl_ospf_rib_cell *cells,
                                               uint32_t *status_out) {
    cells_of<hspf::PlanesNarrow, uint16_t, uint16_t>(t, n_jobs, dist, hops, nh, root_status, border_cells,
                                                     border_status, border_entries, border_entry_status, cells,
                                                     status_out);
    return 0;
}

extern "C" int harness_ospf_abr_asbr_entries(const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                             const void *const *dist, const void *const *hops, const void *const *nh,
                                             const uint32_t *root_status, const void *const *const *border_dist,
                                             const uint32_t *const *const *border_pstatus,
                                             const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                             uint32_t *entries, uint32_t *status_out) {
    entries_of<hspf::PlanesWide, uint32_t, uint64_t>(t, n_jobs, dist, hops, nh, root_status, border_dist,
                                                     border_pstatus, border_n_rows, border_rows, entries, status_out);
    return 0;
}

extern "C" int harness_ospf_abr_asbr_entries16(const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                               const void *const *dist, const void *const *hops, const void *const *nh,
                                               const uint32_t *root_status, const void *const *const *border_dist,
                                               const uint32_t *const *const *border_pstatus,
                                               const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                               uint32_t *entries, uint32_t *status_out) {
    entries_of<hspf::PlanesNarrow, uint16_t, uint16_t>(t, n_jobs, dist, hops, nh, root_status, border_dist,
                                                       border_pstatus, border_n_rows, border_rows, entries, status_out);
    return 0;
}
