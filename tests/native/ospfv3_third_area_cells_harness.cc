// TEST HARNESS (not part of libholo_spf.so): runs the body of the OSPFv3 third-area kernel serially on the CPU, with
// the kernel's job status rule (holo_b200/csrc/ospf_backbone_cells.h):
//   harness_ospfv3_third_area_cells[16]  ospf_backbone_cell_eval with kV3, kAsbr, kNonBackbone and kSlotWinners over
//       an OSPFv3 third-area table (hspf_ospfv3_third_area_table_create), the chain slots reading each border's entries
//       (OspfChainJob).  The arguments are those of ospf_third_area_cells_harness.cc; -1 for a table that is not an
//       OSPFv3 third-area one, as the device calls pick the walk from the marks.
//   harness_third_area_v3_winners_fit  backbone_winners_fit with the OSPFv3 encoding.
// The ASBR entries of an OSPFv3 C table run through ospf_third_area_cells_harness.cc: the loop reads the same records.
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
    for (uint32_t b = 0; b < t->n_borders && t->n_asbr_slots; ++b) {
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
                                         : hspf::ospf_backbone_cell_eval<true, true, true, true>(tpl, v, p, rows);
            hl_ospf_rib_cell &c = cells[(size_t)j * v.P + p];
            c.nh_mask = w.w0; c.aux = w.w1; c.winner = (uint32_t)w.w2; c.mpf = (uint32_t)(w.w2 >> 32);
        }
    }
}

}  // namespace

// the create's check that every slot winner (n_records + (slot index << 8 | options)) fits below kNoRecord
extern "C" int harness_third_area_v3_winners_fit(uint64_t n_recs, uint64_t n_slots) {
    return hspf::backbone_winners_fit(n_recs, n_slots, true) ? 1 : 0;
}

extern "C" int harness_ospfv3_third_area_cells(const hspf_ospfv2_backbone_table *t, uint32_t n_jobs, const void *dist,
                                               const uint16_t *hops, const void *nh, uint32_t root_status,
                                               const hl_ospf_rib_cell *const *border_cells,
                                               const uint32_t *const *border_status,
                                               const uint32_t *const *border_entries,
                                               const uint32_t *const *border_entry_status, hl_ospf_rib_cell *cells,
                                               uint32_t *status_out) {
    if (!t || !t->v3 || !t->third_area) return -1;
    cells_of<hspf::PlanesWide, uint32_t, uint64_t>(t, n_jobs, dist, hops, nh, root_status, border_cells, border_status,
                                                   border_entries, border_entry_status, cells, status_out);
    return 0;
}

extern "C" int harness_ospfv3_third_area_cells16(const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                                 const void *dist, const uint16_t *hops, const void *nh,
                                                 uint32_t root_status, const hl_ospf_rib_cell *const *border_cells,
                                                 const uint32_t *const *border_status,
                                                 const uint32_t *const *border_entries,
                                                 const uint32_t *const *border_entry_status, hl_ospf_rib_cell *cells,
                                                 uint32_t *status_out) {
    if (!t || !t->v3 || !t->third_area) return -1;
    cells_of<hspf::PlanesNarrow, uint16_t, uint16_t>(t, n_jobs, dist, hops, nh, root_status, border_cells,
                                                     border_status, border_entries, border_entry_status, cells,
                                                     status_out);
    return 0;
}
