// Host set-up shared by the OSPF backbone stages (ospfv2_backbone.cu, ospfv2_abr_backbone.cu): binding the
// borders' routing-table cells and the plane sets of the type-4 slots into a stage's cell functor, and an area border
// router's row-0 planes of every area.  nvcc only.
#pragma once
#include "../../include/holo_spf_lsdb.h"
#include "ospf_backbone_cells.h"
#include "route_stage.cuh"

namespace hspf {

// Each border's cells, status words (border_status NULL: none) and K into cell.cells / status / K; the slots past
// the table's borders are NULL.
template <class Table, class Cell>
int bind_ospf_borders(const Table &t, const hl_ospf_rib_cell *const *border_cells, const uint32_t *const *border_status,
                      Cell &cell) {
    for (uint32_t b = 0; b < kOspfBackboneMaxBorders; ++b) {
        cell.cells[b] = nullptr; cell.status[b] = nullptr; cell.K[b] = 0;
        if (b >= t.n_borders) continue;
        // the border's cells, 8-byte words of 24-byte cells
        if (!border_cells[b] || (reinterpret_cast<uintptr_t>(border_cells[b]) & 7u)) return HSPF_E_INVAL;
        cell.cells[b] = border_cells[b];
        cell.status[b] = border_status ? border_status[b] : nullptr;
        cell.K[b] = (uint32_t)t.borders[b]->prefix.size();
    }
    cell.n_borders = t.n_borders;
    return HSPF_OK;
}

// The plane sets the type-4 slots name into cell.sets, from each border's planes, row counts and rows
// (border_planes[b][i], border_n_rows[b][i], border_rows[b]), which may be NULL when the table names none.
template <class Table, class R, class Cell>
int bind_ospf_asbr_sets(const Table &t, const R *const *border_planes, const uint32_t *const *border_n_rows,
                        const uint32_t *const *border_rows, uint32_t n_jobs, Cell &cell) {
    auto &s = cell.sets;
    s.n = (uint32_t)t.asbr_set.size();
    if (s.n && (!border_planes || !border_n_rows || (n_jobs && !border_rows))) return HSPF_E_INVAL;
    for (uint32_t k = 0; k < s.n; ++k) {
        const uint32_t b = t.asbr_set[k].first, i = t.asbr_set[k].second;
        if (!border_planes[b] || !border_n_rows[b] || (n_jobs && !border_rows[b])) return HSPF_E_INVAL;
        ResultPlanes<PlanesOf<R>> p;
        if (result_planes(&border_planes[b][i], t.borders[b]->n_vertices[i], p) || !p.complete()) return HSPF_E_INVAL;
        s.dist[k] = p.dist; s.status[k] = p.status; s.V[k] = p.V;
        s.rows[k] = border_rows[b]; s.n_rows[k] = border_n_rows[b][i];
        s.stride[k] = t.borders[b]->n_areas; s.area[k] = i;
    }
    return HSPF_OK;
}

// An area border router's planes of each area (planes[i], a.n_vertices[i] vertices) into s, one row each (row 0).
template <class AbrTable, class R, class D, class N>
int bind_abr_row0_planes(const AbrTable &a, const R *planes, AbrPlaneSet<D, N> &s) {
    for (uint32_t i = 0; i < a.n_areas; ++i) {
        ResultPlanes<PlanesOf<R>> p;
        if (result_planes(&planes[i], a.n_vertices[i], p) || !p.complete()) return HSPF_E_INVAL;
        s.dist[i] = p.dist; s.hops[i] = p.hops; s.nh[i] = p.nh; s.status[i] = p.status;
        s.V[i] = p.V; s.n_rows[i] = 1;
    }
    return HSPF_OK;
}

}  // namespace hspf
