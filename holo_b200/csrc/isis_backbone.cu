// Device stage for the routing table of an IS-IS backbone router over the L1 what-if jobs of an area
// (include/holo_spf_lsdb.h, "backbone routers over L1 what-if jobs"): compute_routes (holo-isis spf.rs:838-941) at
// the router, for its affected prefixes, with every border's L2 LSP re-originated for the job.
//
// One launch on the ctx stream: one thread per (job, prefix) runs isis_backbone_cell_eval (isis_backbone_cells.h)
// over the router's unperturbed L2 planes (row 0) and the job's row of each border's L1 -> L2 cells, and the shared
// cell kernel or the route-delta stage (route_stage.cuh) stores or compares the 24-byte cells.
#include "../../include/holo_spf_lsdb.h"
#include "isis_backbone_cells.h"
#include "route_stage.cuh"

namespace {

using hspf::IsisBackboneContrib;
using hspf::kIsisBackboneMaxBorders;

template <class Planes>
struct IsisBackboneCell {
    using Rows = hspf::ResultPlanes<Planes>;
    hspf::IsisBackboneView t;
    Rows pl[2];                                          // [topology] of R's L2 batch; only row 0 is read
    const hl_isis_route_cell *cells[kIsisBackboneMaxBorders];   // [n_jobs][K_b] per border
    const uint32_t *status[kIsisBackboneMaxBorders];     // [n_jobs] per border, or NULL
    uint32_t K[kIsisBackboneMaxBorders];
    uint32_t n_borders;
    __device__ __forceinline__ uint32_t status_word(uint32_t j) const {
        uint32_t s = pl[0].status_word(0) | pl[1].status_word(0);
        for (uint32_t b = 0; b < n_borders; ++b)
            if (status[b]) s |= status[b][j];
        return s;
    }
    __device__ __forceinline__ bool refused(uint32_t j) const { return status_word(j) != 0; }
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        hspf::IsisBorderRows rows;
#pragma unroll
        for (uint32_t b = 0; b < kIsisBackboneMaxBorders; ++b) rows.row[b] = cells[b] + (size_t)j * K[b];
        const hl_isis_route_cell c = hspf::isis_backbone_cell_eval(pl[0].job(0), pl[1].job(0), t, p, rows);
        return {c.nh_mask, (uint64_t)c.winner | ((uint64_t)c.metric << 32), c.flags};
    }
    __device__ __forceinline__ uint64_t gather(uint32_t, uint32_t, uint32_t) const { return 0; }   // the decode needs none
    __device__ static hspf::CellWords empty() { return {0, 0xFFFFFFFFu, 0}; }                      // winner none
};

// Blocks per SM of the kernels over this walk: their launch bound and their grid.  No spill at 4 or 8; on an H100,
// timed against 8 in one run, 4 was faster for the cell launch and both delta passes, with byte-identical cells
// (DESIGN.md §4.4, §6).
constexpr uint32_t kBackboneBlocksPerSM = 4;

// The topologies the table has no root in are not read: their planes are ignored.
template <class R>
int make_cell(const hspf_isis_backbone_table *t, const R *l2_std, const R *l2_mt6,
              const hl_isis_route_cell *const *border_cells, const uint32_t *const *border_status,
              IsisBackboneCell<hspf::PlanesOf<R>> &cell) {
    if (!t || !t->dev.blob || !border_cells) return HSPF_E_INVAL;
    const R *pl[2] = {l2_std, l2_mt6};
    for (uint32_t k = 0; k < 2; ++k) {
        const uint32_t V = t->n_vertices[k];
        if (t->root[k] == 0xFFFFFFFFu) cell.pl[k] = {nullptr, nullptr, nullptr, nullptr, V};
        else if (hspf::result_planes(pl[k], V, cell.pl[k]) || !cell.pl[k].complete()) return HSPF_E_INVAL;
    }
    for (uint32_t b = 0; b < kIsisBackboneMaxBorders; ++b) {
        cell.cells[b] = nullptr; cell.status[b] = nullptr; cell.K[b] = 0;
        if (b >= t->n_borders) continue;
        // the border's cells, 8-byte words of 24-byte cells
        if (!border_cells[b] || (reinterpret_cast<uintptr_t>(border_cells[b]) & 7u)) return HSPF_E_INVAL;
        cell.cells[b] = border_cells[b];
        cell.status[b] = border_status ? border_status[b] : nullptr;
        cell.K[b] = t->borders[b]->K;
    }
    cell.n_borders = t->n_borders;
    cell.t = t->view(t->dev.off, static_cast<const IsisBackboneContrib *>(t->dev.contribs));
    return HSPF_OK;
}

template <class R, class Out>
int backbone(hspf_ctx *ctx, const hspf_isis_backbone_table *t, uint32_t n_jobs, const R *l2_std, const R *l2_mt6,
             const hl_isis_route_cell *const *border_cells, const uint32_t *const *border_status, const Out &out) {
    IsisBackboneCell<hspf::PlanesOf<R>> cell{};
    if (const int rc = make_cell(t, l2_std, l2_mt6, border_cells, border_status, cell)) return rc;
    return hspf::launch_route_stage<kBackboneBlocksPerSM>(ctx, t->dev, cell, n_jobs, t->P, out);
}

}  // namespace

extern "C" {

int hspf_isis_backbone_table_upload(hspf_ctx *ctx, hspf_isis_backbone_table *t) {
    return t ? hspf::upload_route_table(ctx, t->dev, t->words, t->contribs.data(),
                                        t->contribs.size() * sizeof(IsisBackboneContrib))
             : HSPF_E_INVAL;
}

int hspf_isis_backbone_cells(hspf_ctx *ctx, const hspf_isis_backbone_table *t, uint32_t n_jobs,
                             const hspf_result *l2_std, const hspf_result *l2_mt6,
                             const hl_isis_route_cell *const *border_cells, const uint32_t *const *border_status,
                             uint32_t *job_status_out, hl_isis_route_cell *cells) {
    return backbone(ctx, t, n_jobs, l2_std, l2_mt6, border_cells, border_status,
                    hspf::CellsOut<hl_isis_route_cell>{cells, job_status_out});
}

int hspf_isis_backbone_cells16(hspf_ctx *ctx, const hspf_isis_backbone_table *t, uint32_t n_jobs,
                               const hspf_result16 *l2_std, const hspf_result16 *l2_mt6,
                               const hl_isis_route_cell *const *border_cells, const uint32_t *const *border_status,
                               uint32_t *job_status_out, hl_isis_route_cell *cells) {
    return backbone(ctx, t, n_jobs, l2_std, l2_mt6, border_cells, border_status,
                    hspf::CellsOut<hl_isis_route_cell>{cells, job_status_out});
}

int hspf_isis_backbone_delta(hspf_ctx *ctx, const hspf_isis_backbone_table *t, uint32_t n_jobs,
                             const hspf_result *l2_std, const hspf_result *l2_mt6,
                             const hl_isis_route_cell *const *border_cells, const uint32_t *const *border_status,
                             const hl_isis_route_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                             hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    return backbone(ctx, t, n_jobs, l2_std, l2_mt6, border_cells, border_status,
                    hspf::DeltaOut<hl_isis_route_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_isis_backbone_delta16(hspf_ctx *ctx, const hspf_isis_backbone_table *t, uint32_t n_jobs,
                               const hspf_result16 *l2_std, const hspf_result16 *l2_mt6,
                               const hl_isis_route_cell *const *border_cells, const uint32_t *const *border_status,
                               const hl_isis_route_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                               hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    return backbone(ctx, t, n_jobs, l2_std, l2_mt6, border_cells, border_status,
                    hspf::DeltaOut<hl_isis_route_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

}  // extern "C"
