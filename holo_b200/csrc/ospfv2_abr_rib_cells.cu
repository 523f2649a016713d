// Device routing-table stage for area border routers (include/holo_spf_lsdb.h, "for one area border router"):
// update_rib_full over every attached area, for every job of a what-if batch.
//
// One thread per (job, prefix) runs abr_rib_cell_eval (ospf_abr_rib_cells.h) over the job's rows of each area's
// planes and writes one 24-byte hl_ospf_rib_cell through the shared warp-tiled store (route_stage.cuh).  The areas'
// plane pointers travel in the kernel parameter (AbrPlaneSet, at most kAbrMaxAreas areas), so a job's row of area i
// is one load of rows[job][i] and the walk's gathers stay inside that row.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/holo_spf_lsdb.h"
#include "ospf_abr_rib_cells.h"
#include "route_stage.cuh"

namespace {

using hspf::RibRec;

template <class Planes, class D, class N>
struct AbrRibCell {
    hspf::AbrRibView t;
    hspf::AbrPlaneSet<D, N> s;
    const uint32_t *rows;            // [n_jobs][t.n_areas]
    __device__ __forceinline__ uint32_t status_word(uint32_t j) const {
        return hspf::abr_job_status(s, t.n_areas, rows + (size_t)j * t.n_areas);
    }
    __device__ __forceinline__ bool refused(uint32_t j) const { return status_word(j) != 0; }
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        const hspf::AbrJobPlanes<Planes, D, N> plane{s, rows + (size_t)j * t.n_areas};
        return hspf::abr_rib_cell_eval<Planes>(plane, t, p);
    }
};

// Blocks per SM of every kernel over this walk: their launch bound and their grid.  At the route kernels' 8 the
// cell kernel spills (32 registers); at 4 neither it nor the delta passes do, and on an H100 4 was faster for the
// cell kernel and both delta passes, with byte-identical cells (DESIGN.md §4.4, §6).
constexpr uint32_t kAbrBlocksPerSM = 4;

template <class Planes, class D, class N>
__global__ void __launch_bounds__(hspf::kRouteThreads, kAbrBlocksPerSM)
ospf_abr_rib_cells_kernel(const __grid_constant__ AbrRibCell<Planes, D, N> cell, uint32_t n_jobs,
                          hl_ospf_rib_cell *__restrict__ cells, uint32_t *__restrict__ status_out, bool aligned16,
                          uint32_t n_gather, const uint32_t *__restrict__ gather_job,
                          const uint32_t *__restrict__ gather_area, const uint32_t *__restrict__ gather_v,
                          uint64_t *__restrict__ gather_nh) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x, first = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (status_out)
        for (uint64_t j = first; j < n_jobs; j += stride) status_out[j] = cell.status_word((uint32_t)j);
    hspf::store_route_cells(n_jobs, cell.t.P, cell, hspf::CellWords{0, 0, hspf::kNoRecord}, cells, aligned16);
    for (uint64_t g = first; g < n_gather; g += stride) {
        const uint32_t job = gather_job[g], i = gather_area[g], v = gather_v[g];
        uint64_t m = 0;
        if (job < n_jobs && i < cell.t.n_areas && v < cell.s.V[i]) {
            const uint32_t r = cell.rows[(size_t)job * cell.t.n_areas + i];
            if (r < cell.s.n_rows[i]) m = (uint64_t)cell.s.nh[i][(size_t)r * cell.s.V[i] + v];
        }
        gather_nh[g] = m;
    }
}

template <class Planes, class D, class N, class Res>
int make_cell(const hspf_ospfv2_abr_ribtable *t, const Res *pl, const uint32_t *n_rows, uint32_t n_jobs,
              const uint32_t *rows, AbrRibCell<Planes, D, N> &cell) {
    if (!t || !t->dev.blob || !pl || !n_rows || (n_jobs && !rows)) return HSPF_E_INVAL;
    cell = AbrRibCell<Planes, D, N>{};
    const RibRec *recs = static_cast<const RibRec *>(t->dev.contribs);
    cell.t = t->view(t->dev.off, recs, reinterpret_cast<const uint32_t *>(recs + t->recs.size()));
    for (uint32_t i = 0; i < t->n_areas; ++i) {
        if (!pl[i].dist || !pl[i].hops || !pl[i].nh_mask) return HSPF_E_INVAL;
        cell.s.dist[i] = pl[i].dist; cell.s.hops[i] = pl[i].hops; cell.s.nh[i] = pl[i].nh_mask;
        cell.s.status[i] = pl[i].job_status;
        cell.s.V[i] = t->n_vertices[i]; cell.s.n_rows[i] = n_rows[i];
    }
    cell.rows = rows;
    return HSPF_OK;
}

template <class Planes, class D, class N, class Res>
int launch_abr_rib_cells(hspf_ctx *ctx, const hspf_ospfv2_abr_ribtable *t, uint32_t n_jobs, const Res *pl,
                         const uint32_t *n_rows, const uint32_t *rows, hl_ospf_rib_cell *cells, uint32_t *status_out,
                         uint32_t n_gather, const uint32_t *gather_job, const uint32_t *gather_area,
                         const uint32_t *gather_v, uint64_t *gather_nh) {
    if (!ctx || !cells) return HSPF_E_INVAL;
    if (n_gather && (!gather_job || !gather_area || !gather_v || !gather_nh)) return HSPF_E_INVAL;
    AbrRibCell<Planes, D, N> cell;
    const int rc = make_cell(t, pl, n_rows, n_jobs, rows, cell);
    if (rc) return rc;
    const uint64_t total = (uint64_t)n_jobs * cell.t.P;
    if (total + n_gather + (status_out ? n_jobs : 0) == 0) return HSPF_OK;
    // the grid covers the cells, or the jobs' status words / the gathers when there are more of those
    return hspf::launch_route_stage(ctx, t->dev, std::max<uint64_t>(std::max<uint64_t>(total, n_jobs), n_gather), cells,
                                    [&](uint32_t blocks, cudaStream_t st, bool aligned16) {
        ospf_abr_rib_cells_kernel<Planes, D, N><<<blocks, hspf::kRouteThreads, 0, st>>>(
            cell, n_jobs, cells, status_out, aligned16, n_gather, gather_job, gather_area, gather_v, gather_nh);
    }, kAbrBlocksPerSM);
}

template <class Planes, class D, class N, class Res>
int launch_abr_rib_delta(hspf_ctx *ctx, const hspf_ospfv2_abr_ribtable *t, uint32_t n_jobs, const Res *pl,
                         const uint32_t *n_rows, const uint32_t *rows, const hl_ospf_rib_cell *base_cells, uint32_t n_base,
                         const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                         uint64_t *n_records) {
    if (!ctx) return HSPF_E_INVAL;
    using Cell = AbrRibCell<Planes, D, N>;
    Cell cell;
    const int rc = make_cell(t, pl, n_rows, n_jobs, rows, cell);
    if (rc) return rc;
    hspf::DeltaArgs a{};
    a.n_jobs = n_jobs; a.P = cell.t.P;
    a.base = reinterpret_cast<const uint64_t *>(base_cells); a.n_base = n_base; a.base_of = base_of;
    a.job_out = job_out; a.n_records = reinterpret_cast<unsigned long long *>(n_records);
    a.records = records; a.cap = cap;
    return hspf::launch_route_delta(ctx, t->dev, a,
        [&](uint32_t blocks, cudaStream_t st, const hspf::DeltaArgs &args) {
            hspf::route_delta_count_kernel<hspf::OspfRibCellLayout, Cell, kAbrBlocksPerSM>
                <<<blocks, hspf::kRouteThreads, 0, st>>>(cell, args);
        },
        [&](uint32_t blocks, cudaStream_t st, const hspf::DeltaArgs &args) {
            hspf::route_delta_store_kernel<hspf::OspfRibCellLayout, Cell, kAbrBlocksPerSM>
                <<<blocks, hspf::kRouteThreads, 0, st>>>(cell, args);
        },
        kAbrBlocksPerSM);
}

}  // namespace

extern "C" {

int hspf_ospfv2_abr_ribtable_upload(hspf_ctx *ctx, hspf_ospfv2_abr_ribtable *t) {
    if (!t) return HSPF_E_INVAL;
    // the records, then the V-flag router vertices of every area
    const size_t rb = t->recs.size() * sizeof(RibRec), vb = t->v_flagged.size() * sizeof(uint32_t);
    std::vector<uint8_t> blob(rb + vb);
    if (rb) std::memcpy(blob.data(), t->recs.data(), rb);
    if (vb) std::memcpy(blob.data() + rb, t->v_flagged.data(), vb);
    return hspf::upload_route_table(ctx, t->dev, t->off, blob.data(), blob.size());
}

int hspf_ospfv2_abr_rib_cells(hspf_ctx *ctx, const hspf_ospfv2_abr_ribtable *t, uint32_t n_jobs, const hspf_result *pl,
                              const uint32_t *n_rows, const uint32_t *rows, hl_ospf_rib_cell *cells,
                              uint32_t *job_status_out, uint32_t n_gather, const uint32_t *gather_job,
                              const uint32_t *gather_area, const uint32_t *gather_v, uint64_t *gather_nh) {
    if (!t || !pl) return HSPF_E_INVAL;
    for (uint32_t i = 0; i < t->n_areas; ++i)
        if (pl[i].nh_words != 1) return HSPF_E_INVAL;
    return launch_abr_rib_cells<hspf::PlanesWide, uint32_t, uint64_t>(ctx, t, n_jobs, pl, n_rows, rows, cells,
                                                                      job_status_out, n_gather, gather_job, gather_area,
                                                                      gather_v, gather_nh);
}

int hspf_ospfv2_abr_rib_cells16(hspf_ctx *ctx, const hspf_ospfv2_abr_ribtable *t, uint32_t n_jobs,
                                const hspf_result16 *pl, const uint32_t *n_rows, const uint32_t *rows,
                                hl_ospf_rib_cell *cells, uint32_t *job_status_out, uint32_t n_gather,
                                const uint32_t *gather_job, const uint32_t *gather_area, const uint32_t *gather_v,
                                uint64_t *gather_nh) {
    return launch_abr_rib_cells<hspf::PlanesNarrow, uint16_t, uint16_t>(ctx, t, n_jobs, pl, n_rows, rows, cells,
                                                                        job_status_out, n_gather, gather_job,
                                                                        gather_area, gather_v, gather_nh);
}

int hspf_ospfv2_abr_rib_delta(hspf_ctx *ctx, const hspf_ospfv2_abr_ribtable *t, uint32_t n_jobs, const hspf_result *pl,
                              const uint32_t *n_rows, const uint32_t *rows, const hl_ospf_rib_cell *base_cells,
                              uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out,
                              hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    if (!t || !pl) return HSPF_E_INVAL;
    for (uint32_t i = 0; i < t->n_areas; ++i)
        if (pl[i].nh_words != 1) return HSPF_E_INVAL;
    return launch_abr_rib_delta<hspf::PlanesWide, uint32_t, uint64_t>(ctx, t, n_jobs, pl, n_rows, rows, base_cells,
                                                                      n_base, base_of, job_out, records, cap, n_records);
}

int hspf_ospfv2_abr_rib_delta16(hspf_ctx *ctx, const hspf_ospfv2_abr_ribtable *t, uint32_t n_jobs,
                                const hspf_result16 *pl, const uint32_t *n_rows, const uint32_t *rows,
                                const hl_ospf_rib_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                                hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    return launch_abr_rib_delta<hspf::PlanesNarrow, uint16_t, uint16_t>(ctx, t, n_jobs, pl, n_rows, rows, base_cells,
                                                                        n_base, base_of, job_out, records, cap, n_records);
}

}  // extern "C"
