// Device route stage for batches of IS-IS SPTs (include/holo_spf_lsdb.h, "batched IS-IS route stage"):
// compute_routes (holo-isis/src/spf.rs:838-941) for every job of a batch.
//
// The SPT planes of both topologies stay in HBM; one thread per (job, prefix) walks the prefix's
// contributors (isis_route_cells.h: isis_route_cell_eval) and writes one 24-byte cell.  Prefix is the fast
// index: contributor records and cells are read / written coalesced, the plane values are gathers inside
// the job's own rows of the prefix's topology.  The stage is bounded by the cell writes.
#include "../../include/holo_spf_lsdb.h"
#include "isis_route_cells.h"
#include "route_stage.cuh"

namespace {

using hspf::IsisContrib;

// The cell of (job, prefix): isis_route_cell_eval over the job's rows of both topologies' planes.
template <class Planes>
struct IsisCell {
    const uint32_t *off; const IsisContrib *contribs; hspf::ResultPlanes<Planes> std_pl, mt6_pl;
    __device__ __forceinline__ bool refused(uint32_t j) const { return std_pl.refused(j) || mt6_pl.refused(j); }
    __device__ __forceinline__ uint32_t status_word(uint32_t j) const { return std_pl.status_word(j) | mt6_pl.status_word(j); }
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        const hl_isis_route_cell c = hspf::isis_route_cell_eval(std_pl.job(j), mt6_pl.job(j), contribs, off[p], off[p + 1]);
        return {c.nh_mask, (uint64_t)c.winner | ((uint64_t)c.metric << 32), c.flags};
    }
    __device__ __forceinline__ uint64_t gather(uint32_t, uint32_t, uint32_t) const { return 0; }   // the decode needs none
    __device__ static hspf::CellWords empty() { return {0, 0xFFFFFFFFu, 0}; }                      // winner none
};

// NULL planes are a topology the table does not read
template <class R>
int make_cell(const hspf_isis_rtable *rt, const R *std_planes, const R *mt6_planes, IsisCell<hspf::PlanesOf<R>> &cell) {
    if (!rt || !rt->dev.blob || hspf::result_planes(std_planes, rt->n_vertices[0], cell.std_pl) ||
        hspf::result_planes(mt6_planes, rt->n_vertices[1], cell.mt6_pl))
        return HSPF_E_INVAL;
    if ((rt->root[0] != 0xFFFFFFFFu && !cell.std_pl.complete()) || (rt->root[1] != 0xFFFFFFFFu && !cell.mt6_pl.complete()))
        return HSPF_E_INVAL;
    cell.off = rt->dev.off;
    cell.contribs = static_cast<const IsisContrib *>(rt->dev.contribs);
    return HSPF_OK;
}

// The cell kernel keeps __launch_bounds__(256) with no minimum (a minimum of 0), the delta passes a minimum of 1;
// the grid is one wave of 8 blocks per SM, as for the OSPF stage.
template <class R, class Out>
int routes(hspf_ctx *ctx, const hspf_isis_rtable *rt, uint32_t n_jobs, const R *std_planes, const R *mt6_planes,
           const Out &out) {
    IsisCell<hspf::PlanesOf<R>> cell{};
    if (const int rc = make_cell(rt, std_planes, mt6_planes, cell)) return rc;
    return hspf::launch_route_stage<Out::kDelta ? 1 : 0, hspf::kRouteBlocksPerSM>(ctx, rt->dev, cell, n_jobs,
                                                                                (uint32_t)rt->prefix.size(), out);
}

}  // namespace

extern "C" {

int hspf_isis_rtable_upload(hspf_ctx *ctx, hspf_isis_rtable *rt) {
    return rt ? hspf::upload_route_table(ctx, rt->dev, rt->off, rt->contribs.data(), rt->contribs.size() * sizeof(IsisContrib))
              : HSPF_E_INVAL;
}

int hspf_isis_routes_batch(hspf_ctx *ctx, const hspf_isis_rtable *rt, uint32_t n_jobs, const hspf_result *std_planes,
                           const hspf_result *mt6_planes, hl_isis_route_cell *cells) {
    return routes(ctx, rt, n_jobs, std_planes, mt6_planes, hspf::CellsOut<hl_isis_route_cell>{cells, nullptr});
}

int hspf_isis_routes_batch16(hspf_ctx *ctx, const hspf_isis_rtable *rt, uint32_t n_jobs, const hspf_result16 *std_planes,
                             const hspf_result16 *mt6_planes, hl_isis_route_cell *cells) {
    return routes(ctx, rt, n_jobs, std_planes, mt6_planes, hspf::CellsOut<hl_isis_route_cell>{cells, nullptr});
}

int hspf_isis_routes_delta(hspf_ctx *ctx, const hspf_isis_rtable *rt, uint32_t n_jobs, const hspf_result *std_planes,
                           const hspf_result *mt6_planes, const hl_isis_route_cell *base_cells, uint32_t n_base,
                           const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                           uint64_t *n_records) {
    return routes(ctx, rt, n_jobs, std_planes, mt6_planes,
                  hspf::DeltaOut<hl_isis_route_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_isis_routes_delta16(hspf_ctx *ctx, const hspf_isis_rtable *rt, uint32_t n_jobs, const hspf_result16 *std_planes,
                             const hspf_result16 *mt6_planes, const hl_isis_route_cell *base_cells, uint32_t n_base,
                             const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                             uint64_t *n_records) {
    return routes(ctx, rt, n_jobs, std_planes, mt6_planes,
                  hspf::DeltaOut<hl_isis_route_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

}  // extern "C"
