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

// One job's rows of one topology's planes: `base` is job * V of that topology.
template <class Planes, class D, class N>
struct TopoPlanes {
    const D *dist; const uint16_t *hops; const N *nh; const uint32_t *status; uint32_t V;
    __device__ __forceinline__ Planes job(uint32_t j) const {
        const size_t base = (size_t)j * V;
        return Planes{dist + base, hops + base, nh + base};
    }
    __device__ __forceinline__ bool refused(uint32_t j) const { return status && status[j] != 0; }
};

// The cell of (job, prefix): isis_route_cell_eval over the job's rows of both topologies' planes.
template <class Planes, class D, class N>
struct IsisCell {
    const uint32_t *off; const IsisContrib *contribs; TopoPlanes<Planes, D, N> std_pl, mt6_pl;
    __device__ __forceinline__ bool refused(uint32_t j) const { return std_pl.refused(j) || mt6_pl.refused(j); }
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        const hl_isis_route_cell c = hspf::isis_route_cell_eval(std_pl.job(j), mt6_pl.job(j), contribs, off[p], off[p + 1]);
        return {c.nh_mask, (uint64_t)c.winner | ((uint64_t)c.metric << 32), c.flags};
    }
};

template <class Planes, class D, class N>
__global__ void __launch_bounds__(hspf::kRouteThreads)
isis_route_cells_kernel(uint32_t n_jobs, uint32_t P, const uint32_t *__restrict__ off,
                        const IsisContrib *__restrict__ contribs, TopoPlanes<Planes, D, N> std_pl,
                        TopoPlanes<Planes, D, N> mt6_pl, hl_isis_route_cell *__restrict__ cells, bool aligned16) {
    const IsisCell<Planes, D, N> cell{off, contribs, std_pl, mt6_pl};
    hspf::store_route_cells(n_jobs, P, cell, hspf::CellWords{0, 0xFFFFFFFFu, 0}, cells, aligned16);   // empty: winner none
}

template <class Planes, class D, class N>
int launch_isis_cells(hspf_ctx *ctx, const hspf_isis_rtable *rt, uint32_t n_jobs, TopoPlanes<Planes, D, N> std_pl,
                      TopoPlanes<Planes, D, N> mt6_pl, hl_isis_route_cell *cells) {
    if (!ctx || !rt || !rt->dev.blob || !cells) return HSPF_E_INVAL;
    // every topology the table reads needs its planes
    if (rt->root[0] != 0xFFFFFFFFu && (!std_pl.dist || !std_pl.hops || !std_pl.nh)) return HSPF_E_INVAL;
    if (rt->root[1] != 0xFFFFFFFFu && (!mt6_pl.dist || !mt6_pl.hops || !mt6_pl.nh)) return HSPF_E_INVAL;
    const uint32_t P = (uint32_t)rt->prefix.size();
    const uint64_t total = (uint64_t)n_jobs * P;
    if (total == 0) return HSPF_OK;
    return hspf::launch_route_stage(ctx, rt->dev, total, cells, [&](uint32_t blocks, cudaStream_t st, bool aligned16) {
        isis_route_cells_kernel<Planes, D, N><<<blocks, hspf::kRouteThreads, 0, st>>>(
            n_jobs, P, rt->dev.off, static_cast<const IsisContrib *>(rt->dev.contribs), std_pl, mt6_pl, cells, aligned16);
    });
}

}  // namespace

extern "C" {

int hspf_isis_rtable_upload(hspf_ctx *ctx, hspf_isis_rtable *rt) {
    return rt ? hspf::upload_route_table(ctx, rt->dev, rt->off, rt->contribs.data(), rt->contribs.size() * sizeof(IsisContrib))
              : HSPF_E_INVAL;
}

int hspf_isis_routes_batch(hspf_ctx *ctx, const hspf_isis_rtable *rt, uint32_t n_jobs, const hspf_result *std_planes,
                           const hspf_result *mt6_planes, hl_isis_route_cell *cells) {
    if (!rt) return HSPF_E_INVAL;
    using TP = TopoPlanes<hspf::PlanesWide, uint32_t, uint64_t>;
    TP s{nullptr, nullptr, nullptr, nullptr, rt->n_vertices[0]}, m{nullptr, nullptr, nullptr, nullptr, rt->n_vertices[1]};
    if (std_planes) {
        if (std_planes->nh_words != 1) return HSPF_E_INVAL;
        s.dist = std_planes->dist; s.hops = std_planes->hops; s.nh = std_planes->nh_mask; s.status = std_planes->job_status;
    }
    if (mt6_planes) {
        if (mt6_planes->nh_words != 1) return HSPF_E_INVAL;
        m.dist = mt6_planes->dist; m.hops = mt6_planes->hops; m.nh = mt6_planes->nh_mask; m.status = mt6_planes->job_status;
    }
    return launch_isis_cells(ctx, rt, n_jobs, s, m, cells);
}

int hspf_isis_routes_batch16(hspf_ctx *ctx, const hspf_isis_rtable *rt, uint32_t n_jobs, const hspf_result16 *std_planes,
                             const hspf_result16 *mt6_planes, hl_isis_route_cell *cells) {
    if (!rt) return HSPF_E_INVAL;
    using TP = TopoPlanes<hspf::PlanesNarrow, uint16_t, uint16_t>;
    TP s{nullptr, nullptr, nullptr, nullptr, rt->n_vertices[0]}, m{nullptr, nullptr, nullptr, nullptr, rt->n_vertices[1]};
    if (std_planes) {
        s.dist = std_planes->dist; s.hops = std_planes->hops; s.nh = std_planes->nh_mask; s.status = std_planes->job_status;
    }
    if (mt6_planes) {
        m.dist = mt6_planes->dist; m.hops = mt6_planes->hops; m.nh = mt6_planes->nh_mask; m.status = mt6_planes->job_status;
    }
    return launch_isis_cells(ctx, rt, n_jobs, s, m, cells);
}

}  // extern "C"
