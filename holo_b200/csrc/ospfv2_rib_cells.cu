// Device routing-table stage for batches of OSPFv2 SPTs whose roots are attached to one area (include/holo_spf_lsdb.h,
// "batched routing-table stage"): update_rib_full (holo-ospf/src/route.rs:146-193) for every job of a batch.
//
// One thread per (job, prefix) walks the prefix's intra-area advertisers, then its type-3 and type-5 records
// (ospf_rib_cells.h: ospf_rib_cell_eval) and writes one 24-byte hl_ospf_rib_cell through the shared warp-tiled
// store (route_stage.cuh).  As in the intra-area stage, prefix is the fast index and the plane values are gathers
// inside the job's own rows; the type-4 lists behind an external prefix are a few records more, read through the
// read-only cache.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/holo_spf_lsdb.h"
#include "ospf_rib_cells.h"
#include "route_stage.cuh"

namespace {

using hspf::RibRec;

// The cell of (job, prefix): ospf_rib_cell_eval over the job's rows of the planes, from the job's root.
template <class Planes, class D, class N>
struct OspfRibCell {
    hspf::RibView t;
    const D *dist; const uint16_t *hops; const N *nh;
    const uint32_t *status; const uint32_t *roots;
    __device__ __forceinline__ bool refused(uint32_t j) const {
        return (status && status[j] != 0) || hspf::rib_job_refusal(t, roots[j]) != 0;
    }
    // what job_status_out of ospf_rib_cells_kernel holds for job j
    __device__ __forceinline__ uint32_t status_word(uint32_t j) const {
        return (status ? status[j] : 0u) | hspf::rib_job_refusal(t, roots[j]);
    }
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        const size_t base = (size_t)j * t.V;
        return hspf::ospf_rib_cell_eval(Planes{dist + base, hops + base, nh + base}, roots[j], t, p);
    }
};

// see DESIGN.md §4.4 for the registers of each instantiation
template <class Planes, class D, class N>
__global__ void __launch_bounds__(hspf::kRouteThreads, hspf::kRouteBlocksPerSM)
ospf_rib_cells_kernel(uint32_t n_jobs, hspf::RibView t, const D *__restrict__ dist, const uint16_t *__restrict__ hops,
                      const N *__restrict__ nh, const uint32_t *__restrict__ job_status, const uint32_t *__restrict__ roots,
                      hl_ospf_rib_cell *__restrict__ cells, uint32_t *__restrict__ status_out, bool aligned16,
                      uint32_t n_gather, const uint32_t *__restrict__ gather_job, const uint32_t *__restrict__ gather_v,
                      uint64_t *__restrict__ gather_nh) {
    const OspfRibCell<Planes, D, N> cell{t, dist, hops, nh, job_status, roots};
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x, first = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (status_out)
        for (uint64_t j = first; j < n_jobs; j += stride)
            status_out[j] = (job_status ? job_status[j] : 0u) | hspf::rib_job_refusal(t, roots[j]);
    hspf::store_route_cells(n_jobs, t.P, cell, hspf::CellWords{0, 0, hspf::kNoRecord}, cells, aligned16);
    for (uint64_t g = first; g < n_gather; g += stride) {
        const uint32_t job = gather_job[g], v = gather_v[g];
        gather_nh[g] = (job < n_jobs && v < t.V) ? (uint64_t)nh[(size_t)job * t.V + v] : 0;
    }
}

template <class Planes, class D, class N>
int launch_rib_cells(hspf_ctx *ctx, const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const D *dist, const uint16_t *hops,
                     const N *nh, const uint32_t *status, const uint32_t *roots, hl_ospf_rib_cell *cells,
                     uint32_t *status_out, uint32_t n_gather, const uint32_t *gather_job, const uint32_t *gather_v,
                     uint64_t *gather_nh) {
    if (!ctx || !rt || !rt->dev.blob || !dist || !hops || !nh || !cells || (n_jobs && !roots)) return HSPF_E_INVAL;
    if (n_gather && (!gather_job || !gather_v || !gather_nh)) return HSPF_E_INVAL;
    const uint32_t P = (uint32_t)rt->prefix.size(), V = (uint32_t)rt->vflags.size();
    const uint64_t total = (uint64_t)n_jobs * P;
    if (total + n_gather + (status_out ? n_jobs : 0) == 0) return HSPF_OK;
    const RibRec *recs = static_cast<const RibRec *>(rt->dev.contribs);
    const hspf::RibView t{rt->dev.off, recs, reinterpret_cast<const uint8_t *>(recs + rt->recs.size()), P, V};
    // the grid covers the cells, or the jobs' status words when there are more jobs than cells
    return hspf::launch_route_stage(ctx, rt->dev, std::max<uint64_t>(total, n_jobs), cells,
                                    [&](uint32_t blocks, cudaStream_t st, bool aligned16) {
        ospf_rib_cells_kernel<Planes, D, N><<<blocks, hspf::kRouteThreads, 0, st>>>(
            n_jobs, t, dist, hops, nh, status, roots, cells, status_out, aligned16, n_gather, gather_job, gather_v, gather_nh);
    });
}

// Blocks per SM of the route-delta passes over this walk: their launch bound and their grid.  At the cell kernels'
// 8 the walk plus the base compare spills 68 bytes in pass A; from 5 down neither pass spills, and of the bounds
// timed on an H100 this one was fastest (DESIGN.md §4.4, §6).
constexpr uint32_t kRibDeltaBlocksPerSM = 4;

// The route-delta stage over the same walk (route_stage.cuh: launch_route_delta), its grid one wave of
// kRibDeltaBlocksPerSM blocks per SM.
template <class Planes, class D, class N>
int launch_rib_delta(hspf_ctx *ctx, const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const D *dist, const uint16_t *hops,
                     const N *nh, const uint32_t *status, const uint32_t *roots, const hl_ospf_rib_cell *base_cells,
                     uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records,
                     uint64_t cap, uint64_t *n_records) {
    if (!ctx || !rt || !rt->dev.blob || !dist || !hops || !nh || (n_jobs && !roots)) return HSPF_E_INVAL;
    using Cell = OspfRibCell<Planes, D, N>;
    const uint32_t P = (uint32_t)rt->prefix.size(), V = (uint32_t)rt->vflags.size();
    const RibRec *recs = static_cast<const RibRec *>(rt->dev.contribs);
    const Cell cell{hspf::RibView{rt->dev.off, recs, reinterpret_cast<const uint8_t *>(recs + rt->recs.size()), P, V},
                    dist, hops, nh, status, roots};
    hspf::DeltaArgs a{};
    a.n_jobs = n_jobs; a.P = P;
    a.base = reinterpret_cast<const uint64_t *>(base_cells); a.n_base = n_base; a.base_of = base_of;
    a.job_out = job_out; a.n_records = reinterpret_cast<unsigned long long *>(n_records);
    a.records = records; a.cap = cap;
    return hspf::launch_route_delta(ctx, rt->dev, a,
        [&](uint32_t blocks, cudaStream_t st, const hspf::DeltaArgs &args) {
            hspf::route_delta_count_kernel<hspf::OspfRibCellLayout, Cell, kRibDeltaBlocksPerSM>
                <<<blocks, hspf::kRouteThreads, 0, st>>>(cell, args);
        },
        [&](uint32_t blocks, cudaStream_t st, const hspf::DeltaArgs &args) {
            hspf::route_delta_store_kernel<hspf::OspfRibCellLayout, Cell, kRibDeltaBlocksPerSM>
                <<<blocks, hspf::kRouteThreads, 0, st>>>(cell, args);
        },
        kRibDeltaBlocksPerSM);
}

}  // namespace

extern "C" {

int hspf_ospfv2_ribtable_upload(hspf_ctx *ctx, hspf_ospfv2_ribtable *rt) {
    if (!rt) return HSPF_E_INVAL;
    // the records, then one flags byte per vertex
    std::vector<uint8_t> blob(rt->recs.size() * sizeof(RibRec) + rt->vflags.size());
    if (!rt->recs.empty()) std::memcpy(blob.data(), rt->recs.data(), rt->recs.size() * sizeof(RibRec));
    if (!rt->vflags.empty()) std::memcpy(blob.data() + rt->recs.size() * sizeof(RibRec), rt->vflags.data(), rt->vflags.size());
    return hspf::upload_route_table(ctx, rt->dev, rt->off, blob.data(), blob.size());
}

int hspf_ospfv2_rib_cells(hspf_ctx *ctx, const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const hspf_result *pl,
                          const uint32_t *roots, hl_ospf_rib_cell *cells, uint32_t *job_status_out, uint32_t n_gather,
                          const uint32_t *gather_job, const uint32_t *gather_v, uint64_t *gather_nh) {
    if (!pl || pl->nh_words != 1) return HSPF_E_INVAL;
    return launch_rib_cells<hspf::PlanesWide, uint32_t, uint64_t>(ctx, rt, n_jobs, pl->dist, pl->hops, pl->nh_mask,
                                                                  pl->job_status, roots, cells, job_status_out, n_gather,
                                                                  gather_job, gather_v, gather_nh);
}

int hspf_ospfv2_rib_cells16(hspf_ctx *ctx, const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const hspf_result16 *pl,
                            const uint32_t *roots, hl_ospf_rib_cell *cells, uint32_t *job_status_out, uint32_t n_gather,
                            const uint32_t *gather_job, const uint32_t *gather_v, uint64_t *gather_nh) {
    if (!pl) return HSPF_E_INVAL;
    return launch_rib_cells<hspf::PlanesNarrow, uint16_t, uint16_t>(ctx, rt, n_jobs, pl->dist, pl->hops, pl->nh_mask,
                                                                    pl->job_status, roots, cells, job_status_out, n_gather,
                                                                    gather_job, gather_v, gather_nh);
}

int hspf_ospfv2_rib_delta(hspf_ctx *ctx, const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const hspf_result *pl,
                          const uint32_t *roots, const hl_ospf_rib_cell *base_cells, uint32_t n_base,
                          const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                          uint64_t *n_records) {
    if (!pl || pl->nh_words != 1) return HSPF_E_INVAL;
    return launch_rib_delta<hspf::PlanesWide, uint32_t, uint64_t>(ctx, rt, n_jobs, pl->dist, pl->hops, pl->nh_mask,
                                                                  pl->job_status, roots, base_cells, n_base, base_of,
                                                                  job_out, records, cap, n_records);
}

int hspf_ospfv2_rib_delta16(hspf_ctx *ctx, const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const hspf_result16 *pl,
                            const uint32_t *roots, const hl_ospf_rib_cell *base_cells, uint32_t n_base,
                            const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                            uint64_t *n_records) {
    if (!pl) return HSPF_E_INVAL;
    return launch_rib_delta<hspf::PlanesNarrow, uint16_t, uint16_t>(ctx, rt, n_jobs, pl->dist, pl->hops, pl->nh_mask,
                                                                    pl->job_status, roots, base_cells, n_base, base_of,
                                                                    job_out, records, cap, n_records);
}

}  // extern "C"
