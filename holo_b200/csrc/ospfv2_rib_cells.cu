// Device routing-table stage for batches of OSPFv2 SPTs whose roots are attached to one area (include/holo_spf_lsdb.h,
// "batched routing-table stage"): update_rib_full (holo-ospf/src/route.rs:146-193) for every job of a batch.
//
// One thread per (job, prefix) walks the prefix's intra-area advertisers, then its type-3 and type-5 records
// (ospf_rib_cells.h: ospf_rib_cell_eval) and writes one 24-byte hl_ospf_rib_cell through the shared warp-tiled
// store (route_stage.cuh).  As in the intra-area stage, prefix is the fast index and the plane values are gathers
// inside the job's own rows; the type-4 lists behind an external prefix are a few records more, read through the
// read-only cache.
#include <cstring>
#include <vector>

#include "../../include/holo_spf_lsdb.h"
#include "ospf_rib_cells.h"
#include "route_stage.cuh"

namespace {

using hspf::RibRec;

// The cell of (job, prefix): ospf_rib_cell_eval over the job's rows of the planes, from the job's root.
template <class Planes>
struct OspfRibCell {
    hspf::RibView t;
    hspf::ResultPlanes<Planes> pl;
    const uint32_t *roots;
    __device__ __forceinline__ bool refused(uint32_t j) const {
        return pl.refused(j) || hspf::rib_job_refusal(t, roots[j]) != 0;
    }
    // what job_status_out holds for job j
    __device__ __forceinline__ uint32_t status_word(uint32_t j) const {
        return pl.status_word(j) | hspf::rib_job_refusal(t, roots[j]);
    }
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        return hspf::ospf_rib_cell_eval(pl.job(j), roots[j], t, p);
    }
    __device__ __forceinline__ uint64_t gather(uint32_t j, uint32_t, uint32_t v) const { return pl.gather(j, v); }
    __device__ static hspf::CellWords empty() { return {0, 0, hspf::kNoRecord}; }
};

template <class R>
int make_cell(const hspf_ospfv2_ribtable *rt, const R *pl, uint32_t n_jobs, const uint32_t *roots,
              OspfRibCell<hspf::PlanesOf<R>> &cell) {
    if (!rt || !rt->dev.blob || (n_jobs && !roots)) return HSPF_E_INVAL;
    const uint32_t P = (uint32_t)rt->prefix.size(), V = (uint32_t)rt->vflags.size();
    if (hspf::result_planes(pl, V, cell.pl) || !cell.pl.complete()) return HSPF_E_INVAL;
    const RibRec *recs = static_cast<const RibRec *>(rt->dev.contribs);
    cell.t = hspf::RibView{rt->dev.off, recs, reinterpret_cast<const uint8_t *>(recs + rt->recs.size()), P, V};
    cell.roots = roots;
    return HSPF_OK;
}

// Blocks per SM of the route-delta passes over this walk: their launch bound and their grid.  At the cell kernels'
// 8 the walk plus the base compare spills 68 bytes in pass A; from 5 down neither pass spills, and of the bounds
// timed on an H100 this one was fastest (DESIGN.md §4.4, §6).
constexpr uint32_t kRibDeltaBlocksPerSM = 4;

// The cell kernel runs under the route kernels' bound of 8 blocks per SM (see DESIGN.md §4.4 for its registers).
template <class R, class Out>
int rib(hspf_ctx *ctx, const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const R *pl, const uint32_t *roots,
        const Out &out) {
    constexpr uint32_t kBlocks = Out::kDelta ? kRibDeltaBlocksPerSM : hspf::kRouteBlocksPerSM;
    OspfRibCell<hspf::PlanesOf<R>> cell{};
    if (const int rc = make_cell(rt, pl, n_jobs, roots, cell)) return rc;
    return hspf::launch_route_stage<kBlocks>(ctx, rt->dev, cell, n_jobs, cell.t.P, out);
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
    return rib(ctx, rt, n_jobs, pl, roots,
               hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out, n_gather, gather_job, nullptr, gather_v, gather_nh});
}

int hspf_ospfv2_rib_cells16(hspf_ctx *ctx, const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const hspf_result16 *pl,
                            const uint32_t *roots, hl_ospf_rib_cell *cells, uint32_t *job_status_out, uint32_t n_gather,
                            const uint32_t *gather_job, const uint32_t *gather_v, uint64_t *gather_nh) {
    return rib(ctx, rt, n_jobs, pl, roots,
               hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out, n_gather, gather_job, nullptr, gather_v, gather_nh});
}

int hspf_ospfv2_rib_delta(hspf_ctx *ctx, const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const hspf_result *pl,
                          const uint32_t *roots, const hl_ospf_rib_cell *base_cells, uint32_t n_base,
                          const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                          uint64_t *n_records) {
    return rib(ctx, rt, n_jobs, pl, roots,
               hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_ospfv2_rib_delta16(hspf_ctx *ctx, const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const hspf_result16 *pl,
                            const uint32_t *roots, const hl_ospf_rib_cell *base_cells, uint32_t n_base,
                            const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                            uint64_t *n_records) {
    return rib(ctx, rt, n_jobs, pl, roots,
               hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

}  // extern "C"
