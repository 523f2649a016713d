// Device routing-table stage for area border routers (include/holo_spf_lsdb.h, "for one area border router"):
// update_rib_full over every attached area, for every job of a what-if batch.
//
// One thread per (job, prefix) runs abr_rib_cell_eval (ospf_abr_rib_cells.h) over the job's rows of each area's
// planes and writes one 24-byte hl_ospf_rib_cell through the shared warp-tiled store (route_stage.cuh).  The areas'
// plane pointers travel in the kernel parameter (AbrPlaneSet, at most kAbrMaxAreas areas), so a job's row of area i
// is one load of rows[job][i] and the walk's gathers stay inside that row.
#include <cstring>
#include <vector>

#include "../../include/holo_spf_lsdb.h"
#include "ospf_abr_rib_cells.h"
#include "route_stage.cuh"

namespace {

using hspf::RibRec;

template <class Planes>
struct AbrRibCell {
    using Rows = hspf::ResultPlanes<Planes>;
    hspf::AbrRibView t;
    hspf::AbrPlaneSet<typename Rows::D, typename Rows::N> s;
    const uint32_t *rows;            // [n_jobs][t.n_areas]
    __device__ __forceinline__ uint32_t status_word(uint32_t j) const {
        return hspf::abr_job_status(s, t.n_areas, rows + (size_t)j * t.n_areas);
    }
    __device__ __forceinline__ bool refused(uint32_t j) const { return status_word(j) != 0; }
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        const hspf::AbrJobPlanes<Planes, typename Rows::D, typename Rows::N> plane{s, rows + (size_t)j * t.n_areas};
        return hspf::abr_rib_cell_eval<Planes>(plane, t, p);
    }
    // next-hop atoms of vertex v in the job's row of area i
    __device__ __forceinline__ uint64_t gather(uint32_t j, uint32_t i, uint32_t v) const {
        if (i >= t.n_areas || v >= s.V[i]) return 0;
        const uint32_t r = rows[(size_t)j * t.n_areas + i];
        return r < s.n_rows[i] ? (uint64_t)s.nh[i][(size_t)r * s.V[i] + v] : 0;
    }
    __device__ static hspf::CellWords empty() { return {0, 0, hspf::kNoRecord}; }
};

// Blocks per SM of every kernel over this walk: their launch bound and their grid.  At the route kernels' 8 the
// cell kernel spills (32 registers); at 4 neither it nor the delta passes do, and on an H100 4 was faster for the
// cell kernel and both delta passes, with byte-identical cells (DESIGN.md §4.4, §6).
constexpr uint32_t kAbrBlocksPerSM = 4;

template <class R>
int make_cell(const hspf_ospfv2_abr_ribtable *t, const R *pl, const uint32_t *n_rows, uint32_t n_jobs,
              const uint32_t *rows, AbrRibCell<hspf::PlanesOf<R>> &cell) {
    if (!t || !t->dev.blob || !pl || !n_rows || (n_jobs && !rows)) return HSPF_E_INVAL;
    const RibRec *recs = static_cast<const RibRec *>(t->dev.contribs);
    cell.t = t->view(t->dev.off, recs, reinterpret_cast<const uint32_t *>(recs + t->recs.size()));
    for (uint32_t i = 0; i < t->n_areas; ++i) {
        typename AbrRibCell<hspf::PlanesOf<R>>::Rows p;
        if (hspf::result_planes(&pl[i], t->n_vertices[i], p) || !p.complete()) return HSPF_E_INVAL;
        cell.s.dist[i] = p.dist; cell.s.hops[i] = p.hops; cell.s.nh[i] = p.nh; cell.s.status[i] = p.status;
        cell.s.V[i] = p.V; cell.s.n_rows[i] = n_rows[i];
    }
    cell.rows = rows;
    return HSPF_OK;
}

template <class R, class Out>
int abr_rib(hspf_ctx *ctx, const hspf_ospfv2_abr_ribtable *t, uint32_t n_jobs, const R *pl, const uint32_t *n_rows,
            const uint32_t *rows, const Out &out) {
    if constexpr (!Out::kDelta)
        if (out.n_gather && !out.gather_area) return HSPF_E_INVAL;     // a gather names the area of its vertex
    AbrRibCell<hspf::PlanesOf<R>> cell{};
    if (const int rc = make_cell(t, pl, n_rows, n_jobs, rows, cell)) return rc;
    return hspf::launch_route_stage<kAbrBlocksPerSM>(ctx, t->dev, cell, n_jobs, cell.t.P, out);
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
    return abr_rib(ctx, t, n_jobs, pl, n_rows, rows,
                   hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out, n_gather, gather_job, gather_area, gather_v,
                                                    gather_nh});
}

int hspf_ospfv2_abr_rib_cells16(hspf_ctx *ctx, const hspf_ospfv2_abr_ribtable *t, uint32_t n_jobs,
                                const hspf_result16 *pl, const uint32_t *n_rows, const uint32_t *rows,
                                hl_ospf_rib_cell *cells, uint32_t *job_status_out, uint32_t n_gather,
                                const uint32_t *gather_job, const uint32_t *gather_area, const uint32_t *gather_v,
                                uint64_t *gather_nh) {
    return abr_rib(ctx, t, n_jobs, pl, n_rows, rows,
                   hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out, n_gather, gather_job, gather_area, gather_v,
                                                    gather_nh});
}

int hspf_ospfv2_abr_rib_delta(hspf_ctx *ctx, const hspf_ospfv2_abr_ribtable *t, uint32_t n_jobs, const hspf_result *pl,
                              const uint32_t *n_rows, const uint32_t *rows, const hl_ospf_rib_cell *base_cells,
                              uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out,
                              hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    return abr_rib(ctx, t, n_jobs, pl, n_rows, rows,
                   hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_ospfv2_abr_rib_delta16(hspf_ctx *ctx, const hspf_ospfv2_abr_ribtable *t, uint32_t n_jobs,
                                const hspf_result16 *pl, const uint32_t *n_rows, const uint32_t *rows,
                                const hl_ospf_rib_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                                hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    return abr_rib(ctx, t, n_jobs, pl, n_rows, rows,
                   hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

}  // extern "C"
