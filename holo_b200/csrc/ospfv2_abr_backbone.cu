// Device stage for the routing table of an OSPF area border router over what-if jobs inside an area it is not
// attached to (include/holo_spf_lsdb.h, hspf_ospfv2_abr_backbone_table_create / hspf_ospfv3_abr_backbone_table_create):
// update_rib_full at the router, for its affected prefixes, with every border's type-3 / Inter-Area-Prefix and type-4
// / Inter-Area-Router LSAs in area 0 re-originated for the job.  The entry points serve OSPFv2 and OSPFv3 tables
// alike: the table's version mark (abr->v3) picks the walk's instantiation.
//
// One launch on the ctx stream: one thread per (job, prefix) runs abr_rib_cell_eval with kSlots (ospf_abr_rib_cells.h,
// ospf_backbone_cells.h: AbrBorderSlots) over the router's row 0 of every area, the job's row of each border's
// routing-table cells and the job's rows of the plane sets its type-4 slots read; the shared cell kernel or the
// route-delta stage (route_stage.cuh) stores or compares the 24-byte cells.
#include <cstring>
#include <vector>

#include "../../include/holo_spf_lsdb.h"
#include "ospf_backbone_cells.h"
#include "ospf_border_bind.cuh"
#include "route_stage.cuh"

namespace {

using hspf::kOspfBackboneMaxBorders;

template <class Planes, bool kV3>
struct OspfAbrBackboneCellOf {
    using Rows = hspf::ResultPlanes<Planes>;
    using D = typename Rows::D;
    using N = typename Rows::N;
    hspf::AbrRibView t;
    hspf::AbrPlaneSet<D, N> s;                                    // R's planes of each area; only row 0 is read
    hspf::OspfAsbrSets<D> sets;                                   // the plane sets the type-4 slots read
    const hl_ospf_rib_cell *cells[kOspfBackboneMaxBorders];       // [n_jobs][K_b] per border
    const uint32_t *status[kOspfBackboneMaxBorders];              // [n_jobs] per border, or NULL
    uint32_t K[kOspfBackboneMaxBorders];
    const uint32_t *border;                                       // the table's border words
    uint32_t n_borders, n_recs;
    __device__ __forceinline__ uint32_t status_word(uint32_t j) const {
        uint32_t st = hspf::abr_row0_status(s, t.n_areas) | hspf::asbr_job_status(sets, j);
        for (uint32_t b = 0; b < n_borders; ++b)
            if (status[b]) st |= status[b][j];
        return st;
    }
    __device__ __forceinline__ bool refused(uint32_t j) const { return status_word(j) != 0; }
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        hspf::AbrBorderSlots<kV3> sl;
#pragma unroll
        for (uint32_t b = 0; b < kOspfBackboneMaxBorders; ++b) sl.rows.row[b] = cells[b] + (size_t)j * K[b];
        sl.border = border;
        sl.n_recs = n_recs;
        const hspf::AbrRow0Planes<Planes, D, N> plane{s, {sets, j}};
        return hspf::abr_rib_cell_eval<Planes, true>(plane, t, p, sl);
    }
    __device__ __forceinline__ uint64_t gather(uint32_t, uint32_t, uint32_t) const { return 0; }   // row 0: host side
    __device__ static hspf::CellWords empty() { return {0, 0, hspf::kNoRecord}; }
};

// The walk over an OSPFv2 table, and over an OSPFv3 one, whose slot winners carry prefix options.  Types of their own,
// so that each has its own kernels and launch bound.
template <class Planes>
struct OspfAbrBackboneCell : OspfAbrBackboneCellOf<Planes, false> {};
template <class Planes>
struct OspfAbrBackboneV3Cell : OspfAbrBackboneCellOf<Planes, true> {};

// Blocks per SM of the kernels over this walk: their launch bound and their grid (DESIGN.md §4.4, §6), for OSPFv2 and
// for OSPFv3 tables.
constexpr uint32_t kAbrBackboneBlocksPerSM = 4;
constexpr uint32_t kAbrBackboneV3BlocksPerSM = 4;

// R's planes, the borders' cells and status words, and the plane sets the type-4 slots name, from each border's
// planes, row counts and rows (border_planes[b][i], border_n_rows[b][i], border_rows[b]), which may be NULL when the
// table has no type-4 slot.
template <class R, class Cell>
int make_cell(const hspf_ospfv2_abr_backbone_table *t, const R *planes, const hl_ospf_rib_cell *const *border_cells,
              const uint32_t *const *border_status, const R *const *border_planes, const uint32_t *const *border_n_rows,
              const uint32_t *const *border_rows, uint32_t n_jobs, Cell &cell) {
    if (!t || !t->abr || !t->dev.blob || !planes || !border_cells) return HSPF_E_INVAL;
    if (const int rc = hspf::bind_abr_row0_planes(*t->abr, planes, cell.s)) return rc;
    if (const int rc = hspf::bind_ospf_borders(*t, border_cells, border_status, cell)) return rc;
    if (const int rc = hspf::bind_ospf_asbr_sets(*t, border_planes, border_n_rows, border_rows, n_jobs, cell))
        return rc;
    cell.n_recs = t->n_recs();
    cell.t = t->view(t->dev.off, static_cast<const hspf::RibRec *>(t->dev.contribs));
    cell.border = t->dev.off + t->border_at();
    return HSPF_OK;
}

template <class Cell, uint32_t kBlocks, class R, class Out>
int abr_backbone_as(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs, const R *planes,
                    const hl_ospf_rib_cell *const *border_cells, const uint32_t *const *border_status,
                    const R *const *border_planes, const uint32_t *const *border_n_rows,
                    const uint32_t *const *border_rows, const Out &out) {
    Cell cell{};
    if (const int rc = make_cell(t, planes, border_cells, border_status, border_planes, border_n_rows, border_rows,
                                 n_jobs, cell))
        return rc;
    return hspf::launch_route_stage<kBlocks>(ctx, t->dev, cell, n_jobs, t->P(), out);
}

// the walk of the table's version
template <class R, class Out>
int abr_backbone(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs, const R *planes,
                 const hl_ospf_rib_cell *const *border_cells, const uint32_t *const *border_status,
                 const R *const *border_planes, const uint32_t *const *border_n_rows,
                 const uint32_t *const *border_rows, const Out &out) {
    if (!t || !t->abr) return HSPF_E_INVAL;
    using P = hspf::PlanesOf<R>;
    return t->abr->v3 ? abr_backbone_as<OspfAbrBackboneV3Cell<P>, kAbrBackboneV3BlocksPerSM>(
                            ctx, t, n_jobs, planes, border_cells, border_status, border_planes, border_n_rows,
                            border_rows, out)
                      : abr_backbone_as<OspfAbrBackboneCell<P>, kAbrBackboneBlocksPerSM>(
                            ctx, t, n_jobs, planes, border_cells, border_status, border_planes, border_n_rows,
                            border_rows, out);
}

// ---- C's ASBR entries per job (hspf_ospfv2_abr_backbone_asbr_entries) ----------------------------------------------
// C's area-0 planes (row 0) and the plane sets its type-4 slots read; group k's entry record is group_rec[k].
template <class D, class N>
struct AbrEntryArgs {
    hspf::AbrPlaneSet<D, N> s;
    hspf::OspfAsbrSets<D> sets;
    const hspf::RibRec *recs;
    const uint32_t *group_rec;
    uint32_t n_areas, area0, G;
};

// One thread per (job, group), then per job its status word: C's row-0 words and the job's rows' words.  A job with a
// non-zero word gets kOspfNoEntry.
template <class Planes, class D, class N>
__global__ void __launch_bounds__(hspf::kRouteThreads)
abr_asbr_entries_kernel(const AbrEntryArgs<D, N> a, uint32_t n_jobs, uint32_t *__restrict__ status_out,
                        uint32_t *__restrict__ entries) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x, first = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t row0 = hspf::abr_row0_status(a.s, a.n_areas);
    if (status_out)
        for (uint64_t j = first; j < n_jobs; j += stride) status_out[j] = row0 | hspf::asbr_job_status(a.sets, (uint32_t)j);
    const uint64_t total = (uint64_t)n_jobs * a.G;
    for (uint64_t idx = first; idx < total; idx += stride) {
        const uint32_t j = (uint32_t)(idx / a.G), k = (uint32_t)(idx - (uint64_t)j * a.G);
        uint32_t m = hspf::kOspfNoEntry;
        if (!(row0 | hspf::asbr_job_status(a.sets, j))) {
            const Planes pl{a.s.dist[a.area0], a.s.hops[a.area0], a.s.nh[a.area0]};
            const hspf::OspfAsbrJob<Planes, D> asbr{a.sets, j};
            m = hspf::abr_asbr_entry(pl, asbr, a.recs, __ldg(a.group_rec + k));
        }
        entries[idx] = m;
    }
}

// Either version's table (v3: the version the call takes): an OSPFv3 table's Inter-Area-Router ranges hold the records
// of OSPFv2's type-4 ranges, so one instantiation of the kernel serves both.
template <class R>
int asbr_entries(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs, const R *planes,
                 const R *const *border_planes, const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                 uint32_t *job_status_out, uint32_t *entries, bool v3) {
    using P = hspf::PlanesOf<R>;
    using Rows = hspf::ResultPlanes<P>;
    if (!ctx || !t || !t->abr || t->abr->v3 != v3 || !t->dev.blob || !planes) return HSPF_E_INVAL;
    const uint32_t G = (uint32_t)t->asbr_group.size();
    if ((n_jobs && G && !entries) || (reinterpret_cast<uintptr_t>(entries) & 3u) ||
        (reinterpret_cast<uintptr_t>(job_status_out) & 3u) || (G && !t->entry_dev.blob))
        return HSPF_E_INVAL;
    AbrEntryArgs<typename Rows::D, typename Rows::N> args{};
    if (const int rc = hspf::bind_abr_row0_planes(*t->abr, planes, args.s)) return rc;
    if (const int rc = hspf::bind_ospf_asbr_sets(*t, border_planes, border_n_rows, border_rows, n_jobs, args)) return rc;
    args.recs = static_cast<const hspf::RibRec *>(t->dev.contribs);
    args.group_rec = t->entry_dev.off;
    args.n_areas = t->abr->n_areas; args.area0 = t->area0; args.G = G;
    const uint64_t items = std::max<uint64_t>((uint64_t)n_jobs * G, job_status_out ? n_jobs : 0u);
    if (items == 0) return HSPF_OK;
    uint32_t blocks = 0;
    if (const int rc = hspf::route_grid(ctx, t->dev, items, hspf::kRouteBlocksPerSM, blocks)) return rc;
    abr_asbr_entries_kernel<P><<<blocks, hspf::kRouteThreads, 0, static_cast<cudaStream_t>(hspf_stream(ctx))>>>(
        args, n_jobs, job_status_out, entries);
    if (cudaGetLastError() != cudaSuccess) return HSPF_E_CUDA;
    hspf_note_launches(ctx, 1);
    return HSPF_OK;
}

}  // namespace

extern "C" {

int hspf_ospfv2_abr_backbone_table_upload(hspf_ctx *ctx, hspf_ospfv2_abr_backbone_table *t) {
    if (!t || !t->abr) return HSPF_E_INVAL;
    const int rc = hspf::upload_route_table(ctx, t->dev, t->words, t->abr->recs.data(),
                                            t->abr->recs.size() * sizeof(hspf::RibRec));
    if (rc || t->asbr_group.empty()) return rc;
    // the entry record of each group with type-4 slots, for hspf_ospfv{2,3}_abr_backbone_asbr_entries
    std::vector<uint32_t> rec;
    for (uint32_t g : t->asbr_group) rec.push_back(t->abr->ext_end + g * t->abr->n_areas + t->area0);
    return hspf::upload_route_table(ctx, t->entry_dev, rec, nullptr, 0);
}

int hspf_ospfv2_abr_backbone_asbr_entries(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                          const hspf_result *planes, const hspf_result *const *border_planes,
                                          const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                          uint32_t *job_status_out, uint32_t *entries) {
    return asbr_entries(ctx, t, n_jobs, planes, border_planes, border_n_rows, border_rows, job_status_out, entries,
                        false);
}

int hspf_ospfv2_abr_backbone_asbr_entries16(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                            const hspf_result16 *planes, const hspf_result16 *const *border_planes,
                                            const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                            uint32_t *job_status_out, uint32_t *entries) {
    return asbr_entries(ctx, t, n_jobs, planes, border_planes, border_n_rows, border_rows, job_status_out, entries,
                        false);
}

int hspf_ospfv3_abr_backbone_asbr_entries(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                          const hspf_result *planes, const hspf_result *const *border_planes,
                                          const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                          uint32_t *job_status_out, uint32_t *entries) {
    return asbr_entries(ctx, t, n_jobs, planes, border_planes, border_n_rows, border_rows, job_status_out, entries,
                        true);
}

int hspf_ospfv3_abr_backbone_asbr_entries16(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                            const hspf_result16 *planes, const hspf_result16 *const *border_planes,
                                            const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                            uint32_t *job_status_out, uint32_t *entries) {
    return asbr_entries(ctx, t, n_jobs, planes, border_planes, border_n_rows, border_rows, job_status_out, entries,
                        true);
}

int hspf_ospfv2_abr_backbone_cells(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                   const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                                   const uint32_t *const *border_status, const hspf_result *const *border_planes,
                                   const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                   uint32_t *job_status_out, hl_ospf_rib_cell *cells) {
    return abr_backbone(ctx, t, n_jobs, planes, border_cells, border_status, border_planes, border_n_rows, border_rows,
                        hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out});
}

int hspf_ospfv2_abr_backbone_cells16(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                     const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                     const uint32_t *const *border_status, const hspf_result16 *const *border_planes,
                                     const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                     uint32_t *job_status_out, hl_ospf_rib_cell *cells) {
    return abr_backbone(ctx, t, n_jobs, planes, border_cells, border_status, border_planes, border_n_rows, border_rows,
                        hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out});
}

int hspf_ospfv2_abr_backbone_delta(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                   const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                                   const uint32_t *const *border_status, const hspf_result *const *border_planes,
                                   const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                   const hl_ospf_rib_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                                   hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                                   uint64_t *n_records) {
    return abr_backbone(ctx, t, n_jobs, planes, border_cells, border_status, border_planes, border_n_rows, border_rows,
                        hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_ospfv2_abr_backbone_delta16(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                     const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                     const uint32_t *const *border_status, const hspf_result16 *const *border_planes,
                                     const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                     const hl_ospf_rib_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                                     hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                                     uint64_t *n_records) {
    return abr_backbone(ctx, t, n_jobs, planes, border_cells, border_status, border_planes, border_n_rows, border_rows,
                        hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

}  // extern "C"
