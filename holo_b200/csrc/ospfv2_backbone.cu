// Device stage for the routing table of an OSPF backbone router over what-if jobs inside other areas
// (include/holo_spf_lsdb.h, "backbone router over what-if jobs inside other areas"): update_rib_full at the router,
// for its affected prefixes, with every border's type-3 / Inter-Area-Prefix LSAs in area 0 re-originated for the job.
// The entry points serve OSPFv2 and OSPFv3 tables alike, tables of an internal router of a non-backbone area over
// jobs on the backbone (hspf_ospfv{2,3}_nonbackbone_table_create) and over jobs inside another non-backbone area
// (hspf_ospfv{2,3}_third_area_table_create): the table's marks (version, target area, third area) pick the walk's
// instantiation.
//
// One launch on the ctx stream: one thread per (job, prefix) runs ospf_backbone_cell_eval (ospf_backbone_cells.h)
// over the router's unperturbed area-0 planes (row 0) and the job's row of each border's routing-table cells, and
// the shared cell kernel or the route-delta stage (route_stage.cuh) stores or compares the 24-byte cells.
#include <cstring>
#include <vector>

#include "../../include/holo_spf_lsdb.h"
#include "ospf_backbone_cells.h"
#include "ospf_border_bind.cuh"
#include "route_stage.cuh"

namespace {

using hspf::kOspfBackboneMaxBorders;

template <class Planes, bool kV3>
struct OspfBackboneCell {
    using Rows = hspf::ResultPlanes<Planes>;
    hspf::OspfBackboneView t;
    Rows pl;                                                      // R's area-0 batch; only row 0 is read
    const hl_ospf_rib_cell *cells[kOspfBackboneMaxBorders];       // [n_jobs][K_b] per border
    const uint32_t *status[kOspfBackboneMaxBorders];              // [n_jobs] per border, or NULL
    uint32_t K[kOspfBackboneMaxBorders];
    uint32_t n_borders;
    __device__ __forceinline__ uint32_t status_word(uint32_t j) const {
        uint32_t s = pl.status_word(0);
        for (uint32_t b = 0; b < n_borders; ++b)
            if (status[b]) s |= status[b][j];
        return s;
    }
    __device__ __forceinline__ bool refused(uint32_t j) const { return status_word(j) != 0; }
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        hspf::OspfBorderRows rows;
#pragma unroll
        for (uint32_t b = 0; b < kOspfBackboneMaxBorders; ++b) rows.row[b] = cells[b] + (size_t)j * K[b];
        return hspf::ospf_backbone_cell_eval<kV3>(pl.job(0), t, p, rows);
    }
    __device__ __forceinline__ uint64_t gather(uint32_t, uint32_t, uint32_t) const { return 0; }   // row 0: host side
    __device__ static hspf::CellWords empty() { return {0, 0, hspf::kNoRecord}; }
};

// The walk over a table with type-4 slots (hspf_ospfv2_backbone_asbr_table_create): the same, plus the plane sets the
// slots read, whose rows enter the job's status word.
template <class Planes>
struct OspfBackboneAsbrCell : OspfBackboneCell<Planes, false> {
    using Base = OspfBackboneCell<Planes, false>;
    hspf::OspfAsbrSets<typename Base::Rows::D> sets;
    __device__ __forceinline__ uint32_t status_word(uint32_t j) const {
        return Base::status_word(j) | hspf::asbr_job_status(sets, j);
    }
    __device__ __forceinline__ bool refused(uint32_t j) const { return status_word(j) != 0; }
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        hspf::OspfBorderRows rows;
#pragma unroll
        for (uint32_t b = 0; b < kOspfBackboneMaxBorders; ++b) rows.row[b] = this->cells[b] + (size_t)j * this->K[b];
        const hspf::OspfAsbrPlanes<Planes, typename Base::Rows::D> pl{this->pl.job(0), {sets, j}};
        return hspf::ospf_backbone_cell_eval<false, true>(pl, this->t, p, rows);
    }
};

// The walk over a table whose target area is not area 0 (hspf_ospfv2_nonbackbone_table_create), with or without
// type-4 slots (the cells and delta calls of both kinds take it): the borders also advertise their inter-area routes, and a plane set may be a border's area 0.
template <class Planes>
struct OspfNonBackboneCell : OspfBackboneAsbrCell<Planes> {
    using Base = OspfBackboneCell<Planes, false>;
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        hspf::OspfBorderRows rows;
#pragma unroll
        for (uint32_t b = 0; b < kOspfBackboneMaxBorders; ++b) rows.row[b] = this->cells[b] + (size_t)j * this->K[b];
        const hspf::OspfAsbrPlanes<Planes, typename Base::Rows::D> pl{this->pl.job(0), {this->sets, j}};
        return hspf::ospf_backbone_cell_eval<false, true, true>(pl, this->t, p, rows);
    }
};

// The same over an OSPFv3 table (hspf_ospfv3_nonbackbone_table_create): slot winners carry prefix options, and a
// plane set is a border's area 0 read for an Inter-Area-Router slot.  A type of its own, so that the OSPFv2 kernels
// above keep their instantiations.
template <class Planes>
struct OspfNonBackboneV3Cell : OspfBackboneAsbrCell<Planes> {
    using Base = OspfBackboneCell<Planes, false>;
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        hspf::OspfBorderRows rows;
#pragma unroll
        for (uint32_t b = 0; b < kOspfBackboneMaxBorders; ++b) rows.row[b] = this->cells[b] + (size_t)j * this->K[b];
        const hspf::OspfAsbrPlanes<Planes, typename Base::Rows::D> pl{this->pl.job(0), {this->sets, j}};
        return hspf::ospf_backbone_cell_eval<true, true, true>(pl, this->t, p, rows);
    }
};

// The walk over an OSPFv3 table of area 0 with Inter-Area-Router slots (hspf_ospfv3_backbone_asbr_table_create): slot
// winners carry prefix options.  A type of its own, so that the kernels above keep their instantiations.
template <class Planes>
struct OspfBackboneAsbrV3Cell : OspfBackboneAsbrCell<Planes> {
    using Base = OspfBackboneCell<Planes, false>;
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        hspf::OspfBorderRows rows;
#pragma unroll
        for (uint32_t b = 0; b < kOspfBackboneMaxBorders; ++b) rows.row[b] = this->cells[b] + (size_t)j * this->K[b];
        const hspf::OspfAsbrPlanes<Planes, typename Base::Rows::D> pl{this->pl.job(0), {this->sets, j}};
        return hspf::ospf_backbone_cell_eval<true, true, false>(pl, this->t, p, rows);
    }
};

// The walk over a third-area table with chain slots (hspf_ospfv2_third_area_table_create): the kNonBackbone walk, with
// each chain slot reading its border's entries of the job, whose status words enter the job's.  A type of its own, so
// that the kernels above keep their instantiations.
template <class Planes>
struct OspfThirdAreaCell : OspfBackboneCell<Planes, false> {
    using Base = OspfBackboneCell<Planes, false>;
    hspf::OspfChainSet chain;
    __device__ __forceinline__ uint32_t status_word(uint32_t j) const {
        uint32_t s = Base::status_word(j);
        for (uint32_t b = 0; b < this->n_borders; ++b)
            if (chain.status[b]) s |= chain.status[b][j];
        return s;
    }
    __device__ __forceinline__ bool refused(uint32_t j) const { return status_word(j) != 0; }
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        hspf::OspfBorderRows rows;
#pragma unroll
        for (uint32_t b = 0; b < kOspfBackboneMaxBorders; ++b) rows.row[b] = this->cells[b] + (size_t)j * this->K[b];
        const hspf::OspfThirdAreaPlanes<Planes> pl{this->pl.job(0), {chain, j}};
        return hspf::ospf_backbone_cell_eval<false, true, true>(pl, this->t, p, rows);
    }
};

// The walk over an OSPFv3 third-area table (hspf_ospfv3_third_area_table_create), with or without chain slots: the C
// cells' inter-area winners may be OSPFv3 slot winners, whose options ride in their low byte (kSlotWinners), and R's
// slot winners carry those options.  A type of its own, so that the kernels above keep their instantiations.
template <class Planes>
struct OspfThirdAreaV3Cell : OspfThirdAreaCell<Planes> {
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        hspf::OspfBorderRows rows;
#pragma unroll
        for (uint32_t b = 0; b < kOspfBackboneMaxBorders; ++b) rows.row[b] = this->cells[b] + (size_t)j * this->K[b];
        const hspf::OspfThirdAreaPlanes<Planes> pl{this->pl.job(0), {this->chain, j}};
        return hspf::ospf_backbone_cell_eval<true, true, true, true>(pl, this->t, p, rows);
    }
};

// Blocks per SM of the kernels over this walk: their launch bound and their grid (DESIGN.md §4.4, §6), for OSPFv2
// and for OSPFv3 tables, for OSPFv2 and OSPFv3 tables with type-4 / Inter-Area-Router slots, for OSPFv2 and OSPFv3
// tables of a non-backbone target area, for OSPFv2 third-area tables with chain slots, and for OSPFv3 third-area
// tables.
constexpr uint32_t kBackboneBlocksPerSM = 4;
constexpr uint32_t kBackboneV3BlocksPerSM = 4;
constexpr uint32_t kBackboneAsbrBlocksPerSM = 4;
constexpr uint32_t kBackboneAsbrV3BlocksPerSM = 4;
constexpr uint32_t kNonBackboneBlocksPerSM = 4;
constexpr uint32_t kNonBackboneV3BlocksPerSM = 4;
constexpr uint32_t kThirdAreaBlocksPerSM = 4;
constexpr uint32_t kThirdAreaV3BlocksPerSM = 4;

template <class R, bool kV3>
int make_cell(const hspf_ospfv2_backbone_table *t, const R *planes, const hl_ospf_rib_cell *const *border_cells,
              const uint32_t *const *border_status, OspfBackboneCell<hspf::PlanesOf<R>, kV3> &cell) {
    if (!t || !t->dev.blob || !border_cells) return HSPF_E_INVAL;
    if (hspf::result_planes(planes, t->n_vertices, cell.pl) || !cell.pl.complete()) return HSPF_E_INVAL;
    if (const int rc = hspf::bind_ospf_borders(*t, border_cells, border_status, cell)) return rc;
    cell.t = t->view(t->dev.off, static_cast<const hspf::RibRec *>(t->dev.contribs));
    return HSPF_OK;
}

template <bool kV3, class R, class Out>
int version(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs, const R *planes,
            const hl_ospf_rib_cell *const *border_cells, const uint32_t *const *border_status, const Out &out) {
    constexpr uint32_t kBlocks = kV3 ? kBackboneV3BlocksPerSM : kBackboneBlocksPerSM;
    OspfBackboneCell<hspf::PlanesOf<R>, kV3> cell{};
    if (const int rc = make_cell(t, planes, border_cells, border_status, cell)) return rc;
    return hspf::launch_route_stage<kBlocks>(ctx, t->dev, cell, n_jobs, t->P(), out);
}

// The launch of a walk over a table with type-4 / Inter-Area-Router slots or of a non-backbone target area (Cell):
// the cell above plus the plane sets the slots name.
template <class Cell, uint32_t kBlocks, class R, class Out>
int asbr_as(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs, const R *planes,
            const hl_ospf_rib_cell *const *border_cells, const uint32_t *const *border_status,
            const R *const *border_planes, const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
            const Out &out) {
    Cell cell{};
    if (const int rc = make_cell(t, planes, border_cells, border_status, cell)) return rc;
    if (const int rc = hspf::bind_ospf_asbr_sets(*t, border_planes, border_n_rows, border_rows, n_jobs, cell))
        return rc;
    return hspf::launch_route_stage<kBlocks>(ctx, t->dev, cell, n_jobs, t->P(), out);
}

// a table of a non-backbone target area: the walk of its version
template <class R, class Out>
int nonbackbone(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs, const R *planes,
                const hl_ospf_rib_cell *const *border_cells, const uint32_t *const *border_status,
                const R *const *border_planes, const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                const Out &out) {
    using P = hspf::PlanesOf<R>;
    return t->v3 ? asbr_as<OspfNonBackboneV3Cell<P>, kNonBackboneV3BlocksPerSM>(
                       ctx, t, n_jobs, planes, border_cells, border_status, border_planes, border_n_rows, border_rows, out)
                 : asbr_as<OspfNonBackboneCell<P>, kNonBackboneBlocksPerSM>(
                       ctx, t, n_jobs, planes, border_cells, border_status, border_planes, border_n_rows, border_rows, out);
}

// The launch of a third-area walk (Cell) over each border's entries (border_entries[b] u32 [n_jobs][G_b], NULL allowed
// for a border with no group; the array may be NULL for a table without chain slots, which reads no entries).
template <class Cell, uint32_t kBlocks, class R, class Out>
int chain_as(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs, const R *planes,
             const hl_ospf_rib_cell *const *border_cells, const uint32_t *const *border_status,
             const uint32_t *const *border_entries, const uint32_t *const *border_entry_status, const Out &out) {
    Cell cell{};
    if (const int rc = make_cell(t, planes, border_cells, border_status, cell)) return rc;
    if (t->n_asbr_slots && !border_entries) return HSPF_E_INVAL;
    for (uint32_t b = 0; b < kOspfBackboneMaxBorders; ++b) {
        cell.chain.entries[b] = nullptr; cell.chain.status[b] = nullptr; cell.chain.G[b] = 0;
        if (b >= t->n_borders || !t->n_asbr_slots) continue;
        cell.chain.G[b] = (uint32_t)t->third[b]->asbr_group.size();
        cell.chain.entries[b] = border_entries[b];
        cell.chain.status[b] = border_entry_status ? border_entry_status[b] : nullptr;
        if (cell.chain.G[b] && (!border_entries[b] || (reinterpret_cast<uintptr_t>(border_entries[b]) & 3u)))
            return HSPF_E_INVAL;
    }
    return hspf::launch_route_stage<kBlocks>(ctx, t->dev, cell, n_jobs, t->P(), out);
}

// A third-area table.  OSPFv2: with chain slots the OspfThirdAreaCell walk, else the plain kNonBackbone walk.  OSPFv3:
// the OspfThirdAreaV3Cell walk, with or without chain slots (the kNonBackbone walks cannot read C's slot winners).
template <class R, class Out>
int third_area(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs, const R *planes,
               const hl_ospf_rib_cell *const *border_cells, const uint32_t *const *border_status,
               const uint32_t *const *border_entries, const uint32_t *const *border_entry_status, const Out &out) {
    if (!t || !t->third_area) return HSPF_E_INVAL;
    using P = hspf::PlanesOf<R>;
    if (t->v3)
        return chain_as<OspfThirdAreaV3Cell<P>, kThirdAreaV3BlocksPerSM>(
            ctx, t, n_jobs, planes, border_cells, border_status, border_entries, border_entry_status, out);
    if (!t->n_asbr_slots)
        return nonbackbone<R>(ctx, t, n_jobs, planes, border_cells, border_status, nullptr, nullptr, nullptr, out);
    return chain_as<OspfThirdAreaCell<P>, kThirdAreaBlocksPerSM>(ctx, t, n_jobs, planes, border_cells, border_status,
                                                                 border_entries, border_entry_status, out);
}

// the walk of the table's version and target area; a table with type-4 slots is backbone_asbr's
template <class R, class Out>
int backbone(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs, const R *planes,
             const hl_ospf_rib_cell *const *border_cells, const uint32_t *const *border_status, const Out &out) {
    // an OSPFv3 third-area table's C cells hold slot winners, which only the third-area calls read
    if (!t || t->n_asbr_slots || (t->third_area && t->v3)) return HSPF_E_INVAL;
    if (t->area_id)
        return nonbackbone<R>(ctx, t, n_jobs, planes, border_cells, border_status, nullptr, nullptr, nullptr, out);
    return t->v3 ? version<true>(ctx, t, n_jobs, planes, border_cells, border_status, out)
                 : version<false>(ctx, t, n_jobs, planes, border_cells, border_status, out);
}

// A table without type-4 slots takes backbone (NULL border planes allowed).  An OSPFv3 table of area 0 is refused
// unless hspf_ospfv3_backbone_asbr_table_create made it.
template <class R, class Out>
int backbone_asbr(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs, const R *planes,
                  const hl_ospf_rib_cell *const *border_cells, const uint32_t *const *border_status,
                  const R *const *border_planes, const uint32_t *const *border_n_rows,
                  const uint32_t *const *border_rows, const Out &out) {
    // a third-area table's type-4 slots are chain slots, and an OSPFv3 one's C cells hold slot winners: only the
    // third-area calls read those
    if (!t || (t->v3 && !t->area_id && !t->asbr) || (t->third_area && (t->n_asbr_slots || t->v3)))
        return HSPF_E_INVAL;
    if (t->area_id)
        return nonbackbone(ctx, t, n_jobs, planes, border_cells, border_status, border_planes, border_n_rows,
                           border_rows, out);
    if (!t->n_asbr_slots) return backbone(ctx, t, n_jobs, planes, border_cells, border_status, out);
    using P = hspf::PlanesOf<R>;
    return t->v3 ? asbr_as<OspfBackboneAsbrV3Cell<P>, kBackboneAsbrV3BlocksPerSM>(
                       ctx, t, n_jobs, planes, border_cells, border_status, border_planes, border_n_rows, border_rows, out)
                 : asbr_as<OspfBackboneAsbrCell<P>, kBackboneAsbrBlocksPerSM>(
                       ctx, t, n_jobs, planes, border_cells, border_status, border_planes, border_n_rows, border_rows, out);
}

}  // namespace

extern "C" {

int hspf_ospfv2_backbone_table_upload(hspf_ctx *ctx, hspf_ospfv2_backbone_table *t) {
    if (!t) return HSPF_E_INVAL;
    return hspf::upload_route_table(ctx, t->dev, t->words, t->recs.data(), t->recs.size() * sizeof(hspf::RibRec));
}

int hspf_ospfv2_backbone_cells(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                               const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                               const uint32_t *const *border_status, uint32_t *job_status_out, hl_ospf_rib_cell *cells) {
    return backbone(ctx, t, n_jobs, planes, border_cells, border_status,
                    hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out});
}

int hspf_ospfv2_backbone_cells16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                 const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                 const uint32_t *const *border_status, uint32_t *job_status_out, hl_ospf_rib_cell *cells) {
    return backbone(ctx, t, n_jobs, planes, border_cells, border_status,
                    hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out});
}

int hspf_ospfv2_backbone_delta(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                               const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                               const uint32_t *const *border_status, const hl_ospf_rib_cell *base_cells, uint32_t n_base,
                               const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records,
                               uint64_t cap, uint64_t *n_records) {
    return backbone(ctx, t, n_jobs, planes, border_cells, border_status,
                    hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_ospfv2_backbone_delta16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                 const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                 const uint32_t *const *border_status, const hl_ospf_rib_cell *base_cells,
                                 uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out,
                                 hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    return backbone(ctx, t, n_jobs, planes, border_cells, border_status,
                    hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_ospfv2_backbone_asbr_cells(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                    const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                                    const uint32_t *const *border_status, const hspf_result *const *border_planes,
                                    const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                    uint32_t *job_status_out, hl_ospf_rib_cell *cells) {
    return backbone_asbr(ctx, t, n_jobs, planes, border_cells, border_status, border_planes, border_n_rows, border_rows,
                         hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out});
}

int hspf_ospfv2_backbone_asbr_cells16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                      const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                      const uint32_t *const *border_status, const hspf_result16 *const *border_planes,
                                      const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                      uint32_t *job_status_out, hl_ospf_rib_cell *cells) {
    return backbone_asbr(ctx, t, n_jobs, planes, border_cells, border_status, border_planes, border_n_rows, border_rows,
                         hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out});
}

int hspf_ospfv2_backbone_asbr_delta(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                    const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                                    const uint32_t *const *border_status, const hspf_result *const *border_planes,
                                    const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                    const hl_ospf_rib_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                                    hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                                    uint64_t *n_records) {
    return backbone_asbr(ctx, t, n_jobs, planes, border_cells, border_status, border_planes, border_n_rows, border_rows,
                         hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_ospfv2_backbone_asbr_delta16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                      const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                      const uint32_t *const *border_status, const hspf_result16 *const *border_planes,
                                      const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                      const hl_ospf_rib_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                                      hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                                      uint64_t *n_records) {
    return backbone_asbr(ctx, t, n_jobs, planes, border_cells, border_status, border_planes, border_n_rows, border_rows,
                         hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_ospfv2_third_area_cells(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                 const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                                 const uint32_t *const *border_status, const uint32_t *const *border_entries,
                                 const uint32_t *const *border_entry_status, uint32_t *job_status_out,
                                 hl_ospf_rib_cell *cells) {
    return third_area(ctx, t, n_jobs, planes, border_cells, border_status, border_entries, border_entry_status,
                      hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out});
}

int hspf_ospfv2_third_area_cells16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                   const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                   const uint32_t *const *border_status, const uint32_t *const *border_entries,
                                   const uint32_t *const *border_entry_status, uint32_t *job_status_out,
                                   hl_ospf_rib_cell *cells) {
    return third_area(ctx, t, n_jobs, planes, border_cells, border_status, border_entries, border_entry_status,
                      hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out});
}

int hspf_ospfv2_third_area_delta(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                 const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                                 const uint32_t *const *border_status, const uint32_t *const *border_entries,
                                 const uint32_t *const *border_entry_status, const hl_ospf_rib_cell *base_cells,
                                 uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out,
                                 hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    return third_area(ctx, t, n_jobs, planes, border_cells, border_status, border_entries, border_entry_status,
                      hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_ospfv2_third_area_delta16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                   const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                   const uint32_t *const *border_status, const uint32_t *const *border_entries,
                                   const uint32_t *const *border_entry_status, const hl_ospf_rib_cell *base_cells,
                                   uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out,
                                   hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    return third_area(ctx, t, n_jobs, planes, border_cells, border_status, border_entries, border_entry_status,
                      hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

}  // extern "C"
