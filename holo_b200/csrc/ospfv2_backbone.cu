// Device stage for the routing table of an OSPF backbone router over what-if jobs inside other areas
// (include/holo_spf_lsdb.h, "backbone router over what-if jobs inside other areas"): update_rib_full at the router,
// for its affected prefixes, with every border's type-3 / Inter-Area-Prefix LSAs in area 0 re-originated for the job.
// The entry points serve OSPFv2 and OSPFv3 tables alike, tables of an internal router of a non-backbone area over
// jobs on the backbone (hspf_ospfv{2,3}_nonbackbone_table_create) and over jobs inside another non-backbone area
// (hspf_ospfv{2,3}_third_area_table_create): the call's family and the table's marks (version, target area, slots,
// third area) pick the walk (pick_walk).
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

// What every walk reads: R's area-0 planes and each border's routing-table cells.
template <class Planes>
struct OspfBackboneCore {
    hspf::OspfBackboneView t;
    hspf::ResultPlanes<Planes> pl;                                // R's area-0 batch; only row 0 is read
    const hl_ospf_rib_cell *cells[kOspfBackboneMaxBorders];       // [n_jobs][K_b] per border
    const uint32_t *status[kOspfBackboneMaxBorders];              // [n_jobs] per border, or NULL
    uint32_t K[kOspfBackboneMaxBorders];
    uint32_t n_borders;
};

// A call's arguments for a side input, NULL where its family takes none: the asbr calls' plane sets per border
// (border_planes[b][i], border_n_rows[b][i], border_rows[b]) and the third-area calls' entries per border
// (border_entries[b] u32 [n_jobs][G_b], border_entry_status[b] [n_jobs]).
template <class R>
struct SideArgs {
    const R *const *border_planes;
    const uint32_t *const *border_n_rows, *const *border_rows;
    const uint32_t *const *border_entries, *const *border_entry_status;
};

// A walk's side input: what rides with R's planes of the job into ospf_backbone_cell_eval, and what it ORs into the
// job's status word after the borders' words.  The plain walks have none.
template <class Planes>
struct NoSide {
    template <class R>
    int bind(const hspf_ospfv2_backbone_table &, const SideArgs<R> &, uint32_t) { return HSPF_OK; }
    __device__ __forceinline__ uint32_t or_status(const OspfBackboneCore<Planes> &, uint32_t s, uint32_t) const {
        return s;
    }
    __device__ __forceinline__ Planes planes(const Planes &pl, uint32_t) const { return pl; }
};

// The plane sets the type-4 / Inter-Area-Router slots read; the job's row of each enters its status word.
template <class Planes>
struct AsbrSide {
    using D = typename hspf::ResultPlanes<Planes>::D;
    hspf::OspfAsbrSets<D> sets;
    template <class R>
    int bind(const hspf_ospfv2_backbone_table &t, const SideArgs<R> &a, uint32_t n_jobs) {
        return hspf::bind_ospf_asbr_sets(t, a.border_planes, a.border_n_rows, a.border_rows, n_jobs, *this);
    }
    __device__ __forceinline__ uint32_t or_status(const OspfBackboneCore<Planes> &, uint32_t s, uint32_t j) const {
        return s | hspf::asbr_job_status(sets, j);
    }
    __device__ __forceinline__ hspf::OspfAsbrPlanes<Planes, D> planes(const Planes &pl, uint32_t j) const {
        return {pl, {sets, j}};
    }
};

// Each border's entries of the job, which its chain slots read (a third-area table); their status words enter the
// job's.  A border with no group may have NULL entries, and a table without chain slots reads none (the array may be
// NULL).
template <class Planes>
struct ChainSide {
    hspf::OspfChainSet chain;
    template <class R>
    int bind(const hspf_ospfv2_backbone_table &t, const SideArgs<R> &a, uint32_t) {
        if (t.n_asbr_slots && !a.border_entries) return HSPF_E_INVAL;
        for (uint32_t b = 0; b < kOspfBackboneMaxBorders; ++b) {
            chain.entries[b] = nullptr; chain.status[b] = nullptr; chain.G[b] = 0;
            if (b >= t.n_borders || !t.n_asbr_slots) continue;
            chain.G[b] = (uint32_t)t.third[b]->asbr_group.size();
            chain.entries[b] = a.border_entries[b];
            chain.status[b] = a.border_entry_status ? a.border_entry_status[b] : nullptr;
            if (chain.G[b] && (!a.border_entries[b] || (reinterpret_cast<uintptr_t>(a.border_entries[b]) & 3u)))
                return HSPF_E_INVAL;
        }
        return HSPF_OK;
    }
    __device__ __forceinline__ uint32_t or_status(const OspfBackboneCore<Planes> &c, uint32_t s, uint32_t j) const {
        for (uint32_t b = 0; b < c.n_borders; ++b)
            if (chain.status[b]) s |= chain.status[b][j];
        return s;
    }
    __device__ __forceinline__ hspf::OspfThirdAreaPlanes<Planes> planes(const Planes &pl, uint32_t j) const {
        return {pl, {chain, j}};
    }
};

// Blocks per SM of each walk's kernels: their launch bound and their grid (DESIGN.md §4.4, §6).
constexpr uint32_t kBackboneBlocksPerSM = 4;
constexpr uint32_t kBackboneV3BlocksPerSM = 4;
constexpr uint32_t kBackboneAsbrBlocksPerSM = 4;
constexpr uint32_t kBackboneAsbrV3BlocksPerSM = 4;
constexpr uint32_t kNonBackboneBlocksPerSM = 4;
constexpr uint32_t kNonBackboneV3BlocksPerSM = 4;
constexpr uint32_t kThirdAreaBlocksPerSM = 4;
constexpr uint32_t kThirdAreaV3BlocksPerSM = 4;

// A walk: the flags it runs ospf_backbone_cell_eval with, its side input and its kernels' launch bound.
template <bool V3, bool Asbr, bool NonBackbone, bool SlotWinners, template <class> class S, uint32_t Blocks>
struct Walk {
    static constexpr bool kV3 = V3, kAsbr = Asbr, kNonBackbone = NonBackbone, kSlotWinners = SlotWinners;
    template <class Planes> using Side = S<Planes>;
    static constexpr uint32_t kBlocks = Blocks;
};

// Tables of area 0 (hspf_ospfv{2,3}_backbone_table_create), and those with type-4 / Inter-Area-Router slots
// (hspf_ospfv{2,3}_backbone_asbr_table_create).
struct WalkBackbone : Walk<false, false, false, false, NoSide, kBackboneBlocksPerSM> {};
struct WalkBackboneV3 : Walk<true, false, false, false, NoSide, kBackboneV3BlocksPerSM> {};
struct WalkBackboneAsbr : Walk<false, true, false, false, AsbrSide, kBackboneAsbrBlocksPerSM> {};
struct WalkBackboneAsbrV3 : Walk<true, true, false, false, AsbrSide, kBackboneAsbrV3BlocksPerSM> {};
// Tables of a non-backbone target area (hspf_ospfv{2,3}_nonbackbone_table_create), with or without slots: the borders
// also advertise their inter-area routes, and a plane set may be a border's area 0.
struct WalkNonBackbone : Walk<false, true, true, false, AsbrSide, kNonBackboneBlocksPerSM> {};
struct WalkNonBackboneV3 : Walk<true, true, true, false, AsbrSide, kNonBackboneV3BlocksPerSM> {};
// Third-area tables (hspf_ospfv{2,3}_third_area_table_create): the kNonBackbone walk over chain slots.  An OSPFv3
// one's C cells may hold OSPFv3 slot winners, whose options ride in their low byte (kSlotWinners).
struct WalkThirdArea : Walk<false, true, true, false, ChainSide, kThirdAreaBlocksPerSM> {};
struct WalkThirdAreaV3 : Walk<true, true, true, true, ChainSide, kThirdAreaV3BlocksPerSM> {};

// The cell functor of walk W (route_stage.cuh).  A job's status word ORs R's row-0 word, the borders' words, then
// the side input's.  Every walk is its own instantiation, with kernels of its own, so a walk added later leaves the
// others' code alone.
template <class Planes, class W>
struct OspfBackboneWalkCell : OspfBackboneCore<Planes>, W::template Side<Planes> {
    __device__ __forceinline__ uint32_t border_status(uint32_t j) const {
        uint32_t s = this->pl.status_word(0);
        for (uint32_t b = 0; b < this->n_borders; ++b)
            if (this->status[b]) s |= this->status[b][j];
        return s;
    }
    __device__ __forceinline__ uint32_t status_word(uint32_t j) const {
        return this->or_status(*this, border_status(j), j);
    }
    __device__ __forceinline__ bool refused(uint32_t j) const { return status_word(j) != 0; }
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        hspf::OspfBorderRows rows;
#pragma unroll
        for (uint32_t b = 0; b < kOspfBackboneMaxBorders; ++b) rows.row[b] = this->cells[b] + (size_t)j * this->K[b];
        return hspf::ospf_backbone_cell_eval<W::kV3, W::kAsbr, W::kNonBackbone, W::kSlotWinners>(
            this->planes(this->pl.job(0), j), this->t, p, rows);
    }
    __device__ __forceinline__ uint64_t gather(uint32_t, uint32_t, uint32_t) const { return 0; }   // row 0: host side
    __device__ static hspf::CellWords empty() { return {0, 0, hspf::kNoRecord}; }
};

// The families of entry points: hspf_ospfv2_backbone_*, hspf_ospfv2_backbone_asbr_* and hspf_ospfv2_third_area_*.
enum class Call { kBackbone, kAsbr, kThirdArea };

// The walk a call of the family runs over t, picked from the table's marks and handed to run as a tag; HSPF_E_INVAL
// for a table the family refuses.
template <class F>
int pick_walk(const hspf_ospfv2_backbone_table *t, Call call, F &&run) {
    if (!t) return HSPF_E_INVAL;
    switch (call) {
    case Call::kBackbone:
        // a table with type-4 slots is the asbr calls'; an OSPFv3 third-area table's C cells hold slot winners, which
        // only the third-area calls read
        if (t->n_asbr_slots || (t->third_area && t->v3)) return HSPF_E_INVAL;
        if (t->area_id) return t->v3 ? run(WalkNonBackboneV3{}) : run(WalkNonBackbone{});
        return t->v3 ? run(WalkBackboneV3{}) : run(WalkBackbone{});
    case Call::kAsbr:
        // an OSPFv3 table of area 0 only from hspf_ospfv3_backbone_asbr_table_create; a third-area table's type-4
        // slots are chain slots, and an OSPFv3 one's C cells hold slot winners
        if ((t->v3 && !t->area_id && !t->asbr) || (t->third_area && (t->n_asbr_slots || t->v3))) return HSPF_E_INVAL;
        if (t->area_id) return t->v3 ? run(WalkNonBackboneV3{}) : run(WalkNonBackbone{});
        if (!t->n_asbr_slots) return t->v3 ? run(WalkBackboneV3{}) : run(WalkBackbone{});   // border planes unread
        return t->v3 ? run(WalkBackboneAsbrV3{}) : run(WalkBackboneAsbr{});
    case Call::kThirdArea:
        // an OSPFv3 table with or without chain slots: the kNonBackbone walks cannot read C's slot winners
        if (!t->third_area) return HSPF_E_INVAL;
        if (t->v3) return run(WalkThirdAreaV3{});
        return t->n_asbr_slots ? run(WalkThirdArea{}) : run(WalkNonBackbone{});
    }
    return HSPF_E_INVAL;
}

// A call: its walk, then R's planes, the borders' cells and status words and the walk's side input into the cell,
// then the launch.
template <class R, class Out>
int stage(hspf_ctx *ctx, Call call, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs, const R *planes,
          const hl_ospf_rib_cell *const *border_cells, const uint32_t *const *border_status, const SideArgs<R> &side,
          const Out &out) {
    return pick_walk(t, call, [&](auto walk) {
        using W = decltype(walk);
        OspfBackboneWalkCell<hspf::PlanesOf<R>, W> cell{};
        if (!t->dev.blob || !border_cells) return HSPF_E_INVAL;
        if (hspf::result_planes(planes, t->n_vertices, cell.pl) || !cell.pl.complete()) return HSPF_E_INVAL;
        if (const int rc = hspf::bind_ospf_borders(*t, border_cells, border_status, cell)) return rc;
        cell.t = t->view(t->dev.off, static_cast<const hspf::RibRec *>(t->dev.contribs));
        if (const int rc = cell.bind(*t, side, n_jobs)) return rc;
        return hspf::launch_route_stage<W::kBlocks>(ctx, t->dev, cell, n_jobs, t->P(), out);
    });
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
    return stage(ctx, Call::kBackbone, t, n_jobs, planes, border_cells, border_status, {},
                 hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out});
}

int hspf_ospfv2_backbone_cells16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                 const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                 const uint32_t *const *border_status, uint32_t *job_status_out, hl_ospf_rib_cell *cells) {
    return stage(ctx, Call::kBackbone, t, n_jobs, planes, border_cells, border_status, {},
                 hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out});
}

int hspf_ospfv2_backbone_delta(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                               const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                               const uint32_t *const *border_status, const hl_ospf_rib_cell *base_cells, uint32_t n_base,
                               const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records,
                               uint64_t cap, uint64_t *n_records) {
    return stage(ctx, Call::kBackbone, t, n_jobs, planes, border_cells, border_status, {},
                 hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_ospfv2_backbone_delta16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                 const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                 const uint32_t *const *border_status, const hl_ospf_rib_cell *base_cells,
                                 uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out,
                                 hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    return stage(ctx, Call::kBackbone, t, n_jobs, planes, border_cells, border_status, {},
                 hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_ospfv2_backbone_asbr_cells(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                    const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                                    const uint32_t *const *border_status, const hspf_result *const *border_planes,
                                    const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                    uint32_t *job_status_out, hl_ospf_rib_cell *cells) {
    return stage(ctx, Call::kAsbr, t, n_jobs, planes, border_cells, border_status,
                 {border_planes, border_n_rows, border_rows}, hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out});
}

int hspf_ospfv2_backbone_asbr_cells16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                      const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                      const uint32_t *const *border_status, const hspf_result16 *const *border_planes,
                                      const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                      uint32_t *job_status_out, hl_ospf_rib_cell *cells) {
    return stage(ctx, Call::kAsbr, t, n_jobs, planes, border_cells, border_status,
                 {border_planes, border_n_rows, border_rows}, hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out});
}

int hspf_ospfv2_backbone_asbr_delta(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                    const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                                    const uint32_t *const *border_status, const hspf_result *const *border_planes,
                                    const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                    const hl_ospf_rib_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                                    hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                                    uint64_t *n_records) {
    return stage(ctx, Call::kAsbr, t, n_jobs, planes, border_cells, border_status,
                 {border_planes, border_n_rows, border_rows},
                 hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_ospfv2_backbone_asbr_delta16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                      const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                      const uint32_t *const *border_status, const hspf_result16 *const *border_planes,
                                      const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                      const hl_ospf_rib_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                                      hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                                      uint64_t *n_records) {
    return stage(ctx, Call::kAsbr, t, n_jobs, planes, border_cells, border_status,
                 {border_planes, border_n_rows, border_rows},
                 hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_ospfv2_third_area_cells(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                 const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                                 const uint32_t *const *border_status, const uint32_t *const *border_entries,
                                 const uint32_t *const *border_entry_status, uint32_t *job_status_out,
                                 hl_ospf_rib_cell *cells) {
    return stage(ctx, Call::kThirdArea, t, n_jobs, planes, border_cells, border_status,
                 {nullptr, nullptr, nullptr, border_entries, border_entry_status},
                 hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out});
}

int hspf_ospfv2_third_area_cells16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                   const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                   const uint32_t *const *border_status, const uint32_t *const *border_entries,
                                   const uint32_t *const *border_entry_status, uint32_t *job_status_out,
                                   hl_ospf_rib_cell *cells) {
    return stage(ctx, Call::kThirdArea, t, n_jobs, planes, border_cells, border_status,
                 {nullptr, nullptr, nullptr, border_entries, border_entry_status},
                 hspf::CellsOut<hl_ospf_rib_cell>{cells, job_status_out});
}

int hspf_ospfv2_third_area_delta(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                 const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                                 const uint32_t *const *border_status, const uint32_t *const *border_entries,
                                 const uint32_t *const *border_entry_status, const hl_ospf_rib_cell *base_cells,
                                 uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out,
                                 hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    return stage(ctx, Call::kThirdArea, t, n_jobs, planes, border_cells, border_status,
                 {nullptr, nullptr, nullptr, border_entries, border_entry_status},
                 hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_ospfv2_third_area_delta16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                   const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                   const uint32_t *const *border_status, const uint32_t *const *border_entries,
                                   const uint32_t *const *border_entry_status, const hl_ospf_rib_cell *base_cells,
                                   uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out,
                                   hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    return stage(ctx, Call::kThirdArea, t, n_jobs, planes, border_cells, border_status,
                 {nullptr, nullptr, nullptr, border_entries, border_entry_status},
                 hspf::DeltaOut<hl_ospf_rib_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

}  // extern "C"
