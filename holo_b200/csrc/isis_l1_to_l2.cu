// Device stage for what an IS-IS L1/L2 router propagates into its L2 LSP (include/holo_spf_lsdb.h, "L1 -> L2
// propagation of an IS-IS L1/L2 router"): lsp_propagate_l1_to_l2 (holo-isis lsdb.rs:1149-1357) for every job of a
// what-if batch.
//
// Two launches on the ctx stream.  The summary pass of the L1/L2 routing-table stage (isis_summary.cuh), over the
// router's hspf_isis_l1l2_ribtable and the job's L1 row, writes each job's summary words.  Then one thread per
// (job, key) runs isis_l1_to_l2_cell_eval (isis_l1_to_l2_cells.h), reading those words, and the shared cell kernel
// or the route-delta stage (route_stage.cuh) stores or compares the 24-byte cells.
#include "../../include/holo_spf_lsdb.h"
#include "isis_l1_to_l2_cells.h"
#include "isis_summary.cuh"
#include "route_stage.cuh"

namespace {

using hspf::IsisPropRecord;

template <class Planes>
struct IsisL1ToL2Cell {
    using Rows = hspf::ResultPlanes<Planes>;
    hspf::IsisL1ToL2View t;
    hspf::IsisL1L2View rib;          // the summaries: cover lists, L1 contributors, configured metrics
    Rows pl[2];                      // [topology] of the L1 batch; MT-IPv6 planes NULL where L1 has no MT-IPv6 root
    uint32_t n_rows;
    const uint32_t *rows;            // [n_jobs]: the job's L1 row
    const uint64_t *words;           // [n_jobs][S], written by the summary pass
    __device__ __forceinline__ uint32_t status_word(uint32_t j) const {
        const uint32_t r = rows[j];
        return r >= n_rows ? HSPF_JS_INVALID : pl[0].status_word(r) | pl[1].status_word(r);
    }
    __device__ __forceinline__ bool refused(uint32_t j) const { return status_word(j) != 0; }
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t k) const {
        const uint32_t r = rows[j];
        const hl_isis_route_cell c =
            hspf::isis_l1_to_l2_cell_eval(pl[0].job(r), pl[1].job(r), t, rib, k, words + (size_t)j * rib.S);
        return {c.nh_mask, (uint64_t)c.winner | ((uint64_t)c.metric << 32), c.flags};
    }
    __host__ __device__ __forceinline__ uint32_t n_summaries() const { return rib.S; }
    __device__ __forceinline__ uint64_t summary_word(uint32_t j, uint32_t s, uint32_t lane) const {
        const uint32_t r = rows[j];
        return hspf::isis_summary_word(pl[0].job(r), pl[1].job(r), rib, s, lane);
    }
    __device__ __forceinline__ uint64_t gather(uint32_t, uint32_t, uint32_t) const { return 0; }   // the decode needs none
    __device__ static hspf::CellWords empty() { return {0, 0xFFFFFFFFu, 0}; }                      // winner none
};

// Blocks per SM of every kernel over this walk (the summary pass included): their launch bound and their grid.  At 8
// only the summary kernel spills (8 / 12 bytes); on an H100, timed against 4 in one run, 8 was faster for the cell
// launch and both delta passes, with byte-identical cells and words (DESIGN.md §4.4, §6).
constexpr uint32_t kL1ToL2BlocksPerSM = 8;

// The L1 topologies the rib table has no root in are not read: their planes are ignored.
template <class R>
int make_cell(const hspf_isis_l1_to_l2_table *t, const R *l1_std, const R *l1_mt6, uint32_t n_rows, uint32_t n_jobs,
              const uint32_t *rows, uint64_t *summary_out, IsisL1ToL2Cell<hspf::PlanesOf<R>> &cell) {
    if (!t || !t->dev.blob || !t->rib || !t->rib->dev.blob || t->rib->dev.device != t->dev.device ||
        (n_jobs && !rows) || (n_jobs && t->rib->S && !summary_out) || (reinterpret_cast<uintptr_t>(summary_out) & 7u))
        return HSPF_E_INVAL;
    const hspf_isis_l1l2_ribtable *rib = t->rib;
    const R *pl[2] = {l1_std, l1_mt6};
    for (uint32_t k = 0; k < 2; ++k) {
        const uint32_t V = rib->n_vertices[0][k];
        if (rib->root[0][k] == 0xFFFFFFFFu) cell.pl[k] = {nullptr, nullptr, nullptr, nullptr, V};
        else if (hspf::result_planes(pl[k], V, cell.pl[k]) || !cell.pl[k].complete()) return HSPF_E_INVAL;
    }
    cell.t = t->view(t->dev.off, static_cast<const IsisPropRecord *>(t->dev.contribs));
    cell.rib = rib->view(rib->dev.off, static_cast<const hspf::IsisContrib *>(rib->dev.contribs));
    cell.n_rows = n_rows;
    cell.rows = rows;
    cell.words = summary_out;
    return HSPF_OK;
}

// The summary pass runs first: the call refuses its output arguments before it.
template <class R, class Out>
int l1_to_l2(hspf_ctx *ctx, const hspf_isis_l1_to_l2_table *t, uint32_t n_jobs, const R *l1_std, const R *l1_mt6,
             uint32_t n_rows, const uint32_t *rows, uint64_t *summary_out, const Out &out) {
    IsisL1ToL2Cell<hspf::PlanesOf<R>> cell{};
    if (const int rc = make_cell(t, l1_std, l1_mt6, n_rows, n_jobs, rows, summary_out, cell)) return rc;
    if (const int rc = hspf::check_route_out(ctx, out, n_jobs, t->K)) return rc;
    if (const int rc = hspf::launch_isis_summaries<kL1ToL2BlocksPerSM>(ctx, t->dev, cell, n_jobs, summary_out)) return rc;
    return hspf::launch_route_stage<kL1ToL2BlocksPerSM>(ctx, t->dev, cell, n_jobs, t->K, out);
}

}  // namespace

extern "C" {

int hspf_isis_l1_to_l2_table_upload(hspf_ctx *ctx, hspf_isis_l1_to_l2_table *t) {
    return t ? hspf::upload_route_table(ctx, t->dev, t->words, t->recs.data(), t->recs.size() * sizeof(IsisPropRecord))
             : HSPF_E_INVAL;
}

int hspf_isis_l1_to_l2_cells(hspf_ctx *ctx, const hspf_isis_l1_to_l2_table *t, uint32_t n_jobs,
                             const hspf_result *l1_std, const hspf_result *l1_mt6, uint32_t n_l1_rows,
                             const uint32_t *rows, uint64_t *summary_out, uint32_t *job_status_out,
                             hl_isis_route_cell *cells) {
    return l1_to_l2(ctx, t, n_jobs, l1_std, l1_mt6, n_l1_rows, rows, summary_out,
                    hspf::CellsOut<hl_isis_route_cell>{cells, job_status_out});
}

int hspf_isis_l1_to_l2_cells16(hspf_ctx *ctx, const hspf_isis_l1_to_l2_table *t, uint32_t n_jobs,
                               const hspf_result16 *l1_std, const hspf_result16 *l1_mt6, uint32_t n_l1_rows,
                               const uint32_t *rows, uint64_t *summary_out, uint32_t *job_status_out,
                               hl_isis_route_cell *cells) {
    return l1_to_l2(ctx, t, n_jobs, l1_std, l1_mt6, n_l1_rows, rows, summary_out,
                    hspf::CellsOut<hl_isis_route_cell>{cells, job_status_out});
}

int hspf_isis_l1_to_l2_delta(hspf_ctx *ctx, const hspf_isis_l1_to_l2_table *t, uint32_t n_jobs,
                             const hspf_result *l1_std, const hspf_result *l1_mt6, uint32_t n_l1_rows,
                             const uint32_t *rows, uint64_t *summary_out, const hl_isis_route_cell *base_cells,
                             uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out,
                             hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    return l1_to_l2(ctx, t, n_jobs, l1_std, l1_mt6, n_l1_rows, rows, summary_out,
                    hspf::DeltaOut<hl_isis_route_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_isis_l1_to_l2_delta16(hspf_ctx *ctx, const hspf_isis_l1_to_l2_table *t, uint32_t n_jobs,
                               const hspf_result16 *l1_std, const hspf_result16 *l1_mt6, uint32_t n_l1_rows,
                               const uint32_t *rows, uint64_t *summary_out, const hl_isis_route_cell *base_cells,
                               uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out,
                               hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    return l1_to_l2(ctx, t, n_jobs, l1_std, l1_mt6, n_l1_rows, rows, summary_out,
                    hspf::DeltaOut<hl_isis_route_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

}  // extern "C"
