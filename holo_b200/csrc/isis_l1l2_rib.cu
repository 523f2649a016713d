// Device routing-table stage for IS-IS L1/L2 routers (include/holo_spf_lsdb.h, "routing table of an IS-IS L1/L2
// router"): update_rib (holo-isis/src/route.rs:182-249) over both levels, for every job of a what-if batch.
//
// Two launches on the ctx stream.  The summary pass (isis_summary.cuh) gives one warp to each (job, summary): the
// lanes stride over the L1 prefixes the summary covers, each runs the prefix's L1 walk, and the warp reduces presence
// and the lowest metric into the job's summary word.  Then one thread per (job, prefix) runs isis_l1l2_cell_eval
// (isis_l1l2_rib_cells.h) over the job's L1 row and L2 row, reading the words the first pass wrote, and the shared
// cell kernel or the route-delta stage (route_stage.cuh) stores or compares the 24-byte cells.
#include "../../include/holo_spf_lsdb.h"
#include "isis_l1l2_rib_cells.h"
#include "isis_summary.cuh"
#include "route_stage.cuh"

namespace {

using hspf::IsisContrib;

template <class Planes>
struct IsisL1L2Cell {
    using Rows = hspf::ResultPlanes<Planes>;
    hspf::IsisL1L2View t;
    Rows pl[2][2];                   // [level - 1][topology]; MT-IPv6 planes NULL where the level has no MT-IPv6 root
    uint32_t n_rows[2];
    const uint32_t *rows;            // [n_jobs][2]: the job's L1 row, L2 row (indexed in size_t: 2 * j wraps at 2^31)
    const uint64_t *words;           // [n_jobs][S], written by the summary pass
    __device__ __forceinline__ uint32_t status_word(uint32_t j) const {
        uint32_t st = 0;
        for (uint32_t l = 0; l < 2; ++l) {
            const uint32_t r = rows[2 * (size_t)j + l];
            if (r >= n_rows[l]) st |= HSPF_JS_INVALID;
            else st |= pl[l][0].status_word(r) | pl[l][1].status_word(r);
        }
        return st;
    }
    __device__ __forceinline__ bool refused(uint32_t j) const { return status_word(j) != 0; }
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        const uint32_t r1 = rows[2 * (size_t)j], r2 = rows[2 * (size_t)j + 1];
        const hl_isis_route_cell c = hspf::isis_l1l2_cell_eval(pl[0][0].job(r1), pl[0][1].job(r1), pl[1][0].job(r2),
                                                               pl[1][1].job(r2), t, p, words + (size_t)j * t.S);
        return {c.nh_mask, (uint64_t)c.winner | ((uint64_t)c.metric << 32), c.flags};
    }
    __host__ __device__ __forceinline__ uint32_t n_summaries() const { return t.S; }
    // the summary word of (job j, summary s) over the job's L1 row (isis_summary.cuh)
    __device__ __forceinline__ uint64_t summary_word(uint32_t j, uint32_t s, uint32_t lane) const {
        const uint32_t r1 = rows[2 * (size_t)j];
        return hspf::isis_summary_word(pl[0][0].job(r1), pl[0][1].job(r1), t, s, lane);
    }
    __device__ __forceinline__ uint64_t gather(uint32_t, uint32_t, uint32_t) const { return 0; }   // the decode needs none
    __device__ static hspf::CellWords empty() { return {0, 0xFFFFFFFFu, 0}; }                      // winner none
};

// Blocks per SM of every kernel over this walk: their launch bound and their grid.  At 8 every kernel is held to 32
// registers and spills a little; on an H100, timed against 4 in one run, 8 was faster for the summary kernel, the
// cell kernel and both delta passes, with byte-identical cells and words (DESIGN.md §4.4, §6).
constexpr uint32_t kL1L2BlocksPerSM = 8;

// A topology the table has no root in is not read: its planes are ignored.
template <class R>
int make_cell(const hspf_isis_l1l2_ribtable *t, const R *l1_std, const R *l1_mt6, const R *l2_std, const R *l2_mt6,
              const uint32_t *n_rows, uint32_t n_jobs, const uint32_t *rows, uint64_t *summary_out,
              IsisL1L2Cell<hspf::PlanesOf<R>> &cell) {
    if (!t || !t->dev.blob || !n_rows || (n_jobs && !rows) || (n_jobs && t->S && !summary_out) ||
        (reinterpret_cast<uintptr_t>(summary_out) & 7u))
        return HSPF_E_INVAL;
    const R *pl[2][2] = {{l1_std, l1_mt6}, {l2_std, l2_mt6}};
    for (uint32_t l = 0; l < 2; ++l)
        for (uint32_t k = 0; k < 2; ++k) {
            const uint32_t V = t->n_vertices[l][k];
            if (t->root[l][k] == 0xFFFFFFFFu) cell.pl[l][k] = {nullptr, nullptr, nullptr, nullptr, V};
            else if (hspf::result_planes(pl[l][k], V, cell.pl[l][k]) || !cell.pl[l][k].complete()) return HSPF_E_INVAL;
        }
    cell.t = t->view(t->dev.off, static_cast<const IsisContrib *>(t->dev.contribs));
    cell.n_rows[0] = n_rows[0];
    cell.n_rows[1] = n_rows[1];
    cell.rows = rows;
    cell.words = summary_out;
    return HSPF_OK;
}

// The summary pass runs first: the call refuses its output arguments before it.
template <class R, class Out>
int l1l2_rib(hspf_ctx *ctx, const hspf_isis_l1l2_ribtable *t, uint32_t n_jobs, const R *l1_std, const R *l1_mt6,
             const R *l2_std, const R *l2_mt6, const uint32_t *n_rows, const uint32_t *rows, uint64_t *summary_out,
             const Out &out) {
    IsisL1L2Cell<hspf::PlanesOf<R>> cell{};
    if (const int rc = make_cell(t, l1_std, l1_mt6, l2_std, l2_mt6, n_rows, n_jobs, rows, summary_out, cell)) return rc;
    if (const int rc = hspf::check_route_out(ctx, out, n_jobs, t->P)) return rc;
    if (const int rc = hspf::launch_isis_summaries<kL1L2BlocksPerSM>(ctx, t->dev, cell, n_jobs, summary_out)) return rc;
    return hspf::launch_route_stage<kL1L2BlocksPerSM>(ctx, t->dev, cell, n_jobs, t->P, out);
}

}  // namespace

extern "C" {

int hspf_isis_l1l2_ribtable_upload(hspf_ctx *ctx, hspf_isis_l1l2_ribtable *t) {
    return t ? hspf::upload_route_table(ctx, t->dev, t->words, t->contribs.data(), t->contribs.size() * sizeof(IsisContrib))
             : HSPF_E_INVAL;
}

int hspf_isis_l1l2_rib_cells(hspf_ctx *ctx, const hspf_isis_l1l2_ribtable *t, uint32_t n_jobs, const hspf_result *l1_std,
                             const hspf_result *l1_mt6, const hspf_result *l2_std, const hspf_result *l2_mt6,
                             const uint32_t *n_rows, const uint32_t *rows, uint64_t *summary_out,
                             uint32_t *job_status_out, hl_isis_route_cell *cells) {
    return l1l2_rib(ctx, t, n_jobs, l1_std, l1_mt6, l2_std, l2_mt6, n_rows, rows, summary_out,
                    hspf::CellsOut<hl_isis_route_cell>{cells, job_status_out});
}

int hspf_isis_l1l2_rib_cells16(hspf_ctx *ctx, const hspf_isis_l1l2_ribtable *t, uint32_t n_jobs,
                               const hspf_result16 *l1_std, const hspf_result16 *l1_mt6, const hspf_result16 *l2_std,
                               const hspf_result16 *l2_mt6, const uint32_t *n_rows, const uint32_t *rows,
                               uint64_t *summary_out, uint32_t *job_status_out, hl_isis_route_cell *cells) {
    return l1l2_rib(ctx, t, n_jobs, l1_std, l1_mt6, l2_std, l2_mt6, n_rows, rows, summary_out,
                    hspf::CellsOut<hl_isis_route_cell>{cells, job_status_out});
}

int hspf_isis_l1l2_rib_delta(hspf_ctx *ctx, const hspf_isis_l1l2_ribtable *t, uint32_t n_jobs, const hspf_result *l1_std,
                             const hspf_result *l1_mt6, const hspf_result *l2_std, const hspf_result *l2_mt6,
                             const uint32_t *n_rows, const uint32_t *rows, uint64_t *summary_out,
                             const hl_isis_route_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                             hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    return l1l2_rib(ctx, t, n_jobs, l1_std, l1_mt6, l2_std, l2_mt6, n_rows, rows, summary_out,
                    hspf::DeltaOut<hl_isis_route_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

int hspf_isis_l1l2_rib_delta16(hspf_ctx *ctx, const hspf_isis_l1l2_ribtable *t, uint32_t n_jobs,
                               const hspf_result16 *l1_std, const hspf_result16 *l1_mt6, const hspf_result16 *l2_std,
                               const hspf_result16 *l2_mt6, const uint32_t *n_rows, const uint32_t *rows,
                               uint64_t *summary_out, const hl_isis_route_cell *base_cells, uint32_t n_base,
                               const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records,
                               uint64_t cap, uint64_t *n_records) {
    return l1l2_rib(ctx, t, n_jobs, l1_std, l1_mt6, l2_std, l2_mt6, n_rows, rows, summary_out,
                    hspf::DeltaOut<hl_isis_route_cell>{base_cells, n_base, base_of, job_out, records, cap, n_records});
}

}  // extern "C"
