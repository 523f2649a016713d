// Device route stage for batches of OSPFv2 SPTs (include/holo_spf_lsdb.h, "batched intra-area
// route stage"): update_rib_intra_area (holo-ospf/src/route.rs:343-446) for every job of a batch.
//
// The SPT planes of a batch stay in HBM; one thread per (job, prefix) walks the prefix's advertisers
// (route_cells.h: route_cell_eval) and writes one 24-byte cell.  Prefix is the fast index: the
// advertiser lists and the cells are read / written coalesced, the plane values are gathers inside
// the job's own rows (200 KB at 10k vertices: L2 hits).  HBM traffic per job is the cells
// (24 B x prefixes) plus one pass over the three planes; the walk itself is a handful of integer
// instructions per advertiser, so the stage is bounded by the cell writes.
#include <algorithm>
#include <cstring>
#include <memory>
#include <new>
#include <vector>

#include "../../include/holo_spf_lsdb.h"
#include "route_stage.cuh"

namespace {

using hspf::RouteContrib;

// The cell of (job, prefix): route_cell_eval over the job's rows of the planes.
template <class Planes, class D, class N>
struct OspfCell {
    const uint32_t *off; const RouteContrib *contribs; const D *dist; const uint16_t *hops; const N *nh;
    const uint32_t *status; uint32_t V;
    __device__ __forceinline__ bool refused(uint32_t j) const { return status && status[j] != 0; }
    __device__ __forceinline__ uint32_t status_word(uint32_t j) const { return status ? status[j] : 0; }
    __device__ __forceinline__ hspf::CellWords operator()(uint32_t j, uint32_t p) const {
        const size_t base = (size_t)j * V;
        const hl_route_cell c = hspf::route_cell_eval(Planes{dist + base, hops + base, nh + base}, contribs, off[p], off[p + 1]);
        return {c.nh_mask, c.lasthop_mask, (uint64_t)c.winner | ((uint64_t)c.metric << 32) | ((uint64_t)c.flags << 48)};
    }
};

// the bound keeps the walk in 32 registers, so the whole grid launch_route_stage sizes is resident at once
template <class Planes, class D, class N>
__global__ void __launch_bounds__(hspf::kRouteThreads, hspf::kRouteBlocksPerSM)
route_cells_kernel(uint32_t n_jobs, uint32_t P, uint32_t V, const uint32_t *__restrict__ off,
                   const RouteContrib *__restrict__ contribs, const D *__restrict__ dist,
                   const uint16_t *__restrict__ hops, const N *__restrict__ nh, const uint32_t *__restrict__ job_status,
                   hl_route_cell *__restrict__ cells, bool aligned16, uint32_t n_gather,
                   const uint32_t *__restrict__ gather_job, const uint32_t *__restrict__ gather_v,
                   uint64_t *__restrict__ gather_nh) {
    const OspfCell<Planes, D, N> cell{off, contribs, dist, hops, nh, job_status, V};
    hspf::store_route_cells(n_jobs, P, cell, hspf::CellWords{0, 0, 0xFFFFFFFFu}, cells, aligned16);   // empty: winner none
    // the few plane values the host decode needs
    for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_gather; g += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t job = gather_job[g], v = gather_v[g];
        gather_nh[g] = (job < n_jobs && v < V) ? (uint64_t)nh[(size_t)job * V + v] : 0;
    }
}

template <class Planes, class D, class N>
int launch_cells(hspf_ctx *ctx, const hspf_ospfv2_rtable *rt, uint32_t n_jobs, const D *dist, const uint16_t *hops,
                 const N *nh, const uint32_t *status, hl_route_cell *cells, uint32_t n_gather,
                 const uint32_t *gather_job, const uint32_t *gather_v, uint64_t *gather_nh) {
    if (!ctx || !rt || !rt->dev.blob || !dist || !hops || !nh || !cells) return HSPF_E_INVAL;
    if (n_gather && (!gather_job || !gather_v || !gather_nh)) return HSPF_E_INVAL;
    const uint32_t P = (uint32_t)rt->t.prefix.size();
    const uint64_t total = (uint64_t)n_jobs * P;
    if (total + n_gather == 0) return HSPF_OK;
    return hspf::launch_route_stage(ctx, rt->dev, total, cells, [&](uint32_t blocks, cudaStream_t st, bool aligned16) {
        route_cells_kernel<Planes, D, N><<<blocks, hspf::kRouteThreads, 0, st>>>(
            n_jobs, P, rt->t.n_vertices, rt->dev.off, static_cast<const RouteContrib *>(rt->dev.contribs), dist, hops, nh,
            status, cells, aligned16, n_gather, gather_job, gather_v, gather_nh);
    });
}

// The route-delta stage over the same walk (route_stage.cuh: launch_route_delta), under the bound of route_cells_kernel
// so that the grid launch_route_stage sizes is resident at once: 32 registers, with a few bytes of spill in pass A.
template <class Planes, class D, class N>
int launch_delta(hspf_ctx *ctx, const hspf_ospfv2_rtable *rt, uint32_t n_jobs, const D *dist, const uint16_t *hops,
                 const N *nh, const uint32_t *status, const hl_route_cell *base_cells, uint32_t n_base,
                 const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                 uint64_t *n_records) {
    if (!ctx || !rt || !rt->dev.blob || !dist || !hops || !nh) return HSPF_E_INVAL;
    using Cell = OspfCell<Planes, D, N>;
    const Cell cell{rt->dev.off, static_cast<const RouteContrib *>(rt->dev.contribs), dist, hops, nh, status, rt->t.n_vertices};
    hspf::DeltaArgs a{};
    a.n_jobs = n_jobs; a.P = (uint32_t)rt->t.prefix.size();
    a.base = reinterpret_cast<const uint64_t *>(base_cells); a.n_base = n_base; a.base_of = base_of;
    a.job_out = job_out; a.n_records = reinterpret_cast<unsigned long long *>(n_records);
    a.records = records; a.cap = cap;
    return hspf::launch_route_delta(ctx, rt->dev, a,
        [&](uint32_t blocks, cudaStream_t st, const hspf::DeltaArgs &args) {
            hspf::route_delta_count_kernel<hspf::OspfCellLayout, Cell, hspf::kRouteBlocksPerSM>
                <<<blocks, hspf::kRouteThreads, 0, st>>>(cell, args);
        },
        [&](uint32_t blocks, cudaStream_t st, const hspf::DeltaArgs &args) {
            hspf::route_delta_store_kernel<hspf::OspfCellLayout, Cell, hspf::kRouteBlocksPerSM>
                <<<blocks, hspf::kRouteThreads, 0, st>>>(cell, args);
        });
}

struct DevBuf {
    void *p = nullptr;
    ~DevBuf() { if (p) cudaFree(p); }
    int alloc(size_t bytes) { return cudaMalloc(&p, std::max<size_t>(bytes, 16)) == cudaSuccess ? 0 : HSPF_E_NOMEM; }
    template <class T> T *as() const { return static_cast<T *>(p); }
};

}  // namespace

extern "C" {

int hspf_ospfv2_rtable_upload(hspf_ctx *ctx, hspf_ospfv2_rtable *rt) {
    return rt ? hspf::upload_route_table(ctx, rt->dev, rt->t.off, rt->t.contribs.data(), rt->t.contribs.size() * sizeof(RouteContrib))
              : HSPF_E_INVAL;
}

int hspf_ospfv2_routes_batch(hspf_ctx *ctx, const hspf_ospfv2_rtable *rt, uint32_t n_jobs, const hspf_result *pl,
                             hl_route_cell *cells, uint32_t n_gather, const uint32_t *gather_job,
                             const uint32_t *gather_v, uint64_t *gather_nh) {
    if (!pl || pl->nh_words != 1) return HSPF_E_INVAL;
    return launch_cells<hspf::PlanesWide, uint32_t, uint64_t>(ctx, rt, n_jobs, pl->dist, pl->hops, pl->nh_mask, pl->job_status,
                                                              cells, n_gather, gather_job, gather_v, gather_nh);
}

int hspf_ospfv2_routes_batch16(hspf_ctx *ctx, const hspf_ospfv2_rtable *rt, uint32_t n_jobs, const hspf_result16 *pl,
                               hl_route_cell *cells, uint32_t n_gather, const uint32_t *gather_job,
                               const uint32_t *gather_v, uint64_t *gather_nh) {
    if (!pl) return HSPF_E_INVAL;
    return launch_cells<hspf::PlanesNarrow, uint16_t, uint16_t>(ctx, rt, n_jobs, pl->dist, pl->hops, pl->nh_mask, pl->job_status,
                                                                cells, n_gather, gather_job, gather_v, gather_nh);
}

int hspf_ospfv2_routes_delta(hspf_ctx *ctx, const hspf_ospfv2_rtable *rt, uint32_t n_jobs, const hspf_result *pl,
                             const hl_route_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                             hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    if (!pl || pl->nh_words != 1) return HSPF_E_INVAL;
    return launch_delta<hspf::PlanesWide, uint32_t, uint64_t>(ctx, rt, n_jobs, pl->dist, pl->hops, pl->nh_mask, pl->job_status,
                                                              base_cells, n_base, base_of, job_out, records, cap, n_records);
}

int hspf_ospfv2_routes_delta16(hspf_ctx *ctx, const hspf_ospfv2_rtable *rt, uint32_t n_jobs, const hspf_result16 *pl,
                               const hl_route_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                               hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    if (!pl) return HSPF_E_INVAL;
    return launch_delta<hspf::PlanesNarrow, uint16_t, uint16_t>(ctx, rt, n_jobs, pl->dist, pl->hops, pl->nh_mask, pl->job_status,
                                                                base_cells, n_base, base_of, job_out, records, cap, n_records);
}

int hspf_ospfv2_run_area_batch(hspf_ctx *ctx, const hl_ospfv2_area *area, const uint32_t *root_router_ids, uint32_t n_roots,
                               hl_route_cell *cells, uint64_t cells_cap, uint32_t *n_prefixes, uint32_t *job_status,
                               uint32_t *gather_off, uint32_t *gather_v, uint64_t *gather_nh, uint32_t gather_cap,
                               double *device_ms) {
    if (!ctx || !area || (n_roots && !root_router_ids) || !n_prefixes || !job_status || !gather_off) return HSPF_E_INVAL;
    hspf_ospfv2_flat *flat = nullptr;
    hspf_ospfv2_rtable *rt = nullptr;
    hspf_graph *g = nullptr;
    cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};
    struct Cleanup {
        hspf_ctx *ctx; hspf_ospfv2_flat *&flat; hspf_ospfv2_rtable *&rt; hspf_graph *&g; cudaEvent_t *ev;
        ~Cleanup() {
            if (g) hspf_graph_free(ctx, g);
            if (rt) hspf_ospfv2_rtable_free(rt);
            if (flat) hspf_ospfv2_flat_free(flat);
            for (int i = 0; i < 3; ++i) if (ev[i]) cudaEventDestroy(ev[i]);
        }
    } cleanup{ctx, flat, rt, g, ev};
    try {
        int rc = hspf_ospfv2_flatten(area, &flat);
        if (rc) return rc;
        rc = hspf_ospfv2_rtable_create(flat, &rt);
        if (rc) return rc;
        const uint32_t P = hspf_ospfv2_rtable_prefixes(rt);
        *n_prefixes = P;
        if ((uint64_t)n_roots * P > cells_cap || (n_roots && P && !cells)) return HSPF_E_NOMEM;
        hspf_csr csr;
        rc = hspf_ospfv2_flat_csr(flat, &csr);
        if (rc) return rc;
        const uint32_t V = csr.n_vertices;
        const uint8_t *is_router = nullptr;
        hspf_ospfv2_flat_vertices(flat, nullptr, &is_router, nullptr);
        // roots, and per root the transit networks next to it (the only plane values the decode needs)
        std::vector<uint32_t> roots(n_roots), gj, gv;
        gather_off[0] = 0;
        for (uint32_t j = 0; j < n_roots; ++j) {
            const uint32_t r = hspf_ospfv2_flat_router_vertex(flat, root_router_ids[j]);
            if (r == 0xFFFFFFFFu) return HSPF_E_INVAL;                       // SpfRootNotFound
            roots[j] = r;
            for (uint32_t e = csr.row_ptr[r]; e < csr.row_ptr[r + 1]; ++e) {
                const uint32_t n = csr.col[e];
                if (is_router[n]) continue;
                bool dup = false;
                for (size_t q = gather_off[j]; q < gv.size() && !dup; ++q) dup = gv[q] == n;
                if (!dup) { gj.push_back(j); gv.push_back(n); }
            }
            gather_off[j + 1] = (uint32_t)gv.size();
        }
        const uint32_t G = (uint32_t)gv.size();
        if (cudaSetDevice(hspf_ctx_device(ctx)) != cudaSuccess) return HSPF_E_CUDA;
        if (G > gather_cap || (G && (!gather_v || !gather_nh))) return HSPF_E_NOMEM;
        rc = hspf_graph_upload(ctx, &csr, &g);
        if (rc) return rc;
        rc = hspf_ospfv2_rtable_upload(ctx, rt);
        if (rc) return rc;
        cudaStream_t st = static_cast<cudaStream_t>(hspf_stream(ctx));
        const size_t NV = (size_t)n_roots * V;
        DevBuf d_roots, d_dist, d_hops, d_nh, d_status, d_cells, d_gj, d_gv, d_gnh;
        if (d_roots.alloc(n_roots * 4) || d_dist.alloc(NV * 4) || d_hops.alloc(NV * 2) || d_nh.alloc(NV * 8) ||
            d_status.alloc(n_roots * 4) || d_cells.alloc((size_t)n_roots * P * sizeof(hl_route_cell)) ||
            d_gj.alloc(G * 4) || d_gv.alloc(G * 4) || d_gnh.alloc(G * 8)) return HSPF_E_NOMEM;
        for (auto &e : ev) if (cudaEventCreate(&e) != cudaSuccess) return HSPF_E_CUDA;
        if (cudaMemcpyAsync(d_roots.p, roots.data(), n_roots * 4, cudaMemcpyHostToDevice, st) != cudaSuccess) return HSPF_E_CUDA;
        if (G) {
            if (cudaMemcpyAsync(d_gj.p, gj.data(), G * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
                cudaMemcpyAsync(d_gv.p, gv.data(), G * 4, cudaMemcpyHostToDevice, st) != cudaSuccess) return HSPF_E_CUDA;
        }
        hspf_jobs jobs{};
        jobs.n_jobs = n_roots;
        jobs.roots = d_roots.as<uint32_t>();
        hspf_result res{};
        res.dist = d_dist.as<uint32_t>(); res.hops = d_hops.as<uint16_t>(); res.nh_mask = d_nh.as<uint64_t>();
        res.nh_words = 1; res.job_status = d_status.as<uint32_t>();
        cudaEventRecord(ev[0], st);
        rc = hspf_run_batch_async(ctx, g, &jobs, &res);
        if (rc) return rc;
        cudaEventRecord(ev[1], st);
        rc = hspf_ospfv2_routes_batch(ctx, rt, n_roots, &res, d_cells.as<hl_route_cell>(), G, d_gj.as<uint32_t>(),
                                      d_gv.as<uint32_t>(), d_gnh.as<uint64_t>());
        if (rc) return rc;
        cudaEventRecord(ev[2], st);
        if (cudaMemcpyAsync(job_status, d_status.p, n_roots * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess) return HSPF_E_CUDA;
        if ((size_t)n_roots * P &&
            cudaMemcpyAsync(cells, d_cells.p, (size_t)n_roots * P * sizeof(hl_route_cell), cudaMemcpyDeviceToHost, st) != cudaSuccess)
            return HSPF_E_CUDA;
        if (G && cudaMemcpyAsync(gather_nh, d_gnh.p, G * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess) return HSPF_E_CUDA;
        if (cudaStreamSynchronize(st) != cudaSuccess) return HSPF_E_CUDA;
        if (G) std::memcpy(gather_v, gv.data(), G * 4);
        if (device_ms) {
            float a = 0, b = 0;
            cudaEventElapsedTime(&a, ev[0], ev[1]);
            cudaEventElapsedTime(&b, ev[1], ev[2]);
            device_ms[0] = a; device_ms[1] = b;
        }
        for (uint32_t j = 0; j < n_roots; ++j) if (job_status[j]) return HSPF_E_JOB_STATUS;
        return HSPF_OK;
    } catch (const std::bad_alloc &) {
        return HSPF_E_NOMEM;
    } catch (...) {
        return HSPF_E_INVAL;
    }
}

}  // extern "C"
