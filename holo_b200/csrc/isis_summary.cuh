// The summary pass of the IS-IS L1/L2 device stages (isis_l1l2_rib.cu, isis_l1_to_l2.cu): which configured
// summaries a job's L1 table makes active, and the lowest L1 metric each covers.  One warp per (job, summary): the
// lanes stride over the L1 prefixes the summary covers (isis_l1l2_rib_cells.h, IsisL1L2View), each runs the
// prefix's L1 walk over the job's L1 planes, and the warp reduces presence and the lowest metric into the job's
// summary word.  nvcc only.
#pragma once
#include "isis_l1l2_rib_cells.h"
#include "route_stage.cuh"

namespace hspf {

// The summary word of summary s over one job's L1 planes (isis_summary_eval, split over the warp's lanes).
template <class Planes>
__device__ __forceinline__ uint64_t isis_summary_word(const Planes &s1, const Planes &m1, const IsisL1L2View &t,
                                                      uint32_t s, uint32_t lane) {
    bool any = false;
    uint32_t low = 0xFFFFFFFFu;
    for (uint32_t i = t.cov_off[s] + lane; i < t.cov_off[s + 1]; i += 32) {
        uint32_t m;
        if (!isis_l1_metric(s1, m1, t, __ldg(t.cov + i), m)) continue;
        any = true;
        low = min(low, m);
    }
    low = __reduce_min_sync(0xFFFFFFFFu, low);
    return __any_sync(0xFFFFFFFFu, any) ? (kIsisSummaryActive | low) : 0;
}

// A stage's cell functor brings n_summaries() (host and device: the launch sizes the grid with it), refused(j) and
// summary_word(j, s, lane).
template <class Cell, int kMinBlocks>
__global__ void __launch_bounds__(kRouteThreads, kMinBlocks)
isis_summary_kernel(const Cell cell, uint32_t n_jobs, uint64_t *__restrict__ out) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n = (uint64_t)n_jobs * cell.n_summaries();
    const uint64_t wstride = (uint64_t)gridDim.x * (kRouteThreads / 32);
    for (uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; w < n; w += wstride) {
        const uint32_t j = (uint32_t)(w / cell.n_summaries()), s = (uint32_t)(w - (uint64_t)j * cell.n_summaries());
        const uint64_t word = cell.refused(j) ? 0 : cell.summary_word(j, s, lane);   // warp-uniform branch
        if (lane == 0) out[w] = word;
    }
}

// Enqueues the summary pass on the ctx stream, launch-bounded and gridded at kMinBlocks blocks per SM: nothing for
// 0 jobs or no summaries.
template <int kMinBlocks, class Cell>
int launch_isis_summaries(hspf_ctx *ctx, const DeviceRouteTable &table, const Cell &cell, uint32_t n_jobs,
                          uint64_t *out) {
    const uint64_t n = (uint64_t)n_jobs * cell.n_summaries();
    if (n == 0) return HSPF_OK;
    uint32_t blocks = 0;
    if (const int rc = route_grid(ctx, table, n * 32, kMinBlocks, blocks)) return rc;
    isis_summary_kernel<Cell, kMinBlocks>
        <<<blocks, kRouteThreads, 0, static_cast<cudaStream_t>(hspf_stream(ctx))>>>(cell, n_jobs, out);
    if (cudaGetLastError() != cudaSuccess) return HSPF_E_CUDA;
    hspf_note_launches(ctx, 1);
    return HSPF_OK;
}

}  // namespace hspf
