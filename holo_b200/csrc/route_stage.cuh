// Device side shared by the batched route stages (ospfv2_routes.cu, isis_routes.cu): the warp-tiled store
// of 24-byte cells, one thread per (job, prefix), and its launch on the ctx stream.  nvcc only.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "holo_spf.h"
#include "route_cells.h"

// counts kernels enqueued on the ctx stream (hspf_capi.cu, hspf_launch_count)
extern "C" void hspf_note_launches(hspf_ctx *ctx, uint32_t n);
extern "C" int hspf_ctx_device(const hspf_ctx *ctx);     // the CUDA device the ctx and its stream belong to

namespace hspf {

constexpr uint32_t kRouteThreads = 256;      // threads per block of a route kernel
constexpr uint32_t kRouteBlocksPerSM = 8;    // the grid: one wave of 8 blocks per SM, at most

struct CellWords { uint64_t w0, w1, w2; };  // one cell, as its three 8-byte words in memory order

// Prefix is the fast index.  A warp owns 32 consecutive cells = one contiguous 768-byte span of the output:
// the cells are staged in shared memory and leave as 48 16-byte stores (full sectors) instead of 96 scattered
// 8-byte ones.  A partial last tile, or a buffer that is not 16-byte aligned, is stored 8 bytes at a time.
// `cell(job, prefix)` gives a cell's words; a job `cell.refused(job)` names gets `empty` (its planes are undefined).
template <class Cell, class F>
__device__ __forceinline__ void store_route_cells(uint32_t n_jobs, uint32_t P, const F &cell, CellWords empty,
                                                  Cell *__restrict__ cells, bool aligned16) {
    static_assert(sizeof(Cell) == 24, "a route cell is three 8-byte words");
    constexpr uint32_t kWarps = kRouteThreads / 32;
    __shared__ __align__(16) uint64_t stage[kWarps][96];
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const uint64_t total = (uint64_t)n_jobs * P;
    const uint64_t n_tiles = (total + 31) / 32;
    const uint64_t wstride = (uint64_t)gridDim.x * kWarps;
    for (uint64_t tile = (uint64_t)blockIdx.x * kWarps + wib; tile < n_tiles; tile += wstride) {
        const uint64_t idx = tile * 32 + lane;
        CellWords c = empty;
        if (idx < total) {
            const uint32_t job = (uint32_t)(idx / P), p = (uint32_t)(idx - (uint64_t)job * P);
            if (!cell.refused(job)) c = cell(job, p);
        }
        if (aligned16 && tile * 32 + 32 <= total) {
            uint64_t *s = stage[wib];
            s[lane * 3 + 0] = c.w0; s[lane * 3 + 1] = c.w1; s[lane * 3 + 2] = c.w2;
            __syncwarp();
            const uint4 *s4 = reinterpret_cast<const uint4 *>(s);
            uint4 *o4 = reinterpret_cast<uint4 *>(cells + tile * 32);
            o4[lane] = s4[lane];
            if (lane < 16) o4[32 + lane] = s4[32 + lane];
            __syncwarp();
        } else if (idx < total) {
            uint64_t *o = reinterpret_cast<uint64_t *>(cells + idx);
            o[0] = c.w0; o[1] = c.w1; o[2] = c.w2;
        }
    }
}

// Enqueues one route kernel on the ctx stream over `total` cells: one wave of kRouteBlocksPerSM blocks per SM,
// warp-tile-stride beyond that.  `launch(blocks, stream, aligned16)` makes the <<<blocks, kRouteThreads>>> call.
template <class Launch>
int launch_route_stage(hspf_ctx *ctx, const DeviceRouteTable &table, uint64_t total, const void *cells, Launch launch) {
    const int dev = hspf_ctx_device(ctx);
    if (table.device != dev) return HSPF_E_INVAL;             // the table was uploaded to another device
    int sms = 0;
    if (cudaSetDevice(dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return HSPF_E_CUDA;
    const uint64_t want = std::max<uint64_t>((total + kRouteThreads - 1) / kRouteThreads, 1);
    const uint32_t blocks = (uint32_t)std::min<uint64_t>(want, (uint64_t)sms * kRouteBlocksPerSM);
    const bool aligned16 = (reinterpret_cast<uintptr_t>(cells) & 15u) == 0;
    launch(blocks, static_cast<cudaStream_t>(hspf_stream(ctx)), aligned16);
    if (cudaGetLastError() != cudaSuccess) return HSPF_E_CUDA;
    hspf_note_launches(ctx, 1);
    return HSPF_OK;
}

}  // namespace hspf
