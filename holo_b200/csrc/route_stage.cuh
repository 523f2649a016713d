// Device side shared by the batched route stages (ospfv2_routes.cu, isis_routes.cu): the warp-tiled store
// of 24-byte cells, one thread per (job, prefix), its launch on the ctx stream, and the fused route-delta stage
// that compares every cell with its job's base cell instead of storing it.  nvcc only.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "holo_spf.h"
#include "route_cells.h"
#include "route_delta.h"

// counts kernels enqueued on the ctx stream (hspf_capi.cu, hspf_launch_count)
extern "C" void hspf_note_launches(hspf_ctx *ctx, uint32_t n);
extern "C" int hspf_ctx_device(const hspf_ctx *ctx);     // the CUDA device the ctx and its stream belong to
// grow-only device workspace of the route-delta stage, owned by the ctx (hspf_capi.cu); NULL when it cannot grow
extern "C" void *hspf_ctx_route_workspace(hspf_ctx *ctx, size_t bytes);

namespace hspf {

constexpr uint32_t kRouteThreads = 256;      // threads per block of a route kernel
constexpr uint32_t kRouteBlocksPerSM = 8;    // the grid: one wave of 8 blocks per SM, at most

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

// ---- route-delta stage (include/holo_spf_lsdb.h, "route-delta stage") ------------------------------------------
// Pass A walks the cells with the same warp tiles as store_route_cells, compares each with its job's base cell
// (route_delta.h) and adds to the per-job summaries: one atomic per counter, job and tile, from the lowest changed
// lane of each job the tile holds.  With records, it also leaves each tile's change count (0..32) in the
// workspace; an exclusive scan turns the counts into record offsets, and pass B re-evaluates only the tiles with
// changes and stores their records at offset + rank among the tile's changed lanes.  Records therefore come out
// in (job, prefix) order without an atomic on their positions, and the cell matrix is never stored.

struct DeltaArgs {
    uint32_t n_jobs, P;
    double inv_p;                     // 1.0 / P (set by launch_route_delta)
    const uint64_t *base;             // base cells [n_base][P] as three words each
    uint32_t n_base;
    const uint32_t *base_of;          // [n_jobs] base row of each job; NULL: row 0
    hl_route_delta_job *job_out;      // [n_jobs], zeroed before pass A
    unsigned long long *n_records;    // total changes, zeroed before pass A
    uint8_t *tile_cnt;                // [n_tiles] changes per warp tile (workspace); NULL: summaries only
    const uint64_t *tile_off;         // [n_tiles] exclusive scan of tile_cnt (workspace)
    hl_route_delta *records;
    uint64_t cap;
};

// warp tiles of the stage; launch_route_delta refuses a batch with 2^32 or more
__host__ __device__ __forceinline__ uint64_t delta_tiles64(uint32_t n_jobs, uint32_t P) {
    return ((uint64_t)n_jobs * P + 31) / 32;
}
__device__ __forceinline__ uint32_t delta_tiles(const DeltaArgs &a) { return (uint32_t)delta_tiles64(a.n_jobs, a.P); }

// The kind of the cell of `lane` in warp tile `tile` (0 past the end, for a job without a valid base row, and for a
// refused job); job / p / metric are set for a changed cell.  The tile counter is 32 bits and the total is
// recomputed from the arguments: the OSPF walk has to fit 32 registers beside this loop.
template <class L, class F>
__device__ __forceinline__ uint32_t delta_eval(const F &cell, const DeltaArgs &a, uint32_t tile, uint32_t lane,
                                               uint32_t &job, uint32_t &p, uint32_t &metric) {
    job = 0xFFFFFFFFu; p = 0; metric = 0;
    const uint64_t idx = (uint64_t)tile * 32 + lane, total = (uint64_t)a.n_jobs * a.P;
    if (idx >= total) return 0;
    // idx / P through the reciprocal: exact after one correction for idx < 2^37, and no division call
    uint64_t q = (uint64_t)((double)idx * a.inv_p);
    int64_t r = (int64_t)(idx - q * a.P);
    if (r < 0) { --q; r += a.P; } else if (r >= (int64_t)a.P) { ++q; r -= a.P; }
    job = (uint32_t)q;
    p = (uint32_t)r;
    const uint32_t b = a.base_of ? a.base_of[job] : 0;
    if (b >= a.n_base || cell.refused(job)) return 0;
    const CellWords c = cell(job, p);
    const uint64_t *w = a.base + ((uint64_t)b * a.P + p) * 3;
    const CellWords base{w[0], w[1], w[2]};
    const uint32_t kind = route_delta_kind<L>(c, base);
    metric = route_delta_metric<L>(c, base, kind);
    return kind;
}

template <class L, class F, int kMinBlocks>
__global__ void __launch_bounds__(kRouteThreads, kMinBlocks) route_delta_count_kernel(F cell, DeltaArgs a) {
    constexpr uint32_t kWarps = kRouteThreads / 32;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < a.n_jobs; j += gridDim.x * blockDim.x) {
        const uint32_t b = a.base_of ? a.base_of[j] : 0;
        a.job_out[j].status = b < a.n_base ? cell.status_word(j) : HSPF_JS_INVALID;
    }
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const uint32_t n_tiles = delta_tiles(a);
    uint32_t warp_changes = 0;      // < 2^32: at most 32 per tile, and a warp walks at most 2^26 of the < 2^32 tiles
    for (uint32_t tile = blockIdx.x * kWarps + wib; tile < n_tiles; tile += gridDim.x * kWarps) {
        uint32_t job, p, metric;
        const uint32_t kind = delta_eval<L>(cell, a, tile, lane, job, p, metric);
        const uint32_t changed = __ballot_sync(0xFFFFFFFFu, kind != 0);
        if (a.tile_cnt && lane == 0) a.tile_cnt[tile] = (uint8_t)__popc(changed);
        if (!changed) continue;
        warp_changes += (uint32_t)__popc(changed);
        // one leader per job in the tile: its lowest changed lane; the counters follow n_changed in bit order
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, job) & changed;
        const bool leader = kind && lane == (uint32_t)(__ffs(peers) - 1);
        if (leader) atomicAdd(&a.job_out[job].n_changed, (uint32_t)__popc(peers));
#pragma unroll
        for (uint32_t b = 0; b < 5; ++b) {
            const uint32_t m = __ballot_sync(0xFFFFFFFFu, kind & (1u << b)) & peers;
            if (leader && m) atomicAdd(&a.job_out[job].n_changed + 1 + b, (uint32_t)__popc(m));
        }
    }
    if (lane == 0 && warp_changes) atomicAdd(a.n_records, (unsigned long long)warp_changes);
}

template <class L, class F, int kMinBlocks>
__global__ void __launch_bounds__(kRouteThreads, kMinBlocks) route_delta_store_kernel(F cell, DeltaArgs a) {
    constexpr uint32_t kWarps = kRouteThreads / 32;
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const uint32_t n_tiles = delta_tiles(a);
    for (uint32_t tile = blockIdx.x * kWarps + wib; tile < n_tiles; tile += gridDim.x * kWarps) {
        if (a.tile_cnt[tile] == 0) continue;
        const uint64_t first = a.tile_off[tile];
        if (first >= a.cap) continue;
        uint32_t job, p, metric;
        const uint32_t kind = delta_eval<L>(cell, a, tile, lane, job, p, metric);
        const uint32_t changed = __ballot_sync(0xFFFFFFFFu, kind != 0);
        const uint64_t pos = first + (uint32_t)__popc(changed & ((1u << lane) - 1u));
        if (kind && pos < a.cap) {
            hl_route_delta r;
            r.job = job; r.prefix = p; r.metric = metric; r.kind = (uint8_t)kind;
            r._pad[0] = r._pad[1] = r._pad[2] = 0;
            a.records[pos] = r;
        }
    }
}

// route_stage.cu: the exclusive scan of the tile counts (CUB), and the temporary storage it needs
size_t route_delta_scan_bytes(uint64_t n_tiles);
cudaError_t route_delta_scan(void *temp, size_t temp_bytes, const uint8_t *cnt, uint64_t *off, uint64_t n_tiles,
                             cudaStream_t st);

// Validates the arguments every route-delta call shares and enqueues the stage on the ctx stream: the summaries and
// the total are zeroed, then `count(blocks, stream, args)` launches pass A; with records, the scan and
// `store(blocks, stream, args)` (pass B) follow.  `a.base` is the caller's base cell buffer.
template <class Count, class Store>
int launch_route_delta(hspf_ctx *ctx, const DeviceRouteTable &table, DeltaArgs a, Count count, Store store) {
    if (!a.base || !a.job_out || !a.n_records || a.n_base == 0) return HSPF_E_INVAL;
    // device buffers at their struct alignment
    if ((reinterpret_cast<uintptr_t>(a.base) & 7u) || (reinterpret_cast<uintptr_t>(a.job_out) & 3u) ||
        (reinterpret_cast<uintptr_t>(a.n_records) & 7u) || (reinterpret_cast<uintptr_t>(a.records) & 3u))
        return HSPF_E_INVAL;
    const int dev = hspf_ctx_device(ctx);
    if (table.device != dev) return HSPF_E_INVAL;
    if (cudaSetDevice(dev) != cudaSuccess) return HSPF_E_CUDA;
    cudaStream_t st = static_cast<cudaStream_t>(hspf_stream(ctx));
    const uint64_t total = (uint64_t)a.n_jobs * a.P, n_tiles = delta_tiles64(a.n_jobs, a.P);
    if (n_tiles > 0xFFFFFFFFull) return HSPF_E_INVAL;
    a.inv_p = a.P ? 1.0 / a.P : 0.0;
    if (cudaMemsetAsync(a.n_records, 0, sizeof(uint64_t), st) != cudaSuccess) return HSPF_E_CUDA;
    if (a.n_jobs == 0) return HSPF_OK;
    if (cudaMemsetAsync(a.job_out, 0, (size_t)a.n_jobs * sizeof(hl_route_delta_job), st) != cudaSuccess) return HSPF_E_CUDA;
    const bool with_records = a.records && a.cap && n_tiles;
    size_t scan_bytes = 0;
    char *ws = nullptr;
    if (with_records) {
        scan_bytes = route_delta_scan_bytes(n_tiles);
        const size_t off_bytes = n_tiles * sizeof(uint64_t), cnt_bytes = (n_tiles + 255) & ~(uint64_t)255;
        ws = static_cast<char *>(hspf_ctx_route_workspace(ctx, off_bytes + cnt_bytes + scan_bytes));
        if (!ws) return HSPF_E_NOMEM;
        a.tile_off = reinterpret_cast<const uint64_t *>(ws);
        a.tile_cnt = reinterpret_cast<uint8_t *>(ws + off_bytes);
        ws += off_bytes + cnt_bytes;
    } else {
        a.tile_cnt = nullptr; a.tile_off = nullptr; a.records = nullptr; a.cap = 0;
    }
    // the grid covers the cells, or the jobs' status words when there are more jobs than cells
    cudaError_t scan = cudaSuccess;
    const int rc = launch_route_stage(ctx, table, std::max<uint64_t>(total, a.n_jobs), a.base,
                                      [&](uint32_t blocks, cudaStream_t s, bool) {
        count(blocks, s, a);
        if (!with_records) return;
        scan = route_delta_scan(ws, scan_bytes, a.tile_cnt, const_cast<uint64_t *>(a.tile_off), n_tiles, s);
        if (scan != cudaSuccess) return;
        store(blocks, s, a);
        hspf_note_launches(ctx, 2);                            // the scan (counted as one) and pass B
    });
    return rc != HSPF_OK ? rc : (scan != cudaSuccess ? HSPF_E_CUDA : HSPF_OK);
}

}  // namespace hspf
