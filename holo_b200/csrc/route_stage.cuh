// Device side shared by the batched route stages (ospfv2_routes.cu, isis_routes.cu, ospfv2_rib_cells.cu,
// ospfv2_abr_rib_cells.cu): the warp-tiled store of 24-byte cells, one thread per (job, prefix), the cell kernel and
// its launch on the ctx stream, and the fused route-delta stage that compares every cell with its job's base cell
// instead of storing it.  A stage brings its cell functor; nvcc only.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <type_traits>

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

// The planes of one result struct (include/holo_spf.h: hspf_result, hspf_result16), rows of V vertices per job.
template <class Planes>
struct ResultPlanes {
    using D = std::remove_const_t<std::remove_pointer_t<decltype(Planes::dist)>>;
    using N = std::remove_const_t<std::remove_pointer_t<decltype(Planes::nh)>>;
    const D *dist; const uint16_t *hops; const N *nh; const uint32_t *status; uint32_t V;
    bool complete() const { return dist && hops && nh; }
    __device__ __forceinline__ Planes job(uint32_t j) const {
        const size_t base = (size_t)j * V;
        return Planes{dist + base, hops + base, nh + base};
    }
    __device__ __forceinline__ bool refused(uint32_t j) const { return status && status[j] != 0; }
    __device__ __forceinline__ uint32_t status_word(uint32_t j) const { return status ? status[j] : 0; }
    __device__ __forceinline__ uint64_t gather(uint32_t j, uint32_t v) const {
        return v < V ? (uint64_t)nh[(size_t)j * V + v] : 0;
    }
};

// the Planes of a result struct type
template <class R>
using PlanesOf = std::conditional_t<std::is_same<R, hspf_result>::value, PlanesWide, PlanesNarrow>;

// The planes of `r` (all NULL when r is NULL: the caller decides whether it needs them).  The route stages read
// one next-hop word: wide planes of more than one are HSPF_E_INVAL.
inline int result_planes(const hspf_result *r, uint32_t V, ResultPlanes<PlanesWide> &p) {
    p = {nullptr, nullptr, nullptr, nullptr, V};
    if (!r) return HSPF_OK;
    if (r->nh_words != 1) return HSPF_E_INVAL;
    p = {r->dist, r->hops, r->nh_mask, r->job_status, V};
    return HSPF_OK;
}
inline int result_planes(const hspf_result16 *r, uint32_t V, ResultPlanes<PlanesNarrow> &p) {
    p = {nullptr, nullptr, nullptr, nullptr, V};
    if (r) p = {r->dist, r->hops, r->nh_mask, r->job_status, V};
    return HSPF_OK;
}

// The grid of a route kernel over `items` threads on the ctx's device: one wave of `blocks_per_sm` blocks per SM
// at most (the kernel's __launch_bounds__ minimum), warp-tile-stride beyond that.  Makes the device current.
inline int route_grid(hspf_ctx *ctx, const DeviceRouteTable &table, uint64_t items, uint32_t blocks_per_sm,
                      uint32_t &blocks) {
    const int dev = hspf_ctx_device(ctx);
    if (table.device != dev) return HSPF_E_INVAL;             // the table was uploaded to another device
    int sms = 0;
    if (cudaSetDevice(dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return HSPF_E_CUDA;
    const uint64_t want = std::max<uint64_t>((items + kRouteThreads - 1) / kRouteThreads, 1);
    blocks = (uint32_t)std::min<uint64_t>(want, (uint64_t)sms * blocks_per_sm);
    return HSPF_OK;
}

// ---- cell kernel ----------------------------------------------------------------------------------------------
// A route stage is a cell functor, passed to every kernel by value as one parameter (as __grid_constant__ it costs the
// IS-IS cell kernel two registers):
//   refused(j)             the job gets Cell::empty() (its planes are undefined)
//   status_word(j)         the job's status word
//   operator()(j, p)       the cell of (job, prefix) as three words
//   gather(j, area, v)     a plane value the host decode needs, 0 when out of range (j < n_jobs is checked here)
//   static empty()         the cell of a refused job

// The jobs' status words and the gathers (when asked for), then the cells.
template <class Cell, int kMinBlocks>
__global__ void __launch_bounds__(kRouteThreads, kMinBlocks)
route_cells_kernel(const Cell cell, uint32_t n_jobs, uint32_t P, CellWords *__restrict__ cells,
                   uint32_t *__restrict__ status_out, bool aligned16, uint32_t n_gather,
                   const uint32_t *__restrict__ gather_job, const uint32_t *__restrict__ gather_area,
                   const uint32_t *__restrict__ gather_v, uint64_t *__restrict__ gather_nh) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x, first = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (status_out)
        for (uint64_t j = first; j < n_jobs; j += stride) status_out[j] = cell.status_word((uint32_t)j);
    for (uint64_t g = first; g < n_gather; g += stride) {
        const uint32_t job = gather_job[g];
        gather_nh[g] = job < n_jobs ? cell.gather(job, gather_area ? gather_area[g] : 0, gather_v[g]) : 0;
    }
    store_route_cells(n_jobs, P, cell, Cell::empty(), cells, aligned16);
}

// ---- what a call writes --------------------------------------------------------------------------------------
// The cells call stores n_jobs x P cells of CellT, the jobs' status words when status_out is set, and n_gather
// gathers of (gather_job, gather_area (NULL: 0), gather_v) into gather_nh.  The delta call compares the cells with
// `base` [n_base][P] instead (the route-delta stage below).  Each descriptor takes its cell layout from CellT.
template <class CellT> struct CellLayoutOf;
template <> struct CellLayoutOf<hl_route_cell> { using type = OspfCellLayout; };
template <> struct CellLayoutOf<hl_ospf_rib_cell> { using type = OspfRibCellLayout; };
template <> struct CellLayoutOf<hl_isis_route_cell> { using type = IsisCellLayout; };

template <class CellT>
struct CellsOut {
    static constexpr bool kDelta = false;
    CellT *cells;
    uint32_t *status_out;
    uint32_t n_gather = 0;
    const uint32_t *gather_job = nullptr, *gather_area = nullptr, *gather_v = nullptr;
    uint64_t *gather_nh = nullptr;
};

template <class CellT>
struct DeltaOut {
    static constexpr bool kDelta = true;
    using Layout = typename CellLayoutOf<CellT>::type;
    const CellT *base;
    uint32_t n_base;
    const uint32_t *base_of;             // [n_jobs] base row of each job; NULL: row 0
    hl_route_delta_job *job_out;
    hl_route_delta *records;
    uint64_t cap;
    uint64_t *n_records;
};

// The output arguments a call refuses (HSPF_E_INVAL) before its first launch, so that a stage with a launch of its
// own before the cells or the compare can check them first.
template <class CellT>
int check_route_out(const hspf_ctx *ctx, const CellsOut<CellT> &o, uint32_t, uint32_t) {
    if (!ctx || !o.cells) return HSPF_E_INVAL;
    if (o.n_gather && (!o.gather_job || !o.gather_v || !o.gather_nh)) return HSPF_E_INVAL;
    return HSPF_OK;
}

// The largest batch of one route-delta call: n_jobs x P <= 2^36 cells, at most 2^31 warp tiles.  The delta kernels
// walk tiles with a 32-bit counter and a stride of the grid's warp count (< 2^31), so tile + stride < 2^32 never
// wraps; the reciprocal in delta_eval is exact below 2^37.
constexpr uint64_t kDeltaMaxCells = 1ull << 36;
inline bool delta_batch_fits(uint32_t n_jobs, uint32_t P) { return (uint64_t)n_jobs * P <= kDeltaMaxCells; }

template <class CellT>
int check_route_out(const hspf_ctx *ctx, const DeltaOut<CellT> &o, uint32_t n_jobs, uint32_t P) {
    if (!ctx || !o.base || !o.job_out || !o.n_records || o.n_base == 0 || !delta_batch_fits(n_jobs, P))
        return HSPF_E_INVAL;
    // device buffers at their struct alignment
    if ((reinterpret_cast<uintptr_t>(o.base) & 7u) || (reinterpret_cast<uintptr_t>(o.job_out) & 3u) ||
        (reinterpret_cast<uintptr_t>(o.n_records) & 7u) || (reinterpret_cast<uintptr_t>(o.records) & 3u))
        return HSPF_E_INVAL;
    return HSPF_OK;
}

// launch_route_stage(ctx, table, cell, n_jobs, P, out) enqueues the cells call or the delta call of `cell` on the
// ctx stream, as `out` is a CellsOut or a DeltaOut.  kMinBlocks is the kernels' launch bound; the grid is one wave
// of kBlocksPerSM blocks per SM at most.

// route_cells_kernel over the largest of the cells, the status words and the gathers.
template <int kMinBlocks, uint32_t kBlocksPerSM = kMinBlocks, class Cell, class CellT>
int launch_route_stage(hspf_ctx *ctx, const DeviceRouteTable &table, const Cell &cell, uint32_t n_jobs, uint32_t P,
                       const CellsOut<CellT> &out) {
    if (const int rc = check_route_out(ctx, out, n_jobs, P)) return rc;
    const uint64_t items = std::max<uint64_t>({(uint64_t)n_jobs * P, out.status_out ? n_jobs : 0u, out.n_gather});
    if (items == 0) return HSPF_OK;
    uint32_t blocks = 0;
    const int rc = route_grid(ctx, table, items, kBlocksPerSM, blocks);
    if (rc != HSPF_OK) return rc;
    const bool aligned16 = (reinterpret_cast<uintptr_t>(out.cells) & 15u) == 0;
    route_cells_kernel<Cell, kMinBlocks><<<blocks, kRouteThreads, 0, static_cast<cudaStream_t>(hspf_stream(ctx))>>>(
        cell, n_jobs, P, reinterpret_cast<CellWords *>(out.cells), out.status_out, aligned16, out.n_gather,
        out.gather_job, out.gather_area, out.gather_v, out.gather_nh);
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
    double inv_p;                     // 1.0 / P
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

// warp tiles of the stage
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
    uint32_t warp_changes = 0;      // < 2^32: at most 32 per tile, and a warp walks at most 2^26 of the <= 2^31 tiles
    // no wrap: n_tiles <= 2^31 (delta_batch_fits) and the stride, the grid's warp count, is far below 2^31
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
    // no wrap, as in pass A
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

// The route-delta stage over `cell`: the summaries and the total are zeroed, then pass A runs; with records, the
// scan and pass B follow.  Both passes are launch-bounded to kMinBlocks blocks per SM.
template <int kMinBlocks, uint32_t kBlocksPerSM = kMinBlocks, class Cell, class CellT>
int launch_route_stage(hspf_ctx *ctx, const DeviceRouteTable &table, const Cell &cell, uint32_t n_jobs, uint32_t P,
                       const DeltaOut<CellT> &out) {
    using Layout = typename DeltaOut<CellT>::Layout;
    if (const int rc = check_route_out(ctx, out, n_jobs, P)) return rc;
    const uint64_t total = (uint64_t)n_jobs * P, n_tiles = delta_tiles64(n_jobs, P);
    // the grid covers the cells, or the jobs' status words when there are more jobs than cells
    uint32_t blocks = 0;
    const int rc = route_grid(ctx, table, std::max<uint64_t>(total, n_jobs), kBlocksPerSM, blocks);
    if (rc != HSPF_OK) return rc;
    DeltaArgs a{};
    a.n_jobs = n_jobs; a.P = P; a.inv_p = P ? 1.0 / P : 0.0;
    a.base = reinterpret_cast<const uint64_t *>(out.base); a.n_base = out.n_base; a.base_of = out.base_of;
    a.job_out = out.job_out; a.n_records = reinterpret_cast<unsigned long long *>(out.n_records);
    cudaStream_t st = static_cast<cudaStream_t>(hspf_stream(ctx));
    if (cudaMemsetAsync(out.n_records, 0, sizeof(uint64_t), st) != cudaSuccess) return HSPF_E_CUDA;
    if (n_jobs == 0) return HSPF_OK;
    if (cudaMemsetAsync(out.job_out, 0, (size_t)n_jobs * sizeof(hl_route_delta_job), st) != cudaSuccess)
        return HSPF_E_CUDA;
    const bool with_records = out.records && out.cap && n_tiles;
    size_t scan_bytes = 0;
    char *ws = nullptr;
    if (with_records) {
        scan_bytes = route_delta_scan_bytes(n_tiles);
        const size_t off_bytes = n_tiles * sizeof(uint64_t), cnt_bytes = (n_tiles + 255) & ~(uint64_t)255;
        ws = static_cast<char *>(hspf_ctx_route_workspace(ctx, off_bytes + cnt_bytes + scan_bytes));
        if (!ws) return HSPF_E_NOMEM;
        a.tile_off = reinterpret_cast<const uint64_t *>(ws);
        a.tile_cnt = reinterpret_cast<uint8_t *>(ws + off_bytes);
        a.records = out.records; a.cap = out.cap;
        ws += off_bytes + cnt_bytes;
    }
    route_delta_count_kernel<Layout, Cell, kMinBlocks><<<blocks, kRouteThreads, 0, st>>>(cell, a);
    if (cudaGetLastError() != cudaSuccess) return HSPF_E_CUDA;
    hspf_note_launches(ctx, 1);
    if (!with_records) return HSPF_OK;
    if (route_delta_scan(ws, scan_bytes, a.tile_cnt, const_cast<uint64_t *>(a.tile_off), n_tiles, st) != cudaSuccess)
        return HSPF_E_CUDA;
    route_delta_store_kernel<Layout, Cell, kMinBlocks><<<blocks, kRouteThreads, 0, st>>>(cell, a);
    if (cudaGetLastError() != cudaSuccess) return HSPF_E_CUDA;
    hspf_note_launches(ctx, 2);                                 // the scan (counted as one) and pass B
    return HSPF_OK;
}

}  // namespace hspf
