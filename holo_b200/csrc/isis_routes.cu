// Device route stage for batches of IS-IS SPTs (include/holo_spf_lsdb.h, "batched IS-IS route stage"):
// compute_routes (holo-isis/src/spf.rs:838-941) for every job of a batch.
//
// The SPT planes of both topologies stay in HBM; one thread per (job, prefix) walks the prefix's
// contributors (isis_route_cells.h: isis_route_cell_eval) and writes one 24-byte cell.  Prefix is the fast
// index: contributor records and cells are read / written coalesced, the plane values are gathers inside
// the job's own rows of the prefix's topology.  The stage is bounded by the cell writes.
#include <cuda_runtime.h>

#include <algorithm>

#include "../../include/holo_spf_lsdb.h"
#include "isis_route_cells.h"

namespace {

using hspf::IsisContrib;

// One job's rows of one topology's planes: `base` is job * V of that topology.
template <class Planes, class D, class N>
struct TopoPlanes {
    const D *dist; const uint16_t *hops; const N *nh; const uint32_t *status; uint32_t V;
    __device__ __forceinline__ Planes job(uint32_t j) const {
        const size_t base = (size_t)j * V;
        return Planes{dist + base, hops + base, nh + base};
    }
    __device__ __forceinline__ bool refused(uint32_t j) const { return status && status[j] != 0; }
};

template <class Planes, class D, class N>
__global__ void __launch_bounds__(256)
isis_route_cells_kernel(uint32_t n_jobs, uint32_t P, const uint32_t *__restrict__ off,
                        const IsisContrib *__restrict__ contribs, TopoPlanes<Planes, D, N> std_pl,
                        TopoPlanes<Planes, D, N> mt6_pl, hl_isis_route_cell *__restrict__ cells, bool aligned16) {
    // a warp owns 32 consecutive cells = one contiguous 768-byte span of the output: the cells are staged in
    // shared memory and leave as 48 16-byte stores (full sectors) instead of 96 scattered 8-byte ones
    __shared__ __align__(16) uint64_t stage[8][96];
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const uint64_t total = (uint64_t)n_jobs * P;
    const uint64_t n_tiles = (total + 31) / 32;
    const uint64_t wstride = (uint64_t)gridDim.x * 8;
    for (uint64_t tile = (uint64_t)blockIdx.x * 8 + wib; tile < n_tiles; tile += wstride) {
        const uint64_t idx = tile * 32 + lane;
        uint64_t w0 = 0, w1 = 0xFFFFFFFFull, w2 = 0;         // an empty cell: no route, winner none
        if (idx < total) {
            const uint32_t job = (uint32_t)(idx / P), p = (uint32_t)(idx - (uint64_t)job * P);
            // planes of a refused job are undefined: empty cells
            if (!std_pl.refused(job) && !mt6_pl.refused(job)) {
                const hl_isis_route_cell c =
                    hspf::isis_route_cell_eval(std_pl.job(job), mt6_pl.job(job), contribs, off[p], off[p + 1]);
                w0 = c.nh_mask;
                w1 = (uint64_t)c.winner | ((uint64_t)c.metric << 32);
                w2 = c.flags;
            }
        }
        if (aligned16 && tile * 32 + 32 <= total) {
            uint64_t *s = stage[wib];
            s[lane * 3 + 0] = w0; s[lane * 3 + 1] = w1; s[lane * 3 + 2] = w2;
            __syncwarp();
            const uint4 *s4 = reinterpret_cast<const uint4 *>(s);
            uint4 *o4 = reinterpret_cast<uint4 *>(cells + tile * 32);
            o4[lane] = s4[lane];
            if (lane < 16) o4[32 + lane] = s4[32 + lane];
            __syncwarp();
        } else if (idx < total) {
            uint64_t *o = reinterpret_cast<uint64_t *>(cells + idx);
            o[0] = w0; o[1] = w1; o[2] = w2;
        }
    }
}
static_assert(sizeof(hl_isis_route_cell) == 24, "hl_isis_route_cell layout");

template <class Planes, class D, class N>
int launch_isis_cells(hspf_ctx *ctx, const hspf_isis_rtable *rt, uint32_t n_jobs, TopoPlanes<Planes, D, N> std_pl,
                      TopoPlanes<Planes, D, N> mt6_pl, hl_isis_route_cell *cells) {
    if (!ctx || !rt || !rt->d_blob || !cells) return HSPF_E_INVAL;
    // every topology the table reads needs its planes
    if (rt->root[0] != 0xFFFFFFFFu && (!std_pl.dist || !std_pl.hops || !std_pl.nh)) return HSPF_E_INVAL;
    if (rt->root[1] != 0xFFFFFFFFu && (!mt6_pl.dist || !mt6_pl.hops || !mt6_pl.nh)) return HSPF_E_INVAL;
    const uint32_t P = (uint32_t)rt->prefix.size();
    const uint64_t total = (uint64_t)n_jobs * P;
    if (total == 0) return HSPF_OK;
    const int dev = hspf_ctx_device(ctx);
    if (rt->device != dev) return HSPF_E_INVAL;               // the table was uploaded to another device
    int sms = 0;
    if (cudaSetDevice(dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return HSPF_E_CUDA;
    // one resident wave (8 blocks of 256 per SM), warp-tile-stride beyond that
    const uint64_t want = std::max<uint64_t>((total + 255) / 256, 1);
    const uint32_t blocks = (uint32_t)std::min<uint64_t>(want, (uint64_t)sms * 8);
    const bool aligned16 = (reinterpret_cast<uintptr_t>(cells) & 15u) == 0;
    cudaStream_t st = static_cast<cudaStream_t>(hspf_stream(ctx));
    isis_route_cells_kernel<Planes, D, N><<<blocks, 256, 0, st>>>(n_jobs, P, rt->d_off, rt->d_contribs, std_pl, mt6_pl,
                                                                  cells, aligned16);
    if (cudaGetLastError() != cudaSuccess) return HSPF_E_CUDA;
    hspf_note_launches(ctx, 1);
    return HSPF_OK;
}

}  // namespace

void hspf_isis_rtable_release_device(hspf_isis_rtable *rt) {
    if (rt && rt->d_blob) {
        cudaFree(rt->d_blob);
        rt->d_blob = nullptr; rt->d_off = nullptr; rt->d_contribs = nullptr;
    }
}

extern "C" {

int hspf_isis_rtable_upload(hspf_ctx *ctx, hspf_isis_rtable *rt) {
    if (!ctx || !rt) return HSPF_E_INVAL;
    hspf_isis_rtable_release_device(rt);
    if (cudaSetDevice(hspf_ctx_device(ctx)) != cudaSuccess) return HSPF_E_CUDA;
    const size_t off_bytes = (rt->off.size() * sizeof(uint32_t) + 15) & ~(size_t)15;
    const size_t con_bytes = rt->contribs.size() * sizeof(IsisContrib);
    void *blob = nullptr;
    if (cudaMalloc(&blob, off_bytes + std::max<size_t>(con_bytes, 16)) != cudaSuccess) return HSPF_E_NOMEM;
    cudaStream_t st = static_cast<cudaStream_t>(hspf_stream(ctx));
    cudaError_t e = cudaMemcpyAsync(blob, rt->off.data(), rt->off.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && con_bytes)
        e = cudaMemcpyAsync(static_cast<char *>(blob) + off_bytes, rt->contribs.data(), con_bytes, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);      // the host vectors may go away after the call
    if (e != cudaSuccess) { cudaFree(blob); return HSPF_E_CUDA; }
    rt->d_blob = blob;
    rt->device = hspf_ctx_device(ctx);
    rt->d_off = static_cast<const uint32_t *>(blob);
    rt->d_contribs = reinterpret_cast<const IsisContrib *>(static_cast<char *>(blob) + off_bytes);
    return HSPF_OK;
}

int hspf_isis_routes_batch(hspf_ctx *ctx, const hspf_isis_rtable *rt, uint32_t n_jobs, const hspf_result *std_planes,
                           const hspf_result *mt6_planes, hl_isis_route_cell *cells) {
    if (!rt) return HSPF_E_INVAL;
    using TP = TopoPlanes<hspf::PlanesWide, uint32_t, uint64_t>;
    TP s{nullptr, nullptr, nullptr, nullptr, rt->n_vertices[0]}, m{nullptr, nullptr, nullptr, nullptr, rt->n_vertices[1]};
    if (std_planes) {
        if (std_planes->nh_words != 1) return HSPF_E_INVAL;
        s.dist = std_planes->dist; s.hops = std_planes->hops; s.nh = std_planes->nh_mask; s.status = std_planes->job_status;
    }
    if (mt6_planes) {
        if (mt6_planes->nh_words != 1) return HSPF_E_INVAL;
        m.dist = mt6_planes->dist; m.hops = mt6_planes->hops; m.nh = mt6_planes->nh_mask; m.status = mt6_planes->job_status;
    }
    return launch_isis_cells(ctx, rt, n_jobs, s, m, cells);
}

int hspf_isis_routes_batch16(hspf_ctx *ctx, const hspf_isis_rtable *rt, uint32_t n_jobs, const hspf_result16 *std_planes,
                             const hspf_result16 *mt6_planes, hl_isis_route_cell *cells) {
    if (!rt) return HSPF_E_INVAL;
    using TP = TopoPlanes<hspf::PlanesNarrow, uint16_t, uint16_t>;
    TP s{nullptr, nullptr, nullptr, nullptr, rt->n_vertices[0]}, m{nullptr, nullptr, nullptr, nullptr, rt->n_vertices[1]};
    if (std_planes) {
        s.dist = std_planes->dist; s.hops = std_planes->hops; s.nh = std_planes->nh_mask; s.status = std_planes->job_status;
    }
    if (mt6_planes) {
        m.dist = mt6_planes->dist; m.hops = mt6_planes->hops; m.nh = mt6_planes->nh_mask; m.status = mt6_planes->job_status;
    }
    return launch_isis_cells(ctx, rt, n_jobs, s, m, cells);
}

}  // extern "C"
