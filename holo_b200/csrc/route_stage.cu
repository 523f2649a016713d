// Device copies of the route tables (route_cells.h: DeviceRouteTable), for both route stages, and the scan of the
// route-delta stage (route_stage.cuh).
#include <cub/device/device_scan.cuh>
#include <cuda/std/functional>

#include "route_stage.cuh"

namespace hspf {

void release_route_table(DeviceRouteTable &d) {
    if (d.blob) cudaFree(d.blob);
    d = DeviceRouteTable{};
}

// `off` and the contributor records in one allocation, the records 16-byte aligned
int upload_route_table(hspf_ctx *ctx, DeviceRouteTable &d, const std::vector<uint32_t> &off, const void *contribs,
                       size_t contrib_bytes) {
    if (!ctx) return HSPF_E_INVAL;
    release_route_table(d);
    const int dev = hspf_ctx_device(ctx);
    if (cudaSetDevice(dev) != cudaSuccess) return HSPF_E_CUDA;
    const size_t off_bytes = (off.size() * sizeof(uint32_t) + 15) & ~(size_t)15;
    void *blob = nullptr;
    if (cudaMalloc(&blob, off_bytes + std::max<size_t>(contrib_bytes, 16)) != cudaSuccess) return HSPF_E_NOMEM;
    cudaStream_t st = static_cast<cudaStream_t>(hspf_stream(ctx));
    cudaError_t e = cudaMemcpyAsync(blob, off.data(), off.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && contrib_bytes)
        e = cudaMemcpyAsync(static_cast<char *>(blob) + off_bytes, contribs, contrib_bytes, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);      // the host vectors may go away after the call
    if (e != cudaSuccess) { cudaFree(blob); return HSPF_E_CUDA; }
    d.blob = blob;
    d.device = dev;
    d.off = static_cast<const uint32_t *>(blob);
    d.contribs = static_cast<char *>(blob) + off_bytes;
    return HSPF_OK;
}

// u8 tile counts -> u64 offsets: the initial value makes the scan accumulate in 64 bits
size_t route_delta_scan_bytes(uint64_t n_tiles) {
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveScan(nullptr, bytes, static_cast<const uint8_t *>(nullptr), static_cast<uint64_t *>(nullptr),
                                   cuda::std::plus<>{}, (uint64_t)0, (int64_t)n_tiles);
    return bytes;
}

cudaError_t route_delta_scan(void *temp, size_t temp_bytes, const uint8_t *cnt, uint64_t *off, uint64_t n_tiles,
                             cudaStream_t st) {
    return cub::DeviceScan::ExclusiveScan(temp, temp_bytes, cnt, off, cuda::std::plus<>{}, (uint64_t)0, (int64_t)n_tiles, st);
}

}  // namespace hspf
