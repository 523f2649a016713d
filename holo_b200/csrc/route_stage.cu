// Device copies of the route tables (route_cells.h: DeviceRouteTable), for both route stages.
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

}  // namespace hspf
