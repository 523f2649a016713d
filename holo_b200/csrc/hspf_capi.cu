// hspf_capi.cu — C ABI of the batched SPF engine (include/holo_spf.h).
//
// Host side: CSR validation, transposition, device residency, batch launch.
// There is no CPU compute path in this file: every result plane is produced by
// spf_batch_kernel on the device.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <numeric>
#include <string>
#include <vector>

#include <cuda.h>
#include <cuda_runtime.h>

#include "holo_spf.h"
#include "quad_layout.h"
#include "spf_kernel.cuh"
#include "spf_quad.cuh"

using namespace hspf;

struct hspf_graph {
    DevGraph d{};
    void *blob = nullptr;      // single device allocation holding every array
    size_t blob_bytes = 0;
    uint32_t max_indeg = 0;
    bool has_leaf = false;     // any HSPF_VF_LEAF / LEAF_UNLESS_ROOT vertex
    bool has_quads = false;    // quad-space image present (spf_quad_kernel eligible, see quad_layout.h)
    QuadDev q{};
    std::string quad_why;      // why the quad image was not built
    std::string fast_why;      // why spf_quad_kernel does not run this graph's batches (empty: it does), see quad_refusal
    // host copies hspf_graph_update_costs validates against
    std::vector<uint32_t> h_row;
    std::vector<uint8_t> h_vflags;
};

struct hspf_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;   // D2H of finished chunks (host-pointer mode)
    cudaEvent_t chunk_done = nullptr;
    int sm_count = 0;
    size_t smem_optin = 0;
    std::string err;
    uint64_t launches = 0;
    uint32_t *d_counter = nullptr;
    // grow-only scratch
    void *ws = nullptr;      size_t ws_bytes = 0;       // global state workspace
    void *stage = nullptr;   size_t stage_bytes = 0;    // device staging of results (host-pointer mode)
    void *h_pin = nullptr;   size_t h_pin_bytes = 0;    // pinned bounce buffer
    void *scratch = nullptr; size_t scratch_bytes = 0;  // planes the caller did not ask for
    void *route_ws = nullptr; size_t route_ws_bytes = 0; // tile counts / offsets of the route-delta stage
    unsigned long long *d_prof = nullptr; int prof_rows = 0;  // optional phase counters (debug)
    bool prof_enabled = false;
    // progress counters of the pipelined host-pointer call (see run_any)
    uint32_t *d_done = nullptr;               // [kMaxDoneChunks]
    uint32_t *prog_done = nullptr;            // set around one enqueue: the launch publishes per-chunk completion
    uint32_t prog_chunk = 0;
    CUresult (*wait_value)(CUstream, CUdeviceptr, cuuint32_t, unsigned int) = nullptr;
    cudaEvent_t prog_reset = nullptr;
    // fused exchange: peer slots the next 16-bit launches also write (hspf_ctx_set_peer_slots)
    uint32_t n_peer_slots = 0;
    long long peer_delta[7] = {0, 0, 0, 0, 0, 0, 0};
    int reserved_sms = 0;     // SMs left free for concurrent kernels (e.g. NCCL), see hspf_ctx_reserve_sms
};

namespace {

int fail(hspf_ctx *ctx, int code, const std::string &msg) {
    if (ctx) ctx->err = msg;
    return code;
}

int cuda_fail(hspf_ctx *ctx, cudaError_t e, const char *what) {
    return fail(ctx, HSPF_E_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

#define CK(call)                                              \
    do {                                                      \
        cudaError_t e_ = (call);                              \
        if (e_ != cudaSuccess) return cuda_fail(ctx, e_, #call); \
    } while (0)

int grow(hspf_ctx *ctx, void **p, size_t *have, size_t need, bool pinned = false) {
    if (*have >= need) return HSPF_OK;
    if (*p) {
        if (pinned) cudaFreeHost(*p); else cudaFree(*p);
        *p = nullptr; *have = 0;
    }
    size_t want = need + need / 4;
    cudaError_t e = pinned ? cudaMallocHost(p, want) : cudaMalloc(p, want);
    if (e != cudaSuccess) { *p = nullptr; return cuda_fail(ctx, e, pinned ? "cudaMallocHost" : "cudaMalloc"); }
    *have = want;
    return HSPF_OK;
}

template <typename VT, bool S, bool F>
int launch(hspf_ctx *ctx, const BatchArgs &args, size_t smem, int grid) {
    if (const char *co = getenv("HSPF_SMEM_CARVEOUT")) {   // tuning knob (experiments only)
        CK(cudaFuncSetAttribute(spf_batch_kernel<VT, S, F>, cudaFuncAttributePreferredSharedMemoryCarveout, atoi(co)));
    }
    if (smem > 0) {
        CK(cudaFuncSetAttribute(spf_batch_kernel<VT, S, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    spf_batch_kernel<VT, S, F><<<grid, kThreads, smem, ctx->stream>>>(args);
    CK(cudaGetLastError());
    ctx->launches++;
    return HSPF_OK;
}

template <typename VT, bool S>
int max_ctas_per_sm(size_t smem) {
    int n = 0;
    if (smem > 0)
        cudaFuncSetAttribute(spf_batch_kernel<VT, S, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, spf_batch_kernel<VT, S, false>, kThreads, smem) != cudaSuccess) n = 1;
    return n < 1 ? 1 : n;
}

// Result planes of either width: hspf_result (dist u32, first_parent u32, nh_mask u64 x nh_words)
// or hspf_result16 (all planes u16, one next-hop word of 16 atoms).
struct AnyResult {
    void *dist = nullptr;
    uint16_t *hops = nullptr;
    void *fp = nullptr;
    uint16_t *npar = nullptr;
    void *nh = nullptr;
    uint32_t nh_words = 1;
    uint32_t *job_status = nullptr;
    bool narrow = false;
    size_t dist_b() const { return narrow ? 2 : 4; }
    size_t fp_b() const { return narrow ? 2 : 4; }
    size_t nh_b() const { return narrow ? 2 : 8 * (size_t)nh_words; }
};

AnyResult any_of(const hspf_result *r) {
    AnyResult a;
    a.dist = r->dist; a.hops = r->hops; a.fp = r->first_parent; a.npar = r->n_parents; a.nh = r->nh_mask;
    a.nh_words = r->nh_words; a.job_status = r->job_status; a.narrow = false;
    return a;
}

AnyResult any_of(const hspf_result16 *r) {
    AnyResult a;
    a.dist = r->dist; a.hops = r->hops; a.fp = r->first_parent; a.npar = r->n_parents; a.nh = r->nh_mask;
    a.nh_words = 1; a.job_status = r->job_status; a.narrow = true;
    return a;
}

template <int T, bool O>
int launch_quad(hspf_ctx *ctx, const QuadArgs &args, size_t smem, int per_sm_cap) {
    CK(cudaFuncSetAttribute(spf_quad_kernel<T, O>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK(cudaFuncSetAttribute(spf_quad_kernel<T, O>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    int per_sm = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, spf_quad_kernel<T, O>, T, smem));
    if (per_sm < 1) return fail(ctx, HSPF_E_CUDA, "spf_quad_kernel does not fit an SM");
    if (per_sm_cap > 0 && per_sm > per_sm_cap) per_sm = per_sm_cap;
    int grid = (ctx->sm_count - ctx->reserved_sms) * per_sm;
    if (const char *mg = getenv("HSPF_MAX_GRID")) {   // tuning knob (experiments only)
        int v = atoi(mg);
        if (v >= 1 && v < grid) grid = v;
    }
    if ((uint32_t)grid > args.n_jobs) grid = (int)args.n_jobs;
    if (grid < 1) grid = 1;
    QuadArgs a = args;
    if (ctx->prof_enabled) {
        if (ctx->prof_rows < grid) {
            if (ctx->d_prof) cudaFree(ctx->d_prof);
            ctx->d_prof = nullptr; ctx->prof_rows = 0;
            CK(cudaMalloc(&ctx->d_prof, (size_t)grid * 16 * sizeof(unsigned long long)));
            ctx->prof_rows = grid;
        }
        CK(cudaMemsetAsync(ctx->d_prof, 0, (size_t)ctx->prof_rows * 16 * sizeof(unsigned long long), ctx->stream));
        a.prof = ctx->d_prof;
    }
    CK(cudaMemsetAsync(ctx->d_counter, 0, sizeof(uint32_t), ctx->stream));
    spf_quad_kernel<T, O><<<grid, T, smem, ctx->stream>>>(a);
    CK(cudaGetLastError());
    ctx->launches++;
    return HSPF_OK;
}

// Launch shape of spf_quad_kernel for one batch: the default CTA size and queue capacity, or the
// tuning knobs (experiments only).
struct QuadPlan {
    int T = (int)kQuadThreads;
    uint32_t qcap = kQuadQcap;
    QuadLayout lay{};
};

// The one decision between the two kernels: spf_quad_kernel runs a batch of graph g with nh_words
// next-hop words when this returns "" (and *plan, if given, holds its launch shape); otherwise the
// returned reason says why spf_batch_kernel runs instead.  enqueue, the pipelined host call of run_any
// (which waits on the quad kernel's progress counters) and hspf_graph_info all ask this function.
std::string quad_refusal(const hspf_ctx *ctx, const hspf_graph *g, uint32_t nh_words, QuadPlan *plan = nullptr) {
    // (a graph without links has an eligible image but no packed in-edges: quad_why is empty then)
    if (!g->has_quads) return g->quad_why.empty() ? std::string("no links") : g->quad_why;
    if (g->has_leaf) return "LEAF vertex flags";
    if (g->d.flags & HSPF_GF_HOPCOUNT) return "hop-count mode";
    if (nh_words != 1) return "more than one next-hop word";
    if (getenv("HSPF_NO_QUAD")) return "HSPF_NO_QUAD is set";           // tuning knob (experiments only)
    QuadPlan p;
    if (const char *qc = getenv("HSPF_QUAD_QCAP")) { int v = atoi(qc); if (v >= 64 && v <= 32768) p.qcap = (uint32_t)v; }
    if (const char *t = getenv("HSPF_QUAD_T")) p.T = atoi(t);            // tuning knobs (experiments only)
    if (p.T != 128 && p.T != 256 && p.T != 384 && p.T != 512) p.T = (int)kQuadThreads;
    p.lay = make_quad_layout(g->d.V, g->q.NQ, p.qcap, (uint32_t)p.T);
    const size_t need = quad_smem_bytes(p.lay);
    if (need > ctx->smem_optin)
        return "the quad kernel's shared memory (" + std::to_string(need) + " B) exceeds the device's " +
               std::to_string(ctx->smem_optin) + " B per block";
    if (plan) *plan = p;
    return "";
}

// The fast path: quad-space kernel (spf_quad.cuh), for a batch quad_refusal accepted.
int enqueue_quad(hspf_ctx *ctx, const hspf_graph *g, const hspf_jobs *jobs, const AnyResult *out, const QuadPlan &p) {
    int cap = 0;
    if (const char *c = getenv("HSPF_CTAS_PER_SM")) cap = atoi(c);       // tuning knob (experiments only)
    const int T = p.T;
    const QuadLayout &lay = p.lay;
    QuadArgs a{};
    a.g = g->d; a.q = g->q; a.lay = lay;
    a.n_jobs = jobs->n_jobs; a.roots = jobs->roots;
    a.ov_off = jobs->ov_off; a.ov_edge = jobs->ov_edge; a.ov_cost = jobs->ov_cost;
    a.out_dist = static_cast<uint32_t *>(out->dist); a.out_hops = out->hops;
    a.out_fp = static_cast<uint32_t *>(out->fp); a.out_npar = out->npar;
    a.out_nh = static_cast<uint64_t *>(out->nh); a.out_status = out->job_status;
    a.narrow = out->narrow ? 1u : 0u;
    a.n_peers = out->narrow ? ctx->n_peer_slots : 0u;
    for (uint32_t k = 0; k < 7; ++k) a.peer_delta[k] = ctx->peer_delta[k];
    a.done = ctx->prog_done;
    a.done_chunk = ctx->prog_chunk ? ctx->prog_chunk : 1u;
    a.job_counter = ctx->d_counter;
    a.sub_rounds = 1;
    if (const char *sr = getenv("HSPF_QUAD_SUB")) { int v = atoi(sr); if (v >= 1 && v <= 8) a.sub_rounds = (uint32_t)v; }   // tuning knob
    const bool ov = jobs->ov_off != nullptr;
    switch (T) {
    case 128: return ov ? launch_quad<128, true>(ctx, a, lay.total, cap) : launch_quad<128, false>(ctx, a, lay.total, cap);
    case 256: return ov ? launch_quad<256, true>(ctx, a, lay.total, cap) : launch_quad<256, false>(ctx, a, lay.total, cap);
    case 512: return ov ? launch_quad<512, true>(ctx, a, lay.total, cap) : launch_quad<512, false>(ctx, a, lay.total, cap);
    default: return ov ? launch_quad<384, true>(ctx, a, lay.total, cap) : launch_quad<384, false>(ctx, a, lay.total, cap);
    }
}

// Enqueue one batch.  All pointers in `jobs`/`out` are device pointers here.
int enqueue(hspf_ctx *ctx, const hspf_graph *g, const hspf_jobs *jobs, const AnyResult *out) {
    QuadPlan qp;
    const std::string why = quad_refusal(ctx, g, out->nh_words, &qp);
    if (why.empty()) return enqueue_quad(ctx, g, jobs, out, qp);
    if (out->narrow)
        return fail(ctx, HSPF_E_UNSUPPORTED, "16-bit result planes need the packed fast path (" + why + ")");
    const uint32_t V = g->d.V;
    const bool q16 = V <= 0xFFFFu;
    const Layout lay = make_layout(V, g->d.E, q16 ? 2 : 4);
    const size_t sb = lay.total;
    // static smem of the kernel (Small) is ~4.5 KB; leave headroom
    const size_t smem_cap = ctx->smem_optin > 6144 ? ctx->smem_optin - 6144 : 0;
    const bool in_smem = sb <= smem_cap;

    BatchArgs a{};
    a.g = g->d;
    a.lay = lay;
    a.n_jobs = jobs->n_jobs;
    a.roots = jobs->roots;
    a.ov_off = jobs->ov_off;
    a.ov_edge = jobs->ov_edge;
    a.ov_cost = jobs->ov_cost;
    a.out_dist = static_cast<uint32_t *>(out->dist);
    a.out_hops = out->hops;
    a.out_fp = static_cast<uint32_t *>(out->fp);
    a.out_npar = out->npar;
    a.out_nh = static_cast<uint64_t *>(out->nh);
    a.out_status = out->job_status;
    a.nhw = out->nh_words;
    a.job_counter = ctx->d_counter;
    // pointer-jumping next-hop phase: needs the aliased layout (dagbit in qa, words over dist)
    a.jump_ok = (in_smem && q16 && g->d.iedge16 && g->d.edge16 && g->d.iquad && lay.dagbit == lay.qa && lay.kq0 == lay.dist && !getenv("HSPF_NO_JUMP")) ? 1u : 0u;
    if (getenv("HSPF_NO_ROW16")) a.g.row16 = nullptr;   // tuning knob (experiments only)

    int per_sm = in_smem ? (q16 ? max_ctas_per_sm<uint16_t, true>(sb) : max_ctas_per_sm<uint32_t, true>(sb))
                         : (q16 ? max_ctas_per_sm<uint16_t, false>(0) : max_ctas_per_sm<uint32_t, false>(0));
    if (const char *lim = getenv("HSPF_CTAS_PER_SM")) {   // tuning knob (experiments only)
        int v = atoi(lim);
        if (v >= 1 && v < per_sm) per_sm = v;
    }
    // SMs reserved for a concurrent kernel: launch fewer persistent CTAs (job fetch is dynamic)
    int grid = (ctx->sm_count - ctx->reserved_sms) * per_sm;
    if (const char *mg = getenv("HSPF_MAX_GRID")) {   // tuning knob (experiments only)
        int v = atoi(mg);
        if (v >= 1 && v < grid) grid = v;
    }
    if ((uint32_t)grid > jobs->n_jobs) grid = (int)jobs->n_jobs;
    if (grid < 1) grid = 1;

    if (!in_smem) {
        int rc = grow(ctx, &ctx->ws, &ctx->ws_bytes, sb * (size_t)grid);
        if (rc) return rc;
        a.ws = static_cast<uint8_t *>(ctx->ws);
        a.ws_stride = sb;
    }
    if (ctx->prof_enabled) {
        if (ctx->prof_rows < grid) {
            if (ctx->d_prof) cudaFree(ctx->d_prof);
            CK(cudaMalloc(&ctx->d_prof, (size_t)grid * 16 * sizeof(unsigned long long)));
            ctx->prof_rows = grid;
        }
        CK(cudaMemsetAsync(ctx->d_prof, 0, (size_t)ctx->prof_rows * 16 * sizeof(unsigned long long), ctx->stream));
        a.prof = ctx->d_prof;
    }
    CK(cudaMemsetAsync(ctx->d_counter, 0, sizeof(uint32_t), ctx->stream));
    const bool fast = !jobs->ov_off && !(g->d.flags & HSPF_GF_HOPCOUNT) && !g->has_leaf && out->nh_words == 1;
    if (in_smem) {
        if (fast) return q16 ? launch<uint16_t, true, true>(ctx, a, sb, grid) : launch<uint32_t, true, true>(ctx, a, sb, grid);
        return q16 ? launch<uint16_t, true, false>(ctx, a, sb, grid) : launch<uint32_t, true, false>(ctx, a, sb, grid);
    }
    return q16 ? launch<uint16_t, false, false>(ctx, a, 0, grid) : launch<uint32_t, false, false>(ctx, a, 0, grid);
}

struct Planes {   // byte sizes of the result planes of a batch
    size_t dist, hops, fp, npar, nh, status;
    size_t total() const { return dist + hops + fp + npar + nh + status; }
};

Planes plane_sizes(uint32_t n_jobs, uint32_t V, const AnyResult &r) {
    auto al = [](size_t x) { return (x + 255) / 256 * 256; };
    size_t n = (size_t)n_jobs * V;
    Planes p;
    p.dist = al(n * r.dist_b()); p.hops = al(n * 2); p.fp = al(n * r.fp_b()); p.npar = al(n * 2);
    p.nh = al(n * r.nh_b()); p.status = al((size_t)n_jobs * 4);
    return p;
}

int check_result_args(hspf_ctx *ctx, const AnyResult &out) {
    if (out.nh_words < 1 || out.nh_words > 4) return fail(ctx, HSPF_E_INVAL, "nh_words must be 1..4");
    return HSPF_OK;
}

int run_async_any(hspf_ctx *ctx, const hspf_graph *g, const hspf_jobs *jobs, const AnyResult &out);
int run_any(hspf_ctx *ctx, const hspf_graph *g, const hspf_jobs *jobs, const AnyResult &out, uint32_t flags);

int run_async_any(hspf_ctx *ctx, const hspf_graph *g, const hspf_jobs *jobs, const AnyResult &out) {
    int rc = check_result_args(ctx, out);
    if (rc) return rc;
    if (jobs->n_jobs == 0) return HSPF_OK;
    if (!jobs->roots) return fail(ctx, HSPF_E_INVAL, "null roots");
    try {
        CK(cudaSetDevice(ctx->device));
        // planes the caller skipped still have to exist on the device
        AnyResult r = out;
        Planes ps = plane_sizes(jobs->n_jobs, g->d.V, r);
        size_t need = 0;
        if (!r.dist) need += ps.dist;
        if (!r.hops) need += ps.hops;
        if (!r.fp) need += ps.fp;
        if (!r.npar) need += ps.npar;
        if (!r.nh) need += ps.nh;
        if (!r.job_status) need += ps.status;
        if (need) {
            rc = grow(ctx, &ctx->scratch, &ctx->scratch_bytes, need);
            if (rc) return rc;
            uint8_t *p = static_cast<uint8_t *>(ctx->scratch);
            if (!r.dist) { r.dist = p; p += ps.dist; }
            if (!r.hops) { r.hops = reinterpret_cast<uint16_t *>(p); p += ps.hops; }
            if (!r.fp) { r.fp = p; p += ps.fp; }
            if (!r.npar) { r.npar = reinterpret_cast<uint16_t *>(p); p += ps.npar; }
            if (!r.nh) { r.nh = p; p += ps.nh; }
            if (!r.job_status) { r.job_status = reinterpret_cast<uint32_t *>(p); p += ps.status; }
        }
        return enqueue(ctx, g, jobs, &r);
    } catch (...) {
        return fail(ctx, HSPF_E_INVAL, "unexpected exception");
    }
}

int run_any(hspf_ctx *ctx, const hspf_graph *g, const hspf_jobs *jobs, const AnyResult &out, uint32_t flags) {
    int rc = check_result_args(ctx, out);
    if (rc) return rc;
    if (jobs->n_jobs == 0) return HSPF_OK;
    if (!jobs->roots) return fail(ctx, HSPF_E_INVAL, "null roots");
    try {
        CK(cudaSetDevice(ctx->device));
        const uint32_t n = jobs->n_jobs, V = g->d.V;
        if (flags & HSPF_RUN_DEVICE_PTRS) {
            rc = run_async_any(ctx, g, jobs, out);
            if (rc) return rc;
            CK(cudaStreamSynchronize(ctx->stream));
            return HSPF_OK;   // job_status stays on the device in this mode
        }
        // ---- host-pointer mode: validate, stage in, run, stage out --------------
        uint32_t n_ov = 0;
        for (uint32_t j = 0; j < n; ++j)
            if (jobs->roots[j] >= V) return fail(ctx, HSPF_E_INVAL, "root out of range");
        if (jobs->ov_off) {
            if (!jobs->ov_edge || !jobs->ov_cost) {
                if (jobs->ov_off[n] != 0) return fail(ctx, HSPF_E_INVAL, "null override arrays");
            }
            for (uint32_t j = 0; j < n; ++j) {
                if (jobs->ov_off[j + 1] < jobs->ov_off[j]) return fail(ctx, HSPF_E_INVAL, "ov_off not monotone");
                if (jobs->ov_off[j + 1] - jobs->ov_off[j] > HSPF_MAX_OVERRIDES)
                    return fail(ctx, HSPF_E_UNSUPPORTED, "more than HSPF_MAX_OVERRIDES overrides in a job");
            }
            n_ov = jobs->ov_off[n];
            for (uint32_t i = 0; i < n_ov; ++i)
                if (jobs->ov_edge[i] >= g->d.E) return fail(ctx, HSPF_E_INVAL, "override edge out of range");
        }
        auto al = [](size_t x) { return (x + 255) / 256 * 256; };
        const size_t in_roots = al((size_t)n * 4);
        const size_t in_off = jobs->ov_off ? al((size_t)(n + 1) * 4) : 0;
        const size_t in_ove = al((size_t)n_ov * 4 + 4), in_ovc = al((size_t)n_ov * 4 + 4);
        const size_t in_total = in_roots + in_off + in_ove + in_ovc;
        Planes ps = plane_sizes(n, V, out);
        const size_t dev_total = in_total + ps.total();
        rc = grow(ctx, &ctx->stage, &ctx->stage_bytes, dev_total);
        if (rc) return rc;
        rc = grow(ctx, &ctx->h_pin, &ctx->h_pin_bytes, in_total, true);
        if (rc) return rc;
        uint8_t *hp = static_cast<uint8_t *>(ctx->h_pin);
        uint8_t *dp = static_cast<uint8_t *>(ctx->stage);
        std::memcpy(hp, jobs->roots, (size_t)n * 4);
        if (jobs->ov_off) {
            std::memcpy(hp + in_roots, jobs->ov_off, (size_t)(n + 1) * 4);
            if (n_ov) {
                std::memcpy(hp + in_roots + in_off, jobs->ov_edge, (size_t)n_ov * 4);
                std::memcpy(hp + in_roots + in_off + in_ove, jobs->ov_cost, (size_t)n_ov * 4);
            }
        }
        CK(cudaMemcpyAsync(dp, hp, in_total, cudaMemcpyHostToDevice, ctx->stream));
        hspf_jobs dj{};
        dj.n_jobs = n;
        dj.roots = reinterpret_cast<const uint32_t *>(dp);
        dj.ov_off = jobs->ov_off ? reinterpret_cast<const uint32_t *>(dp + in_roots) : nullptr;
        dj.ov_edge = reinterpret_cast<const uint32_t *>(dp + in_roots + in_off);
        dj.ov_cost = reinterpret_cast<const uint32_t *>(dp + in_roots + in_off + in_ove);
        uint8_t *rp = dp + in_total;
        AnyResult dr = out;
        dr.dist = rp; rp += ps.dist;
        dr.hops = reinterpret_cast<uint16_t *>(rp); rp += ps.hops;
        dr.fp = rp; rp += ps.fp;
        dr.npar = reinterpret_cast<uint16_t *>(rp); rp += ps.npar;
        dr.nh = rp; rp += ps.nh;
        dr.job_status = reinterpret_cast<uint32_t *>(rp); rp += ps.status;
        std::vector<uint32_t> st(n);
        const size_t db = out.dist_b(), fb = out.fp_b(), nb = out.nh_b();
        // Fast path: ONE launch for the whole batch; the kernel counts finished jobs per chunk
        // (release ordered behind their planes) and the copy stream waits on those counters with
        // stream memory operations, so a chunk's planes travel to the host while the rest of the
        // batch still computes.  (Launching the batch in pieces instead costs more than it hides:
        // a launch cannot finish faster than one job's latency.)
        // (only spf_quad_kernel counts finished jobs: the waits below would never end behind spf_batch_kernel)
        if (ctx->wait_value && n >= 256 && !getenv("HSPF_E2E_CHUNK") && quad_refusal(ctx, g, out.nh_words).empty()) {
            uint32_t pieces = 4;       // few, large copies: every cudaMemcpyAsync costs ~10 us here
            if (const char *pc = getenv("HSPF_E2E_PIECES")) { int v = atoi(pc); if (v >= 1 && v <= 64) pieces = (uint32_t)v; }   // tuning knob
            const uint32_t pchunk = std::max<uint32_t>(1, (n + pieces - 1) / pieces);
            const uint32_t n_chunks = (n + pchunk - 1) / pchunk;
            CK(cudaMemsetAsync(ctx->d_done, 0, 64 * sizeof(uint32_t), ctx->stream));
            CK(cudaEventRecord(ctx->prog_reset, ctx->stream));
            ctx->prog_done = ctx->d_done; ctx->prog_chunk = pchunk;
            rc = enqueue(ctx, g, &dj, &dr);
            ctx->prog_done = nullptr; ctx->prog_chunk = 0;
            if (rc) return rc;
            CK(cudaEventRecord(ctx->chunk_done, ctx->stream));
            cudaStream_t cs = ctx->copy_stream;
            CK(cudaStreamWaitEvent(cs, ctx->prog_reset, 0));       // the counters of this call, not of the last one
            for (uint32_t c = 0; c < n_chunks; ++c) {
                const uint32_t c0 = c * pchunk, cn = std::min(pchunk, n - c0);
                if (ctx->wait_value(reinterpret_cast<CUstream>(cs), reinterpret_cast<CUdeviceptr>(ctx->d_done + c), cn,
                                    CU_STREAM_WAIT_VALUE_GEQ) != CUDA_SUCCESS)
                    return fail(ctx, HSPF_E_CUDA, "cuStreamWaitValue32 failed");
                const size_t o = (size_t)c0 * V, cv = (size_t)cn * V;
                if (out.dist) CK(cudaMemcpyAsync(static_cast<uint8_t *>(out.dist) + o * db, static_cast<uint8_t *>(dr.dist) + o * db, cv * db, cudaMemcpyDeviceToHost, cs));
                if (out.hops) CK(cudaMemcpyAsync(out.hops + o, dr.hops + o, cv * 2, cudaMemcpyDeviceToHost, cs));
                if (out.fp) CK(cudaMemcpyAsync(static_cast<uint8_t *>(out.fp) + o * fb, static_cast<uint8_t *>(dr.fp) + o * fb, cv * fb, cudaMemcpyDeviceToHost, cs));
                if (out.npar) CK(cudaMemcpyAsync(out.npar + o, dr.npar + o, cv * 2, cudaMemcpyDeviceToHost, cs));
                if (out.nh) CK(cudaMemcpyAsync(static_cast<uint8_t *>(out.nh) + o * nb, static_cast<uint8_t *>(dr.nh) + o * nb, cv * nb, cudaMemcpyDeviceToHost, cs));
            }
            CK(cudaStreamWaitEvent(cs, ctx->chunk_done, 0));
            CK(cudaMemcpyAsync(st.data(), dr.job_status, (size_t)n * 4, cudaMemcpyDeviceToHost, cs));
            CK(cudaStreamSynchronize(cs));
            CK(cudaStreamSynchronize(ctx->stream));
            bool any = false;
            for (uint32_t j = 0; j < n; ++j) any |= (st[j] != 0);
            if (out.job_status) std::memcpy(out.job_status, st.data(), (size_t)n * 4);
            if (any) return fail(ctx, HSPF_E_JOB_STATUS, "one or more jobs need the CPU path (see job_status)");
            return HSPF_OK;
        }
        // General path: one launch (HSPF_E2E_CHUNK: pieces, each copied back on a second stream
        // while the next one computes).
        uint32_t chunk = n;
        if (const char *cs = getenv("HSPF_E2E_CHUNK")) { int v = atoi(cs); if (v > 0) chunk = (uint32_t)v; }
        for (uint32_t c0 = 0; c0 < n; c0 += chunk) {
            const uint32_t cn = std::min(chunk, n - c0);
            hspf_jobs cj = dj;
            cj.n_jobs = cn;
            cj.roots = dj.roots + c0;
            if (dj.ov_off) cj.ov_off = dj.ov_off + c0;    // offsets stay absolute into ov_edge/ov_cost
            AnyResult cr = dr;
            const size_t o = (size_t)c0 * V;
            cr.dist = static_cast<uint8_t *>(dr.dist) + o * db; cr.hops = dr.hops + o;
            cr.fp = static_cast<uint8_t *>(dr.fp) + o * fb; cr.npar = dr.npar + o;
            cr.nh = static_cast<uint8_t *>(dr.nh) + o * nb;
            cr.job_status = dr.job_status + c0;
            rc = enqueue(ctx, g, &cj, &cr);
            if (rc) return rc;
            CK(cudaEventRecord(ctx->chunk_done, ctx->stream));
            CK(cudaStreamWaitEvent(ctx->copy_stream, ctx->chunk_done, 0));
            const size_t cv = (size_t)cn * V;
            cudaStream_t cs = ctx->copy_stream;
            if (out.dist) CK(cudaMemcpyAsync(static_cast<uint8_t *>(out.dist) + o * db, cr.dist, cv * db, cudaMemcpyDeviceToHost, cs));
            if (out.hops) CK(cudaMemcpyAsync(out.hops + o, cr.hops, cv * 2, cudaMemcpyDeviceToHost, cs));
            if (out.fp) CK(cudaMemcpyAsync(static_cast<uint8_t *>(out.fp) + o * fb, cr.fp, cv * fb, cudaMemcpyDeviceToHost, cs));
            if (out.npar) CK(cudaMemcpyAsync(out.npar + o, cr.npar, cv * 2, cudaMemcpyDeviceToHost, cs));
            if (out.nh) CK(cudaMemcpyAsync(static_cast<uint8_t *>(out.nh) + o * nb, cr.nh, cv * nb, cudaMemcpyDeviceToHost, cs));
            CK(cudaMemcpyAsync(st.data() + c0, cr.job_status, (size_t)cn * 4, cudaMemcpyDeviceToHost, cs));
        }
        CK(cudaStreamSynchronize(ctx->copy_stream));
        CK(cudaStreamSynchronize(ctx->stream));
        bool any = false;
        for (uint32_t j = 0; j < n; ++j) any |= (st[j] != 0);
        if (out.job_status) std::memcpy(out.job_status, st.data(), (size_t)n * 4);
        if (any) return fail(ctx, HSPF_E_JOB_STATUS, "one or more jobs need the CPU path (see job_status)");
        return HSPF_OK;
    } catch (const std::bad_alloc &) {
        return fail(ctx, HSPF_E_NOMEM, "host allocation failed");
    } catch (...) {
        return fail(ctx, HSPF_E_INVAL, "unexpected exception");
    }
}

}  // namespace

extern "C" {

const char *hspf_version(void) { return "holo_spf 0.1 sm_90a"; }

int hspf_ctx_create(int device, hspf_ctx **out) {
    if (!out) return HSPF_E_INVAL;
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0 || device < 0 || device >= n) return HSPF_E_CUDA;
    hspf_ctx *ctx = new (std::nothrow) hspf_ctx();
    if (!ctx) return HSPF_E_NOMEM;
    ctx->device = device;
    if (cudaSetDevice(device) != cudaSuccess) { delete ctx; return HSPF_E_CUDA; }
    cudaDeviceProp prop{};
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { delete ctx; return HSPF_E_CUDA; }
    ctx->sm_count = prop.multiProcessorCount;
    ctx->smem_optin = prop.sharedMemPerBlockOptin;
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return HSPF_E_CUDA; }
    if (cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->chunk_done, cudaEventDisableTiming) != cudaSuccess ||
        cudaMalloc(&ctx->d_counter, sizeof(uint32_t)) != cudaSuccess) {
        if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
        if (ctx->chunk_done) cudaEventDestroy(ctx->chunk_done);
        cudaStreamDestroy(ctx->stream); delete ctx; return HSPF_E_CUDA;
    }
    // optional: stream memory operations for the pipelined host-pointer call
    {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuStreamWaitValue32", &fn, cudaEnableDefault, &q) == cudaSuccess && fn &&
            q == cudaDriverEntryPointSuccess &&
            cudaMalloc(&ctx->d_done, 64 * sizeof(uint32_t)) == cudaSuccess &&
            cudaEventCreateWithFlags(&ctx->prog_reset, cudaEventDisableTiming) == cudaSuccess)
            ctx->wait_value = reinterpret_cast<decltype(ctx->wait_value)>(fn);
    }
    *out = ctx;
    return HSPF_OK;
}

void hspf_ctx_destroy(hspf_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) { cudaStreamSynchronize(ctx->stream); cudaStreamDestroy(ctx->stream); }
    if (ctx->copy_stream) { cudaStreamSynchronize(ctx->copy_stream); cudaStreamDestroy(ctx->copy_stream); }
    if (ctx->chunk_done) cudaEventDestroy(ctx->chunk_done);
    if (ctx->d_counter) cudaFree(ctx->d_counter);
    if (ctx->d_done) cudaFree(ctx->d_done);
    if (ctx->prog_reset) cudaEventDestroy(ctx->prog_reset);
    if (ctx->d_prof) cudaFree(ctx->d_prof);
    if (ctx->ws) cudaFree(ctx->ws);
    if (ctx->stage) cudaFree(ctx->stage);
    if (ctx->scratch) cudaFree(ctx->scratch);
    if (ctx->route_ws) cudaFree(ctx->route_ws);
    if (ctx->h_pin) cudaFreeHost(ctx->h_pin);
    delete ctx;
}

const char *hspf_last_error(const hspf_ctx *ctx) { return ctx ? ctx->err.c_str() : "null ctx"; }

void *hspf_stream(hspf_ctx *ctx) { return ctx ? (void *)ctx->stream : nullptr; }

uint64_t hspf_launch_count(const hspf_ctx *ctx) { return ctx ? ctx->launches : 0; }
/* kernels other translation units of the library enqueue on the ctx stream (route_cells.h) */
void hspf_note_launches(hspf_ctx *ctx, uint32_t n) { if (ctx) ctx->launches += n; }
int hspf_ctx_device(const hspf_ctx *ctx) { return ctx ? ctx->device : -1; }
void *hspf_ctx_route_workspace(hspf_ctx *ctx, size_t bytes) {
    if (!ctx) return nullptr;
    return grow(ctx, &ctx->route_ws, &ctx->route_ws_bytes, bytes) == HSPF_OK ? ctx->route_ws : nullptr;
}

int hspf_ctx_set_peer_slots(hspf_ctx *ctx, uint32_t n_peers, const int64_t *deltas) {
    if (!ctx || n_peers > 7 || (n_peers && !deltas)) return HSPF_E_INVAL;
    ctx->n_peer_slots = n_peers;
    for (uint32_t k = 0; k < n_peers; ++k) ctx->peer_delta[k] = (long long)deltas[k];
    return HSPF_OK;
}

int hspf_ctx_reserve_sms(hspf_ctx *ctx, int n_sms) {
    if (!ctx || n_sms < 0 || n_sms >= ctx->sm_count) return HSPF_E_INVAL;
    ctx->reserved_sms = n_sms;
    return HSPF_OK;
}

int hspf_debug_phase_profile(hspf_ctx *ctx, int enable, uint64_t out[16]) {
    if (!ctx) return HSPF_E_INVAL;
    if (out) {
        for (int k = 0; k < 16; ++k) out[k] = 0;
        if (ctx->d_prof && ctx->prof_rows > 0) {
            CK(cudaStreamSynchronize(ctx->stream));
            std::vector<unsigned long long> h((size_t)ctx->prof_rows * 16);
            CK(cudaMemcpy(h.data(), ctx->d_prof, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
            for (int r = 0; r < ctx->prof_rows; ++r)
                for (int k = 0; k < 16; ++k) out[k] += h[(size_t)r * 16 + k];
        }
    }
    ctx->prof_enabled = enable != 0;
    return HSPF_OK;
}

int hspf_graph_upload(hspf_ctx *ctx, const hspf_csr *g, hspf_graph **out) {
    if (!ctx || !g || !out) return HSPF_E_INVAL;
    *out = nullptr;
    try {
        const uint32_t V = g->n_vertices, E = g->n_edges;
        if (V == 0 || V >= 0xFFFFFFF0u) return fail(ctx, HSPF_E_INVAL, "n_vertices out of range");
        if (!g->row_ptr || !g->vflags || (E && (!g->col || !g->cost))) return fail(ctx, HSPF_E_INVAL, "null CSR array");
        if (g->row_ptr[0] != 0 || g->row_ptr[V] != E) return fail(ctx, HSPF_E_INVAL, "row_ptr[0]!=0 or row_ptr[V]!=E");
        bool zero_cost_hop_tail = false;
        uint64_t cost_sum = 0;
        std::vector<uint32_t> indeg(V + 1, 0);
        for (uint32_t u = 0; u < V; ++u) {
            if (g->row_ptr[u + 1] < g->row_ptr[u]) return fail(ctx, HSPF_E_INVAL, "row_ptr not monotone");
            const bool uh = g->vflags[u] & HSPF_VF_HOP;
            for (uint32_t e = g->row_ptr[u]; e < g->row_ptr[u + 1]; ++e) {
                const uint32_t v = g->col[e];
                if (v >= V) return fail(ctx, HSPF_E_INVAL, "col out of range");
                if (v == u) return fail(ctx, HSPF_E_INVAL, "self loop");
                if (g->cost[e] == HSPF_COST_DISABLED) return fail(ctx, HSPF_E_INVAL, "cost 0xFFFFFFFF is reserved");
                if (!uh && !(g->vflags[v] & HSPF_VF_HOP)) return fail(ctx, HSPF_E_INVAL, "edge joins two non-HOP vertices");
                if (uh && g->cost[e] == 0) zero_cost_hop_tail = true;
                cost_sum += g->cost[e];
                indeg[v + 1]++;
            }
        }
        if (g->flags & HSPF_GF_HOPCOUNT) {
            for (uint32_t u = 0; u < V; ++u)
                for (uint32_t e = g->row_ptr[u]; e < g->row_ptr[u + 1]; ++e) {
                    const bool zero = (g->vflags[u] & HSPF_VF_HOP) && !(g->vflags[g->col[e]] & HSPF_VF_HOP);
                    if (g->cost[e] != (zero ? 0u : 1u))
                        return fail(ctx, HSPF_E_INVAL, "HSPF_GF_HOPCOUNT: costs must be 0 (HOP->non-HOP) or 1");
                }
        } else if (zero_cost_hop_tail)
            return fail(ctx, HSPF_E_NEEDS_ORACLE,
                        "zero-cost link out of a hop-counting vertex: ECMP DAG depends on pop order");
        uint32_t max_indeg = 0;
        for (uint32_t v = 0; v < V; ++v) max_indeg = std::max(max_indeg, indeg[v + 1]);
        if (max_indeg >= 0xFFFFu) return fail(ctx, HSPF_E_UNSUPPORTED, "in-degree >= 65535");

        // transposed CSR: in-edges of v ordered by (source, forward edge index)
        std::vector<uint32_t> irow(V + 1, 0);
        for (uint32_t v = 0; v < V; ++v) irow[v + 1] = irow[v] + indeg[v + 1];
        std::vector<uint32_t> fill(irow.begin(), irow.end() - 1);
        std::vector<uint4> iedge(E);
        std::vector<uint2> fedge(E);
        for (uint32_t u = 0; u < V; ++u)
            for (uint32_t e = g->row_ptr[u]; e < g->row_ptr[u + 1]; ++e) {
                const uint32_t v = g->col[e];
                const uint32_t k = fill[v]++;
                iedge[k] = make_uint4(u, g->cost[e], e, 0u);
                fedge[e] = make_uint2(v, g->cost[e]);
            }

        // compact twins used by the jump phase when ids and costs fit 16 bits: row offsets
        // (kept in shared memory during the SSSP) and in-edges as (source | cost << 16)
        uint32_t max_cost = 0;
        for (uint32_t e = 0; e < E; ++e) max_cost = std::max(max_cost, g->cost[e]);
        const bool pack_rows = V <= 0xFFFFu && E <= 0xFFFFu;
        const bool pack_in = V <= 0xFFFFu && max_cost <= 0xFFFFu;
        std::vector<uint16_t> row16(pack_rows ? V : 0);
        for (uint32_t v = 0; v < (uint32_t)row16.size(); ++v) row16[v] = (uint16_t)g->row_ptr[v];
        std::vector<uint32_t> iedge16(pack_in ? E : 0);
        for (uint32_t k = 0; k < (uint32_t)iedge16.size(); ++k) iedge16[k] = iedge[k].x | (iedge[k].y << 16);
        // ... and the same in-edge records padded per vertex to whole 16-byte quads (pad record:
        // the vertex itself with cost 0xFFFF, which can never be a parent), so the parents pass reads the usual
        // four in-edges of a vertex with one 128-bit load
        std::vector<uint32_t> iquad_row(pack_in ? V + 1 : 0);
        std::vector<uint32_t> iquad;
        if (pack_in) {
            for (uint32_t v = 0; v < V; ++v) {
                iquad_row[v] = (uint32_t)(iquad.size() / 4);
                for (uint32_t k = irow[v]; k < irow[v + 1]; ++k) iquad.push_back(iedge16[k]);
                while (iquad.size() % 4) iquad.push_back(v | 0xFFFF0000u);   // pad: self-loop, never a parent
            }
            iquad_row[V] = (uint32_t)(iquad.size() / 4);
        }
        std::vector<uint32_t> edge16(pack_in ? E : 0);     // forward edges as (head | cost << 16)
        for (uint32_t e = 0; e < (uint32_t)edge16.size(); ++e) edge16[e] = fedge[e].x | (fedge[e].y << 16);

        // quad-space image for spf_quad_kernel (quad_layout.h), when ids and costs pack
        QuadHost QH;
        {
            std::vector<uint32_t> isrc(E), icost(E), ifwd(E);
            for (uint32_t k = 0; k < E; ++k) { isrc[k] = iedge[k].x; icost[k] = iedge[k].y; ifwd[k] = iedge[k].z; }
            QH = build_quads(V, E, g->row_ptr, g->col, g->cost, g->vflags, irow.data(), isrc.data(), icost.data(),
                             ifwd.data(), g->delta);
        }

        auto al = [](size_t x) { return (x + 255) / 256 * 256; };
        const size_t o_row = 0;
        const size_t o_edge = o_row + al((size_t)(V + 1) * 4);
        const size_t o_irow = o_edge + al((size_t)E * 8);
        const size_t o_iedge = o_irow + al((size_t)(V + 1) * 4);
        const size_t o_vf = o_iedge + al((size_t)E * 16);
        const size_t o_row16 = o_vf + al(V);
        const size_t o_iedge16 = o_row16 + al(row16.size() * 2);
        const size_t o_edge16 = o_iedge16 + al(iedge16.size() * 4);
        const size_t o_iqrow = o_edge16 + al(edge16.size() * 4);
        const size_t o_iquad = o_iqrow + al(iquad_row.size() * 4);
        const size_t o_fq = o_iquad + al(iquad.size() * 4);
        const size_t o_fcont = o_fq + al(QH.fq.size() * 4);
        const size_t o_slot = o_fcont + al(QH.fcont.size() * 4);
        const size_t o_vert = o_slot + al(QH.slot_of.size() * 2);
        const size_t o_iq = o_vert + al(QH.vert_of.size() * 2);
        const size_t o_imeta = o_iq + al(QH.iq.size() * 4);
        const size_t o_fpos = o_imeta + al(QH.imeta.size() * 4);
        const size_t o_ipos = o_fpos + al(QH.fpos.size() * 4);
        const size_t total = o_ipos + al(QH.ipos.size() * 4);

        hspf_graph *G = new hspf_graph();
        cudaError_t e = cudaSetDevice(ctx->device);
        if (e == cudaSuccess) e = cudaMalloc(&G->blob, total);
        if (e != cudaSuccess) { delete G; return cuda_fail(ctx, e, "cudaMalloc(graph)"); }
        G->blob_bytes = total;
        uint8_t *b = static_cast<uint8_t *>(G->blob);
        std::vector<uint8_t> host(total, 0);
        std::memcpy(host.data() + o_row, g->row_ptr, (size_t)(V + 1) * 4);
        if (E) {
            std::memcpy(host.data() + o_edge, fedge.data(), (size_t)E * 8);
            std::memcpy(host.data() + o_iedge, iedge.data(), (size_t)E * 16);
        }
        std::memcpy(host.data() + o_irow, irow.data(), (size_t)(V + 1) * 4);
        std::memcpy(host.data() + o_vf, g->vflags, V);
        if (!row16.empty()) std::memcpy(host.data() + o_row16, row16.data(), row16.size() * 2);
        if (!iedge16.empty()) std::memcpy(host.data() + o_iedge16, iedge16.data(), iedge16.size() * 4);
        if (!edge16.empty()) std::memcpy(host.data() + o_edge16, edge16.data(), edge16.size() * 4);
        if (!iquad_row.empty()) std::memcpy(host.data() + o_iqrow, iquad_row.data(), iquad_row.size() * 4);
        if (!iquad.empty()) std::memcpy(host.data() + o_iquad, iquad.data(), iquad.size() * 4);
        if (QH.eligible) {
            std::memcpy(host.data() + o_fq, QH.fq.data(), QH.fq.size() * 4);
            std::memcpy(host.data() + o_fcont, QH.fcont.data(), QH.fcont.size() * 4);
            std::memcpy(host.data() + o_slot, QH.slot_of.data(), QH.slot_of.size() * 2);
            std::memcpy(host.data() + o_vert, QH.vert_of.data(), QH.vert_of.size() * 2);
            std::memcpy(host.data() + o_iq, QH.iq.data(), QH.iq.size() * 4);
            std::memcpy(host.data() + o_imeta, QH.imeta.data(), QH.imeta.size() * 4);
            if (E) {
                std::memcpy(host.data() + o_fpos, QH.fpos.data(), QH.fpos.size() * 4);
                std::memcpy(host.data() + o_ipos, QH.ipos.data(), QH.ipos.size() * 4);
            }
        }
        e = cudaMemcpyAsync(b, host.data(), total, cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) { cudaFree(G->blob); delete G; return cuda_fail(ctx, e, "graph H2D"); }

        G->d.V = V; G->d.E = E;
        G->d.row = reinterpret_cast<const uint32_t *>(b + o_row);
        G->d.edge = reinterpret_cast<const uint2 *>(b + o_edge);
        G->d.irow = reinterpret_cast<const uint32_t *>(b + o_irow);
        G->d.iedge = reinterpret_cast<const uint4 *>(b + o_iedge);
        G->d.vflags = b + o_vf;
        G->d.row16 = row16.empty() ? nullptr : reinterpret_cast<const uint16_t *>(b + o_row16);
        G->d.iedge16 = iedge16.empty() ? nullptr : reinterpret_cast<const uint32_t *>(b + o_iedge16);
        G->d.edge16 = edge16.empty() ? nullptr : reinterpret_cast<const uint32_t *>(b + o_edge16);
        G->d.iquad_row = iquad_row.empty() ? nullptr : reinterpret_cast<const uint32_t *>(b + o_iqrow);
        G->d.iquad = iquad.empty() ? nullptr : reinterpret_cast<const uint4 *>(b + o_iquad);
        G->has_quads = QH.eligible && G->d.iedge16 != nullptr;
        G->quad_why = QH.why;
        if (G->has_quads) {
            G->q.NQ = QH.NQ; G->q.NIQ = QH.NIQ; G->q.shift = QH.shift;
            uint32_t st = 0;
            while ((1u << st) < QH.max_ichain) ++st;
            G->q.isteps = st;
            G->q.fq = reinterpret_cast<const uint4 *>(b + o_fq);
            G->q.fcont = reinterpret_cast<const uint32_t *>(b + o_fcont);
            G->q.slot_of = reinterpret_cast<const uint16_t *>(b + o_slot);
            G->q.vert_of = reinterpret_cast<const uint16_t *>(b + o_vert);
            G->q.iq = reinterpret_cast<const uint4 *>(b + o_iq);
            G->q.imeta = reinterpret_cast<const uint2 *>(b + o_imeta);
            G->q.fpos = reinterpret_cast<const uint32_t *>(b + o_fpos);
            G->q.ipos = reinterpret_cast<const uint32_t *>(b + o_ipos);
        }
        G->d.reject_above = g->reject_above;
        G->d.saturate_at = g->saturate_at;
        G->d.flags = g->flags;
        uint32_t delta = g->delta;
        if (delta == 0) {
            // near/far bucket width: ~4x the mean link cost keeps the SSSP at a few buckets
            // (fewer barrier rounds) with ~1.3x re-expansion on the BASELINE shapes
            uint64_t mean = E ? cost_sum / E : 1;
            delta = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(4 * mean, 1), 0x7FFFFFFFu);
        }
        G->d.delta = delta;
        G->max_indeg = max_indeg;
        G->h_row.assign(g->row_ptr, g->row_ptr + V + 1);
        G->h_vflags.assign(g->vflags, g->vflags + V);
        for (uint32_t v = 0; v < V; ++v)
            if (g->vflags[v] & (HSPF_VF_LEAF | HSPF_VF_LEAF_UNLESS_ROOT)) G->has_leaf = true;
        G->fast_why = quad_refusal(ctx, G, 1);
        *out = G;
        return HSPF_OK;
    } catch (const std::bad_alloc &) {
        return fail(ctx, HSPF_E_NOMEM, "host allocation failed");
    } catch (...) {
        return fail(ctx, HSPF_E_INVAL, "unexpected exception");
    }
}

int hspf_graph_update_costs(hspf_ctx *ctx, hspf_graph *g, uint32_t n, const uint32_t *edges, const uint32_t *costs) {
    if (!ctx || !g || (n && (!edges || !costs))) return HSPF_E_INVAL;
    if (n == 0) return HSPF_OK;
    try {
        if (g->d.flags & HSPF_GF_HOPCOUNT) return fail(ctx, HSPF_E_UNSUPPORTED, "hop-count graphs have fixed costs");
        for (uint32_t i = 0; i < n; ++i) {
            const uint32_t e = edges[i], c = costs[i];
            if (e >= g->d.E) return fail(ctx, HSPF_E_INVAL, "edge out of range");
            if (c == HSPF_COST_DISABLED) return fail(ctx, HSPF_E_INVAL, "cost 0xFFFFFFFF is reserved");
            const uint32_t tail = (uint32_t)(std::upper_bound(g->h_row.begin(), g->h_row.end(), e) - g->h_row.begin()) - 1;
            if (c == 0 && (g->h_vflags[tail] & HSPF_VF_HOP))
                return fail(ctx, HSPF_E_NEEDS_ORACLE, "zero-cost link out of a hop-counting vertex");
            if (g->d.iedge16 && c > 0xFFFFu) return fail(ctx, HSPF_E_UNSUPPORTED, "cost does not fit the packed image");
            if (g->has_quads && (c > 65534u || (unsigned long long)c > (3ull << g->q.shift)))
                return fail(ctx, HSPF_E_UNSUPPORTED, "cost outside the bucket ring of the uploaded image");
        }
        cudaError_t er = cudaSetDevice(ctx->device);
        uint32_t *d = nullptr;
        if (er == cudaSuccess) er = cudaMalloc(&d, (size_t)n * 8);
        if (er != cudaSuccess) return cuda_fail(ctx, er, "cudaMalloc(cost patch)");
        er = cudaMemcpyAsync(d, edges, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream);
        if (er == cudaSuccess) er = cudaMemcpyAsync(d + n, costs, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream);
        if (er == cudaSuccess) {
            hspf::patch_costs_kernel<<<(n + 127) / 128, 128, 0, ctx->stream>>>(g->d, g->q, g->has_quads, n, d, d + n);
            er = cudaGetLastError();
            ctx->launches++;
        }
        if (er == cudaSuccess) er = cudaStreamSynchronize(ctx->stream);
        cudaFree(d);
        if (er != cudaSuccess) return cuda_fail(ctx, er, "cost patch");
        return HSPF_OK;
    } catch (const std::bad_alloc &) {
        return fail(ctx, HSPF_E_NOMEM, "host allocation failed");
    }
}

void hspf_graph_free(hspf_ctx *ctx, hspf_graph *g) {
    if (!g) return;
    if (ctx) { cudaSetDevice(ctx->device); cudaStreamSynchronize(ctx->stream); }
    if (g->blob) cudaFree(g->blob);
    delete g;
}

int hspf_sync(hspf_ctx *ctx) {
    if (!ctx) return HSPF_E_INVAL;
    CK(cudaStreamSynchronize(ctx->stream));
    return HSPF_OK;
}

int hspf_run_batch_async(hspf_ctx *ctx, const hspf_graph *g, const hspf_jobs *jobs, const hspf_result *out) {
    if (!ctx || !g || !jobs) return HSPF_E_INVAL;
    if (!out) return fail(ctx, HSPF_E_INVAL, "null result");
    return run_async_any(ctx, g, jobs, any_of(out));
}

int hspf_run_batch(hspf_ctx *ctx, const hspf_graph *g, const hspf_jobs *jobs, const hspf_result *out, uint32_t flags) {
    if (!ctx || !g || !jobs) return HSPF_E_INVAL;
    if (!out) return fail(ctx, HSPF_E_INVAL, "null result");
    return run_any(ctx, g, jobs, any_of(out), flags);
}

int hspf_run_batch16_async(hspf_ctx *ctx, const hspf_graph *g, const hspf_jobs *jobs, const hspf_result16 *out) {
    if (!ctx || !g || !jobs) return HSPF_E_INVAL;
    if (!out) return fail(ctx, HSPF_E_INVAL, "null result");
    return run_async_any(ctx, g, jobs, any_of(out));
}

int hspf_run_batch16(hspf_ctx *ctx, const hspf_graph *g, const hspf_jobs *jobs, const hspf_result16 *out, uint32_t flags) {
    if (!ctx || !g || !jobs) return HSPF_E_INVAL;
    if (!out) return fail(ctx, HSPF_E_INVAL, "null result");
    return run_any(ctx, g, jobs, any_of(out), flags);
}

int hspf_graph_info(const hspf_graph *g, uint32_t info[8]) {
    if (!g || !info) return HSPF_E_INVAL;
    info[0] = g->fast_why.empty() ? 1u : 0u;   // spf_quad_kernel runs one-word batches / 16-bit planes available
    info[1] = g->has_quads ? g->q.NQ : 0u;
    info[2] = g->has_quads ? g->q.NIQ : 0u;
    info[3] = g->has_quads ? g->q.shift : 0u;
    info[4] = g->d.V; info[5] = g->d.E; info[6] = g->max_indeg; info[7] = 0;
    return HSPF_OK;
}

int hspf_debug_quad_image(const hspf_csr *g, uint32_t hdr[8], uint32_t *fq, uint32_t *fcont, uint16_t *slot_of,
                          uint16_t *vert_of, uint32_t *iq, uint32_t *imeta, uint32_t *fpos, uint32_t *ipos) {
    if (!g || !hdr) return HSPF_E_INVAL;
    try {
        const uint32_t V = g->n_vertices, E = g->n_edges;
        std::vector<uint32_t> irow(V + 1, 0), isrc(E), icost(E), ifwd(E);
        for (uint32_t e = 0; e < E; ++e) {
            if (g->col[e] >= V) return HSPF_E_INVAL;
            irow[g->col[e] + 1]++;
        }
        for (uint32_t v = 0; v < V; ++v) irow[v + 1] += irow[v];
        std::vector<uint32_t> fill(irow.begin(), irow.end() - 1);
        for (uint32_t u = 0; u < V; ++u)
            for (uint32_t e = g->row_ptr[u]; e < g->row_ptr[u + 1]; ++e) {
                const uint32_t k = fill[g->col[e]]++;
                isrc[k] = u; icost[k] = g->cost[e]; ifwd[k] = e;
            }
        QuadHost Q = build_quads(V, E, g->row_ptr, g->col, g->cost, g->vflags, irow.data(), isrc.data(), icost.data(),
                                 ifwd.data(), g->delta);
        hdr[0] = Q.eligible ? 1u : 0u; hdr[1] = Q.NQ; hdr[2] = Q.NIQ; hdr[3] = Q.shift;
        hdr[4] = Q.max_ichain; hdr[5] = Q.max_atoms; hdr[6] = 0; hdr[7] = 0;
        if (!Q.eligible) return HSPF_OK;
        hdr[6] = (uint32_t)quad_smem_bytes(make_quad_layout(V, Q.NQ, kQuadQcap, kQuadThreads));
        auto cp = [](auto *dst, const auto &v) { if (dst && !v.empty()) std::memcpy(dst, v.data(), v.size() * sizeof(v[0])); };
        cp(fq, Q.fq); cp(fcont, Q.fcont); cp(slot_of, Q.slot_of); cp(vert_of, Q.vert_of);
        cp(iq, Q.iq); cp(imeta, Q.imeta); cp(fpos, Q.fpos); cp(ipos, Q.ipos);
        return HSPF_OK;
    } catch (...) {
        return HSPF_E_NOMEM;
    }
}

int hspf_atom_count(const hspf_csr *g, uint32_t root, uint32_t *n_atoms) {
    if (!g || !n_atoms || root >= g->n_vertices) return HSPF_E_INVAL;
    uint32_t rb = g->row_ptr[root], re = g->row_ptr[root + 1];
    uint32_t n = re - rb;
    for (uint32_t e = rb; e < re; ++e) {
        uint32_t h = g->col[e];
        if (!(g->vflags[h] & HSPF_VF_HOP)) n += g->row_ptr[h + 1] - g->row_ptr[h];
    }
    *n_atoms = n;
    return HSPF_OK;
}

int hspf_atom_decode(const hspf_csr *g, uint32_t root, uint32_t atom, uint32_t *tail, uint32_t *edge) {
    if (!g || !tail || !edge || root >= g->n_vertices) return HSPF_E_INVAL;
    uint32_t rb = g->row_ptr[root], re = g->row_ptr[root + 1];
    uint32_t deg = re - rb;
    if (atom < deg) { *tail = root; *edge = rb + atom; return HSPF_OK; }
    uint32_t base = deg;
    for (uint32_t e = rb; e < re; ++e) {
        uint32_t h = g->col[e];
        if (g->vflags[h] & HSPF_VF_HOP) continue;
        uint32_t d = g->row_ptr[h + 1] - g->row_ptr[h];
        if (atom < base + d) { *tail = h; *edge = g->row_ptr[h] + (atom - base); return HSPF_OK; }
        base += d;
    }
    return HSPF_E_INVAL;
}

}  // extern "C"
