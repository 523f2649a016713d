// TEST HARNESS (not part of libholo_spf.so): the route-delta stage on the CPU — route_delta_kind, the classification
// the device stage compiles (holo_b200/csrc/route_delta.h), applied to cells the test supplies, with the stage's
// summaries, record order and capacity — so that the classification can be checked without a GPU.
#include <cstdint>
#include <cstring>

#include "holo_spf.h"
#include "../../holo_b200/csrc/route_delta.h"

namespace {

template <class L>
void stage(const uint64_t *cells, uint32_t n_jobs, uint32_t P, const uint64_t *base, uint32_t n_base,
           const uint32_t *base_of, const uint32_t *status, hl_route_delta_job *job_out, hl_route_delta *records,
           uint64_t cap, uint64_t *n_records) {
    uint64_t n = 0;
    for (uint32_t j = 0; j < n_jobs; ++j) {
        hl_route_delta_job &o = job_out[j];
        std::memset(&o, 0, sizeof o);
        const uint32_t b = base_of ? base_of[j] : 0;
        o.status = b < n_base ? (status ? status[j] : 0) : HSPF_JS_INVALID;
        if (o.status) continue;
        for (uint32_t p = 0; p < P; ++p) {
            const uint64_t *w = cells + ((uint64_t)j * P + p) * 3, *v = base + ((uint64_t)b * P + p) * 3;
            const hspf::CellWords J{w[0], w[1], w[2]}, B{v[0], v[1], v[2]};
            const uint32_t kind = hspf::route_delta_kind<L>(J, B);
            if (!kind) continue;
            ++o.n_changed;
            o.n_lost += !!(kind & HL_DELTA_LOST);
            o.n_gained += !!(kind & HL_DELTA_GAINED);
            o.n_metric += !!(kind & HL_DELTA_METRIC);
            o.n_nexthops += !!(kind & HL_DELTA_NEXTHOPS);
            o.n_other += !!(kind & HL_DELTA_OTHER);
            if (records && n < cap) {
                hl_route_delta &r = records[n];
                std::memset(&r, 0, sizeof r);
                r.job = j; r.prefix = p; r.metric = hspf::route_delta_metric<L>(J, B, kind); r.kind = (uint8_t)kind;
            }
            ++n;
        }
    }
    *n_records = n;
}

}  // namespace

// kind of one cell pair; isis: 0 hl_route_cell layout, 1 hl_isis_route_cell layout
extern "C" uint32_t harness_delta_kind(int isis, const uint64_t *job_cell, const uint64_t *base_cell) {
    const hspf::CellWords J{job_cell[0], job_cell[1], job_cell[2]}, B{base_cell[0], base_cell[1], base_cell[2]};
    return isis ? hspf::route_delta_kind<hspf::IsisCellLayout>(J, B) : hspf::route_delta_kind<hspf::OspfCellLayout>(J, B);
}

// the whole stage over cells [n_jobs][P]; status: [n_jobs] status words (NULL: all 0)
extern "C" int harness_route_delta(int isis, const uint64_t *cells, uint32_t n_jobs, uint32_t P, const uint64_t *base,
                                   uint32_t n_base, const uint32_t *base_of, const uint32_t *status,
                                   hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap, uint64_t *n_records) {
    if (isis)
        stage<hspf::IsisCellLayout>(cells, n_jobs, P, base, n_base, base_of, status, job_out, records, cap, n_records);
    else
        stage<hspf::OspfCellLayout>(cells, n_jobs, P, base, n_base, base_of, status, job_out, records, cap, n_records);
    return 0;
}
