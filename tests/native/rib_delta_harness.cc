// TEST HARNESS (not part of libholo_spf.so): the route-delta stage on the CPU over OSPFv2 routing-table cells
// (hl_ospf_rib_cell) — route_delta_kind with OspfRibCellLayout, the classification hspf_ospfv2_rib_delta[16]
// compiles (holo_b200/csrc/route_delta.h).  The stage itself (summaries, record order, capacity) is the one of
// route_delta_harness.cc, included here so that both harnesses run the same CPU restatement.
#include "route_delta_harness.cc"

// kind of one pair of routing-table cells
extern "C" uint32_t harness_rib_delta_kind(const uint64_t *job_cell, const uint64_t *base_cell) {
    const hspf::CellWords J{job_cell[0], job_cell[1], job_cell[2]}, B{base_cell[0], base_cell[1], base_cell[2]};
    return hspf::route_delta_kind<hspf::OspfRibCellLayout>(J, B);
}

// the whole stage over routing-table cells [n_jobs][P]; status: [n_jobs] status words (NULL: all 0)
extern "C" int harness_rib_route_delta(const uint64_t *cells, uint32_t n_jobs, uint32_t P, const uint64_t *base,
                                       uint32_t n_base, const uint32_t *base_of, const uint32_t *status,
                                       hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                                       uint64_t *n_records) {
    stage<hspf::OspfRibCellLayout>(cells, n_jobs, P, base, n_base, base_of, status, job_out, records, cap, n_records);
    return 0;
}
