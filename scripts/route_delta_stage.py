#!/usr/bin/env python
"""Route-delta stage on the C3 what-if workload, against the route-cell kernel it replaces; device only.

C3 routes exactly as scripts/isis_route_stage.py builds it (10 000 systems, 40 000 directed adjacencies, wide metrics
U[1,1000], seed SEED_BASE+3, 10 000 jobs of one root, job j removing adjacency j mod 20 000, two /32 prefixes per
system).  The base row is the root's plain SPT (one job without overrides, through hspf_isis_routes_batch).  After
one SPT batch, with CUDA events over warmed launches on the engine's stream, alternating:
  (a) hspf_isis_routes_batch: every cell stored (4.8 GB);
  (b) hspf_isis_routes_delta, summaries only (records NULL);
  (c) hspf_isis_routes_delta with records (cap = the total).
Records the card's name and power limit, the times, the total changes and how they spread over jobs, and the bytes
each variant moves.  Outside the timed region the delta is checked against a comparison of (a)'s cells with the base
row done with torch on the device, for every job: summaries, total and every record.  Fails without a GPU.

    python scripts/route_delta_stage.py [--out FILE] [--jobs N] [--reps R]
"""
import argparse
import sys

import numpy as np

import stage_bench

DATASHEET_GBS = 3350.0        # H100 SXM HBM3, NVIDIA data sheet


def torch_delta(cells_u8, base_u8, n, P):
    """The stage restated with torch over stored IS-IS cells: (per-job counts [n, 6], records (job, prefix, metric, kind))."""
    import torch
    from holo_b200.route_table import DELTA_GAINED, DELTA_LOST, DELTA_METRIC, DELTA_NEXTHOPS, DELTA_OTHER
    w = cells_u8.view(torch.int64).view(n, P, 3)
    b = base_u8.view(torch.int64).view(1, P, 3)
    lo32 = 0xFFFFFFFF

    def fields(x):
        return (x[..., 2] & 1) != 0, (x[..., 1] >> 32) & lo32, x[..., 0], x[..., 1] & lo32, x[..., 2]

    jp, jm, jn, jw, jf = fields(w)
    bp, bm, bn, bw, bf = fields(b)
    both = jp & bp
    kind = torch.zeros((n, P), dtype=torch.int32, device=w.device)
    kind |= torch.where(bp & ~jp, DELTA_LOST, 0).to(torch.int32)
    kind |= torch.where(jp & ~bp, DELTA_GAINED, 0).to(torch.int32)
    kind |= torch.where(both & (jm != bm), DELTA_METRIC, 0).to(torch.int32)
    kind |= torch.where(both & (jn != bn), DELTA_NEXTHOPS, 0).to(torch.int32)
    kind |= torch.where(both & ((jw != bw) | (jf != bf)), DELTA_OTHER, 0).to(torch.int32)
    counts = torch.stack([(kind != 0).sum(1)] + [((kind & bit) != 0).sum(1) for bit in
                                                (DELTA_LOST, DELTA_GAINED, DELTA_METRIC, DELTA_NEXTHOPS, DELTA_OTHER)], 1)
    nz = torch.nonzero(kind)                              # row-major: (job, prefix) order
    k = kind[nz[:, 0], nz[:, 1]]
    metric = torch.where(k == DELTA_LOST, bm.expand(n, P)[nz[:, 0], nz[:, 1]], jm[nz[:, 0], nz[:, 1]])
    return counts, nz, metric, k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--jobs", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch = stage_bench.require_gpu("route_delta_stage.py")
    from bench import adjacency_edges
    from holo_b200 import capi, isis, synth
    from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
    from isis_synth import synth_instance
    from test_isis_route_cells_gpu import DeviceTopology

    t = synth.random_topology(10000, 40000, synth.SEED_BASE + 3, cost_lo=1, cost_hi=1000)
    inst = synth_instance(t, 0)
    f = isis.Flat(isis.synth_level(t))
    csr = f.csr
    root = f.vertex(isis.sysid(0) << 8)
    pair = adjacency_edges(csr, t, lambda i: f.vertex(isis.sysid(int(i)) << 8))
    n = args.jobs
    ov = [[(pair[j % len(pair)][0], capi.COST_DISABLED), (pair[j % len(pair)][1], capi.COST_DISABLED)] for j in range(n)]

    ctx = capi.Context(0)
    dev = torch.device("cuda", 0)
    rt = isis.RouteTable(inst)
    assert rt.root[isis.TOPO_STD] == root and rt.n_vertices[isis.TOPO_STD] == csr.n_vertices
    assert rt.root[isis.TOPO_MT6] == isis.NO_ROOT
    rt.upload(ctx)
    V, P, K = csr.n_vertices, rt.n_prefixes, rt.n_contributors
    base_top = DeviceTopology(ctx, csr, root, 1)
    base_top.run()
    base = torch.empty(P * 24, dtype=torch.uint8, device=dev)
    isis.routes_batch_device(ctx, rt, 1, base_top.rs, None, base.data_ptr())
    top = DeviceTopology(ctx, csr, root, n, ov)
    top.run()
    rs, status = top.rs, top.status
    cells = torch.empty(n * P * 24, dtype=torch.uint8, device=dev)
    job_out = torch.empty(n * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device=dev)
    total = torch.zeros(1, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()

    def run_cells():
        isis.routes_batch_device(ctx, rt, n, rs, None, cells.data_ptr())

    def run_delta(records=None, cap=0):
        isis.routes_delta_device(ctx, rt, n, rs, None, base.data_ptr(), 1, 0, job_out.data_ptr(),
                                 records.data_ptr() if records is not None else 0, cap, total.data_ptr())

    run_delta()
    ctx.sync()
    n_changes = int(total.item())
    records = torch.empty(max(n_changes, 1) * DELTA_DT.itemsize, dtype=torch.uint8, device=dev)
    variants = {"cells": run_cells, "delta_summary": run_delta, "delta_records": lambda: run_delta(records, n_changes)}
    ms = stage_bench.time_alternating(ctx, variants, args.reps, 3)

    # ---- outside the timed region: the delta against torch's comparison of the stored cells, every job
    run_cells()
    run_delta(records, n_changes)
    ctx.sync()
    counts, nz, metric, kind = torch_delta(cells, base, n, P)
    jo = job_out.view(torch.int32).view(n, 8)
    rec = records[: n_changes * DELTA_DT.itemsize].view(torch.int32).view(n_changes, 4)
    check = {
        "total": int(total.item()) == len(kind),
        "summaries": bool((jo[:, :6] == counts.to(torch.int32)).all().item()) and bool((jo[:, 6] == status).all().item()),
        "records": (len(kind) == n_changes and bool((rec[:, 0] == nz[:, 0].to(torch.int32)).all().item())
                    and bool((rec[:, 1] == nz[:, 1].to(torch.int32)).all().item())
                    and bool((rec[:, 2] == metric.to(torch.int32)).all().item())
                    and bool(((rec[:, 3] & 0xFF) == kind).all().item())),
    }
    check["jobs"] = n
    ok = check["total"] and check["summaries"] and check["records"]
    per_job = jo[:, 0].cpu().numpy()
    kinds = {name: int(jo[:, i].sum().item()) for i, name in enumerate(("changed", "lost", "gained", "metric", "nexthops", "other"))}

    card, power = stage_bench.card_and_power()
    n_tiles = (n * P + 31) // 32
    contrib = n * (K * 16 + P * 8)                            # every job reads its prefixes' records and offsets
    gathers = n * K * 14                                      # dist + hops + nh_mask of each contributor's vertex
    cell_bytes = n * P * 24
    base_reads = n * P * 24                                   # each job's cells are compared with a base row (L2)
    summary_bytes = n * DELTA_JOB_DT.itemsize
    bytes_moved = {
        "cells": {"contributors": contrib, "plane_gathers": gathers, "cell_writes": cell_bytes},
        "delta_summary": {"contributors": contrib, "plane_gathers": gathers, "base_reads": base_reads,
                          "summaries": summary_bytes},
        "delta_records": {"contributors": 2 * contrib, "plane_gathers": 2 * gathers, "base_reads": 2 * base_reads,
                          "summaries": summary_bytes, "tile_counts_and_offsets": n_tiles * (1 + 8) * 2,
                          "records": n_changes * DELTA_DT.itemsize,
                          "note": "pass B re-reads contributors, planes and base only for tiles with changes; "
                                  "the factor 2 is the upper bound"},
    }
    med = {k: float(np.median(v)) for k, v in ms.items()}
    out = {
        "workload": f"C3 routes delta: IS-IS L2 synthetic LSDB, 10000 systems / 40000 directed adjacencies, wide metrics "
                    f"U[1,1000], {n} what-if jobs of one root (job j removes adjacency j mod {len(pair)}), "
                    f"2 /32 prefixes per system, base row = the root's plain SPT",
        "seed": hex(synth.SEED_BASE + 3),
        "card": card, "power_limit": power,
        "jobs": n, "prefixes": P, "contributors": K, "vertices": V, "reps": args.reps,
        "refused_jobs": int((status != 0).sum().item()),
        "ms": {k: {"median": med[k], "min": float(min(v)), "max": float(max(v))} for k, v in ms.items()},
        "delta_over_cells": {"summary": med["delta_summary"] / med["cells"], "records": med["delta_records"] / med["cells"]},
        "changes": {"total": n_changes, **kinds,
                    "jobs_with_changes": int((per_job > 0).sum()),
                    "per_job": {"min": int(per_job.min()), "median": float(np.median(per_job)),
                                "p90": float(np.percentile(per_job, 90)), "p99": float(np.percentile(per_job, 99)),
                                "max": int(per_job.max())}},
        "bytes_per_launch": bytes_moved,
        "datasheet_bw_GBps": DATASHEET_GBS,
        "cross_check_against_torch": check,
    }
    stage_bench.write_json(out, args.out)
    del base_top, top
    ctx.close()
    if not ok:
        sys.exit("the delta differs from torch's comparison of the stored cells")


if __name__ == "__main__":
    main()
