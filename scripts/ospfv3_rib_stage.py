#!/usr/bin/env python
"""The routing-table stages over an OSPFv3 area on a C5 what-if batch (hspf_ospfv3_ribtable_create's table through
hspf_ospfv2_rib_cells and hspf_ospfv2_rib_delta); device only.

C5's topology as OSPFv3 area 0.0.0.1 (ospfv3.synth_area) with inter-area and external load (ospfv3.inter_area_view,
seed 0xC5, the sizes scripts/ospf_rib_delta_stage.py gives the OSPFv2 batch).  One internal router whose atoms fit wide
planes with nh_words == 1 is the root of every job: job 0 has no override, job j > 0 disables one router-to-router link
in both directions, the links drawn with a fixed seed.  The base row is job 0's cells.  After one SPT batch, with CUDA
events over warmed launches on the engine's stream, alternating:
  (a) the SPT batch;
  (b) hspf_ospfv2_rib_cells (ospf_rib_cells_kernel): every cell stored;
  (c) hspf_ospfv2_rib_delta, summaries only (records NULL);
  (d) hspf_ospfv2_rib_delta with records (cap = the total).
Records the card's name and power limit, the times, and how the changes spread over jobs and kinds.  Outside the timed
region the delta is checked against a torch comparison of (b)'s cells with the base row, for every job (summaries,
total, every record), and sampled jobs are decoded (hspf_ospfv3_rib_from_cells) and their records tied to the decoded
tables.  Fails without a GPU.

    python scripts/ospfv3_rib_stage.py [--out FILE] [--jobs N] [--reps R]
"""
import argparse
import ctypes as C
import sys

import numpy as np

import stage_bench


def link_pairs(flat):
    """(e, reverse e) of every router-to-router link, each link once."""
    csr = flat.csr
    src = np.repeat(np.arange(csr.n_vertices), np.diff(csr.row_ptr)).tolist()
    col = csr.col.tolist()
    rtr = [bool(flat.is_router[src[e]] and flat.is_router[col[e]]) for e in range(csr.n_edges)]
    at = {(src[e], col[e]): e for e in range(csr.n_edges) if rtr[e]}
    return [(e, at[(col[e], src[e])]) for e in range(csr.n_edges) if rtr[e] and src[e] < col[e] and (col[e], src[e]) in at]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--jobs", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch = stage_bench.require_gpu("ospfv3_rib_stage.py")
    from holo_b200 import capi, ospf_rib, ospfv3, synth
    from ospf_rib_delta_stage import torch_delta
    from holo_b200.route_table import DELTA_DT, DELTA_GAINED, DELTA_JOB_DT, DELTA_LOST, DELTA_METRIC
    from test_isis_route_cells_gpu import DeviceTopology

    kw = dict(n_abr=16, n_asbr=16, n_inter=10000, n_ext=5000, n_overlap=3000, n_fresh=2000, n_ext_only=1000)
    t = synth.random_topology(10000, 40000, synth.SEED_BASE + 5, cost_choices=[10, 20], lan_fraction=0.05)

    def view(i):
        return ospfv3.inter_area_view(ospfv3.synth_area(t, root=i, area_id=1), 0xC5, **kw)

    area0, _, _ = view(0)
    flat0 = ospfv3.Flat(area0)
    flags = dict(zip(area0.router_lsas["adv_rtr"].tolist(), area0.router_lsas["flags"].tolist()))
    root_index = next(i for i in range(t.n_routers) if not flags[ospfv3.RID_BASE + i] & 1
                      and capi.atom_count(flat0.csr, flat0.router_vertex(ospfv3.RID_BASE + i)) <= 64)
    area, sums, ext = view(root_index)
    flat = ospfv3.Flat(area)
    csr = flat.csr
    V = csr.n_vertices
    rv = flat.router_vertex(area.router_id)
    pairs = link_pairs(flat)
    rng = np.random.default_rng(0xC5)
    n = args.jobs
    cut = [pairs[int(i)] for i in rng.integers(len(pairs), size=n - 1)]

    ctx = capi.Context(0)
    dev = torch.device("cuda", 0)
    rt = ospf_rib.RibTable(flat, 1, sums, ext)
    rt.upload(ctx)
    P = rt.n_prefixes
    top = DeviceTopology(ctx, csr, rv, n, [[]] + [[(e, capi.COST_DISABLED) for e in pr] for pr in cut])
    rs = top.rs
    d_roots = torch.full((n,), rv, dtype=torch.int32, device=dev)
    cells = torch.empty(n * P * 24, dtype=torch.uint8, device=dev)
    st_out = torch.zeros(n, dtype=torch.int32, device=dev)
    job_out = torch.empty(n * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device=dev)
    total = torch.zeros(1, dtype=torch.int64, device=dev)
    top.run()
    ctx.sync()
    # the base row: job 0's cells (no override)
    ospf_rib.rib_cells_device(ctx, rt, n, rs, d_roots.data_ptr(), cells.data_ptr(), st_out.data_ptr())
    base = cells[: P * 24].clone()

    def run_cells():
        ospf_rib.rib_cells_device(ctx, rt, n, rs, d_roots.data_ptr(), cells.data_ptr(), st_out.data_ptr())

    def delta_call(fn, records=None, cap=0):
        rc = fn(ctx.handle, rt.handle, n, C.byref(rs), d_roots.data_ptr(), base.data_ptr(), 1, None, job_out.data_ptr(),
                records.data_ptr() if records is not None else None, cap, total.data_ptr())
        if rc != capi.HSPF_OK:
            raise capi.HspfError(rc, ctx.last_error())

    fn_a = ctx.lib.hspf_ospfv2_rib_delta
    delta_call(fn_a)
    ctx.sync()
    n_changes = int(total.item())
    records = torch.empty(max(n_changes, 1) * DELTA_DT.itemsize, dtype=torch.uint8, device=dev)
    variants = {
        "spt_batch": lambda: ctx.run_device(top.g, top.js, rs, sync=False),
        "ospf_rib_cells_kernel": run_cells,
        "delta_summary": lambda: delta_call(fn_a),
        "delta_records": lambda: delta_call(fn_a, records, n_changes),
    }
    ms = stage_bench.time_alternating(ctx, variants, args.reps, 3)
    med = {k: float(np.median(v)) for k, v in ms.items()}

    # ---- outside the timed region: the delta against torch's comparison of the stored cells, every job
    check = {"jobs": n}
    ctx.run_device(top.g, top.js, rs, sync=True)
    run_cells()
    records.fill_(0xAB)
    delta_call(fn_a, records, n_changes)
    ctx.sync()
    jo_t, rec_t, tot = job_out.clone(), records.clone(), int(total.item())
    status = top.status.clone()
    counts, want = torch_delta(cells, base, n, P)
    jo = jo_t.view(torch.int32).view(n, 8)
    rec = rec_t[: n_changes * DELTA_DT.itemsize].view(torch.int32).view(n_changes, 4)
    check["total"] = tot == len(want) == n_changes
    check["summaries"] = (bool((jo[:, :6] == counts.to(torch.int32)).all().item())
                          and bool((jo[:, 6] == st_out).all().item()))
    check["records"] = len(want) == n_changes and bool((rec[:, :3] == want[:, :3]).all().item()) and \
        bool(((rec[:, 3] & 0xFF) == want[:, 3]).all().item())

    # ---- sampled jobs decoded; their records tied to the decoded tables
    host_cells = lambda j: cells[j * P * 24:(j + 1) * P * 24].cpu().numpy().view(ospf_rib.RIB_CELL_DT)
    nets = sorted({int(v) for v in csr.col[csr.row_ptr[rv]: csr.row_ptr[rv + 1]] if not flat.is_router[v]})
    nh = top.nh.view(n, V)
    key = lambda p, ln: (bytes(p["bytes"].tolist()), int(ln))
    index = {key(p, ln): i for i, (p, ln) in enumerate(zip(rt.prefix, rt.plen))}

    def table(j):
        m = nh[j].cpu().numpy().view(np.uint64)
        rib = ospf_rib.rib_from_cells_v3(area, rt, host_cells(j), np.asarray(nets, np.uint32), m[nets])
        if rib.rc != capi.HSPF_OK:
            return None
        return {index[key(r["prefix"], r["len"])]: int(r["metric"]) for r in rib.routes}

    rec_np = rec.cpu().numpy().view(np.uint32)
    base_rows = table(0)
    per_job = jo[:, 0].cpu().numpy()
    sample = sorted({1, 2, n // 3, n // 2, n - 1} | set(np.nonzero(per_job)[0][:3].tolist()))
    ties = []
    for j in sample:
        rows = table(j)
        if rows is None or base_rows is None:
            ties.append({"job": int(j), "decoded": False})
            continue
        r = rec_np[rec_np[:, 0] == j]
        kind = r[:, 3] & 0xFF
        ok = (set(r[kind == DELTA_LOST, 1].tolist()) == set(base_rows) - set(rows)
              and set(r[kind == DELTA_GAINED, 1].tolist()) == set(rows) - set(base_rows)
              and set(r[(kind & DELTA_METRIC) != 0, 1].tolist())
              == {p for p in set(base_rows) & set(rows) if base_rows[p] != rows[p]})
        ties.append({"job": int(j), "decoded": True, "records": int(len(r)), "equal": bool(ok)})
    check["sampled_decodes_tie"] = all(x.get("equal", False) for x in ties)

    card, power = stage_bench.card_and_power()
    kinds = {name: int(jo[:, i].sum().item()) for i, name in enumerate(("changed", "lost", "gained", "metric", "nexthops",
                                                                        "other"))}
    out = {
        "workload": f"C5 topology as OSPFv3 area 0.0.0.1 (ospfv3.synth_area: 10000 routers, 40000 directed adjacencies, "
                    f"costs {{10, 20}}, 5 % on LANs) with ospfv3.inter_area_view(seed 0xC5, {kw}); {n} what-if jobs of "
                    f"internal router {root_index} "
                    f"(vertex {rv}): job 0 plain, job j > 0 disables one router-to-router link in both directions "
                    f"(numpy default_rng(0xC5) over {len(pairs)} links); base row = job 0's cells",
        "card": card, "power_limit": power,
        "jobs": n, "vertices": V, "prefixes": P, "records_in_table": rt.n_contributors, "reps": args.reps,
        "refused_jobs": int((status != 0).sum().item()),
        "ms": {k: {"median": med[k], "min": float(min(v)), "max": float(max(v))} for k, v in ms.items()},
        "delta_over_cells": {k: med[k] / med["ospf_rib_cells_kernel"] for k in med if "delta" in k},
        "bytes": {"cells_stored": n * P * 24, "summaries": n * DELTA_JOB_DT.itemsize,
                  "records": n_changes * DELTA_DT.itemsize},
        "changes": {"total": n_changes, **kinds, "jobs_with_changes": int((per_job > 0).sum()),
                    "per_job": {"median": float(np.median(per_job)), "p99": float(np.percentile(per_job, 99)),
                                "max": int(per_job.max())}},
        "cross_check_against_torch": check,
        "sampled_decodes": ties,
    }
    stage_bench.write_json(out, args.out)
    ctx.close()
    if not (check["total"] and check["summaries"] and check["records"] and check["sampled_decodes_tie"]):
        sys.exit("ospfv3_rib_stage.py: a cross-check failed")


if __name__ == "__main__":
    main()
