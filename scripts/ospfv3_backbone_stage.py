#!/usr/bin/env python
"""The backbone-router stage over OSPFv3 tables (hspf_ospfv2_backbone_cells / hspf_ospfv2_backbone_delta on a table of
hspf_ospfv3_backbone_table_create) on a 10 000-job what-if batch inside one non-backbone area; device only:
python scripts/ospfv3_backbone_stage.py [--jobs 10000] [--reps 10] [--out profiles/h100_C5v3_backbone.json]

Domain (ospfv3.backbone_view, seed 0xC5): C5's topology (10 000 routers, 5 % of adjacencies on LANs, costs {10, 20}) as
OSPFv3 area 0, one 2 000-router area, three area border routers ("borders", the first also in a 12-router area 2),
backbone router R = router 0 of area 0.  Job 0 is unperturbed; job j > 0 disables one router-to-router link of area 1
(both directions).  Each border runs its areas' SPT batches (one row per job in area 1, one row elsewhere) and its ABR
cells (hspf_ospfv2_abr_rib_cells over its OSPFv3 ABR table); the backbone calls read those cells in place with R's one
area-0 row.

The launch bound of the OSPFv3 instantiation (kBackboneV3BlocksPerSM in csrc/ospfv2_backbone.cu) is timed against the
other bound in the same run: a second copy of the library, built into a temporary directory with the other value (and
-Xptxas -v, whose register and spill lines for the OSPFv3 kernels are recorded), runs the same calls on the same table
data, planes and border cells, alternating with the first.  CUDA-event medians over `--reps` alternating launches after
warm-up; the card's name and power limit are read (not set) in the same run.  Outside the timed region: both builds'
cells are byte-identical and the delta's total equals a count over the stored cells.  Host figure (a CPU
measurement): per job, the host chain the stage replaces (each border's area_from_planes + update_rib_full_v3 +
net_summaries_v3, then R's update_rib_full_v3), timed over a few jobs."""
import argparse
import ctypes as C
import time

import numpy as np

import stage_bench

BOUND = ("ospfv2_backbone.cu", "kBackboneV3BlocksPerSM")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--jobs", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--host-jobs", type=int, default=2)
    args = ap.parse_args()
    torch = stage_bench.require_gpu("ospfv3_backbone_stage.py")
    from holo_b200 import capi, ospf_rib, ospfv3, route_table, synth
    from holo_b200.route_table import DELTA_JOB_DT, DELTA_DT
    from test_isis_route_cells_gpu import DeviceTopology

    t0 = synth.random_topology(10000, 40000, synth.SEED_BASE + 5, cost_choices=[10, 20], lan_fraction=0.05)
    t1 = synth.random_topology(2000, 8000, synth.SEED_BASE + 850, cost_choices=[10, 20], lan_fraction=0.05)
    v = ospfv3.backbone_view(t0, t1, 0xC5)
    ctx = capi.Context(0)
    dev = torch.device("cuda", 0)
    n = args.jobs
    rng = np.random.default_rng(0xC5)
    keep = []

    # the jobs: one link of the area per job, named by its end points' ids
    bareas = [b[0] for b in v["borders"]]
    i1 = [b[1].index(1) for b in v["borders"]]
    f1 = ospfv3.Flat(bareas[0][i1[0]])
    src = np.repeat(np.arange(f1.csr.n_vertices), np.diff(f1.csr.row_ptr))
    links = sorted({tuple(sorted((int(f1.router_ids[src[e]]), int(f1.router_ids[f1.csr.col[e]]))))
                    for e in range(f1.csr.n_edges) if f1.is_router[src[e]] and f1.is_router[f1.csr.col[e]]})
    job_links = [None] + [links[int(rng.integers(len(links)))] for _ in range(n - 1)]
    tables, border_cells, flats_all, tops_all = [], [], [], []
    for b, (areas, ids, sums) in enumerate(v["borders"]):
        flats = [ospfv3.Flat(a) for a in areas]
        rt = ospf_rib.AbrRibTable(areas[0].router_id, flats, ids, sums, None, v["externals"])
        rt.upload(ctx)
        f = flats[i1[b]]
        s = np.repeat(np.arange(f.csr.n_vertices), np.diff(f.csr.row_ptr))
        by_pair = {}
        for e in range(f.csr.n_edges):
            if f.is_router[s[e]] and f.is_router[f.csr.col[e]]:
                by_pair.setdefault(tuple(sorted((int(f.router_ids[s[e]]), int(f.router_ids[f.csr.col[e]])))), []).append(e)
        rs_list, n_rows, tops = [], [], []
        for i, fl in enumerate(flats):
            root = fl.router_vertex(areas[0].router_id)
            ov = [[]] if i != i1[b] else [[(e, capi.COST_DISABLED) for e in by_pair.get(l, [])] if l else [] for l in job_links]
            top = DeviceTopology(ctx, fl.csr, root, len(ov), ov)
            top.run()
            rs_list.append(top.rs); n_rows.append(top.n); tops.append(top)
        rows = np.zeros((n, len(areas)), np.uint32)
        rows[:, i1[b]] = np.arange(n)
        d_rows = torch.from_numpy(rows.view(np.int32).reshape(-1).copy()).to(dev)
        cells = torch.empty(n * rt.n_prefixes * 24, dtype=torch.uint8, device=dev)
        ospf_rib.abr_rib_cells_device(ctx, rt, n, rs_list, n_rows, d_rows.data_ptr(), cells.data_ptr())
        keep += [d_rows, rs_list]
        tables.append(rt); border_cells.append(cells); flats_all.append(flats); tops_all.append(tops)
    r_area = v["r_area"]
    r_flat = ospfv3.Flat(r_area)
    rv = r_flat.router_vertex(r_area.router_id)
    rtop = DeviceTopology(ctx, r_flat.csr, rv, 1, [[]])
    rtop.run()
    rs_r = rtop.rs
    bt = ospf_rib.BackboneTable(r_flat, r_area.router_id, v["summaries0"], v["externals"], tables)
    bt.upload(ctx)
    ctx.sync()
    P = bt.n_prefixes
    bc = [c.data_ptr() for c in border_cells]

    cur = stage_bench.launch_bound(*BOUND)
    other = 8 if cur == 4 else 4
    lib_path, log = stage_bench.build_variant(*BOUND, other, "backbone_v3_bound_", ptxas=True)
    regs_other = stage_bench.ptxas_registers(log, lambda k: "WalkBackboneV3" in k)
    libv = C.CDLL(str(lib_path))
    route_table.declare(libv)
    # the variant's own tables over the same images
    vt = []
    for b, (areas, ids, sums) in enumerate(v["borders"]):
        rt = tables[b]
        fl_, ids_, sp_, ns_, act_, _s, ext_, _f = rt._keep
        h = C.c_void_p()
        assert libv.hspf_ospfv3_abr_ribtable_create(rt.router_id, len(areas), fl_, ids_.ctypes.data, sp_, ns_.ctypes.data,
                                                    act_.ctypes.data, ext_.ctypes.data, len(ext_), C.byref(h)) == 0
        vt.append(h)
    hv = C.c_void_p()
    sm, ex = bt.summaries, bt.externals
    arr = (C.c_void_p * len(vt))(*[h.value for h in vt])
    assert libv.hspf_ospfv3_backbone_table_create(r_flat.handle, r_area.router_id, sm.ctypes.data, len(sm), ex.ctypes.data,
                                                  len(ex), arr, len(vt), C.byref(hv)) == 0
    assert libv.hspf_ospfv2_backbone_table_upload(ctx.handle, hv) == 0
    handles = {cur: (ctx.lib, bt.handle), other: (libv, hv)}
    cells = {b: torch.empty(n * P * 24, dtype=torch.uint8, device=dev) for b in (4, 8)}
    job_out = torch.zeros(n * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device=dev)
    total = torch.zeros(1, dtype=torch.int64, device=dev)
    bca = (C.c_void_p * len(bc))(*bc)

    def cell_launch(b):
        lib, h = handles[b]
        return lambda: lib.hspf_ospfv2_backbone_cells(ctx.handle, h, n, C.byref(rs_r), bca, None, None, cells[b].data_ptr())

    cell_launch(4)(); cell_launch(8)()
    ctx.sync()
    same_bounds = bool(torch.equal(cells[4], cells[8]))
    base = cells[cur][: P * 24].clone()
    lib, h = handles[cur]
    assert lib.hspf_ospfv2_backbone_delta(ctx.handle, h, n, C.byref(rs_r), bca, None, base.data_ptr(), 1, None,
                                          job_out.data_ptr(), None, 0, total.data_ptr()) == 0
    ctx.sync()
    cap = int(total.cpu()[0])
    w = cells[cur].view(torch.int64).reshape(n, P, 3)
    changed = int((w != w[0:1]).any(dim=2).sum().item())
    recs = torch.empty(max(cap, 1) * DELTA_DT.itemsize, dtype=torch.uint8, device=dev)

    def delta(b, with_records):
        lib, h = handles[b]
        return lambda: lib.hspf_ospfv2_backbone_delta(ctx.handle, h, n, C.byref(rs_r), bca, None, base.data_ptr(), 1, None,
                                                      job_out.data_ptr(), recs.data_ptr() if with_records else None,
                                                      cap if with_records else 0, total.data_ptr())

    work = {}
    for b in (4, 8):
        work[f"backbone_cells_bound{b}"] = cell_launch(b)
        work[f"backbone_delta_summaries_bound{b}"] = delta(b, False)
        work[f"backbone_delta_records_bound{b}"] = delta(b, True)
    med = {k: float(np.median(x)) for k, x in stage_bench.time_alternating(ctx, work, args.reps, 2).items()}

    # host chain per job (CPU), over the device planes read back
    host_ms = []
    rp = rtop.planes(0)
    for j in range(1, 1 + args.host_jobs):
        t = time.perf_counter()
        new = [s for s in v["summaries0"] if int(s["adv_rtr"]) not in {int(x.router_id) for x in tables}]
        for b, (areas, ids, sums) in enumerate(v["borders"]):
            ra = []
            for i, a in enumerate(areas):
                spf = stage_bench.spf_from_planes("ospfv3", a, tops_all[b][i].planes(j if i == i1[b] else 0))
                ra.append(ospf_rib.RibArea(a.area_id, spf, a.ifaces, sums[i], True))
            rid = areas[0].router_id
            rib = ospf_rib.update_rib_full_v3(rid, areas[0].max_paths, ra, v["externals"])
            new += list(ospf_rib.net_summaries_v3(rid, rib, ra, [ospf_rib.area_config()] * len(areas), ids.index(0)))
        s = np.array(new, ospf_rib.INTER_AREA_LSA_DT)
        s = s[np.lexsort((s["lsa_id"], s["adv_rtr"], s["lsa_type"]))]
        r_spf = stage_bench.spf_from_planes("ospfv3", r_area, rp)
        ospf_rib.update_rib_full_v3(r_area.router_id, r_area.max_paths, [ospf_rib.RibArea(0, r_spf, r_area.ifaces, s, True)],
                                    v["externals"])
        host_ms.append((time.perf_counter() - t) * 1e3)

    card, power = stage_bench.card_and_power()
    out = {
        "stage": "hspf_ospfv2_backbone_cells / hspf_ospfv2_backbone_delta over an hspf_ospfv3_backbone_table_create table",
        "workload": {"area0": "C5 as OSPFv3: 10000 routers, 40000 links, costs {10, 20}, 5 % LANs",
                     "area1": "2000 routers", "area2": "12 routers, first border only",
                     "borders": len(tables), "jobs": n, "affected_prefixes": P, "slots": bt.n_slots,
                     "border_keys": [t.n_prefixes for t in tables]},
        "card": card, "power_limit": power, "reps": args.reps, "median_ms": med, "launch_bound": cur,
        "other_bound": other, "cells_equal_other_bound": same_bounds, "ptxas_other_bound": regs_other,
        "delta_total": cap, "delta_total_equals_changed_cells": cap == changed,
        "host_chain_ms_per_job": float(np.median(host_ms)), "host_jobs_timed": len(host_ms),
        "note": "device figures are CUDA-event medians of alternating launches; the host chain is a CPU figure",
    }
    stage_bench.write_json(out, args.out)


if __name__ == "__main__":
    main()
