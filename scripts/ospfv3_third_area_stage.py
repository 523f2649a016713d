#!/usr/bin/env python
"""The OSPFv3 stage of an internal router of a non-backbone area over what-if jobs inside another non-backbone area
(hspf_ospfv3_abr_backbone_asbr_entries, hspf_ospfv2_third_area_cells / hspf_ospfv2_third_area_delta over an
hspf_ospfv3_third_area_table_create table) on a 10 000-job what-if batch inside area 1; device only:
python scripts/ospfv3_third_area_stage.py [--jobs 10000] [--reps 10] [--out profiles/h100_C5v3_third_area.json]

Domain (ospfv3.third_area_view, seed 0xC5, n_c=2, area1_asbrs=2, area1_ext=1000): C5's topology as OSPFv3 area 0, a
2 000-router area 1 with three area border routers (B, the first also in a small area 2) and two ASBRs with about
1 000 AS-external LSAs each, and a 2 000-router area 3 (R's area; area 2 is the first B's) with two area border routers
(C) and R, an internal router of area 3.  Job 0 is unperturbed; job j > 0 disables one router-to-router link of area 1
(both directions).  The whole chain runs on the device: each B's area SPT batches (one row per job in area 1) and ABR
cells (hspf_ospfv2_abr_rib_cells); each C's row 0, OSPFv3 abr_backbone cells and ASBR entries over them; R's row 0,
then R's calls over the C's cells and entries.

The launch bound of R's kernels (kThirdAreaV3BlocksPerSM in csrc/ospfv2_backbone.cu) is timed against the other bound
in the same run: a second copy of the library, built into a temporary directory with the other value, runs the same
calls on its own copy of R's table over the same C tables, planes, cells and entries, alternating with the first.
The entries call is timed in the same loop.  CUDA-event medians over `--reps` alternating launches after warm-up; the
card's name and power limit are read (not set) in the same run, with the device memory the run holds.  Outside the
timed region: both builds' cells are byte-identical and the delta's total equals a count over the stored cells.  Host
figure (a CPU measurement): per job, the host chain the stage replaces (each B's area_from_planes + update_rib_full_v3
+ net and rtr summaries into area 0, each C's over those into area 3, then R's update_rib_full_v3), timed over a few
jobs."""
import argparse
import ctypes as C
import time

import numpy as np

import stage_bench

BOUND = ("ospfv2_backbone.cu", "kThirdAreaV3BlocksPerSM")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--jobs", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--host-jobs", type=int, default=2)
    args = ap.parse_args()
    torch = stage_bench.require_gpu("ospfv3_third_area_stage.py")
    from holo_b200 import capi, ospf_rib, ospfv3, route_table, synth
    from holo_b200.route_table import DELTA_JOB_DT, DELTA_DT
    from test_isis_route_cells_gpu import DeviceTopology

    ctx = capi.Context(0)
    dev = torch.device("cuda", 0)
    n = args.jobs
    rng = np.random.default_rng(0xC5)
    keep = []

    t0 = synth.random_topology(10000, 40000, synth.SEED_BASE + 5, cost_choices=[10, 20], lan_fraction=0.05)
    t1 = synth.random_topology(2000, 8000, synth.SEED_BASE + 850, cost_choices=[10, 20], lan_fraction=0.05)
    t3 = synth.random_topology(2000, 8000, synth.SEED_BASE + 851, cost_choices=[10, 20], lan_fraction=0.05)
    v = ospfv3.third_area_view(t0, t1, t3, 0xC5, stage_bench.root_spf(ctx), n_c=2, area1_asbrs=2, area1_ext=1000)

    # the jobs: one router-to-router link of area 1 per job, named by its end points' ids
    i1 = [b[1].index(1) for b in v["borders"]]
    f1 = ospfv3.Flat(v["borders"][0][0][i1[0]])
    src = np.repeat(np.arange(f1.csr.n_vertices), np.diff(f1.csr.row_ptr))
    links = sorted({tuple(sorted((int(f1.router_ids[src[e]]), int(f1.router_ids[f1.csr.col[e]]))))
                    for e in range(f1.csr.n_edges) if f1.is_router[src[e]] and f1.is_router[f1.csr.col[e]]})
    job_links = [None] + [links[int(rng.integers(len(links)))] for _ in range(n - 1)]
    tables, border_cells, tops_all, border_rs, border_nrows, border_rows = [], [], [], [], [], []
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
        border_rs.append(rs_list)
        border_nrows.append(n_rows)
        border_rows.append(d_rows.data_ptr())
        tables.append(rt); border_cells.append(cells); tops_all.append(tops)
    bc = [c.data_ptr() for c in border_cells]
    # the C's: row 0 of each area, OSPFv3 abr_backbone cells over the B's, and their ASBR entries
    ctables, c_rs, c_tops, c_cells, c_ent, c_est = [], [], [], [], [], []
    for areas, ids, sums in v["c_areas"]:
        flats = [ospfv3.Flat(a) for a in areas]
        tops = [DeviceTopology(ctx, f.csr, f.router_vertex(a.router_id), 1, [[]]) for a, f in zip(areas, flats)]
        for top in tops:
            top.run()
        rl = [top.rs for top in tops]
        ct = ospf_rib.AbrBackboneTable(areas[0].router_id, flats, ids, sums, None, v["externals"], tables)
        assert ct.v3
        ct.upload(ctx)
        out = torch.empty(n * ct.n_prefixes * 24, dtype=torch.uint8, device=dev)
        ospf_rib.abr_backbone_cells_device(ctx, ct, n, rl, bc, None, border_rs, border_nrows, border_rows, 0,
                                           out.data_ptr())
        G = len(ct.asbr_ids)
        assert G > 0
        ent = torch.empty(n * G, dtype=torch.int32, device=dev)
        est = torch.empty(n, dtype=torch.int32, device=dev)
        ospf_rib.abr_backbone_asbr_entries_device(ctx, ct, n, rl, border_rs, border_nrows, border_rows, est.data_ptr(),
                                                  ent.data_ptr())
        ctables.append(ct); c_rs.append(rl); c_tops.append(tops); c_cells.append(out); c_ent.append(ent); c_est.append(est)
    ra = v["r_area"]
    rf = ospfv3.Flat(ra)
    rtop = DeviceTopology(ctx, rf.csr, rf.router_vertex(ra.router_id), 1, [[]])
    rtop.run()
    r_rs = rtop.rs
    tt = ospf_rib.BackboneTable(rf, ra.router_id, v["summaries3"], v["externals"], ctables,
                                config=ospf_rib.area_config())
    assert tt.v3 and tt.third_area and tt.n_asbr_slots > 0
    tt.upload(ctx)
    ctx.sync()
    assert not any(x.any().item() for x in c_est)
    P = tt.n_prefixes

    cur = stage_bench.launch_bound(*BOUND)
    other = 8 if cur == 4 else 4
    libv = C.CDLL(str(stage_bench.build_variant(*BOUND, other, "third_area_v3_bound_")))
    route_table.declare(libv)
    # the variant's own copy of R's table, over the same flat and C tables
    hv = C.c_void_p()
    carr = (C.c_void_p * len(ctables))(*[x.handle.value for x in ctables])
    sm, ext = tt.summaries, tt.externals
    assert libv.hspf_ospfv3_third_area_table_create(rf.handle, ra.router_id, tt.config.ctypes.data, sm.ctypes.data,
                                                    len(sm), ext.ctypes.data, len(ext), carr, len(ctables),
                                                    C.byref(hv)) == 0
    assert libv.hspf_ospfv2_backbone_table_upload(ctx.handle, hv) == 0
    handles = {cur: (ctx.lib, tt.handle), other: (libv, hv)}
    cells = {b: torch.empty(n * P * 24, dtype=torch.uint8, device=dev) for b in (4, 8)}
    job_out = torch.zeros(n * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device=dev)
    total = torch.zeros(1, dtype=torch.int64, device=dev)
    cca = (C.c_void_p * len(c_cells))(*[x.data_ptr() for x in c_cells])
    cea = (C.c_void_p * len(c_ent))(*[x.data_ptr() for x in c_ent])
    cesa = (C.c_void_p * len(c_est))(*[x.data_ptr() for x in c_est])

    def cell_launch(b):
        lib, h = handles[b]
        return lambda: lib.hspf_ospfv2_third_area_cells(ctx.handle, h, n, C.byref(r_rs), cca, None, cea, cesa, None,
                                                        cells[b].data_ptr())

    assert cell_launch(4)() == 0 and cell_launch(8)() == 0
    ctx.sync()
    same_bounds = bool(torch.equal(cells[4], cells[8]))
    base = cells[cur][: P * 24].clone()
    lib, h = handles[cur]
    assert lib.hspf_ospfv2_third_area_delta(ctx.handle, h, n, C.byref(r_rs), cca, None, cea, cesa, base.data_ptr(), 1,
                                            None, job_out.data_ptr(), None, 0, total.data_ptr()) == 0
    ctx.sync()
    cap = int(total.cpu()[0])
    w = cells[cur].view(torch.int64).reshape(n, P, 3)
    changed = int((w != w[0:1]).any(dim=2).sum().item())
    recs = torch.empty(max(cap, 1) * DELTA_DT.itemsize, dtype=torch.uint8, device=dev)
    entries_moved = int(sum(int((e.reshape(n, -1) != e.reshape(n, -1)[0:1]).any(dim=1).sum().item()) for e in c_ent))
    # cells whose winner differs from job 0's at an equal metric and path (the two-hop options chain among them)
    wi = cells[cur].view(torch.int32).reshape(n, P, 6)
    same_mpf = (wi[:, :, 5] == wi[0:1, :, 5]) & (wi[:, :, 4] != wi[0:1, :, 4])
    options_moved = int(same_mpf.sum().item())

    def delta(b, with_records):
        lib, h = handles[b]
        return lambda: lib.hspf_ospfv2_third_area_delta(ctx.handle, h, n, C.byref(r_rs), cca, None, cea, cesa,
                                                        base.data_ptr(), 1, None, job_out.data_ptr(),
                                                        recs.data_ptr() if with_records else None,
                                                        cap if with_records else 0, total.data_ptr())

    def entries(k):
        ct, rl = ctables[k], c_rs[k]
        return lambda: ospf_rib.abr_backbone_asbr_entries_device(ctx, ct, n, rl, border_rs, border_nrows, border_rows,
                                                                 c_est[k].data_ptr(), c_ent[k].data_ptr())

    work = {f"asbr_entries_c{k}": entries(k) for k in range(len(ctables))}
    for b in (4, 8):
        work[f"third_area_cells_bound{b}"] = cell_launch(b)
        work[f"third_area_delta_summaries_bound{b}"] = delta(b, False)
        work[f"third_area_delta_records_bound{b}"] = delta(b, True)
    med = {k: float(np.median(x)) for k, x in stage_bench.time_alternating(ctx, work, args.reps, 2).items()}
    held = torch.cuda.memory_allocated(dev)
    free, total_mem = torch.cuda.mem_get_info()

    # host chain per job (CPU), over the device planes read back
    host_ms = []
    cp = [[top.planes(0) for top in tops] for tops in c_tops]
    rp = rtop.planes(0)
    bids = {int(x.router_id) for x in tables}
    cids = {int(x.router_id) for x in ctables}
    for j in range(1, 1 + args.host_jobs):
        t = time.perf_counter()
        new0 = [tuple(s) for s in v["c_areas"][0][2][0].tolist() if int(s[0]) not in bids]
        for b, (areas, ids, sums) in enumerate(v["borders"]):
            rab = []
            for i, a in enumerate(areas):
                spf = stage_bench.spf_from_planes("ospfv3", a, tops_all[b][i].planes(j if i == i1[b] else 0))
                rab.append(ospf_rib.RibArea(a.area_id, spf, a.ifaces, sums[i], True))
            rid = areas[0].router_id
            new0 += ospfv3.nonbackbone_lsas(rid, areas[0].max_paths, rab, v["externals"], ids.index(0))
        s0 = np.array(new0, ospf_rib.INTER_AREA_LSA_DT)
        s0 = s0[np.lexsort((s0["lsa_id"], s0["adv_rtr"], s0["lsa_type"]))]
        new3 = [tuple(s) for s in v["summaries3"].tolist() if int(s[0]) not in cids]
        for (areas, ids, sums), pls in zip(v["c_areas"], cp):
            rac = [ospf_rib.RibArea(a.area_id, stage_bench.spf_from_planes("ospfv3", a, p), a.ifaces,
                                    s0 if a.area_id == 0 else ss, True) for a, p, ss in zip(areas, pls, sums)]
            rid = areas[0].router_id
            new3 += ospfv3.nonbackbone_lsas(rid, areas[0].max_paths, rac, v["externals"], ids.index(3))
        s3 = np.array(new3, ospf_rib.INTER_AREA_LSA_DT)
        s3 = s3[np.lexsort((s3["lsa_id"], s3["adv_rtr"], s3["lsa_type"]))]
        r_spf = stage_bench.spf_from_planes("ospfv3", ra, rp)
        ospf_rib.update_rib_full_v3(ra.router_id, ra.max_paths, [ospf_rib.RibArea(3, r_spf, ra.ifaces, s3, True)],
                                    v["externals"])
        host_ms.append((time.perf_counter() - t) * 1e3)

    card, power = stage_bench.card_and_power()
    out = {
        "stage": "hspf_ospfv3_abr_backbone_asbr_entries, hspf_ospfv2_third_area_cells / hspf_ospfv2_third_area_delta "
                 "(hspf_ospfv3_third_area_table_create)",
        "workload": {"area0": "C5: 10000 routers, 40000 links, costs {10, 20}, 5 % LANs", "area1": "2000 routers",
                     "area3": "2000 routers (R's area)", "area1_asbrs": len(v["area1_asbrs"]),
                     "externals": len(v["externals"]), "b_borders": len(tables), "c_borders": len(ctables),
                     "jobs": n, "affected_prefixes": P, "slots": tt.n_slots, "chain_slots": tt.n_asbr_slots,
                     "c_keys": [x.n_prefixes for x in ctables], "c_asbr_groups": [len(x.asbr_ids) for x in ctables],
                     "b_keys": [x.n_prefixes for x in tables]},
        "card": card, "power_limit": power, "reps": args.reps, "median_ms": med, "launch_bound": cur,
        "other_bound": other, "cells_equal_other_bound": same_bounds,
        "delta_total": cap, "delta_total_equals_changed_cells": cap == changed,
        "jobs_with_moved_entries": entries_moved, "cells_with_other_winner_at_equal_mpf": options_moved,
        "device_memory_allocated_gib": held / 2**30, "device_memory_in_use_gib": (total_mem - free) / 2**30,
        "host_chain_ms_per_job": float(np.median(host_ms)), "host_jobs_timed": len(host_ms),
        "note": "device figures are CUDA-event medians of alternating launches; the host chain is a CPU figure",
    }
    stage_bench.write_json(out, args.out)


if __name__ == "__main__":
    main()
