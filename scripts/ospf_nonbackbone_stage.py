#!/usr/bin/env python
"""The OSPFv2 stage of an internal router of a non-backbone area over what-if jobs on the backbone
(hspf_ospfv2_nonbackbone_table_create through hspf_ospfv2_backbone_asbr_cells / _delta) on a what-if batch of area-0
link failures and re-costings; device only:
python scripts/ospf_nonbackbone_stage.py [--jobs 10000] [--reps 10] [--out profiles/h100_C5_nonbackbone.json]

Domain (ospfv2.nonbackbone_view, seed 0xC5, n_ext=2000): scripts/ospf_backbone_stage.py's C5 domain (C5's LSDB as
area 0, one 2 000-router area 1, three area border routers ("borders")) seen from R = the first non-border router of
area 1.  The area-0 ASBR advertises about 2 000 type-5 LSAs of both E-bit values, so that R's type-4 slots read the
borders' area-0 rows; area 1's type-3/4 LSAs are the borders' net_summaries at the unperturbed job.  (The area-1
ASBRs of scripts/ospf_backbone_asbr_stage.py are left out: another border's type-4 LSA for them in area 0 would be an
inter-area router entry at a border, which the create refuses.)  Job 0 is unperturbed; job j > 0 disables one
router-to-router link of area 0 (both directions) or re-costs it to 35, seeded.  The jobs run as far as the borders'
cells fit beside the planes and two copies of R's cells; the run prints the device memory it holds.  Each border runs
its area-0 SPT batch (one row per job) and one row of area 1, then its ABR cells (hspf_ospfv2_abr_rib_cells); R's
calls read those cells and the borders' area-0 rows in place with R's one area-1 row.

The launch bound of the new kernels (kNonBackboneBlocksPerSM in csrc/ospfv2_backbone.cu) is timed against the other
bound in the same run: a second copy of the library, built into a temporary directory with the other value, runs the
same calls on the same table data, planes and border cells, alternating with the first.  CUDA-event medians over
`--reps` alternating launches after warm-up, also for the borders' area-0 SPT batch and their ABR cells; the card's
name and power limit are read (not set) in the same run.  Outside the timed region: both builds' cells are
byte-identical and the delta's total equals a count over the stored cells.  Host figure (a CPU measurement): per job,
the host chain the stage replaces (each border's area_from_planes + update_rib_full + router tables + net_summaries
into area 1, type 3 and type 4, then R's update_rib_full), timed over a few jobs."""
import argparse
import ctypes as C
import sys
import time

import numpy as np

import stage_bench

BOUND = ("ospfv2_backbone.cu", "kNonBackboneBlocksPerSM")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--jobs", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--host-jobs", type=int, default=2)
    ap.add_argument("--v0", type=int, default=10000, help="area-0 routers (C5: 10000)")
    ap.add_argument("--v1", type=int, default=2000, help="area-1 routers")
    args = ap.parse_args()
    torch = stage_bench.require_gpu("ospf_nonbackbone_stage.py")
    from holo_b200 import capi, ospf_rib, ospfv2, route_table, synth
    from holo_b200.route_table import DELTA_JOB_DT, DELTA_DT
    from test_isis_route_cells_gpu import DeviceTopology

    ctx = capi.Context(0)
    dev = torch.device("cuda", 0)

    t0 = synth.random_topology(args.v0, 4 * args.v0, synth.SEED_BASE + 5, cost_choices=[10, 20], lan_fraction=0.05)
    t1 = synth.random_topology(args.v1, 4 * args.v1, synth.SEED_BASE + 850, cost_choices=[10, 20], lan_fraction=0.05)
    v = ospfv2.nonbackbone_view(t0, t1, 0xC5, stage_bench.root_spf(ctx), n_ext=2000)
    rng = np.random.default_rng(0xC5)
    keep = []

    # the tables, R's table and the jobs' size before any batch: how many jobs fit
    tables, flats_all = [], []
    for areas, ids, sums in v["borders"]:
        flats = [ospfv2.Flat(a) for a in areas]
        rt = ospf_rib.AbrRibTable(areas[0].router_id, flats, ids, sums, None, v["externals"])
        rt.upload(ctx)
        tables.append(rt); flats_all.append(flats)
    r_area = v["r_area"]
    r_flat = ospfv2.Flat(r_area)
    rv = r_flat.router_vertex(r_area.router_id)
    bt = ospf_rib.BackboneTable(r_flat, r_area.router_id, v["summaries1"], v["externals"], tables,
                                config=ospf_rib.area_config())
    assert bt.n_asbr_slots > 0
    bt.upload(ctx)
    P = bt.n_prefixes
    i0 = [b[1].index(0) for b in v["borders"]]
    per_job = sum(f[i].csr.n_vertices * 14 + t.n_prefixes * 24 for f, i, t in zip(flats_all, i0, tables)) + 2 * P * 24
    free, _total = torch.cuda.mem_get_info()
    n = max(2, min(args.jobs, int(0.85 * free) // per_job))

    # the jobs: one area-0 router link per job, named by its end points' ids, disabled or re-costed to 35
    f0 = flats_all[0][i0[0]]
    src = np.repeat(np.arange(f0.csr.n_vertices), np.diff(f0.csr.row_ptr))
    links = sorted({tuple(sorted((int(f0.ids[src[e]]), int(f0.ids[f0.csr.col[e]])))) for e in range(f0.csr.n_edges)
                    if f0.link_index[e] != 0xFFFFFFFF and f0.is_router[f0.csr.col[e]]})
    job_links = [None] + [(links[int(rng.integers(len(links)))], int(rng.choice([capi.COST_DISABLED, 35])))
                          for _ in range(n - 1)]
    border_cells, tops_all, border_rs, border_nrows, border_rows, spt_runs, abr_runs = [], [], [], [], [], [], []
    for b, (areas, ids, sums) in enumerate(v["borders"]):
        flats, rt = flats_all[b], tables[b]
        f = flats[i0[b]]
        s = np.repeat(np.arange(f.csr.n_vertices), np.diff(f.csr.row_ptr))
        by_pair = {}
        for e in range(f.csr.n_edges):
            by_pair.setdefault(tuple(sorted((int(f.ids[s[e]]), int(f.ids[f.csr.col[e]])))), []).append(e)
        rs_list, n_rows, tops = [], [], []
        for i, fl in enumerate(flats):
            root = fl.router_vertex(areas[0].router_id)
            ov = [[]] if i != i0[b] else [[(e, jl[1]) for e in by_pair.get(jl[0], [])] if jl else [] for jl in job_links]
            top = DeviceTopology(ctx, fl.csr, root, len(ov), ov)
            top.run()
            if i == i0[b]:
                spt_runs.append(lambda t=top: ctx.run_device(t.g, t.js, t.rs, sync=False))
            rs_list.append(top.rs); n_rows.append(top.n); tops.append(top)
        rows = np.zeros((n, len(areas)), np.uint32)
        rows[:, i0[b]] = np.arange(n)
        d_rows = torch.from_numpy(rows.view(np.int32).reshape(-1).copy()).to(dev)
        cells = torch.empty(n * rt.n_prefixes * 24, dtype=torch.uint8, device=dev)
        abr_run = (lambda rt=rt, rs_list=rs_list, n_rows=n_rows, d_rows=d_rows, cells=cells:
                   ospf_rib.abr_rib_cells_device(ctx, rt, n, rs_list, n_rows, d_rows.data_ptr(), cells.data_ptr()))
        abr_run()
        abr_runs.append(abr_run)
        keep += [d_rows, rs_list]
        border_rs.append((capi.ResultStruct * len(rs_list))(*rs_list))
        border_nrows.append(np.asarray(n_rows, np.uint32))
        border_rows.append(d_rows.data_ptr())
        border_cells.append(cells); tops_all.append(tops)
    rtop = DeviceTopology(ctx, r_flat.csr, rv, 1, [[]])
    rtop.run()
    rs_r = rtop.rs
    ctx.sync()
    bc = [c.data_ptr() for c in border_cells]

    cur = stage_bench.launch_bound(*BOUND)
    other = 8 if cur == 4 else 4
    libv = C.CDLL(str(stage_bench.build_variant(*BOUND, other, "nonbackbone_bound_")))
    route_table.declare(libv)
    # the variant's own tables over the same images
    vt = []
    for b, (areas, ids, sums) in enumerate(v["borders"]):
        rt = tables[b]
        fl_, ids_, sp_, ns_, act_, _s, ext_, _f = rt._keep
        h = C.c_void_p()
        assert libv.hspf_ospfv2_abr_ribtable_create(rt.router_id, len(areas), fl_, ids_.ctypes.data, sp_,
                                                    ns_.ctypes.data, act_.ctypes.data, ext_.ctypes.data, len(ext_),
                                                    C.byref(h)) == 0
        vt.append(h)
    hv = C.c_void_p()
    sm, ex = bt.summaries, bt.externals
    arr = (C.c_void_p * len(vt))(*[h.value for h in vt])
    assert libv.hspf_ospfv2_nonbackbone_table_create(r_flat.handle, r_area.router_id, bt.config.ctypes.data,
                                                     sm.ctypes.data, len(sm), ex.ctypes.data, len(ex), arr, len(vt),
                                                     C.byref(hv)) == 0
    assert libv.hspf_ospfv2_backbone_table_upload(ctx.handle, hv) == 0
    handles = {cur: (ctx.lib, bt.handle), other: (libv, hv)}
    cells = {b: torch.empty(n * P * 24, dtype=torch.uint8, device=dev) for b in (4, 8)}
    job_out = torch.zeros(n * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device=dev)
    total = torch.zeros(1, dtype=torch.int64, device=dev)
    bca = (C.c_void_p * len(bc))(*bc)
    bpa = (C.c_void_p * len(border_rs))(*[C.addressof(x) for x in border_rs])
    bna = (C.c_void_p * len(border_nrows))(*[x.ctypes.data for x in border_nrows])
    bra = (C.c_void_p * len(border_rows))(*border_rows)

    def cell_launch(b):
        lib, h = handles[b]
        return lambda: lib.hspf_ospfv2_backbone_asbr_cells(ctx.handle, h, n, C.byref(rs_r), bca, None, bpa, bna, bra, None,
                                                          cells[b].data_ptr())

    assert cell_launch(4)() == 0 and cell_launch(8)() == 0
    ctx.sync()
    same_bounds = bool(torch.equal(cells[4], cells[8]))
    base = cells[cur][: P * 24].clone()
    lib, h = handles[cur]
    assert lib.hspf_ospfv2_backbone_asbr_delta(ctx.handle, h, n, C.byref(rs_r), bca, None, bpa, bna, bra,
                                               base.data_ptr(), 1, None, job_out.data_ptr(), None, 0,
                                               total.data_ptr()) == 0
    ctx.sync()
    cap = int(total.cpu()[0])
    w = cells[cur].view(torch.int64).reshape(n, P, 3)
    changed = int((w != w[0:1]).any(dim=2).sum().item())
    recs = torch.empty(max(cap, 1) * DELTA_DT.itemsize, dtype=torch.uint8, device=dev)
    held = torch.cuda.memory_allocated(dev)

    def delta(b, with_records):
        lib, h = handles[b]
        return lambda: lib.hspf_ospfv2_backbone_asbr_delta(ctx.handle, h, n, C.byref(rs_r), bca, None, bpa, bna, bra,
                                                           base.data_ptr(), 1, None, job_out.data_ptr(),
                                                           recs.data_ptr() if with_records else None,
                                                           cap if with_records else 0, total.data_ptr())

    work = {"border_area0_spt_batch": lambda: [r() for r in spt_runs],
            "border_abr_cells": lambda: [r() for r in abr_runs]}
    for b in (4, 8):
        work[f"nonbackbone_cells_bound{b}"] = cell_launch(b)
        work[f"nonbackbone_delta_summaries_bound{b}"] = delta(b, False)
        work[f"nonbackbone_delta_records_bound{b}"] = delta(b, True)
    med = {k: float(np.median(x)) for k, x in stage_bench.time_alternating(ctx, work, args.reps, 2).items()}
    same_after = bool(torch.equal(cells[4], cells[8]))

    # host chain per job (CPU), over the device planes read back
    host_ms = []
    rp = rtop.planes(0)
    bids = {int(x.router_id) for x in tables}
    for j in range(1, 1 + min(args.host_jobs, n - 1)):
        t = time.perf_counter()
        new = [s for s in v["summaries1"] if int(s["adv_rtr"]) not in bids]
        for b, (areas, ids, sums) in enumerate(v["borders"]):
            ra = []
            for i, a in enumerate(areas):
                spf = stage_bench.spf_from_planes("ospfv2", a, tops_all[b][i].planes(j if i == i0[b] else 0))
                ra.append(ospf_rib.RibArea(a.area_id, spf, a.ifaces, sums[i], True))
            rid = areas[0].router_id
            rib = ospf_rib.update_rib_full(rid, areas[0].max_paths, ra, v["externals"])
            new += list(ospf_rib.net_summaries(rid, rib, ospf_rib.router_tables(rid, ra), ra,
                                               [ospf_rib.area_config()] * len(areas), ids.index(1)))
        s = np.array(new, ospf_rib.SUMMARY_LSA_DT)
        s = s[np.lexsort((s["lsa_id"], s["adv_rtr"], s["lsa_type"]))]
        r_spf = stage_bench.spf_from_planes("ospfv2", r_area, rp)
        ospf_rib.update_rib_full(r_area.router_id, r_area.max_paths, [ospf_rib.RibArea(1, r_spf, r_area.ifaces, s, True)],
                                 v["externals"])
        host_ms.append((time.perf_counter() - t) * 1e3)

    card, power = stage_bench.card_and_power()
    out = {
        "stage": "hspf_ospfv2_nonbackbone_table_create + hspf_ospfv2_backbone_asbr_cells / _delta",
        "workload": {"area0": f"{args.v0} routers, {4 * args.v0} links, costs {{10, 20}}, 5 % LANs",
                     "area1": f"{args.v1} routers", "externals": len(v["externals"]), "borders": len(tables),
                     "jobs": n, "jobs_asked": args.jobs, "affected_prefixes": P, "slots": bt.n_slots,
                     "type4_slots": bt.n_asbr_slots, "plane_sets": bt.n_asbr_sets,
                     "border_keys": [t.n_prefixes for t in tables],
                     "border_cells_bytes": sum(t.n_prefixes for t in tables) * 24 * n,
                     "device_bytes_held": int(held)},
        "card": card, "power_limit": power, "reps": args.reps, "median_ms": med, "launch_bound": cur,
        "other_bound": other, "cells_equal_other_bound": same_bounds and same_after,
        "delta_total": cap, "delta_total_equals_changed_cells": cap == changed,
        "host_chain_ms_per_job": float(np.median(host_ms)) if host_ms else None, "host_jobs_timed": len(host_ms),
        "note": "device figures are CUDA-event medians of alternating launches; the host chain is a CPU figure",
    }
    print(f"device memory held: {held / 2**30:.1f} GiB ({n} jobs)", file=sys.stderr)
    stage_bench.write_json(out, args.out)


if __name__ == "__main__":
    main()
