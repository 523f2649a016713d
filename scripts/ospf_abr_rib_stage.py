#!/usr/bin/env python
"""The routing-table stage for an area border router (hspf_ospfv2_abr_rib_cells / hspf_ospfv2_abr_rib_delta) on a
10 000-job what-if batch, beside each area's SPT batch and the one-area stage (ospf_rib_cells_kernel) of an internal
router of area 0; device only:
python scripts/ospf_abr_rib_stage.py [--jobs 10000] [--reps 10] [--out profiles/h100_C5_abr_rib.json]

Areas (ospfv2.abr_view, seed 0xC5): C5's LSDB (10 000 routers, 5 % of adjacencies on LANs, costs {10, 20}) as area 0
with C5's routing-table load (inter_area_view as in scripts/ospf_rib_stage.py), plus two synth_area areas of 2 000
routers; one ABR root attached to all three.  Job 0 is unperturbed; job j > 0 disables one router-to-router link (both
directions) in area (j - 1) mod 3, whose row it takes; its other rows are their row 0.

The launch bound of the stage's kernels (kAbrBlocksPerSM in csrc/ospfv2_abr_rib_cells.cu) is timed against 8 in the
same run: a second copy of the library, built into a temporary directory with that constant set to 8, runs the same
calls on the same table data and planes, alternating with the first.  CUDA-event medians over `--reps` alternating
launches after warm-up; the card's name and power limit are read in the same run.  Outside the timed region: both
builds' cells are byte-identical, the delta equals a torch comparison of the stored cells for every job (summaries,
total and every record), and sampled jobs decode to the host stages (area_from_planes + update_rib_full) over the same
planes."""
import argparse
import ctypes as C
import shutil
import time

import numpy as np

import stage_bench

BOUND = ("ospfv2_abr_rib_cells.cu", "kAbrBlocksPerSM")


def torch_delta(cells, base, status, chunk=256):
    """(per-job summaries [n, 8] u32 as DELTA_JOB_DT, records as (job, prefix, metric, kind) int64 [R, 4]) of cells
    [n, P, 3] int64 words against base [P, 3], on the device."""
    import torch
    n, P = cells.shape[0], cells.shape[1]
    summ = torch.zeros((n, 8), dtype=torch.int64, device=cells.device)
    recs = []
    b = base
    bm = (b[:, 2] >> 32) & 0xFFFFFFFF
    bp = ((bm >> 28) & 1) != 0
    for j0 in range(0, n, chunk):
        c = cells[j0: j0 + chunk]
        cm = (c[:, :, 2] >> 32) & 0xFFFFFFFF
        cp = ((cm >> 28) & 1) != 0
        both = cp & bp
        k = torch.zeros(cp.shape, dtype=torch.int64, device=c.device)
        k |= (bp & ~cp).long() * 0x01
        k |= (cp & ~bp).long() * 0x02
        k |= (both & ((cm & 0x03FFFFFF) != (bm & 0x03FFFFFF))).long() * 0x04
        k |= (both & (c[:, :, 0] != b[:, 0])).long() * 0x08
        other = (c[:, :, 1] != b[:, 1]) | ((c[:, :, 2] & 0xFFFFFFFF) != (b[:, 2] & 0xFFFFFFFF)) | ((cm >> 26) != (bm >> 26))
        k |= (both & other).long() * 0x10
        st = status[j0: j0 + chunk]
        k[st != 0] = 0
        summ[j0: j0 + chunk, 0] = (k != 0).sum(1)
        for q, bit in enumerate((0x01, 0x02, 0x04, 0x08, 0x10)):
            summ[j0: j0 + chunk, 1 + q] = ((k & bit) != 0).sum(1)
        summ[j0: j0 + chunk, 6] = st
        jj, pp = torch.nonzero(k, as_tuple=True)
        kk = k[jj, pp]
        met = torch.where(kk == 0x01, bm[pp] & 0x03FFFFFF, cm[jj, pp] & 0x03FFFFFF)
        recs.append(torch.stack([jj + j0, pp, met, kk], 1))
    return summ, torch.cat(recs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--jobs", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch = stage_bench.require_gpu("ospf_abr_rib_stage.py")
    from holo_b200 import capi, ospf_rib, ospfv2, route_table, synth
    from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
    from test_isis_route_cells_gpu import DeviceTopology

    t_setup = time.perf_counter()
    kw = dict(n_abr=16, n_asbr=16, n_inter=10000, n_ext=5000, n_overlap=3000, n_fresh=2000, n_ext_only=1000)
    topos = [synth.random_topology(10000, 40000, synth.SEED_BASE + 5, cost_choices=[10, 20], lan_fraction=0.05)]
    topos += [synth.random_topology(2000, 8000, synth.SEED_BASE + 850 + k, cost_choices=[10, 20], lan_fraction=0.05)
              for k in range(2)]
    areas, sums, ext = ospfv2.abr_view(topos, 0xC5, roots=[0, 0, 0], **kw)
    A = len(areas)
    flats = [ospfv2.Flat(a) for a in areas]
    rvs = [f.router_vertex(ospfv2.ABR_ROUTER_ID) for f in flats]
    rt = ospf_rib.AbrRibTable(ospfv2.ABR_ROUTER_ID, flats, [a.area_id for a in areas], sums, None, ext)
    ctx = capi.Context(0)
    dev = torch.device("cuda", 0)
    rt.upload(ctx)
    n, P = args.jobs, rt.n_prefixes
    rng = np.random.default_rng(0xC5)
    # per area: row 0 plain, then one row per job of that area (one link cut, both directions)
    rows = np.zeros((n, A), np.uint32)
    ovs = [[[]] for _ in range(A)]
    for i, f in enumerate(flats):
        c = f.csr
        src = np.repeat(np.arange(c.n_vertices), np.diff(c.row_ptr))
        fwd = {(int(src[e]), int(c.col[e])): e for e in range(c.n_edges) if f.link_index[e] != 0xFFFFFFFF}
        pairs = [(e, fwd[(v, u)]) for (u, v), e in fwd.items() if u < v and (v, u) in fwd]
        for j in range(1 + i, n, A):
            e, r = pairs[int(rng.integers(len(pairs)))]
            rows[j, i] = len(ovs[i])
            ovs[i].append([(e, capi.COST_DISABLED), (r, capi.COST_DISABLED)])
    tops = [DeviceTopology(ctx, flats[i].csr, rvs[i], len(ovs[i]), ovs[i]) for i in range(A)]
    rs_list, n_rows = [top.rs for top in tops], [top.n for top in tops]
    # the one-area stage for comparison: area 0's rows rooted at an internal router of area 0
    a0 = areas[0]
    internal = next(int(r) for r, fl in zip(a0.router_lsas["adv_rtr"], a0.router_lsas["flags"])
                    if not fl & 0x01 and flats[0].router_vertex(int(r)) != 0xFFFFFFFF)
    iv = flats[0].router_vertex(internal)
    top_in = DeviceTopology(ctx, flats[0].csr, iv, len(ovs[0]), ovs[0])
    rt1 = ospf_rib.RibTable(flats[0], a0.area_id, sums[0], ext)
    rt1.upload(ctx)
    m0 = len(ovs[0])
    d_roots_in = torch.full((m0,), iv, dtype=torch.int32, device=dev)
    cells1 = torch.empty(m0 * rt1.n_prefixes * 24, dtype=torch.uint8, device=dev)
    for top in tops + [top_in]:
        top.run()
    ctx.sync()
    d_rows = torch.from_numpy(rows.view(np.int32).reshape(-1).copy()).to(dev)

    # the other launch bound, from a copy of the library
    lib8_path = stage_bench.build_variant(*BOUND, 8, "abr_bound_")
    lib8 = C.CDLL(str(lib8_path))
    route_table.declare(lib8)
    fl_, ids_, sp_, ns_, act_, _s, ext_, _f = rt._keep
    h8 = C.c_void_p()
    rc = lib8.hspf_ospfv2_abr_ribtable_create(rt.router_id, A, fl_, ids_.ctypes.data, sp_, ns_.ctypes.data, act_.ctypes.data,
                                              ext_.ctypes.data if len(ext_) else None, len(ext_), C.byref(h8))
    assert rc == 0
    assert lib8.hspf_ospfv2_abr_ribtable_upload(ctx.handle, h8) == 0
    arr = (capi.ResultStruct * A)(*rs_list)
    nr = np.asarray(n_rows, np.uint32)
    cells = {b: torch.empty(n * P * 24, dtype=torch.uint8, device=dev) for b in (4, 8)}
    st_out = torch.zeros(n, dtype=torch.int32, device=dev)
    job_out = torch.zeros(n * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device=dev)
    total = torch.zeros(1, dtype=torch.int64, device=dev)
    lib4 = ctx.lib

    def abr_cells(lib, h, b):
        return lambda: lib.hspf_ospfv2_abr_rib_cells(ctx.handle, h, n, arr, nr.ctypes.data, d_rows.data_ptr(),
                                                     cells[b].data_ptr(), st_out.data_ptr(), 0, None, None, None, None)

    base = torch.empty(P * 24, dtype=torch.uint8, device=dev)
    abr_cells(lib4, rt.handle, 4)()
    ctx.sync()
    base.copy_(cells[4][: P * 24])
    # summaries first, to size the record buffer
    assert lib4.hspf_ospfv2_abr_rib_delta(ctx.handle, rt.handle, n, arr, nr.ctypes.data, d_rows.data_ptr(), base.data_ptr(), 1,
                                          None, job_out.data_ptr(), None, 0, total.data_ptr()) == 0
    ctx.sync()
    cap = int(total.cpu()[0])
    recs = torch.empty(max(cap, 1) * DELTA_DT.itemsize, dtype=torch.uint8, device=dev)

    def delta(lib, h, with_records):
        return lambda: lib.hspf_ospfv2_abr_rib_delta(ctx.handle, h, n, arr, nr.ctypes.data, d_rows.data_ptr(), base.data_ptr(),
                                                     1, None, job_out.data_ptr(), recs.data_ptr() if with_records else None,
                                                     cap if with_records else 0, total.data_ptr())

    variants = {f"spt_batch_area{i}": (lambda t=top: ctx.run_device(t.g, t.js, t.rs, sync=False))
                for i, top in enumerate(tops)}
    variants.update({
        "abr_rib_cells_kernel_bound4": abr_cells(lib4, rt.handle, 4),
        "abr_rib_cells_kernel_bound8": abr_cells(lib8, h8, 8),
        "abr_rib_delta_summaries_bound4": delta(lib4, rt.handle, False),
        "abr_rib_delta_summaries_bound8": delta(lib8, h8, False),
        "abr_rib_delta_records_bound4": delta(lib4, rt.handle, True),
        "abr_rib_delta_records_bound8": delta(lib8, h8, True),
        "ospf_rib_cells_kernel_area0_internal_root": lambda: ospf_rib.rib_cells_device(
            ctx, rt1, m0, top_in.rs, d_roots_in.data_ptr(), cells1.data_ptr()),
    })
    ms = stage_bench.time_alternating(ctx, variants, args.reps, 2)
    med = {k: float(np.median(v)) for k, v in ms.items()}

    # ---- outside the timed region
    abr_cells(lib4, rt.handle, 4)()
    abr_cells(lib8, h8, 8)()
    ctx.sync()
    same_bounds = bool(torch.equal(cells[4], cells[8]))
    checks = {}
    for b, (lib, h) in ((4, (lib4, rt.handle)), (8, (lib8, h8))):
        job_out.zero_(); recs.zero_()
        delta(lib, h, True)()
        ctx.sync()
        words = cells[b].view(torch.int64).view(n, P, 3)
        summ, want = torch_delta(words, base.view(torch.int64).view(P, 3), st_out.long())
        got_j = torch.from_numpy(job_out.cpu().numpy().view(np.uint32).astype(np.int64).reshape(n, 8)).to(dev)
        got_r = recs.cpu().numpy()[: cap * DELTA_DT.itemsize].view(DELTA_DT)
        gr = torch.from_numpy(np.stack([got_r[k].astype(np.int64) for k in ("job", "prefix", "metric", "kind")], 1)).to(dev)
        checks[f"bound{b}"] = {"summaries_equal": bool(torch.equal(got_j[:, :7], summ[:, :7])),
                               "total": int(total.cpu()[0]), "records_equal": bool(torch.equal(gr, want))}
    status = st_out.cpu().numpy().view(np.uint32)
    sample = sorted({0, 1, 2, 3, n // 2, n - 1})
    decoded = []
    for j in sample:
        cj = cells[4][j * P * 24: (j + 1) * P * 24].cpu().numpy().view(ospf_rib.RIB_CELL_DT)
        p, ga, gv, gn = [], [], [], []
        for i in range(A):
            d, h, m = tops[i].planes(int(rows[j, i]))
            p.append((d, h, m))
            f, rv = flats[i], rvs[i]
            nets = sorted({int(v) for v in f.csr.col[f.csr.row_ptr[rv]: f.csr.row_ptr[rv + 1]] if not f.is_router[v]})
            ga += [i] * len(nets); gv += nets; gn += [int(m[v]) for v in nets]
        t0 = time.perf_counter()
        got = ospf_rib.abr_rib_from_cells(areas, rt, cj, ga, gv, gn)
        t_dec = time.perf_counter() - t0
        t0 = time.perf_counter()
        ra = [ospf_rib.RibArea(a.area_id, stage_bench.spf_from_planes("ospfv2", a, p[i]), a.ifaces, sums[i])
              for i, a in enumerate(areas)]
        want = ospf_rib.update_rib_full(ospfv2.ABR_ROUTER_ID, a0.max_paths, ra, ext)
        t_host = time.perf_counter() - t0
        ok = (status[j] == 0 and got.rc == 0 and got.routes.tobytes() == want.routes.tobytes()
              and got.nexthops.tobytes() == want.nexthops.tobytes())
        decoded.append({"job": int(j), "rows": [int(x) for x in rows[j]], "routes": int(len(got.routes)), "equal": bool(ok),
                        "decode_s": round(t_dec, 4), "host_stages_s": round(t_host, 4)})
    card, power = stage_bench.card_and_power()
    out = {
        "workload": f"ABR {ospfv2.ABR_ROUTER_ID:#x} of ospfv2.abr_view(seed 0xC5): area 0 = C5 (10000 routers, 40000 directed "
                    f"adjacencies, costs {{10, 20}}, 5 % on LANs) with inter_area_view({kw}); areas 1, 2 = synth_area of "
                    f"2000 routers / 8000 adjacencies; {n} jobs (job 0 plain, job j > 0 one link cut in area (j - 1) % 3)",
        "areas": [{"area_id": int(a.area_id), "vertices": int(f.csr.n_vertices), "rows": int(r), "atoms": int(na)}
                  for a, f, r, na in zip(areas, flats, n_rows, rt.n_atoms)],
        "prefixes": int(P), "records": int(rt.n_contributors), "ospf_rib_table_prefixes_area0": int(rt1.n_prefixes),
        "jobs": n, "changes": int(cap), "jobs_changed": int((job_out.cpu().numpy().view(DELTA_JOB_DT)["n_changed"] > 0).sum()),
        "card": card, "power_limit": power, "reps": args.reps,
        "median_ms": med, "ms": ms,
        "cells_bound4_equal_bound8": same_bounds, "delta_checks": checks, "sampled_decodes": decoded,
        "setup_s": round(time.perf_counter() - t_setup, 1),
    }
    stage_bench.write_json(out, args.out)
    print("decodes equal:", all(d["equal"] for d in decoded))
    shutil.rmtree(lib8_path.parent, ignore_errors=True)


if __name__ == "__main__":
    main()
