#!/usr/bin/env python
"""The routing-table stage for an OSPFv3 area border router (hspf_ospfv2_abr_rib_cells / hspf_ospfv2_abr_rib_delta over
a table of hspf_ospfv3_abr_ribtable_create) on a 10 000-job what-if batch, beside each area's SPT batch; device only:
python scripts/ospfv3_abr_rib_stage.py [--jobs 10000] [--reps 10] [--out profiles/h100_C5v3_abr_rib.json]

Areas (ospfv3.abr_view, seed 0xC5): C5's topology as the OSPFv3 backbone (10 000 routers, 5 % of adjacencies on LANs,
costs {10, 20}) with C5's routing-table load (ospfv3.inter_area_view as in scripts/ospfv3_rib_stage.py), plus two
synth_area areas of 2 000 routers; one ABR root attached to all three.  Job 0 is unperturbed; job j > 0 disables one
router-to-router link (both directions) in area (j - 1) mod 3, whose row it takes; its other rows are their row 0.

CUDA-event medians over `--reps` alternating launches after warm-up; the card's name and power limit are read in the
same run.  Outside the timed region: the delta equals a torch comparison of the stored cells for every job (summaries,
total and every record), and sampled jobs decode to the host stages (ospfv3.area_from_planes + update_rib_full_v3) over
the same planes."""
import argparse
import time

import numpy as np

import stage_bench


def router_link_pairs(flat):
    """(e, reverse e) of every router-to-router link of an ospfv3.Flat's CSR, each link once."""
    c = flat.csr
    src = np.repeat(np.arange(c.n_vertices), np.diff(c.row_ptr))
    fwd = {(int(src[e]), int(c.col[e])): e for e in range(c.n_edges)
           if flat.is_router[int(src[e])] and flat.is_router[int(c.col[e])]}
    return [(e, fwd[(v, u)]) for (u, v), e in fwd.items() if u < v and (v, u) in fwd]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--jobs", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch = stage_bench.require_gpu("ospfv3_abr_rib_stage.py")
    from holo_b200 import capi, ospf_rib, ospfv3, synth
    from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
    from ospf_abr_rib_stage import torch_delta
    from test_isis_route_cells_gpu import DeviceTopology

    t_setup = time.perf_counter()
    kw = dict(n_abr=16, n_asbr=16, n_inter=10000, n_ext=5000, n_overlap=3000, n_fresh=2000, n_ext_only=1000)
    topos = [synth.random_topology(10000, 40000, synth.SEED_BASE + 5, cost_choices=[10, 20], lan_fraction=0.05)]
    topos += [synth.random_topology(2000, 8000, synth.SEED_BASE + 850 + k, cost_choices=[10, 20], lan_fraction=0.05)
              for k in range(2)]
    areas, sums, ext = ospfv3.abr_view(topos, 0xC5, roots=[0, 0, 0], **kw)
    A = len(areas)
    flats = [ospfv3.Flat(a) for a in areas]
    rvs = [f.router_vertex(ospfv3.ABR_ROUTER_ID) for f in flats]
    rt = ospf_rib.AbrRibTable(ospfv3.ABR_ROUTER_ID, flats, [a.area_id for a in areas], sums, None, ext)
    assert rt.v3
    ctx = capi.Context(0)
    dev = torch.device("cuda", 0)
    rt.upload(ctx)
    n, P = args.jobs, rt.n_prefixes
    rng = np.random.default_rng(0xC5)
    rows = np.zeros((n, A), np.uint32)
    ovs = [[[]] for _ in range(A)]
    for i, f in enumerate(flats):
        pairs = router_link_pairs(f)
        for j in range(1 + i, n, A):
            e, r = pairs[int(rng.integers(len(pairs)))]
            rows[j, i] = len(ovs[i])
            ovs[i].append([(e, capi.COST_DISABLED), (r, capi.COST_DISABLED)])
    tops = [DeviceTopology(ctx, flats[i].csr, rvs[i], len(ovs[i]), ovs[i]) for i in range(A)]
    for top in tops:
        top.run()
    rs_list, n_rows = [top.rs for top in tops], [top.n for top in tops]
    ctx.sync()
    d_rows = torch.from_numpy(rows.view(np.int32).reshape(-1).copy()).to(dev)
    arr = (capi.ResultStruct * A)(*rs_list)
    nr = np.asarray(n_rows, np.uint32)
    cells = torch.empty(n * P * 24, dtype=torch.uint8, device=dev)
    st_out = torch.zeros(n, dtype=torch.int32, device=dev)
    job_out = torch.zeros(n * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device=dev)
    total = torch.zeros(1, dtype=torch.int64, device=dev)
    lib = ctx.lib

    def abr_cells():
        assert lib.hspf_ospfv2_abr_rib_cells(ctx.handle, rt.handle, n, arr, nr.ctypes.data, d_rows.data_ptr(),
                                             cells.data_ptr(), st_out.data_ptr(), 0, None, None, None, None) == 0

    base = torch.empty(P * 24, dtype=torch.uint8, device=dev)
    abr_cells()
    ctx.sync()
    base.copy_(cells[: P * 24])
    # summaries first, to size the record buffer
    assert lib.hspf_ospfv2_abr_rib_delta(ctx.handle, rt.handle, n, arr, nr.ctypes.data, d_rows.data_ptr(), base.data_ptr(),
                                         1, None, job_out.data_ptr(), None, 0, total.data_ptr()) == 0
    ctx.sync()
    cap = int(total.cpu()[0])
    recs = torch.empty(max(cap, 1) * DELTA_DT.itemsize, dtype=torch.uint8, device=dev)

    def delta(with_records):
        return lambda: lib.hspf_ospfv2_abr_rib_delta(ctx.handle, rt.handle, n, arr, nr.ctypes.data, d_rows.data_ptr(),
                                                     base.data_ptr(), 1, None, job_out.data_ptr(),
                                                     recs.data_ptr() if with_records else None,
                                                     cap if with_records else 0, total.data_ptr())

    variants = {f"spt_batch_area{i}": (lambda t=top: ctx.run_device(t.g, t.js, t.rs, sync=False))
                for i, top in enumerate(tops)}
    variants.update({"abr_rib_cells_kernel": abr_cells, "abr_rib_delta_summaries": delta(False),
                     "abr_rib_delta_records": delta(True)})
    ms = stage_bench.time_alternating(ctx, variants, args.reps, 2)
    med = {k: float(np.median(v)) for k, v in ms.items()}

    # ---- outside the timed region
    abr_cells()
    job_out.zero_(); recs.zero_()
    delta(True)()
    ctx.sync()
    words = cells.view(torch.int64).view(n, P, 3)
    summ, want_r = torch_delta(words, base.view(torch.int64).view(P, 3), st_out.long())
    got_j = torch.from_numpy(job_out.cpu().numpy().view(np.uint32).astype(np.int64).reshape(n, 8)).to(dev)
    got_r = recs.cpu().numpy()[: cap * DELTA_DT.itemsize].view(DELTA_DT)
    gr = torch.from_numpy(np.stack([got_r[k].astype(np.int64) for k in ("job", "prefix", "metric", "kind")], 1)).to(dev)
    checks = {"summaries_equal": bool(torch.equal(got_j[:, :7], summ[:, :7])), "total": int(total.cpu()[0]),
              "records_equal": bool(torch.equal(gr, want_r))}
    status = st_out.cpu().numpy().view(np.uint32)
    sample = sorted({0, 1, 2, 3, n // 2, n - 1})
    decoded = []
    for j in sample:
        cj = cells[j * P * 24: (j + 1) * P * 24].cpu().numpy().view(ospf_rib.RIB_CELL_DT)
        p, ga, gv, gn = [], [], [], []
        for i in range(A):
            d, h, m = tops[i].planes(int(rows[j, i]))
            p.append((d, h, m))
            f, rv = flats[i], rvs[i]
            nets = sorted({int(v) for v in f.csr.col[f.csr.row_ptr[rv]: f.csr.row_ptr[rv + 1]] if not f.is_router[v]})
            ga += [i] * len(nets); gv += nets; gn += [int(m[v]) for v in nets]
        t0 = time.perf_counter()
        got = ospf_rib.abr_rib_from_cells_v3(areas, rt, cj, ga, gv, gn)
        t_dec = time.perf_counter() - t0
        t0 = time.perf_counter()
        ra = [ospf_rib.RibArea(a.area_id, stage_bench.spf_from_planes("ospfv3", a, p[i]), a.ifaces, sums[i])
              for i, a in enumerate(areas)]
        want = ospf_rib.update_rib_full_v3(ospfv3.ABR_ROUTER_ID, areas[0].max_paths, ra, ext)
        t_host = time.perf_counter() - t0
        ok = (status[j] == 0 and got.rc == 0 and got.routes.tobytes() == want.routes.tobytes()
              and got.nexthops.tobytes() == want.nexthops.tobytes())
        decoded.append({"job": int(j), "rows": [int(x) for x in rows[j]], "routes": int(len(got.routes)), "equal": bool(ok),
                        "decode_s": round(t_dec, 4), "host_stages_s": round(t_host, 4)})
    card, power = stage_bench.card_and_power()
    out = {
        "workload": f"OSPFv3 ABR {ospfv3.ABR_ROUTER_ID:#x} of ospfv3.abr_view(seed 0xC5): area 0 = C5's topology (10000 "
                    f"routers, 40000 directed adjacencies, costs {{10, 20}}, 5 % on LANs) with ospfv3.inter_area_view({kw}); "
                    f"areas 1, 2 = synth_area of 2000 routers / 8000 adjacencies; {n} jobs (job 0 plain, job j > 0 one "
                    f"link cut in area (j - 1) % 3)",
        "areas": [{"area_id": int(a.area_id), "vertices": int(f.csr.n_vertices), "rows": int(r), "atoms": int(na)}
                  for a, f, r, na in zip(areas, flats, n_rows, rt.n_atoms)],
        "prefixes": int(P), "records": int(rt.n_contributors), "jobs": n, "changes": int(cap),
        "jobs_changed": int((job_out.cpu().numpy().view(DELTA_JOB_DT)["n_changed"] > 0).sum()),
        "card": card, "power_limit": power, "reps": args.reps,
        "median_ms": med, "ms": ms, "delta_checks": checks, "sampled_decodes": decoded,
        "setup_s": round(time.perf_counter() - t_setup, 1),
    }
    stage_bench.write_json(out, args.out)
    print("decodes equal:", all(d["equal"] for d in decoded))


if __name__ == "__main__":
    main()
