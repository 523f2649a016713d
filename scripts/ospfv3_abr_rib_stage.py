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
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))


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
    import torch
    if not torch.cuda.is_available():
        sys.exit("ospfv3_abr_rib_stage.py: no CUDA device; this measurement runs on the GPU only")
    from holo_b200 import capi, ospf_rib, ospfv3, synth
    from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
    from ospf_abr_rib_stage import torch_delta

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
    u32p, u16p, u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint16), C.POINTER(C.c_uint64)
    keep, spt, rs_list, planes, n_rows = [], [], [], [], []
    for i in range(A):
        csr, root, ov = flats[i].csr, rvs[i], ovs[i]
        m = len(ov)
        g = ctx.upload(csr)
        off = np.zeros(m + 1, np.int64)
        ed, co = [], []
        for j, o in enumerate(ov):
            for e, cst in o:
                ed.append(e); co.append(cst)
            off[j + 1] = len(ed)
        t = [torch.full((m,), root, dtype=torch.int32, device=dev), torch.from_numpy(off.astype(np.int32)).to(dev),
             torch.from_numpy(np.asarray(ed or [0], np.uint32).view(np.int32).copy()).to(dev),
             torch.from_numpy(np.asarray(co or [0], np.uint32).view(np.int32).copy()).to(dev)]
        js = capi.JobsStruct()
        js.n_jobs, js.roots, js.ov_off, js.ov_edge, js.ov_cost = m, *(C.cast(x.data_ptr(), u32p) for x in t)
        V = csr.n_vertices
        pl = [torch.empty(m * V, dtype=torch.int32, device=dev), torch.empty(m * V, dtype=torch.int16, device=dev),
              torch.empty(m * V, dtype=torch.int64, device=dev), torch.zeros(m, dtype=torch.int32, device=dev)]
        rs = capi.ResultStruct()
        rs.dist, rs.hops = C.cast(pl[0].data_ptr(), u32p), C.cast(pl[1].data_ptr(), u16p)
        rs.nh_mask, rs.nh_words = C.cast(pl[2].data_ptr(), u64p), 1
        rs.job_status = C.cast(pl[3].data_ptr(), u32p)
        keep.extend([g, t, pl, js])
        spt.append((g, js, rs))
        rs_list.append(rs)
        planes.append(pl)
        n_rows.append(m)
        ctx.run_device(g, js, rs, sync=False)
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

    variants = {f"spt_batch_area{i}": (lambda g=g, js=js, rs=rs: ctx.run_device(g, js, rs, sync=False))
                for i, (g, js, rs) in enumerate(spt)}
    variants.update({"abr_rib_cells_kernel": abr_cells, "abr_rib_delta_summaries": delta(False),
                     "abr_rib_delta_records": delta(True)})
    stream = torch.cuda.ExternalStream(ctx.stream, device=dev)
    for _ in range(2):
        for fn in variants.values():
            fn()
    ctx.sync()
    ev = {k: [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.reps)]
          for k in variants}
    for r in range(args.reps):
        for k, fn in variants.items():
            ev[k][r][0].record(stream)
            fn()
            ev[k][r][1].record(stream)
    ctx.sync()
    ms = {k: [a.elapsed_time(b) for a, b in e] for k, e in ev.items()}
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
            V = flats[i].csr.n_vertices
            r = int(rows[j, i])
            d = planes[i][0][r * V: (r + 1) * V].cpu().numpy().view(np.uint32).copy()
            h = planes[i][1][r * V: (r + 1) * V].cpu().numpy().view(np.uint16).copy()
            m = planes[i][2][r * V: (r + 1) * V].cpu().numpy().view(np.uint64).copy()
            p.append((d, h, m))
            f, rv = flats[i], rvs[i]
            nets = sorted({int(v) for v in f.csr.col[f.csr.row_ptr[rv]: f.csr.row_ptr[rv + 1]] if not f.is_router[v]})
            ga += [i] * len(nets); gv += nets; gn += [int(m[v]) for v in nets]
        t0 = time.perf_counter()
        got = ospf_rib.abr_rib_from_cells_v3(areas, rt, cj, ga, gv, gn)
        t_dec = time.perf_counter() - t0
        t0 = time.perf_counter()
        ra = []
        for i, a in enumerate(areas):
            m4 = np.zeros((len(p[i][0]), 4), np.uint64)
            m4[:, 0] = p[i][2]
            spf = ospfv3.area_from_planes(a, lambda c, r, w, d=p[i][0], h=p[i][1], m4=m4: (d, h, m4[:, :w]))
            ra.append(ospf_rib.RibArea(a.area_id, spf, a.ifaces, sums[i]))
        want = ospf_rib.update_rib_full_v3(ospfv3.ABR_ROUTER_ID, areas[0].max_paths, ra, ext)
        t_host = time.perf_counter() - t0
        ok = (status[j] == 0 and got.rc == 0 and got.routes.tobytes() == want.routes.tobytes()
              and got.nexthops.tobytes() == want.nexthops.tobytes())
        decoded.append({"job": int(j), "rows": [int(x) for x in rows[j]], "routes": int(len(got.routes)), "equal": bool(ok),
                        "decode_s": round(t_dec, 4), "host_stages_s": round(t_host, 4)})
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    card, power = (q[0].split(", ") + ["?"])[:2] if q else (torch.cuda.get_device_name(0), "?")
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
    print(json.dumps({k: out[k] for k in ("card", "power_limit", "median_ms", "delta_checks", "changes", "prefixes",
                                          "areas")}, indent=1))
    print("decodes equal:", all(d["equal"] for d in decoded))
    if args.out:
        Path(args.out).write_text(json.dumps(out, indent=1) + "\n")


if __name__ == "__main__":
    main()
