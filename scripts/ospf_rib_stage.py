#!/usr/bin/env python
"""The OSPFv2 routing-table stage (hspf_ospfv2_rib_cells) on C5 with generated inter-area and external load, beside the
SPT batch and the intra-area cell kernel (route_cells_kernel) over the same planes:
python scripts/ospf_rib_stage.py [--roots 1000] [--reps 10] [--out profiles/h100_C5_rib.json]

C5's LSDB (10 000 routers, 5 % of adjacencies on LANs, costs {10, 20}) as area 0.0.0.1, with
ospfv2.inter_area_view: 16 ABRs and 16 ASBRs, 10 000 type-3, 10 type-4 and 5 000 type-5 LSAs over 3 000 of the area's
prefixes, 2 000 new ones (and three with host bits or the default route), plus 1 000 named by externals only.  Jobs: the first `--roots` internal routers as roots.
CUDA-event medians over `--reps` alternating launches after warm-up; the card's name and power limit are read in the
same run; the host stages (area_from_planes + update_rib_full) are timed per root; outside the timed region sampled
jobs are decoded and compared with the host stages over the same planes."""
import argparse
import ctypes as C
import sys
import time

import numpy as np

import stage_bench

DATASHEET_GBS = 3350.0            # H100 SXM5 HBM3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--roots", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch = stage_bench.require_gpu("ospf_rib_stage.py")
    from holo_b200 import capi, ospf_rib, ospfv2, synth

    kw = dict(n_abr=16, n_asbr=16, n_inter=10000, n_ext=5000, n_overlap=3000, n_fresh=2000, n_ext_only=1000)
    t = synth.random_topology(10000, 40000, synth.SEED_BASE + 5, cost_choices=[10, 20], lan_fraction=0.05)

    def view(i):
        a = ospfv2.synth_area(t, root=i)
        a.area_id = 1
        return ospfv2.inter_area_view(a, 0xC5, **kw)

    area, sums, ext = view(0)
    flat = ospfv2.Flat(area)
    csr = flat.csr
    V = csr.n_vertices
    flags = dict(zip(area.router_lsas["adv_rtr"].tolist(), area.router_lsas["flags"].tolist()))
    internal = [i for i in range(t.n_routers) if not flags[ospfv2.RID_BASE + i] & 1]
    idx = internal[: args.roots]
    roots = [flat.router_vertex(ospfv2.RID_BASE + i) for i in idx]
    n = len(roots)
    ctx = capi.Context(0)
    dev = torch.device("cuda", 0)
    rt = ospf_rib.RibTable(flat, 1, sums, ext)
    rt.upload(ctx)
    it = ospfv2.RouteTable(flat)
    it.upload(ctx)
    g = ctx.upload(csr)
    u16p, u32p, u64p = C.POINTER(C.c_uint16), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
    d_roots = torch.tensor(np.asarray(roots, np.int32), device=dev)
    js = capi.JobsStruct()
    js.n_jobs, js.roots = n, C.cast(d_roots.data_ptr(), u32p)
    planes = [torch.empty(n * V, dtype=torch.int32, device=dev), torch.empty(n * V, dtype=torch.int16, device=dev),
              torch.empty(n * V, dtype=torch.int64, device=dev), torch.zeros(n, dtype=torch.int32, device=dev)]
    rs = capi.ResultStruct()
    rs.dist, rs.hops = C.cast(planes[0].data_ptr(), u32p), C.cast(planes[1].data_ptr(), u16p)
    rs.nh_mask, rs.nh_words = C.cast(planes[2].data_ptr(), u64p), 1
    rs.job_status = C.cast(planes[3].data_ptr(), u32p)
    P, PI = rt.n_prefixes, it.n_prefixes
    rib_cells = torch.empty(n * P * 24, dtype=torch.uint8, device=dev)
    intra_cells = torch.empty(n * PI * 24, dtype=torch.uint8, device=dev)
    st_out = torch.zeros(n, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    variants = {
        "spt_batch": lambda: ctx.run_device(g, js, rs, sync=False),
        "route_cells_kernel": lambda: ospfv2.routes_batch_device(ctx, it, n, rs, intra_cells.data_ptr()),
        "ospf_rib_cells_kernel": lambda: ospf_rib.rib_cells_device(ctx, rt, n, rs, d_roots.data_ptr(), rib_cells.data_ptr(),
                                                                   st_out.data_ptr()),
    }
    ms = stage_bench.time_alternating(ctx, variants, args.reps, 3)
    med = {k: float(np.median(v)) for k, v in ms.items()}

    # ---- outside the timed region: sampled jobs decoded against the host stages over the same planes
    status = st_out.cpu().numpy().view(np.uint32)
    cells = rib_cells.cpu().numpy().view(ospf_rib.RIB_CELL_DT).reshape(n, P)
    dist = planes[0].view(n, V)
    hops = planes[1].view(n, V)
    nh = planes[2].view(n, V)
    sample = sorted({0, 1, n // 3, n // 2, n - 1})
    checks, host_s, decode_s, kinds = [], [], [], np.zeros(4, np.int64)
    for j in sample:
        a, s, e = view(idx[j])
        f = ospfv2.Flat(a)
        rv = f.router_vertex(a.router_id)
        d = dist[j].cpu().numpy().view(np.uint32).copy()
        h = hops[j].cpu().numpy().view(np.uint16).copy()
        m = nh[j].cpu().numpy().view(np.uint64).copy()
        nets = sorted({int(v) for v in f.csr.col[f.csr.row_ptr[rv]: f.csr.row_ptr[rv + 1]] if not f.is_router[v]})
        t0 = time.perf_counter()
        got = ospf_rib.rib_from_cells(a, rt, cells[j], np.asarray(nets, np.uint32), m[nets])
        decode_s.append(time.perf_counter() - t0)
        m4 = np.zeros((V, 4), np.uint64)
        m4[:, 0] = m
        t0 = time.perf_counter()
        spf = ospfv2.area_from_planes(a, lambda c, r, w: (d, h, m4[:, :w]))
        want = ospf_rib.update_rib_full(a.router_id, a.max_paths, [ospf_rib.RibArea(1, spf, a.ifaces, s)], e)
        host_s.append(time.perf_counter() - t0)
        ok = (status[j] == 0 and got.rc == 0 and got.routes.tobytes() == want.routes.tobytes()
              and got.nexthops.tobytes() == want.nexthops.tobytes())
        kinds += np.bincount(got.routes["path_type"], minlength=4)[:4]
        checks.append({"job": int(j), "root": int(a.router_id), "routes": int(len(got.routes)), "equal": bool(ok)})

    card, power = stage_bench.card_and_power()
    K = rt.n_contributors
    rib_bytes = {"cell_writes": n * P * 24, "records": n * K * 16, "offsets": n * P * 12,
                 "note": "records and offsets are re-read by every job and mostly stay in L2; plane gathers not counted"}
    intra_bytes = {"cell_writes": n * PI * 24, "records": n * it.n_contributors * 16, "offsets": n * PI * 4}
    gbs = lambda b, k: sum(v for v in b.values() if isinstance(v, int)) / med[k] / 1e6
    out = {
        "workload": f"C5 LSDB as area 0.0.0.1 (10000 routers, 40000 directed adjacencies, costs {{10, 20}}, 5 % on LANs) "
                    f"with ospfv2.inter_area_view(seed 0xC5, {kw}): {int((sums['lsa_type'] == 3).sum())} type-3, "
                    f"{int((sums['lsa_type'] == 4).sum())} type-4, {len(ext)} type-5 LSAs; {n} internal routers as roots",
        "card": card, "power_limit": power,
        "jobs": n, "vertices": V, "prefixes": P, "records": K, "intra_prefixes": PI, "intra_records": it.n_contributors,
        "refused_jobs": int((status != 0).sum()), "reps": args.reps,
        "ms": {k: {"median": med[k], "min": float(min(v)), "max": float(max(v))} for k, v in ms.items()},
        "bytes_per_launch": {"ospf_rib_cells_kernel": rib_bytes, "route_cells_kernel": intra_bytes},
        "GBps": {"ospf_rib_cells_kernel": gbs(rib_bytes, "ospf_rib_cells_kernel"),
                 "route_cells_kernel": gbs(intra_bytes, "route_cells_kernel")},
        "cell_write_GBps_over_datasheet": {"ospf_rib_cells_kernel": n * P * 24 / med["ospf_rib_cells_kernel"] / 1e6 / DATASHEET_GBS,
                                           "route_cells_kernel": n * PI * 24 / med["route_cells_kernel"] / 1e6 / DATASHEET_GBS},
        "datasheet_bw_GBps": DATASHEET_GBS,
        "host_per_root_s": {"area_from_planes_plus_update_rib_full": float(np.median(host_s)),
                            "rib_from_cells": float(np.median(decode_s))},
        "decoded_route_types_in_sample": {"intra": int(kinds[0]), "inter": int(kinds[1]), "type1": int(kinds[2]),
                                          "type2": int(kinds[3])},
        "cross_check_against_host_stages": checks,
    }
    stage_bench.write_json(out, args.out)
    ctx.close()
    if not all(c["equal"] for c in checks):
        sys.exit("ospf_rib_stage.py: a decoded job differs from the host stages")


if __name__ == "__main__":
    main()
