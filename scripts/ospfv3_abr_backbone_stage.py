#!/usr/bin/env python
"""The OSPFv3 area-border-router stage over what-if jobs inside an area the router is not attached to
(hspf_ospfv3_abr_backbone_table_create through hspf_ospfv2_abr_backbone_cells / hspf_ospfv2_abr_backbone_delta) on a
10 000-job what-if batch inside one non-backbone area; device only:
python scripts/ospfv3_abr_backbone_stage.py [--jobs 10000] [--reps 10] [--out profiles/h100_C5v3_abr_backbone.json]

Domain (ospfv3.abr_backbone_view, seed 0xC5, area1_asbrs=2, area1_ext=1000): C5's topology as OSPFv3 area 0, a
2 000-router area 1 with three area border routers ("borders", the first also in backbone_view's small area 2) and
two ASBRs with about 1 000 AS-external LSAs each, and R = router 0 of area 0, also the ABR of a 2 000-router area 3.
Job 0 is unperturbed; job j > 0 disables one router-to-router link of area 1 (both directions).  Each border runs its
area SPT batches (one row per job in area 1) and its OSPFv3 ABR cells (hspf_ospfv2_abr_rib_cells); R's calls read
those cells and the borders' area-1 rows in place with R's row 0 of areas 0 and 3.

The launch bound of the OSPFv3 kernels (kAbrBackboneV3BlocksPerSM in csrc/ospfv2_abr_backbone.cu) is timed against
the other bound in the same run: a second copy of the library, built into a temporary directory with the other value, runs the
same calls on the same table data, planes and border cells, alternating with the first.  CUDA-event medians over
`--reps` alternating launches after warm-up; the card's name and power limit are read (not set) in the same run.
Outside the timed region: both builds' cells are byte-identical and the delta's total equals a count over the stored
cells.  Host figure (a CPU measurement): per job, the host chain the stage replaces (each border's area_from_planes +
update_rib_full_v3 + net_summaries_v3 + rtr_summaries_v3, then R's update_rib_full_v3 over its two areas), timed over
a few jobs."""
import argparse
import ctypes as C
import json
import re
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
CONST = "kAbrBackboneV3BlocksPerSM"


def build_variant(bound: int, tmp: Path) -> Path:
    """libholo_spf.so with kAbrBackboneV3BlocksPerSM = bound, built from a copy of the sources in `tmp`."""
    from holo_b200 import build
    src = tmp / "holo_b200" / "csrc"
    shutil.copytree(build.CSRC, src)
    shutil.copytree(build.ROOT / "include", tmp / "include")
    cu = src / "ospfv2_abr_backbone.cu"
    text, n = re.subn(rf"constexpr uint32_t {CONST} = \d+;", f"constexpr uint32_t {CONST} = {bound};", cu.read_text())
    assert n == 1
    cu.write_text(text)
    out = tmp / "libholo_spf_variant.so"
    srcs = sorted(list(src.glob("*.cu")) + list(src.glob("*.cc")))
    subprocess.run([build.os.environ.get("NVCC", "nvcc"), *build.NVCC_FLAGS, "-o", str(out), *map(str, srcs)], check=True,
                   capture_output=True)
    return out


def current_bound() -> int:
    return int(re.search(rf"constexpr uint32_t {CONST} = (\d+);",
                         (ROOT / "holo_b200" / "csrc" / "ospfv2_abr_backbone.cu").read_text()).group(1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--jobs", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--host-jobs", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("ospfv3_abr_backbone_stage.py: no CUDA device; this measurement runs on the GPU only")
    from holo_b200 import capi, ospf_rib, ospfv3, route_table, synth
    from holo_b200.route_table import DELTA_JOB_DT, DELTA_DT

    t0 = synth.random_topology(10000, 40000, synth.SEED_BASE + 5, cost_choices=[10, 20], lan_fraction=0.05)
    t1 = synth.random_topology(2000, 8000, synth.SEED_BASE + 850, cost_choices=[10, 20], lan_fraction=0.05)
    t2 = synth.random_topology(2000, 8000, synth.SEED_BASE + 851, cost_choices=[10, 20], lan_fraction=0.05)
    v = ospfv3.abr_backbone_view(t0, t1, t2, 0xC5, area1_asbrs=2, area1_ext=1000)
    ctx = capi.Context(0)
    dev = torch.device("cuda", 0)
    n = args.jobs
    rng = np.random.default_rng(0xC5)
    u32p, u16p, u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint16), C.POINTER(C.c_uint64)
    keep = []

    def spt_batch(csr, root, ov):
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
        ctx.run_device(g, js, rs, sync=False)
        return rs, pl

    # the jobs: one link of the area per job, named by its end points' ids
    bareas = [b[0] for b in v["borders"]]
    i1 = [b[1].index(1) for b in v["borders"]]
    f1 = ospfv3.Flat(bareas[0][i1[0]])
    src = np.repeat(np.arange(f1.csr.n_vertices), np.diff(f1.csr.row_ptr))
    links = sorted({tuple(sorted((int(f1.router_ids[src[e]]), int(f1.router_ids[f1.csr.col[e]]))))
                    for e in range(f1.csr.n_edges) if f1.is_router[src[e]] and f1.is_router[f1.csr.col[e]]})
    job_links = [None] + [links[int(rng.integers(len(links)))] for _ in range(n - 1)]
    tables, border_cells, flats_all, planes_all, border_rs, border_nrows, border_rows = [], [], [], [], [], [], []
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
        rs_list, n_rows, pls = [], [], []
        for i, fl in enumerate(flats):
            root = fl.router_vertex(areas[0].router_id)
            ov = [[]] if i != i1[b] else [[(e, capi.COST_DISABLED) for e in by_pair.get(l, [])] if l else [] for l in job_links]
            rs, pl = spt_batch(fl.csr, root, ov)
            rs_list.append(rs); n_rows.append(len(ov)); pls.append(pl)
        rows = np.zeros((n, len(areas)), np.uint32)
        rows[:, i1[b]] = np.arange(n)
        d_rows = torch.from_numpy(rows.view(np.int32).reshape(-1).copy()).to(dev)
        cells = torch.empty(n * rt.n_prefixes * 24, dtype=torch.uint8, device=dev)
        ospf_rib.abr_rib_cells_device(ctx, rt, n, rs_list, n_rows, d_rows.data_ptr(), cells.data_ptr())
        keep += [d_rows, rs_list]
        border_rs.append((capi.ResultStruct * len(rs_list))(*rs_list))
        border_nrows.append(np.asarray(n_rows, np.uint32))
        border_rows.append(d_rows.data_ptr())
        tables.append(rt); border_cells.append(cells); flats_all.append(flats); planes_all.append(pls)
    r_areas = v["r_areas"]
    r_flats = [ospfv3.Flat(a) for a in r_areas]
    r_rs, r_pl = [], []
    for a, f in zip(r_areas, r_flats):
        rs, pl = spt_batch(f.csr, f.router_vertex(a.router_id), [[]])
        r_rs.append(rs); r_pl.append(pl)
    bt = ospf_rib.AbrBackboneTable(r_areas[0].router_id, r_flats, v["area_ids"], v["summaries"], None, v["externals"],
                                   tables)
    assert bt.v3 and bt.n_asbr_slots > 0
    bt.upload(ctx)
    r_arr = (capi.ResultStruct * len(r_rs))(*r_rs)
    ctx.sync()
    P = bt.n_prefixes
    bc = [c.data_ptr() for c in border_cells]

    cur = current_bound()
    other = 8 if cur == 4 else 4
    libv = C.CDLL(str(build_variant(other, Path(tempfile.mkdtemp(prefix="abr_backbone_v3_bound_")))))
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
    arr = (C.c_void_p * len(vt))(*[h.value for h in vt])
    fl_, ids_, sp_, ns_, act_, _s, ext_, _f = bt._keep
    assert libv.hspf_ospfv3_abr_backbone_table_create(bt.router_id, len(r_areas), fl_, ids_.ctypes.data, sp_,
                                                      ns_.ctypes.data, act_.ctypes.data, ext_.ctypes.data, len(ext_),
                                                      arr, len(vt), C.byref(hv)) == 0
    assert libv.hspf_ospfv2_abr_backbone_table_upload(ctx.handle, hv) == 0
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
        return lambda: lib.hspf_ospfv2_abr_backbone_cells(ctx.handle, h, n, r_arr, bca, None, bpa, bna, bra, None,
                                                          cells[b].data_ptr())

    cell_launch(4)(); cell_launch(8)()
    ctx.sync()
    same_bounds = bool(torch.equal(cells[4], cells[8]))
    base = cells[cur][: P * 24].clone()
    lib, h = handles[cur]
    assert lib.hspf_ospfv2_abr_backbone_delta(ctx.handle, h, n, r_arr, bca, None, bpa, bna, bra,
                                               base.data_ptr(), 1, None, job_out.data_ptr(), None, 0,
                                               total.data_ptr()) == 0
    ctx.sync()
    cap = int(total.cpu()[0])
    w = cells[cur].view(torch.int64).reshape(n, P, 3)
    changed = int((w != w[0:1]).any(dim=2).sum().item())
    recs = torch.empty(max(cap, 1) * DELTA_DT.itemsize, dtype=torch.uint8, device=dev)

    def delta(b, with_records):
        lib, h = handles[b]
        return lambda: lib.hspf_ospfv2_abr_backbone_delta(ctx.handle, h, n, r_arr, bca, None, bpa, bna, bra,
                                                           base.data_ptr(), 1, None, job_out.data_ptr(),
                                                           recs.data_ptr() if with_records else None,
                                                           cap if with_records else 0, total.data_ptr())

    work = {}
    for b in (4, 8):
        work[f"abr_backbone_cells_bound{b}"] = cell_launch(b)
        work[f"abr_backbone_delta_summaries_bound{b}"] = delta(b, False)
        work[f"abr_backbone_delta_records_bound{b}"] = delta(b, True)
    stream = torch.cuda.ExternalStream(ctx.stream, device=dev)
    for _ in range(2):
        for fn in work.values():
            fn()
    ctx.sync()
    ev = {k: [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.reps)]
          for k in work}
    for r in range(args.reps):
        for k, fn in work.items():
            ev[k][r][0].record(stream)
            fn()
            ev[k][r][1].record(stream)
    ctx.sync()
    med = {k: float(np.median([a.elapsed_time(b) for a, b in ev[k]])) for k in work}

    # host chain per job (CPU), over the device planes read back
    def host_planes(pl, row, V):
        d = pl[0].view(torch.int32).reshape(-1, V)[row].cpu().numpy().view(np.uint32)
        hh = pl[1].reshape(-1, V)[row].cpu().numpy().view(np.uint16)
        m = pl[2].reshape(-1, V)[row].cpu().numpy().view(np.uint64)
        return d, hh, m

    def spf_of(a, p):
        return ospfv3.area_from_planes(a, lambda csr, root, nhw: (p[0], p[1], np.pad(p[2][:, None], ((0, 0), (0, nhw - 1)))))

    host_ms = []
    rp = [host_planes(pl, 0, f.csr.n_vertices) for pl, f in zip(r_pl, r_flats)]
    bids = {int(x.router_id) for x in tables}
    for j in range(1, 1 + args.host_jobs):
        t = time.perf_counter()
        new = [tuple(s) for s in v["summaries"][0].tolist() if int(s[0]) not in bids]   # Inter-Area-Prefix and -Router
        for b, (areas, ids, sums) in enumerate(v["borders"]):
            ra = []
            for i, a in enumerate(areas):
                p = host_planes(planes_all[b][i], j if i == i1[b] else 0, flats_all[b][i].csr.n_vertices)
                ra.append(ospf_rib.RibArea(a.area_id, spf_of(a, p), a.ifaces, sums[i], True))
            new += ospfv3.nonbackbone_lsas(areas[0].router_id, areas[0].max_paths, ra, v["externals"], ids.index(0))
        s = np.array(new, ospf_rib.INTER_AREA_LSA_DT)
        s = s[np.lexsort((s["lsa_id"], s["adv_rtr"], s["lsa_type"]))]
        ospf_rib.update_rib_full_v3(r_areas[0].router_id, r_areas[0].max_paths,
                                 [ospf_rib.RibArea(a.area_id, spf_of(a, p), a.ifaces, s if a.area_id == 0 else ss, True)
                                  for a, p, ss in zip(r_areas, rp, v["summaries"])], v["externals"])
        host_ms.append((time.perf_counter() - t) * 1e3)

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    card, power = (q[0].split(", ") + ["?"])[:2] if q else (torch.cuda.get_device_name(0), "?")
    out = {
        "stage": "hspf_ospfv3_abr_backbone_table_create, hspf_ospfv2_abr_backbone_cells / _delta (OSPFv3 table)",
        "workload": {"area0": "C5 as OSPFv3: 10000 routers, 40000 links, costs {10, 20}, 5 % LANs",
                     "area1": "2000 routers", "area3": "2000 routers (R's other area)",
                     "area1_asbrs": len(v["area1_asbrs"]), "externals": len(v["externals"]),
                     "borders": len(tables), "jobs": n, "affected_prefixes": P, "slots": bt.n_slots,
                     "inter_area_router_slots": bt.n_asbr_slots, "plane_sets": bt.n_asbr_sets,
                     "border_keys": [t.n_prefixes for t in tables]},
        "card": card, "power_limit": power, "reps": args.reps, "median_ms": med, "launch_bound": cur,
        "other_bound": other, "cells_equal_other_bound": same_bounds,
        "delta_total": cap, "delta_total_equals_changed_cells": cap == changed,
        "host_chain_ms_per_job": float(np.median(host_ms)), "host_jobs_timed": len(host_ms),
        "note": "device figures are CUDA-event medians of alternating launches; the host chain is a CPU figure",
    }
    print(json.dumps(out))
    if args.out:
        Path(args.out).write_text(json.dumps(out, indent=1) + "\n")


if __name__ == "__main__":
    main()
