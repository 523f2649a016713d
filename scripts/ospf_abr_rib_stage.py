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


def build_variant(bound: int, tmp: Path) -> Path:
    """libholo_spf.so with kAbrBlocksPerSM = bound, built from a copy of the sources in `tmp`."""
    from holo_b200 import build
    src = tmp / "holo_b200" / "csrc"                 # the sources include ../../include
    shutil.copytree(build.CSRC, src)
    shutil.copytree(build.ROOT / "include", tmp / "include")
    cu = src / "ospfv2_abr_rib_cells.cu"
    text, n = re.subn(r"constexpr uint32_t kAbrBlocksPerSM = \d+;", f"constexpr uint32_t kAbrBlocksPerSM = {bound};",
                      cu.read_text())
    assert n == 1
    cu.write_text(text)
    out = tmp / "libholo_spf_variant.so"
    flags = [f for f in build.NVCC_FLAGS]
    srcs = sorted(list(src.glob("*.cu")) + list(src.glob("*.cc")))
    subprocess.run([build.os.environ.get("NVCC", "nvcc"), *flags, "-o", str(out), *map(str, srcs)], check=True,
                   capture_output=True)
    return out


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
    import torch
    if not torch.cuda.is_available():
        sys.exit("ospf_abr_rib_stage.py: no CUDA device; this measurement runs on the GPU only")
    from holo_b200 import capi, ospf_rib, ospfv2, route_table, synth
    from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT

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
    u32p, u16p, u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint16), C.POINTER(C.c_uint64)
    keep, spt, rs_list, n_rows = [], [], [], []

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
        return g, js, rs, pl

    planes = []
    for i in range(A):
        g, js, rs, pl = spt_batch(flats[i].csr, rvs[i], ovs[i])
        spt.append((g, js, rs))
        rs_list.append(rs)
        planes.append(pl)
        n_rows.append(len(ovs[i]))
    # the one-area stage for comparison: area 0's rows rooted at an internal router of area 0
    a0 = areas[0]
    internal = next(int(r) for r, fl in zip(a0.router_lsas["adv_rtr"], a0.router_lsas["flags"])
                    if not fl & 0x01 and flats[0].router_vertex(int(r)) != 0xFFFFFFFF)
    iv = flats[0].router_vertex(internal)
    g_in, js_in, rs_in, pl_in = spt_batch(flats[0].csr, iv, ovs[0])
    rt1 = ospf_rib.RibTable(flats[0], a0.area_id, sums[0], ext)
    rt1.upload(ctx)
    m0 = len(ovs[0])
    d_roots_in = torch.full((m0,), iv, dtype=torch.int32, device=dev)
    cells1 = torch.empty(m0 * rt1.n_prefixes * 24, dtype=torch.uint8, device=dev)
    for g, js, rs in spt:
        ctx.run_device(g, js, rs, sync=False)
    ctx.run_device(g_in, js_in, rs_in, sync=False)
    ctx.sync()
    d_rows = torch.from_numpy(rows.view(np.int32).reshape(-1).copy()).to(dev)

    # the other launch bound, from a copy of the library
    tmp = Path(tempfile.mkdtemp(prefix="abr_bound_"))
    lib8 = C.CDLL(str(build_variant(8, tmp)))
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

    variants = {f"spt_batch_area{i}": (lambda g=g, js=js, rs=rs: ctx.run_device(g, js, rs, sync=False))
                for i, (g, js, rs) in enumerate(spt)}
    variants.update({
        "abr_rib_cells_kernel_bound4": abr_cells(lib4, rt.handle, 4),
        "abr_rib_cells_kernel_bound8": abr_cells(lib8, h8, 8),
        "abr_rib_delta_summaries_bound4": delta(lib4, rt.handle, False),
        "abr_rib_delta_summaries_bound8": delta(lib8, h8, False),
        "abr_rib_delta_records_bound4": delta(lib4, rt.handle, True),
        "abr_rib_delta_records_bound8": delta(lib8, h8, True),
        "ospf_rib_cells_kernel_area0_internal_root": lambda: ospf_rib.rib_cells_device(
            ctx, rt1, m0, rs_in, d_roots_in.data_ptr(), cells1.data_ptr()),
    })
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
        got = ospf_rib.abr_rib_from_cells(areas, rt, cj, ga, gv, gn)
        t_dec = time.perf_counter() - t0
        t0 = time.perf_counter()
        ra = []
        for i, a in enumerate(areas):
            m4 = np.zeros((len(p[i][0]), 4), np.uint64)
            m4[:, 0] = p[i][2]
            spf = ospfv2.area_from_planes(a, lambda c, r, w, d=p[i][0], h=p[i][1], m4=m4: (d, h, m4[:, :w]))
            ra.append(ospf_rib.RibArea(a.area_id, spf, a.ifaces, sums[i]))
        want = ospf_rib.update_rib_full(ospfv2.ABR_ROUTER_ID, a0.max_paths, ra, ext)
        t_host = time.perf_counter() - t0
        ok = (status[j] == 0 and got.rc == 0 and got.routes.tobytes() == want.routes.tobytes()
              and got.nexthops.tobytes() == want.nexthops.tobytes())
        decoded.append({"job": int(j), "rows": [int(x) for x in rows[j]], "routes": int(len(got.routes)), "equal": bool(ok),
                        "decode_s": round(t_dec, 4), "host_stages_s": round(t_host, 4)})
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    card, power = (q[0].split(", ") + ["?"])[:2] if q else (torch.cuda.get_device_name(0), "?")
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
    text = json.dumps(out, indent=1)
    print(json.dumps({k: out[k] for k in ("card", "power_limit", "median_ms", "cells_bound4_equal_bound8", "delta_checks",
                                          "changes", "prefixes", "areas")}, indent=1))
    print("decodes equal:", all(d["equal"] for d in decoded))
    if args.out:
        Path(args.out).write_text(text + "\n")
    shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
