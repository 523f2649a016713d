#!/usr/bin/env python
"""IS-IS route stage on the C3 what-if workload: SPT batch + route kernel, device only.

C3 as bench.py builds it (10 000 systems, 40 000 directed adjacencies, wide metrics U[1,1000], seed SEED_BASE+3,
10 000 jobs of the same root, job j removing adjacency j mod 20 000), with two /32 prefixes per system as
tests/isis_synth.py::synth_instance advertises them.  Records, with CUDA events over warmed repeated launches on
the engine's stream: the SPT batch and the route kernel (hspf_isis_routes_batch) per launch, the cell and
contributor bytes per launch and what they come to against the H100 SXM data-sheet bandwidth; the host
hspf_isis_routes_from_planes and hspf_isis_routes_from_cells per job; the card's name and power limit.  Outside
the timed region one job's device cells are decoded and compared with compute_routes on the LSDB that lacks that
job's adjacency.  Fails without a GPU.

    python scripts/isis_route_stage.py [--out FILE] [--jobs N] [--reps R]
"""
import argparse
import ctypes as C
import sys
import time

import numpy as np

import stage_bench

DATASHEET_GBS = 3350.0        # H100 SXM HBM3, NVIDIA data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--jobs", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch = stage_bench.require_gpu("isis_route_stage.py")
    from bench import adjacency_edges
    from holo_b200 import capi, isis, synth
    from isis_synth import synth_instance
    from test_isis_route_cells_gpu import DeviceTopology

    t = synth.random_topology(10000, 40000, synth.SEED_BASE + 3, cost_lo=1, cost_hi=1000)
    inst = synth_instance(t, 0)
    lv = isis.synth_level(t)
    f = isis.Flat(lv)
    csr = f.csr
    root = f.vertex(isis.sysid(0) << 8)
    pair = adjacency_edges(csr, t, lambda i: f.vertex(isis.sysid(int(i)) << 8))
    n = args.jobs
    ov = [[(pair[j % len(pair)][0], capi.COST_DISABLED), (pair[j % len(pair)][1], capi.COST_DISABLED)] for j in range(n)]

    ctx = capi.Context(0)
    dev = torch.device("cuda", 0)
    rt = isis.RouteTable(inst)
    assert rt.root[isis.TOPO_STD] == root and rt.n_vertices[isis.TOPO_STD] == csr.n_vertices
    assert rt.root[isis.TOPO_MT6] == isis.NO_ROOT
    rt.upload(ctx)
    top = DeviceTopology(ctx, csr, root, n, ov)
    V, P, K = csr.n_vertices, rt.n_prefixes, rt.n_contributors
    u16p, u32p = C.POINTER(C.c_uint16), C.POINTER(C.c_uint32)
    cells = torch.empty(n * P * isis.CELL_DT.itemsize, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()

    stream = torch.cuda.ExternalStream(ctx.stream, device=dev)
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(args.reps)]

    def launch(e=None):
        if e:
            e[0].record(stream)
        ctx.run_device(top.g, top.js, top.rs, sync=False)
        if e:
            e[1].record(stream)
        isis.routes_batch_device(ctx, rt, n, top.rs, None, cells.data_ptr())
        if e:
            e[2].record(stream)

    for _ in range(3):                                       # warm-up: modules, both kernels, caches
        launch()
    ctx.sync()
    for e in ev:
        launch(e)
    ctx.sync()
    spt = [a.elapsed_time(b) for a, b, _ in ev]
    rk = [b.elapsed_time(c) for _, b, c in ev]

    # ---- outside the timed region: status, one job decoded against compute_routes on the changed LSDB
    st = top.status.cpu().numpy()
    single = {}
    for k in range(t.n_p2p):
        key = tuple(sorted((int(t.p2p_a[k]), int(t.p2p_b[k]))))
        single[key] = single.get(key, 0) + 1
    j = next(j for j in range(n) if single[tuple(sorted((int(t.p2p_a[j % len(pair)]), int(t.p2p_b[j % len(pair)]))))] == 1)
    a, b = int(t.p2p_a[j % len(pair)]), int(t.p2p_b[j % len(pair)])
    row = np.frombuffer(cells[j * P * 24:(j + 1) * P * 24].cpu().numpy().tobytes(), isis.CELL_DT)
    dj, hj, _ = top.planes(j)
    t0 = time.perf_counter()
    got = isis.routes_from_cells(inst, rt, row, (dj, hj), None, ov[j])
    decode_ms = (time.perf_counter() - t0) * 1e3
    cut = dict(inst, level=_without_adjacency(inst["level"], a, b, isis))
    want = isis.compute_routes(ctx, cut)
    decode_ok = (got.rc == capi.HSPF_OK and got.routes.tobytes() == want.routes.tobytes()
                 and got.nexthops.tobytes() == want.nexthops.tobytes())

    # host route stage over the same job's planes, for comparison (flatten included, as the call does it)
    lib = capi.load_library()
    lib.hspf_isis_routes_from_planes.argtypes = [C.POINTER(isis.InstanceStruct), u32p, u16p, u32p, u16p,
                                                 C.POINTER(isis.RibStruct)]
    host_ms = []
    for _ in range(3):
        t0 = time.perf_counter()
        r = isis._call_rib(lib.hspf_isis_routes_from_planes, inst, (),
                           tail_args=(dj.ctypes.data_as(u32p), hj.ctypes.data_as(u16p), C.cast(None, u32p), C.cast(None, u16p)))
        host_ms.append((time.perf_counter() - t0) * 1e3)
    assert r.rc == capi.HSPF_OK

    card, power = stage_bench.card_and_power()
    cell_bytes = n * P * isis.CELL_DT.itemsize
    contrib_bytes = n * (K * 16 + P * 8)                      # every job reads its prefixes' records and offsets
    rk_ms, spt_ms = float(np.median(rk)), float(np.median(spt))
    out = {
        "workload": f"C3 routes: IS-IS L2 synthetic LSDB, 10000 systems / 40000 directed adjacencies, wide metrics U[1,1000], "
                    f"{n} what-if jobs of one root (job j removes adjacency j mod {len(pair)}), 2 /32 prefixes per system",
        "seed": hex(synth.SEED_BASE + 3),
        "card": card, "power_limit": power,
        "jobs": n, "prefixes": P, "contributors": K, "vertices": V,
        "refused_jobs": int((st != 0).sum()),
        "reps": args.reps,
        "spt_batch_ms": {"median": spt_ms, "min": float(min(spt)), "max": float(max(spt))},
        "route_kernel_ms": {"median": rk_ms, "min": float(min(rk)), "max": float(max(rk))},
        "route_over_spt": rk_ms / spt_ms,
        "cell_bytes_per_launch": cell_bytes,
        "contributor_bytes_per_launch": contrib_bytes,
        "route_kernel_GBps": (cell_bytes + contrib_bytes) / rk_ms / 1e6,
        "route_kernel_share_of_datasheet_bw": (cell_bytes + contrib_bytes) / rk_ms / 1e6 / DATASHEET_GBS,
        "datasheet_bw_GBps": DATASHEET_GBS,
        "host_routes_from_planes_ms_per_job": float(np.median(host_ms)),
        "host_routes_from_cells_ms_per_job": decode_ms,
        "decode_check": {"job": j, "removed_adjacency": [a, b], "equal_to_compute_routes": bool(decode_ok),
                         "routes": int(len(got.routes))},
    }
    stage_bench.write_json(out, args.out)
    ctx.close()
    if not decode_ok:
        sys.exit("decoded cells differ from compute_routes")


def _without_adjacency(level, a, b, isis):
    """The level with the IS reachability between systems a and b removed (both directions)."""
    import copy
    lv = copy.copy(level)
    reaches = lv.reaches.copy()
    for owner, nbr in ((a, b), (b, a)):
        for i in np.nonzero(lv.lsps["lan_id"] == (isis.sysid(owner) << 8))[0]:
            lo, k = int(lv.lsps["reach_off"][i]), int(lv.lsps["n_reach"][i])
            hit = lo + np.nonzero(reaches["neighbor"][lo:lo + k] == (isis.sysid(nbr) << 8))[0]
            reaches["neighbor"][hit] = 0xFFFFFF0000              # a system without LSP: no adjacency
    lv.reaches = reaches
    return lv


if __name__ == "__main__":
    main()
