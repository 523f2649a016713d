#!/usr/bin/env python
"""The routes an IS-IS backbone router gets from an area's L1/L2 routers on an L1 what-if batch, device and host.

Workload: the L1 -> L2 script's domain (C3's LSDB as the L2 backbone, a 2 000-system L1 area from isis.l1l2_view
joined by three L1/L2 routers, summaries 10.1.4.0/22 and 10.2.0.0/16), every border with its own L1 batch and L1 -> L2
table, and backbone router R = 100 of C3.  10 000 jobs: job 0 is plain, job j > 0 disables one L1 adjacency (both
directions), row j of every border's L1 batch.

The launch bound of the backbone kernels (kBackboneBlocksPerSM in csrc/isis_backbone.cu) is timed against the other of
4 and 8 in the same run: that build is a copy of the library with the constant changed (built by this script, or given
with --variant), with its own tables over the same instances, reading the same device border cells.  Records, with
CUDA events over warmed alternating launches on the engine's stream: the three borders' L1 -> L2 cell launches
(summary pass + cell kernel), the backbone cell launch (every cell stored) and the backbone delta with summaries only
and with records, the last three for both bounds; the card's name and power limit.  Host figure (a host measurement): per job, the
chain the device replaces, hspf_isis_spt_from_planes + hspf_isis_l1_to_l2 for each border and
hspf_isis_routes_from_planes over R's LSDB with the borders' LSPs re-originated, over a sample of jobs.  Outside the
timed region: the delta is checked against the stored cells for all jobs, and sampled jobs are decoded and compared
with that chain.  Fails without a GPU.

    python scripts/isis_backbone_stage.py [--out FILE] [--jobs N] [--reps R] [--variant LIB]
"""
import argparse
import ctypes as C
import time

import numpy as np

import stage_bench

BOUND = ("isis_backbone.cu", "kBackboneBlocksPerSM")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--jobs", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--l1", type=int, default=2000)
    ap.add_argument("--backbone", type=int, default=100)
    ap.add_argument("--host-sample", type=int, default=5)
    ap.add_argument("--variant", default="", help="a prebuilt library with the other launch bound")
    args = ap.parse_args()
    torch = stage_bench.require_gpu("isis_backbone_stage.py")
    from holo_b200 import capi, isis, route_table, synth
    from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
    from test_isis_backbone_cells import restrict, same_rib, spliced
    from test_isis_l1l2_rib_cells import topology_flat
    from test_isis_route_cells_gpu import DeviceTopology
    from test_route_delta import reference

    summ = [("10.1.4.0/22", None), ("10.2.0.0/16", None)]
    c3 = synth.random_topology(10000, 40000, synth.SEED_BASE + 3, cost_lo=1, cost_hi=1000)
    vs = [isis.l1l2_view(1, n_l1=args.l1, l2_topology=c3, summaries=summ, cost_choices=[1, 5, 10, 20], root=b)
          for b in range(3)]
    ctx = capi.Context(0)
    n = args.jobs
    rng = np.random.default_rng(7)
    f = topology_flat(vs[0]["l1"], isis.MT_STANDARD)
    row, col = f.csr.row_ptr, f.csr.col
    src_of = np.repeat(np.arange(f.csr.n_vertices), np.diff(row))
    ovs = [[]]
    for e in rng.integers(0, f.csr.n_edges, n - 1):                 # one adjacency: the edge and its reverse
        u, w = int(src_of[e]), int(col[e])
        back = [int(x) for x in range(int(row[w]), int(row[w + 1])) if int(col[x]) == u]
        ovs.append([(int(e), capi.COST_DISABLED)] + [(x, capi.COST_DISABLED) for x in back])
    d_rows = torch.tensor(np.arange(n, dtype=np.uint32).view(np.int32), device="cuda")
    borders = []
    for v in vs:
        rib = isis.L1L2RibTable(v["l1"], v["l2"], v["cfg"], v["l2_derived"])
        rib.upload(ctx)
        t = isis.L1ToL2Table(v["l1"], v["l2"], rib)
        t.upload(ctx)
        top = DeviceTopology(ctx, topology_flat(v["l1"], isis.MT_STANDARD).csr, rib.root[0][isis.TOPO_STD], n, ovs)
        cells = torch.zeros(n * t.n_keys * 3, dtype=torch.int64, device="cuda")
        words = torch.zeros(max(n * t.n_summaries, 1), dtype=torch.int64, device="cuda")
        borders.append(dict(v=v, rib=rib, t=t, top=top, cells=cells, words=words, lid=v["l1"]["system_id"] << 8))
    r = isis.l1l2_backbone(vs[0], args.backbone)
    derived = vs[0]["derived_all"]
    bt = isis.BackboneTable(r, [b["t"] for b in borders], derived)
    bt.upload(ctx)
    fr = topology_flat(r, isis.MT_STANDARD)
    rtop = DeviceTopology(ctx, fr.csr, fr.vertex(r["system_id"] << 8), 1, [[]])
    P = bt.n_prefixes
    cells = torch.zeros(n * P * 3, dtype=torch.int64, device="cuda")
    job_out = torch.zeros(n * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device="cuda")
    cap = n * 64
    recs = torch.zeros(cap * DELTA_DT.itemsize, dtype=torch.uint8, device="cuda")
    total = torch.zeros(1, dtype=torch.int64, device="cuda")
    base_cells = torch.zeros(P * 3, dtype=torch.int64, device="cuda")
    st = torch.cuda.ExternalStream(ctx.lib.hspf_stream(ctx.handle))
    bcells = [b["cells"].data_ptr() for b in borders]

    # the other launch bound, from a copy of the library, with its own tables over the same instances
    cur = stage_bench.launch_bound(*BOUND)
    other = 4 if cur == 8 else 8
    libv = C.CDLL(args.variant or str(stage_bench.build_variant(*BOUND, other, "backbone_bound_")))
    route_table.declare(libv)
    keep = []
    for b in borders:
        s1, s2 = isis.instance_struct(b["v"]["l1"]), isis.instance_struct(b["v"]["l2"])
        m = np.ascontiguousarray(b["v"]["l2_derived"], np.uint8)
        rv, tv = C.c_void_p(), C.c_void_p()
        assert libv.hspf_isis_l1l2_ribtable_create(C.byref(s1), C.byref(s2), m.ctypes.data, b["rib"].cfg.ctypes.data,
                                                   len(b["rib"].cfg), C.byref(rv)) == 0
        assert libv.hspf_isis_l1_to_l2_table_create(C.byref(s1), C.byref(s2), None, rv, C.byref(tv)) == 0
        keep.append((rv, tv))
    sr = isis.instance_struct(r)
    der = np.ascontiguousarray(derived, np.uint8)
    btv = C.c_void_p()
    assert libv.hspf_isis_backbone_table_create(C.byref(sr), der.ctypes.data, 3, (C.c_void_p * 3)(*[t for _, t in keep]),
                                                C.byref(btv)) == 0
    assert libv.hspf_isis_backbone_table_upload(ctx.handle, btv) == 0
    cellsv = torch.zeros(n * P * 3, dtype=torch.int64, device="cuda")
    bcp = (C.c_void_p * 3)(*bcells)
    libs = {cur: (ctx.lib, bt.handle, cells), other: (libv, btv, cellsv)}

    def border_launch():
        for b in borders:
            isis.l1_to_l2_cells_device(ctx, b["t"], n, (b["top"].rs, None), n, d_rows.data_ptr(), b["words"].data_ptr(),
                                       0, b["cells"].data_ptr())

    def cell_launch(b=cur):
        lib, h, c = libs[b]
        assert lib.hspf_isis_backbone_cells(ctx.handle, h, n, C.byref(rtop.rs), None, bcp, None, None, c.data_ptr()) == 0

    def delta(with_records, b=cur):
        lib, h, _ = libs[b]
        assert lib.hspf_isis_backbone_delta(ctx.handle, h, n, C.byref(rtop.rs), None, bcp, None, base_cells.data_ptr(), 1,
                                            None, job_out.data_ptr(), recs.data_ptr() if with_records else None,
                                            cap if with_records else 0, total.data_ptr()) == 0

    for b in borders:
        b["top"].run()
    rtop.run()
    ctx.sync()
    border_launch()
    cell_launch()
    ctx.sync()
    base_cells.copy_(cells[: P * 3])                 # job 0, plain
    work = {"border_l1_to_l2_cells_x3": border_launch}
    for b in (cur, other):
        work[f"backbone_cells_bound{b}"] = lambda b=b: cell_launch(b)
        work[f"backbone_delta_summaries_bound{b}"] = lambda b=b: delta(False, b)
        work[f"backbone_delta_records_bound{b}"] = lambda b=b: delta(True, b)
    for fn in work.values():
        fn()
    ctx.sync()
    times = {k: [] for k in work}
    for _ in range(args.reps):
        for k, fn in work.items():
            a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(st)
            fn()
            z.record(st)
            z.synchronize()
            times[k].append(a.elapsed_time(z))
    med = {k: float(np.median(x)) for k, x in times.items()}
    gpu = ", ".join(stage_bench.card_and_power())
    # outside the timed region: the delta against the stored cells, sampled jobs against the host chain
    border_launch()
    cell_launch(cur)
    cell_launch(other)
    ctx.sync()
    same_bounds = bool(torch.equal(cells, cellsv))
    ch = cells.cpu().numpy().view(np.uint8).view(isis.CELL_DT).reshape(n, P)
    delta(True)
    ctx.sync()
    jw, rw, tw = reference(ch, ch[:1], None, cap=cap)
    assert job_out.cpu().numpy().view(DELTA_JOB_DT).tobytes() == jw.tobytes() and int(total.item()) == tw
    assert recs.cpu().numpy().view(DELTA_DT)[: min(cap, tw)].tobytes() == rw.tobytes()
    for b in borders:
        t = b["t"]
        b["ch"] = b["cells"].cpu().numpy().view(np.uint8).view(isis.CELL_DT).reshape(n, t.n_keys)
        b["wh"] = b["words"].cpu().numpy().view(np.uint64)[: n * t.n_summaries].reshape(n, t.n_summaries)
        b["dist"] = b["top"].dist.cpu().numpy().view(np.uint32).reshape(n, b["top"].V)
        b["hops"] = b["top"].hops.cpu().numpy().view(np.uint16).reshape(n, b["top"].V)
    rd = rtop.dist.cpu().numpy().view(np.uint32).reshape(1, rtop.V)[0]
    rh = rtop.hops.cpu().numpy().view(np.uint16).reshape(1, rtop.V)[0]
    affected = {(int(p["is_v6"]), bytes(p["bytes"]), int(k)) for p, k in zip(bt.prefix, bt.len)}

    class Entries:
        pass

    def chain(j, entries):
        bs = []
        for b, e in zip(borders, entries):
            x = Entries()
            x.lid, x.entries = b["lid"], {j: e}
            bs.append(x)
        return isis.routes_from_planes(spliced(r, derived, bs, j), lambda csr, root: (rd, rh))

    sample = [0, 1, n // 2, n - 1]
    for j in sample:
        entries = [isis.l1_to_l2_from_cells(b["v"]["l1"], b["t"], b["ch"][j], b["wh"][j]) for b in borders]
        got = isis.backbone_from_cells(r, bt, ch[j], [(rd, rh), None], entries)
        same_rib(got, restrict(chain(j, entries), lambda k: k in affected))
    # host figure: per border the SPT from the job's planes and the propagation, then R's routes over the spliced LSDB
    jobs = rng.choice(np.arange(1, n), args.host_sample, replace=False)

    def active(cfg, w):
        a = cfg.copy()
        a["metric"] = w & np.uint64(0xFFFFFFFF)
        return a[(w >> np.uint64(32)) == 1].copy()
    acts = {(k, int(j)): active(b["v"]["cfg"], b["wh"][j]) for k, b in enumerate(borders) for j in jobs}
    t0 = time.perf_counter()
    for j in jobs:
        entries = []
        for k, b in enumerate(borders):
            l1 = b["v"]["l1"]
            spt = f.spt_from_planes(b["rib"].root[0][isis.TOPO_STD], b["dist"][j], b["hops"][j], ovs[j])
            entries.append(isis.l1_to_l2(l1["level"], l1["system_id"], spt, None, l1["level"].metric_type,
                                         r["level"].metric_type, b["v"]["cfg"], acts[(k, int(j))]))
        chain(int(j), entries)
    host_ms = (time.perf_counter() - t0) * 1000.0 / len(jobs)
    out = dict(gpu=gpu, workload="C3 as the L2 backbone + a 2 000-system L1 area, three borders, backbone router "
                                 f"{args.backbone}, two summaries over part of the area",
               jobs=n, affected_prefixes=P, border_keys=[b["t"].n_keys for b in borders], l2_vertices=rtop.V,
               reps=args.reps, median_ms=med, launch_bound=cur, other_bound=other, cells_equal_other_bound=same_bounds,
               delta_records=tw, delta_checked_jobs=n, sampled_jobs_decoded=len(sample),
               host_ms_per_job_chain=host_ms, host_sample_jobs=len(jobs),
               host_note="host measurement (CPU of the GPU machine), not an H100 figure")
    stage_bench.write_json(out, args.out)
    for rv, tv in keep:
        libv.hspf_isis_l1_to_l2_table_free(tv)
        libv.hspf_isis_l1l2_ribtable_free(rv)
    libv.hspf_isis_backbone_table_free(btv)
    ctx.close()


if __name__ == "__main__":
    main()
