#!/usr/bin/env python
"""What an IS-IS L1/L2 router propagates into its L2 LSP on a what-if batch, device and host.

Workload: the L1/L2 routing-table script's domain (C3's LSDB as the L2 backbone, a 2 000-system L1 area from
isis.l1l2_view joined by three L1/L2 routers), with summaries over part of the area only (10.1.4.0/22 and 10.2.0.0/16),
so that the other /32s of the area, about 1 000 keys, propagate one by one.  10 000 jobs of root 0: job 0 is plain,
job j > 0 disables one L1 adjacency (both directions), row j of the L1 batch.

The launch bound of the stage's kernels (kL1ToL2BlocksPerSM in csrc/isis_l1_to_l2.cu) is timed against the other of 4
and 8 in the same run: that build is a copy of the library with the constant changed (built by this script, or given
with --variant), run on the same table data and planes.  Records, with CUDA events over warmed alternating launches on
the engine's stream: the L1 SPT batch, the cell launch (summary pass + cell kernel, every cell stored) and the delta
with summaries only and with records, for both bounds; the card's name and power limit.  Host figure (a host
measurement): the per-job time of hspf_isis_spt_from_planes + hspf_isis_l1_to_l2 over a sample of jobs.  Outside the
timed region: both builds' cells and words are compared, the delta is checked against the stored cells for all jobs,
and sampled jobs are decoded and compared with the host function.  Fails without a GPU.

    python scripts/isis_l1_to_l2_stage.py [--out FILE] [--jobs N] [--reps R] [--variant LIB]
"""
import argparse
import ctypes as C
import time

import numpy as np

import stage_bench

BOUND = ("isis_l1_to_l2.cu", "kL1ToL2BlocksPerSM")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--jobs", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--l1", type=int, default=2000)
    ap.add_argument("--host-sample", type=int, default=20)
    ap.add_argument("--variant", default="", help="a prebuilt library with the other launch bound")
    args = ap.parse_args()
    torch = stage_bench.require_gpu("isis_l1_to_l2_stage.py")
    from holo_b200 import capi, isis, route_table, synth
    from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
    from test_isis_l1_to_l2_cells import host
    from test_isis_l1l2_rib_cells import topology_flat
    from test_isis_route_cells_gpu import DeviceTopology
    from test_route_delta import reference

    summ = [("10.1.4.0/22", None), ("10.2.0.0/16", None)]
    c3 = synth.random_topology(10000, 40000, synth.SEED_BASE + 3, cost_lo=1, cost_hi=1000)
    v = isis.l1l2_view(1, n_l1=args.l1, l2_topology=c3, summaries=summ, cost_choices=[1, 5, 10, 20])
    ctx = capi.Context(0)
    rib = isis.L1L2RibTable(v["l1"], v["l2"], v["cfg"])
    rib.upload(ctx)
    t = isis.L1ToL2Table(v["l1"], v["l2"], rib)
    t.upload(ctx)
    n = args.jobs
    rng = np.random.default_rng(7)
    f = topology_flat(v["l1"], isis.MT_STANDARD)
    row, col = f.csr.row_ptr, f.csr.col
    src_of = np.repeat(np.arange(f.csr.n_vertices), np.diff(row))
    ovs = [[]]
    for e in rng.integers(0, f.csr.n_edges, n - 1):                 # one adjacency: the edge and its reverse
        u, w = int(src_of[e]), int(col[e])
        back = [int(x) for x in range(int(row[w]), int(row[w + 1])) if int(col[x]) == u]
        ovs.append([(int(e), capi.COST_DISABLED)] + [(x, capi.COST_DISABLED) for x in back])
    top = DeviceTopology(ctx, f.csr, rib.root[0][isis.TOPO_STD], n, ovs)
    rows = np.arange(n, dtype=np.uint32)
    d_rows = torch.tensor(rows.view(np.int32), device="cuda")
    K, S = t.n_keys, t.n_summaries
    cells = torch.zeros(n * K * 3, dtype=torch.int64, device="cuda")
    words = torch.zeros(n * S, dtype=torch.int64, device="cuda")
    job_out = torch.zeros(n * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device="cuda")
    cap = n * 64
    recs = torch.zeros(cap * DELTA_DT.itemsize, dtype=torch.uint8, device="cuda")
    total = torch.zeros(1, dtype=torch.int64, device="cuda")
    st = torch.cuda.ExternalStream(ctx.lib.hspf_stream(ctx.handle))

    # the other launch bound, from a copy of the library, with its own tables over the same instances
    cur = stage_bench.launch_bound(*BOUND)
    other = 4 if cur == 8 else 8
    libv = C.CDLL(args.variant or str(stage_bench.build_variant(*BOUND, other, "l1_to_l2_bound_")))
    route_table.declare(libv)
    s1, s2 = isis.instance_struct(v["l1"]), isis.instance_struct(v["l2"])
    rv, tv = C.c_void_p(), C.c_void_p()
    assert libv.hspf_isis_l1l2_ribtable_create(C.byref(s1), C.byref(s2), None, rib.cfg.ctypes.data, len(rib.cfg),
                                               C.byref(rv)) == 0
    assert libv.hspf_isis_l1l2_ribtable_upload(ctx.handle, rv) == 0
    assert libv.hspf_isis_l1_to_l2_table_create(C.byref(s1), C.byref(s2), None, rv, C.byref(tv)) == 0
    assert libv.hspf_isis_l1_to_l2_table_upload(ctx.handle, tv) == 0
    libs = {cur: (ctx.lib, t.handle), other: (libv, tv)}
    cellsv = torch.zeros(n * K * 3, dtype=torch.int64, device="cuda")
    wordsv = torch.zeros(n * S, dtype=torch.int64, device="cuda")
    rs = [C.byref(top.rs), None]
    base_cells = torch.zeros(K * 3, dtype=torch.int64, device="cuda")

    def cell_launch(b=cur):
        lib, h = libs[b]
        c, w = (cells, words) if b == cur else (cellsv, wordsv)
        assert lib.hspf_isis_l1_to_l2_cells(ctx.handle, h, n, *rs, top.n, d_rows.data_ptr(), w.data_ptr(), None,
                                            c.data_ptr()) == 0

    def delta(with_records, b=cur):
        lib, h = libs[b]
        assert lib.hspf_isis_l1_to_l2_delta(ctx.handle, h, n, *rs, top.n, d_rows.data_ptr(), words.data_ptr(),
                                            base_cells.data_ptr(), 1, None, job_out.data_ptr(),
                                            recs.data_ptr() if with_records else None, cap if with_records else 0,
                                            total.data_ptr()) == 0

    top.run()
    ctx.sync()
    cell_launch()
    ctx.sync()
    base_cells.copy_(cells[: K * 3])                 # job 0, plain
    work = {"spt_l1": top.run}
    for b in (cur, other):
        work[f"cells_bound{b}"] = lambda b=b: cell_launch(b)
        work[f"delta_summaries_bound{b}"] = lambda b=b: delta(False, b)
        work[f"delta_records_bound{b}"] = lambda b=b: delta(True, b)
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
    cell_launch(cur)
    cell_launch(other)
    ctx.sync()
    same_bounds = bool(torch.equal(cells, cellsv) and torch.equal(words, wordsv))
    # outside the timed region: the delta against the stored cells, sampled jobs against the host function
    ch = cells.cpu().numpy().view(np.uint8).view(isis.CELL_DT).reshape(n, K)
    wh = words.cpu().numpy().view(np.uint64).reshape(n, S)
    delta(True)
    ctx.sync()
    jw, rw, tw = reference(ch, ch[:1], None, cap=cap)
    assert job_out.cpu().numpy().view(DELTA_JOB_DT).tobytes() == jw.tobytes() and int(total.item()) == tw
    assert recs.cpu().numpy().view(DELTA_DT)[: min(cap, tw)].tobytes() == rw.tobytes()
    dist = top.dist.cpu().numpy().view(np.uint32).reshape(top.n, top.V)
    hops = top.hops.cpu().numpy().view(np.uint16).reshape(top.n, top.V)
    sample = [0, 1, n // 2, n - 1]
    for j in sample:
        got = isis.l1_to_l2_from_cells(v["l1"], t, ch[j], wh[j])
        want = host(v["l1"], v["l2"], t, [(dist[j], hops[j]), None], [ovs[j], []], v["cfg"], None)
        assert got.tobytes() == want.tobytes(), j
    # host figure: the SPT from the job's planes, then the propagation (the job's active summaries, from its words)
    lv, sysid, mt = v["l1"]["level"], v["l1"]["system_id"], v["l1"]["level"].metric_type
    jobs = rng.choice(np.arange(1, n), args.host_sample, replace=False)
    def active(w):
        a = v["cfg"].copy()
        a["metric"] = w & np.uint64(0xFFFFFFFF)
        return a[(w >> np.uint64(32)) == 1].copy()
    acts = {int(j): active(wh[j]) for j in jobs}
    t0 = time.perf_counter()
    for j in jobs:
        spt = f.spt_from_planes(rib.root[0][isis.TOPO_STD], dist[j], hops[j], ovs[j])
        isis.l1_to_l2(lv, sysid, spt, None, mt, v["l2"]["level"].metric_type, v["cfg"], acts[int(j)])
    host_ms = (time.perf_counter() - t0) * 1000.0 / len(jobs)
    out = dict(gpu=gpu, workload="C3 as the L2 backbone + a 2 000-system L1 area, two summaries over part of the area",
               jobs=n, keys=K, records=t.n_records, summaries=S, l1_vertices=rib.n_vertices[0][0], spt_rows=top.n,
               reps=args.reps, median_ms=med, launch_bound=cur, other_bound=other, cells_equal_other_bound=same_bounds,
               delta_records=tw, delta_checked_jobs=n, sampled_jobs_decoded=len(sample),
               host_ms_per_job_spt_from_planes_plus_l1_to_l2=host_ms, host_sample_jobs=len(jobs),
               host_note="host measurement (CPU of the GPU machine), not an H100 figure")
    stage_bench.write_json(out, args.out)
    ctx.close()


if __name__ == "__main__":
    main()
