#!/usr/bin/env python
"""Routing table of an IS-IS L1/L2 router on a what-if batch, device only.

Workload: C3's LSDB as the L2 backbone (10 000 systems, 40 000 directed adjacencies, wide metrics U[1,1000], seed
SEED_BASE+3, as bench.py builds it) and a 2 000-system L1 area from isis.l1l2_view, joined by three L1/L2 routers
(C3's routers 0-2), 16 summaries over the area (10.1.0.0/20 .. 10.1.240.0/20, so the area's /32s fall under them)
and 10 000 jobs of root 0: job j < 5 000 disables one L1 adjacency (L1 row j + 1), the others one L2 adjacency
(L2 row j - 4 999).

The launch bound of the stage's kernels (kL1L2BlocksPerSM in csrc/isis_l1l2_rib.cu) is timed against the other of 4
and 8 in the same run: that build is a copy of the library with the constant changed, built by this script, run on
the same table data and planes.  Records, with CUDA events over warmed alternating launches on the engine's stream: the two
SPT batches, the cell launch (summary pass + cell kernel, every cell stored) and the delta with summaries only and
with records, for both bounds; then, in a separate torch.profiler run, the summary kernel and the cell kernel on
their own; the card's name and power limit.  Outside the timed region, both builds' cells and words are compared,
the delta is checked against the stored cells for all jobs, and three sampled jobs are decoded and compared with the
host chain.  Fails without a GPU.

    python scripts/isis_l1l2_rib_stage.py [--out FILE] [--jobs N] [--reps R]
"""
import argparse
import ctypes as C

import numpy as np

import stage_bench

BOUND = ("isis_l1l2_rib.cu", "kL1L2BlocksPerSM")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--jobs", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--l1", type=int, default=2000)
    args = ap.parse_args()
    torch = stage_bench.require_gpu("isis_l1l2_rib_stage.py")
    from holo_b200 import capi, isis, route_table, synth
    from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
    from test_isis_l1l2_rib_cells import chain, level_routes, same_rib, topology_flat, without
    from test_isis_route_cells_gpu import DeviceTopology
    from test_route_delta import reference

    summ = [(f"10.1.{16 * i}.0/20", None) for i in range(16)]
    c3 = synth.random_topology(10000, 40000, synth.SEED_BASE + 3, cost_lo=1, cost_hi=1000)
    v = isis.l1l2_view(1, n_l1=args.l1, l2_topology=c3, summaries=summ, cost_choices=[1, 5, 10, 20])
    ctx = capi.Context(0)
    t = isis.L1L2RibTable(v["l1"], v["l2"], v["cfg"], v["l2_derived"])
    t.upload(ctx)
    n = args.jobs
    half = n // 2
    rng = np.random.default_rng(7)
    tops, ovs = [], []
    for l, inst, rows in ((0, v["l1"], half + 1), (1, v["l2"], n - half + 1)):
        f = topology_flat(inst, isis.MT_STANDARD)
        ov = [[]] + [[(int(e), capi.COST_DISABLED)] for e in rng.integers(0, f.csr.n_edges, rows - 1)]
        tops.append(DeviceTopology(ctx, f.csr, t.root[l][isis.TOPO_STD], rows, ov))
        ovs.append(ov)
    rows = np.zeros((n, 2), np.uint32)
    rows[:half, 0] = np.arange(1, half + 1)
    rows[half:, 1] = np.arange(1, n - half + 1)
    d_rows = torch.tensor(rows.view(np.int32).reshape(-1), device="cuda")
    P, S = t.n_prefixes, t.n_summaries
    cells = torch.zeros(n * P * 3, dtype=torch.int64, device="cuda")
    words = torch.zeros(n * S, dtype=torch.int64, device="cuda")
    base_cells = torch.zeros(P * 3, dtype=torch.int64, device="cuda")
    base_words = torch.zeros(S, dtype=torch.int64, device="cuda")
    base_rows = torch.zeros(2, dtype=torch.int32, device="cuda")
    job_out = torch.zeros(n * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device="cuda")
    cap = n * 64
    recs = torch.zeros(cap * DELTA_DT.itemsize, dtype=torch.uint8, device="cuda")
    total = torch.zeros(1, dtype=torch.int64, device="cuda")
    n_rows = [tops[0].n, tops[1].n]
    lv = (tops[0].rs, None), (tops[1].rs, None)
    st = torch.cuda.ExternalStream(ctx.lib.hspf_stream(ctx.handle))

    def spt(k):
        tops[k].run()

    # the other launch bound, from a copy of the library, with its own table over the same instances
    cur = stage_bench.launch_bound(*BOUND)
    other = 4 if cur == 8 else 8
    libv = C.CDLL(str(stage_bench.build_variant(*BOUND, other, "l1l2_bound_")))
    route_table.declare(libv)
    s1, s2 = isis.instance_struct(v["l1"]), isis.instance_struct(v["l2"])
    hv = C.c_void_p()
    assert libv.hspf_isis_l1l2_ribtable_create(C.byref(s1), C.byref(s2), v["l2_derived"].ctypes.data, t.cfg.ctypes.data,
                                               len(t.cfg), C.byref(hv)) == 0
    assert libv.hspf_isis_l1l2_ribtable_upload(ctx.handle, hv) == 0
    libs = {cur: (ctx.lib, t.handle), other: (libv, hv)}
    cellsv = torch.zeros(n * P * 3, dtype=torch.int64, device="cuda")
    wordsv = torch.zeros(n * S, dtype=torch.int64, device="cuda")
    nr = (C.c_uint32 * 2)(*n_rows)
    rs = [C.byref(tops[0].rs), None, C.byref(tops[1].rs), None]

    def cell_launch(b=cur):
        lib, h = libs[b]
        c, w = (cells, words) if b == cur else (cellsv, wordsv)
        assert lib.hspf_isis_l1l2_rib_cells(ctx.handle, h, n, *rs, nr, d_rows.data_ptr(), w.data_ptr(), None,
                                            c.data_ptr()) == 0

    def delta(c, b=cur):
        lib, h = libs[b]
        assert lib.hspf_isis_l1l2_rib_delta(ctx.handle, h, n, *rs, nr, d_rows.data_ptr(), words.data_ptr(),
                                            base_cells.data_ptr(), 1, None, job_out.data_ptr(),
                                            recs.data_ptr() if c else None, cap if c else 0, total.data_ptr()) == 0

    for k in (0, 1):
        spt(k)
    ctx.sync()
    isis.l1l2_rib_cells_device(ctx, t, 1, *lv, n_rows, base_rows.data_ptr(), base_words.data_ptr(), 0, base_cells.data_ptr())
    ctx.sync()
    work = {"spt_l1": lambda: spt(0), "spt_l2": lambda: spt(1)}
    for b in (cur, other):
        work[f"cells_bound{b}"] = lambda b=b: cell_launch(b)
        work[f"delta_summaries_bound{b}"] = lambda b=b: delta(False, b)
        work[f"delta_records_bound{b}"] = lambda b=b: delta(True, b)
    for f in work.values():
        f()
    ctx.sync()
    times = {k: [] for k in work}
    for _ in range(args.reps):
        for k, f in work.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(st)
            f()
            b.record(st)
            b.synchronize()
            times[k].append(a.elapsed_time(b))
    med = {k: float(np.median(x)) for k, x in times.items()}
    # the summary kernel and the cell kernel on their own: kernel times from a profiler run of its own
    from torch.profiler import ProfilerActivity, profile
    kern = {}
    for b in (cur, other):
        ctx.sync()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                cell_launch(b)
            ctx.sync()
        for e in prof.key_averages():
            for key, pat in (("summary_kernel", "isis_summary_kernel"), ("cell_kernel", "route_cells_kernel")):
                if pat in e.key:
                    kern[f"{key}_bound{b}"] = e.device_time_total / max(e.count, 1) / 1000.0
    cell_launch(cur)
    cell_launch(other)
    ctx.sync()
    same_bounds = bool(torch.equal(cells, cellsv) and torch.equal(words, wordsv))
    # outside the timed region: the delta against the stored cells, sampled jobs against the host chain
    cell_launch()
    ctx.sync()
    ch = cells.cpu().numpy().view(np.uint8).view(isis.CELL_DT).reshape(n, P)
    wh = words.cpu().numpy().view(np.uint64).reshape(n, S)
    bh = base_cells.cpu().numpy().view(np.uint8).view(isis.CELL_DT).reshape(1, P)
    delta(True)
    ctx.sync()
    jw, rw, tw = reference(ch, bh, None, cap=cap)
    assert job_out.cpu().numpy().view(DELTA_JOB_DT).tobytes() == jw.tobytes() and int(total.item()) == tw
    assert recs.cpu().numpy().view(DELTA_DT)[: min(cap, tw)].tobytes() == rw.tobytes()
    for j in (0, half - 1, n - 1):
        planes = []
        for k in range(2):
            r = int(rows[j, k])
            tp = tops[k]
            planes += [(tp.dist.cpu().numpy().view(np.uint32).reshape(tp.n, tp.V)[r],
                        tp.hops.cpu().numpy().view(np.uint16).reshape(tp.n, tp.V)[r]), None]
        o = [ovs[0][rows[j, 0]], (), ovs[1][rows[j, 1]], ()]
        got = isis.l1l2_rib_from_cells(v["l1"], v["l2"], t, ch[j], wh[j], planes, o)
        want, _ = chain(level_routes(v["l1"], o[0]), level_routes(without(v["l2"], v["l2_derived"]), o[2]), v["cfg"])
        same_rib(got, want)
    gpu = ", ".join(stage_bench.card_and_power())
    out = dict(gpu=gpu, workload="C3 as the L2 backbone + a 2 000-system L1 area, 16 summaries", jobs=n, prefixes=P, summaries=S, l1_vertices=t.n_vertices[0][0], l2_vertices=t.n_vertices[1][0],
               spt_rows=n_rows, reps=args.reps, median_ms=med,
               profiler_kernel_ms=kern, launch_bound=cur, other_bound=other, cells_equal_other_bound=same_bounds, delta_records=tw, sampled_jobs_decoded=3,
               delta_checked_jobs=n)
    stage_bench.write_json(out, args.out)
    ctx.close()


if __name__ == "__main__":
    main()
