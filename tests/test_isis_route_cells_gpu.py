"""GPU: the batched IS-IS route stage on the device (hspf_isis_routes_batch / _batch16 behind the SPT batches).

SPT planes are written by hspf_run_batch[16]_async into device buffers and never leave the device before the
route kernel reads them; the cells must equal the CPU harness's cells over the same planes, and decode to the
engine's compute_routes (goldens) or to the oracle's table on an LSDB carrying each job's change (what-if)."""
import ctypes as C

import numpy as np
import pytest

import golden_util as gu
from holo_b200 import capi, isis, synth
from isis_synth import synth_instance
from oracle import pyoracle
from test_isis_route_cells import (harness, cells_on_cpu, decode, mt6_instance, same_rib, set_reach_metric,  # noqa: F401
                                   single_p2p, topology_flat)

pytestmark = pytest.mark.gpu

u16p, u32p, u64p = C.POINTER(C.c_uint16), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)


class DeviceTopology:
    """One topology's graph and a batch of jobs of the local root on the device (device roots, overrides,
    planes); `run()` enqueues the SPT batch."""

    def __init__(self, ctx, csr, root, n_jobs, overrides=None, narrow=False):
        import torch
        self.ctx, self.n, self.V, self.narrow = ctx, n_jobs, csr.n_vertices, narrow
        self.g = ctx.upload(csr)
        dev = "cuda"
        self.keep = [torch.full((n_jobs,), root, dtype=torch.int32, device=dev)]
        js = capi.JobsStruct()
        js.n_jobs = n_jobs
        js.roots = C.cast(self.keep[0].data_ptr(), u32p)
        if overrides is not None:
            off = np.zeros(n_jobs + 1, np.int64)
            ed, co = [], []
            for j, ov in enumerate(overrides):
                for e, c in ov:
                    ed.append(e)
                    co.append(c)
                off[j + 1] = len(ed)
            t_off = torch.from_numpy(off).to(torch.int32).to(dev)
            t_ed = torch.from_numpy(np.asarray(ed or [0], np.uint32).view(np.int32).copy()).to(dev)
            t_co = torch.from_numpy(np.asarray(co or [0], np.uint32).view(np.int32).copy()).to(dev)
            js.ov_off, js.ov_edge, js.ov_cost = (C.cast(x.data_ptr(), u32p) for x in (t_off, t_ed, t_co))
            self.keep += [t_off, t_ed, t_co]
        self.js = js
        NV = n_jobs * self.V
        self.dist = torch.zeros(NV, dtype=torch.int16 if narrow else torch.int32, device=dev)
        self.hops = torch.zeros(NV, dtype=torch.int16, device=dev)
        self.nh = torch.zeros(NV, dtype=torch.int16 if narrow else torch.int64, device=dev)
        self.status = torch.zeros(n_jobs, dtype=torch.int32, device=dev)
        if narrow:
            rs = capi.Result16Struct()
            rs.dist, rs.nh_mask = C.cast(self.dist.data_ptr(), u16p), C.cast(self.nh.data_ptr(), u16p)
        else:
            rs = capi.ResultStruct()
            rs.dist, rs.nh_mask = C.cast(self.dist.data_ptr(), u32p), C.cast(self.nh.data_ptr(), u64p)
            rs.nh_words = 1
        rs.hops = C.cast(self.hops.data_ptr(), u16p)
        rs.job_status = C.cast(self.status.data_ptr(), u32p)
        self.rs = rs

    def run(self):
        import torch
        torch.cuda.synchronize()                  # the buffers were filled on torch's stream
        (self.ctx.run_device16 if self.narrow else self.ctx.run_device)(self.g, self.js, self.rs, sync=False)

    def planes(self, j):
        """Job j's (dist u32, hops u16, nh u64) on the host, narrow planes widened."""
        sl = slice(j * self.V, (j + 1) * self.V)
        d = self.dist[sl].cpu().numpy()
        h = self.hops[sl].cpu().numpy().view(np.uint16).copy()
        m = self.nh[sl].cpu().numpy()
        if self.narrow:
            d = d.view(np.uint16).astype(np.uint32)
            d[d == 0xFFFF] = 0xFFFFFFFF
            m = m.view(np.uint16).astype(np.uint64)
        else:
            d, m = d.view(np.uint32).copy(), m.view(np.uint64).copy()
        return d, h, m


def device_cells(ctx, inst, rt, n_jobs, ov_std=None, narrow=False, offset=0, poke_status=None):
    """SPT batches of both topologies and the route kernel behind them, all on the device; cells written at
    `offset` bytes into the output buffer.  poke_status: {topology: [jobs]} whose status words are set between
    the batches and the route kernel."""
    import torch
    tops = {}
    for t, mt in ((isis.TOPO_STD, isis.MT_STANDARD), (isis.TOPO_MT6, isis.MT_IPV6)):
        if rt.root[t] != isis.NO_ROOT:
            f = topology_flat(inst, mt)
            tops[t] = DeviceTopology(ctx, f.csr, rt.root[t], n_jobs, ov_std if t == isis.TOPO_STD else None, narrow)
            tops[t].run()
    if poke_status:
        ctx.sync()
        for t, jobs in poke_status.items():
            for j in jobs:
                tops[t].status[j] = 2
    P = rt.n_prefixes
    buf = torch.full((offset + n_jobs * P * isis.CELL_DT.itemsize,), 0xAB, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    isis.routes_batch_device(ctx, rt, n_jobs, tops[isis.TOPO_STD].rs if isis.TOPO_STD in tops else None,
                             tops[isis.TOPO_MT6].rs if isis.TOPO_MT6 in tops else None, buf.data_ptr() + offset)
    ctx.sync()
    cells = np.frombuffer(buf.cpu().numpy()[offset:].tobytes(), isis.CELL_DT).reshape(n_jobs, P)
    return cells, tops


def harness_cells(harness, rt, tops, j):
    return cells_on_cpu(harness, rt, {t: d.planes(j) for t, d in tops.items()})


def job_planes(tops, j):
    return {t: d.planes(j) for t, d in tops.items()}


SNAPS = gu.load_isis()
LEVELS = [(s, i) for s in SNAPS for i in range(len(s["levels"]))]


def test_goldens_through_the_device_path(ctx, harness):
    """Every level of every IS-IS golden snapshot: flatten, upload, a one-job batch at the local root, the route
    kernel, and a decode equal to compute_routes."""
    n = 0
    for snap, li in LEVELS:
        inst = gu.isis_instance_image(snap, snap["levels"][li])
        rt = isis.RouteTable(inst)
        if rt.n_prefixes == 0 or rt.root[isis.TOPO_STD] == isis.NO_ROOT:
            continue
        rt.upload(ctx)
        cells, tops = device_cells(ctx, inst, rt, 1)
        assert cells[0].tobytes() == harness_cells(harness, rt, tops, 0).tobytes()
        got = decode(inst, rt, cells[0], job_planes(tops, 0))
        same_rib(got, isis.compute_routes(ctx, inst))
        n += 1
    assert n >= 30


@pytest.fixture(scope="module")
def c3_small():
    t = synth.random_topology(2000, 8000, synth.SEED_BASE + 3, cost_lo=1, cost_hi=1000)
    inst = synth_instance(t, 0)
    f = topology_flat(inst, isis.MT_STANDARD)
    adj = []
    for k, a, b in single_p2p(t):
        va, vb = f.vertex(isis.sysid(a) << 8), f.vertex(isis.sysid(b) << 8)
        row, col = f.csr.row_ptr, f.csr.col
        ab = [e for e in range(row[va], row[va + 1]) if col[e] == vb]
        ba = [e for e in range(row[vb], row[vb + 1]) if col[e] == va]
        adj.append((a, b, ab[0], ba[0]))
    return t, inst, adj


def test_c3_shape_whatif_batch(ctx, harness, c3_small):
    """2 000 systems, 64 jobs each removing one adjacency (every 7th, the root's own included), wide planes:
    every job's device cells equal the harness's over that job's device planes; a sample of jobs decodes to the
    oracle's table on the LSDB without that adjacency."""
    t, inst, adj = c3_small
    pick = [adj[(7 * j) % len(adj)] for j in range(63)] + [next(x for x in adj if 0 in x[:2])]
    ov = [[(ab, capi.COST_DISABLED), (ba, capi.COST_DISABLED)] for (_a, _b, ab, ba) in pick]
    rt = isis.RouteTable(inst)
    rt.upload(ctx)
    cells, tops = device_cells(ctx, inst, rt, len(pick), ov)
    assert not tops[isis.TOPO_STD].status.any().item()
    for j in range(len(pick)):
        assert cells[j].tobytes() == harness_cells(harness, rt, tops, j).tobytes(), j
    assert (cells["flags"] & isis.CELL_PRESENT != 0).sum() > 60 * (rt.n_prefixes - 10)
    for j in (0, 5, 31, 63):
        a, b = pick[j][:2]
        got = decode(inst, rt, cells[j], job_planes(tops, j), {isis.TOPO_STD: ov[j]})
        want = pyoracle.isis_compute_routes(set_reach_metric(set_reach_metric(inst, a, b, None), b, a, None))
        same_rib(got, want)


def test_narrow_planes_give_the_wide_cells(ctx, harness):
    t = synth.random_topology(300, 1200, synth.SEED_BASE + 41, cost_lo=1, cost_hi=20, lan_fraction=0.1)
    n_ok = 0
    for root in (0, 11, 150):
        inst = synth_instance(t, root, sr=True)
        rt = isis.RouteTable(inst)
        rt.upload(ctx)
        f = topology_flat(inst, isis.MT_STANDARD)
        adj = [x for x in single_p2p(t) if root not in x[1:]][:6]
        row, col = f.csr.row_ptr, f.csr.col
        ov = [[]]
        for _k, a, b in adj:
            va, vb = f.vertex(isis.sysid(a) << 8), f.vertex(isis.sysid(b) << 8)
            ov.append([(e, capi.COST_DISABLED) for e in range(row[va], row[va + 1]) if col[e] == vb])
        wide, _ = device_cells(ctx, inst, rt, len(ov), ov)
        narrow, tops = device_cells(ctx, inst, rt, len(ov), ov, narrow=True)
        ok = tops[isis.TOPO_STD].status.cpu().numpy() == 0          # more than 16 atoms: no narrow planes
        assert not narrow[~ok]["flags"].any()
        assert narrow[ok].tobytes() == wide[ok].tobytes()
        for j in np.nonzero(ok)[0]:
            assert narrow[j].tobytes() == harness_cells(harness, rt, tops, int(j)).tobytes()
        n_ok += int(ok.sum())
    assert n_ok >= 10


def test_overload_bits_use_the_general_kernel(ctx, harness):
    t = synth.random_topology(300, 1200, synth.SEED_BASE + 43, cost_choices=[5, 10], lan_fraction=0.1)
    inst = synth_instance(t, 4, isis.METRIC_BOTH, 2, sr=True)
    lsps = inst["level"].lsps
    over = (lsps["fragment"] == 0) & np.isin(lsps["lan_id"], [isis.sysid(r) << 8 for r in range(20, 300, 9)])
    lsps["flags"][over] |= isis.LSPF_OL
    rt = isis.RouteTable(inst)
    rt.upload(ctx)
    f = topology_flat(inst, isis.MT_STANDARD)
    assert not ctx.graph_info(ctx.upload(f.csr))["fast_path"]           # leaf flags: spf_batch_kernel
    cells, tops = device_cells(ctx, inst, rt, 2, [[], [(int(f.csr.row_ptr[f.vertex(isis.sysid(4) << 8)]), 50)]])
    for j in range(2):
        assert cells[j].tobytes() == harness_cells(harness, rt, tops, j).tobytes()
    same_rib(decode(inst, rt, cells[0], job_planes(tops, 0)), isis.compute_routes(ctx, inst))


def test_refused_jobs_get_empty_cells(ctx, harness):
    """A non-zero status word in either topology empties that job's cells; the others are untouched."""
    t = synth.random_topology(150, 600, synth.SEED_BASE + 45, cost_lo=1, cost_hi=20)
    inst = mt6_instance(t, 0)
    rt = isis.RouteTable(inst)
    rt.upload(ctx)
    cells, tops = device_cells(ctx, inst, rt, 3, poke_status={isis.TOPO_STD: [1], isis.TOPO_MT6: [2]})
    empty = np.zeros(1, isis.CELL_DT)
    empty["winner"] = 0xFFFFFFFF
    assert (cells[1] == empty[0]).all() and (cells[2] == empty[0]).all()
    assert cells[0].tobytes() == harness_cells(harness, rt, tops, 0).tobytes()
    same_rib(decode(inst, rt, cells[0], job_planes(tops, 0)), isis.compute_routes(ctx, inst))


def test_partial_warp_tiles_and_a_misaligned_cell_buffer(ctx, harness):
    t = synth.random_topology(150, 600, synth.SEED_BASE + 47, cost_choices=[5, 10], lan_fraction=0.1)
    inst = synth_instance(t, 2, sr=True)
    rt = isis.RouteTable(inst)
    rt.upload(ctx)
    n = next(k for k in range(3, 40) if (k * rt.n_prefixes) % 32)
    aligned, tops = device_cells(ctx, inst, rt, n)
    for off in (8, 24):
        cells, _ = device_cells(ctx, inst, rt, n, offset=off)
        assert cells.tobytes() == aligned.tobytes()
    for j in range(n):
        assert aligned[j].tobytes() == harness_cells(harness, rt, tops, j).tobytes()
