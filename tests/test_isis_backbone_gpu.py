"""GPU: the routes a backbone router gets from an IS-IS area's L1/L2 routers for every L1 what-if job
(hspf_isis_backbone_cells[16], _delta[16]).  Each border runs its L1 batch and hspf_isis_l1_to_l2_cells on the
device, and the backbone call reads those cells where they are.  The device cells must equal, byte for byte, the CPU
harness (the same walk compiled for the host) over the same planes and border cells; sampled jobs decode to the
reference chain; the delta equals the reference comparison of the stored cells."""
import numpy as np
import pytest

from holo_b200 import capi, isis
from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT, DELTA_NEXTHOPS
from test_isis_backbone_cells import backbone_cells, harness, level_routes, restrict, same_rib, spliced  # noqa: F401
from test_isis_l1l2_rib_cells import TOPOS, p2p_links, topology_flat
from test_isis_route_cells_gpu import DeviceTopology
from test_route_delta import reference

pytestmark = pytest.mark.gpu

SENTINEL = 0xAB
GUARD = 64


def dev_u32(a):
    import torch
    return torch.tensor(np.asarray(a, np.uint32).view(np.int32).reshape(-1), device="cuda")


def host_planes(t, row, narrow):
    d = t.dist.cpu().numpy().view(np.uint16 if narrow else np.uint32).reshape(t.n, t.V)[row]
    h = t.hops.cpu().numpy().view(np.uint16).reshape(t.n, t.V)[row]
    m = t.nh.cpu().numpy().view(np.uint16 if narrow else np.uint64).reshape(t.n, t.V)[row]
    if narrow:                 # the harnesses read wide planes: widen, unreached stays unreached
        d = d.astype(np.uint32)
        d[d == 0xFFFF] = 0xFFFFFFFF
        m = m.astype(np.uint64)
    return np.ascontiguousarray(d), np.ascontiguousarray(h), np.ascontiguousarray(m)


class DeviceBorder:
    """One border's tables, its L1 batch (row j: job j) and its L1 -> L2 cells on the device."""

    def __init__(self, ctx, v, narrow, ovs, up_down=None):
        import torch
        self.v, self.narrow = v, narrow
        self.lid = v["l1"]["system_id"] << 8
        self.rib = isis.L1L2RibTable(v["l1"], v["l2"], v["cfg"], v["l2_derived"])
        self.rib.upload(ctx)
        self.t = isis.L1ToL2Table(v["l1"], v["l2"], self.rib, up_down)
        self.t.upload(ctx)
        n = len(ovs)
        self.top = []
        for tt, mt in TOPOS:
            if self.rib.root[0][tt] == isis.NO_ROOT:
                self.top.append(None)
                continue
            d = DeviceTopology(ctx, topology_flat(v["l1"], mt).csr, self.rib.root[0][tt], n, [o[tt] for o in ovs], narrow)
            d.run()
            self.top.append(d)
        self.cells = torch.zeros(n * self.t.n_keys * 3, dtype=torch.int64, device="cuda")
        self.words = torch.zeros(max(n * self.t.n_summaries, 1), dtype=torch.int64, device="cuda")
        self.status = torch.zeros(n, dtype=torch.int32, device="cuda")
        rows = dev_u32(np.arange(n))
        isis.l1_to_l2_cells_device(ctx, self.t, n, tuple(x.rs if x is not None else None for x in self.top), n,
                                   rows.data_ptr(), self.words.data_ptr(), self.status.data_ptr(), self.cells.data_ptr())
        ctx.sync()
        self.host_cells = self.cells.cpu().numpy().view(isis.CELL_DT).reshape(n, self.t.n_keys).copy()
        w = self.words.cpu().numpy().view(np.uint64)[: n * self.t.n_summaries].reshape(n, self.t.n_summaries)
        self.entries = [isis.l1_to_l2_from_cells(v["l1"], self.t, self.host_cells[j], w[j]) for j in range(n)]


class Domain:
    """A synthetic domain, its three borders on the device and backbone router i's L2 batch (one row)."""

    def __init__(self, ctx, seed, i, n_jobs=24, narrow=False, **kw):
        import torch
        self.ctx, self.narrow = ctx, narrow
        vs = [isis.l1l2_view(seed, root=b, **kw) for b in range(3)]
        self.v = vs[0]
        l1 = self.v["l1"]
        links = p2p_links(self.v["t1"], 0, self.v["t1"].n_routers, isis.sysid)
        rng = np.random.default_rng(seed)
        pick = rng.choice(len(links), n_jobs - 1, replace=len(links) < n_jobs - 1)
        self.ovs = [[[], []]]
        for k in pick:
            ov = []
            for tt, mt in TOPOS:
                if tt == isis.TOPO_MT6 and not l1["mt_ipv6"]:
                    ov.append([])
                    continue
                f = topology_flat(l1, mt)
                a, b = (f.vertex(x << 8) for x in links[k])
                row, col = f.csr.row_ptr, f.csr.col
                ov.append([(e, capi.COST_DISABLED) for x, y in ((a, b), (b, a)) for e in range(int(row[x]), int(row[x + 1]))
                           if int(col[e]) == y])
            self.ovs.append(ov)
        # border 0 with up/down bits on a fifth of the L1 entries: fewer keys than the others
        ud = (rng.random(len(l1["level"].ipreaches)) < 0.2).astype(np.uint8)
        self.borders = [DeviceBorder(ctx, v, narrow, self.ovs, ud if k == 0 else None) for k, v in enumerate(vs)]
        self.r = isis.l1l2_backbone(self.v, i)
        self.derived = self.v["derived_all"].copy()
        # border 0's entries it no longer propagates stay in its LSP as configured ones
        lv, b0 = self.r["level"], self.borders[0]
        keys = {(int(k), bytes(p["bytes"]), int(n)) for k, p, n in zip(b0.t.kind, b0.t.prefix, b0.t.len)}
        for x in np.nonzero(lv.lsps["lan_id"] == b0.lid)[0]:
            a = int(lv.lsps["ipreach_off"][x])
            for k in range(a, a + int(lv.lsps["n_ipreach"][x])):
                e = lv.ipreaches[k]
                if (int(e["kind"]), bytes(e["prefix"]["bytes"]), int(e["len"])) not in keys:
                    self.derived[k] = 0
        self.bt = isis.BackboneTable(self.r, [b.t for b in self.borders], self.derived)
        self.bt.upload(ctx)
        self.rtop = []
        for tt, mt in TOPOS:
            if tt == isis.TOPO_MT6 and not self.r["mt_ipv6"]:
                self.rtop.append(None)
                continue
            f = topology_flat(self.r, mt)
            d = DeviceTopology(ctx, f.csr, f.vertex(self.r["system_id"] << 8), 1, [[]], narrow)
            d.run()
            self.rtop.append(d)
        ctx.sync()
        self.n = n_jobs
        torch.cuda.synchronize()

    def rs(self):
        return tuple(t.rs if t is not None else None for t in self.rtop)

    def planes(self):
        return [host_planes(t, 0, self.narrow) if t is not None else None for t in self.rtop]

    def launch(self, status=True, offset=8):
        import torch
        n, P = self.n, self.bt.n_prefixes
        nbytes = n * P * isis.CELL_DT.itemsize
        buf = torch.full((offset + nbytes + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
        st = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        isis.backbone_cells_device(self.ctx, self.bt, n, self.rs(), [b.cells.data_ptr() for b in self.borders],
                                   [b.status.data_ptr() for b in self.borders] if status else None, st.data_ptr(),
                                   buf.data_ptr() + offset)
        self.ctx.sync()
        host = buf.cpu().numpy()
        assert (host[:offset] == SENTINEL).all() and (host[offset + nbytes:] == SENTINEL).all()
        return host[offset: offset + nbytes].copy().view(isis.CELL_DT).reshape(n, P), st.cpu().numpy().view(np.uint32)[:n]

    def harness(self, harness):
        class B:
            pass
        bs = []
        for b in self.borders:
            x = B()
            x.cells = np.ascontiguousarray(b.host_cells)
            bs.append(x)
        return backbone_cells(harness[1], self.bt, bs, self.planes(), self.n)


KW = dict(n_l1=50, n_l2=30, l1_degree=2, cost_choices=[10], summaries=[("10.2.0.0/16", None), ("10.1.0.5/32", None)])


@pytest.mark.parametrize("narrow", [False, True])
@pytest.mark.parametrize("mt6", [False, True])
def test_device_cells_equal_harness(ctx, harness, narrow, mt6):
    d = Domain(ctx, 61, 15, narrow=narrow, mt6=mt6, **KW)        # 11 / 16 first-hop atoms: fits 16-bit planes
    assert len({b.t.n_keys for b in d.borders}) > 1            # borders with different K
    cells, st = d.launch()
    want = d.harness(harness)
    assert not st.any()
    assert cells.tobytes() == want.tobytes()
    assert (cells["flags"] & isis.CELL_PRESENT).any() and (cells["winner"] >= 0).all()


@pytest.mark.parametrize("narrow", [False, True])
def test_sampled_jobs_decode_to_the_chain(ctx, harness, narrow):
    d = Domain(ctx, 62, 9, narrow=narrow, **KW)
    cells, st = d.launch()
    planes = [p[:2] if p is not None else None for p in d.planes()]
    affected = {(int(p["is_v6"]), bytes(p["bytes"]), int(n)) for p, n in zip(d.bt.prefix, d.bt.len)}

    class B:
        pass
    bs = []
    for b in d.borders:
        x = B()
        x.lid, x.entries = b.lid, b.entries
        bs.append(x)
    for j in (0, 1, d.n // 2, d.n - 1):
        got = isis.backbone_from_cells(d.r, d.bt, cells[j], planes, [b.entries[j] for b in d.borders])
        want = level_routes(spliced(d.r, d.derived, bs, j))
        same_rib(got, restrict(want, lambda k: k in affected))


def test_refused_jobs(ctx, harness):
    import torch
    d = Domain(ctx, 63, 7, n_jobs=8, **KW)
    want = d.harness(harness)
    d.borders[1].status[3] = 5                 # a border's job refused
    torch.cuda.synchronize()
    cells, st = d.launch()
    assert st[3] == 5 and not np.delete(st, 3).any()
    assert np.delete(cells, 3, axis=0).tobytes() == np.delete(want, 3, axis=0).tobytes()
    assert not cells[3]["flags"].any() and (cells[3]["winner"] == 0xFFFFFFFF).all()
    cells, st = d.launch(status=False)         # no border status words: not refused
    assert cells.tobytes() == want.tobytes()
    d.rtop[0].status[0] = capi.JS_INVALID      # R's row refused: every job
    torch.cuda.synchronize()
    cells, st = d.launch()
    assert (st == (capi.JS_INVALID | np.where(np.arange(d.n) == 3, 5, 0))).all()
    assert not cells["flags"].any()
    d.rtop[0].status[0] = 0
    d.borders[1].status[3] = 0


@pytest.mark.parametrize("narrow", [False, True])
def test_delta_equals_comparison_of_stored_cells(ctx, harness, narrow):
    import torch
    d = Domain(ctx, 64, 11, n_jobs=40, narrow=narrow, **KW)
    d.borders[0].status[5] = 1                 # refused: status set, nothing compared
    torch.cuda.synchronize()
    cells, st = d.launch()
    n, P = d.n, d.bt.n_prefixes
    base = cells[:1].copy()
    base_of = np.zeros(n, np.uint32)
    base_of[-1] = 1                            # out of range: HSPF_JS_INVALID, not compared
    d_base = torch.from_numpy(base.view(np.uint8).reshape(-1).copy()).cuda()
    d_of = dev_u32(base_of)
    for cap in (0, 7, n * P):
        job_out = torch.zeros(n * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device="cuda")
        recs = torch.zeros(max(cap, 1) * DELTA_DT.itemsize, dtype=torch.uint8, device="cuda")
        total = torch.zeros(1, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        isis.backbone_delta_device(ctx, d.bt, n, d.rs(), [b.cells.data_ptr() for b in d.borders],
                                   [b.status.data_ptr() for b in d.borders], d_base.data_ptr(), 1, d_of.data_ptr(),
                                   job_out.data_ptr(), recs.data_ptr() if cap else 0, cap, total.data_ptr())
        ctx.sync()
        jw, rw, tw = reference(cells, base, base_of, cap=cap, status=st)
        got_job = job_out.cpu().numpy().view(DELTA_JOB_DT)
        assert got_job.tobytes() == jw.tobytes()
        assert got_job[5]["status"] == 1 and got_job[5]["n_changed"] == 0
        assert got_job[-1]["status"] == capi.JS_INVALID
        assert int(total.item()) == tw and tw > 0
        if cap:
            got = recs.cpu().numpy().view(DELTA_DT)[: min(cap, tw)]
            assert got.tobytes() == rw.tobytes()
            if cap == n * P:
                assert (got["kind"] & DELTA_NEXTHOPS).any()
    d.borders[0].status[5] = 0
