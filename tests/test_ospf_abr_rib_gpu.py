"""GPU: the batched routing-table stage for area border routers (hspf_ospfv2_abr_rib_cells[16], _delta[16]).  Each
area's SPT planes are written on the device by one SPT batch per area; a job picks one row per area.  The device cells
must equal, byte for byte, the CPU harness (the same walk compiled for the host) over those planes; sampled jobs decode
to what the host stages give; the delta equals the numpy reference over the stored cells."""
import ctypes as C

import numpy as np
import pytest

from holo_b200 import capi, ospf_rib
from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
from test_isis_route_cells_gpu import DeviceTopology
from test_ospf_abr_rib_cells import domain, harness, harness_cells, router_edges, same_rib  # noqa: F401
from test_ospf_rib_delta import reference
from test_ospfv2_route_cells import gather_for

pytestmark = pytest.mark.gpu

SENTINEL = 0xAB
GUARD = 64


def dev_u32(a):
    import torch
    return torch.tensor(np.asarray(a, np.uint32).view(np.int32).reshape(-1), device="cuda")


class AbrBatch:
    """A domain's table on the device and, per area, a batch of rows computed on the device: row 0 unperturbed, the
    others disabling one router-to-router link each.  `rows` [n_jobs, n_areas] pick one row per area."""

    def __init__(self, ctx, seed, n_rows=6, narrow=False, **kw):
        self.ctx, self.narrow = ctx, narrow
        self.dom = domain(seed, **kw)
        self.rt = self.dom.rt
        self.rt.upload(ctx)
        rng = np.random.default_rng(seed)
        self.ov = [[[]] + [router_edges(self.dom, i, rng) for _ in range(n_rows - 1)] for i in range(self.rt.n_areas)]
        self.top = [DeviceTopology(ctx, f.csr, rv, n_rows, self.ov[i], narrow)
                    for i, (f, rv) in enumerate(zip(self.dom.flats, self.dom.rv))]
        for t in self.top:
            t.run()
        ctx.sync()
        self.n_rows = [n_rows] * self.rt.n_areas
        A = self.rt.n_areas
        jobs = [[0] * A]
        for i in range(A):
            jobs += [[r if k == i else 0 for k in range(A)] for r in range(1, n_rows)]
        jobs += [[int(rng.integers(0, n_rows)) for _ in range(A)] for _ in range(5)]
        self.rows = np.asarray(jobs, np.uint32)

    def host_planes(self, i):
        t = self.top[i]
        d = t.dist.cpu().numpy().view(np.uint16 if self.narrow else np.uint32).reshape(t.n, t.V)
        h = t.hops.cpu().numpy().view(np.uint16).reshape(t.n, t.V)
        m = t.nh.cpu().numpy().view(np.uint16 if self.narrow else np.uint64).reshape(t.n, t.V)
        return d, h, m

    def launch(self, rows=None, offset=0, gather=()):
        import torch
        rows = self.rows if rows is None else np.asarray(rows, np.uint32)
        n, P = rows.shape[0], self.rt.n_prefixes
        nbytes = n * P * ospf_rib.RIB_CELL_DT.itemsize
        buf = torch.full((offset + nbytes + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
        st = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
        d_rows = dev_u32(rows)
        g = np.asarray(gather or [(0, 0, 0)], np.uint32)
        gj, ga, gv = dev_u32(g[:, 0]), dev_u32(g[:, 1]), dev_u32(g[:, 2])
        gnh = torch.zeros(len(g), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        ospf_rib.abr_rib_cells_device(self.ctx, self.rt, n, [t.rs for t in self.top], self.n_rows, d_rows.data_ptr(),
                                      buf.data_ptr() + offset, st.data_ptr(), len(gather), gj.data_ptr(), ga.data_ptr(),
                                      gv.data_ptr(), gnh.data_ptr())
        self.ctx.sync()
        host = buf.cpu().numpy()
        assert (host[:offset] == SENTINEL).all() and (host[offset + nbytes:] == SENTINEL).all()
        cells = host[offset: offset + nbytes].copy().view(ospf_rib.RIB_CELL_DT).reshape(n, P)
        return cells, st.cpu().numpy().view(np.uint32)[:n], gnh.cpu().numpy().view(np.uint64)[: len(gather)]

    def harness(self, harness, rows=None, status=None):
        rows = self.rows if rows is None else rows
        area_rows = [self.host_planes(i) for i in range(self.rt.n_areas)]
        return harness_cells(harness, self.rt, area_rows, rows, status=status, narrow_planes=self.narrow)


@pytest.mark.parametrize("narrow", [False, True])
@pytest.mark.parametrize("offset", [0, 8, 24])
def test_device_cells_equal_harness(ctx, harness, narrow, offset):
    b = AbrBatch(ctx, 1, narrow=narrow, V=30, E=90)
    cells, st, _ = b.launch(offset=offset)
    want, wst = b.harness(harness)
    assert (st == wst).all() and not st.any()
    assert cells.tobytes() == want.tobytes()
    again, _, _ = b.launch(offset=offset)
    assert again.tobytes() == cells.tobytes()                                      # repeat launches
    # a batch whose cells end in a partial warp tile, with the guard after it untouched
    m = next(m for m in range(len(b.rows), 0, -1) if (m * b.rt.n_prefixes) % 32)
    part, _, _ = b.launch(rows=b.rows[:m], offset=offset)
    assert part.tobytes() == want[:m].tobytes()


def test_sampled_jobs_decode_to_the_host_pipeline(ctx, harness):
    b = AbrBatch(ctx, 2)
    A = b.rt.n_areas
    nets = [sorted({int(v) for v in f.csr.col[f.csr.row_ptr[r]: f.csr.row_ptr[r + 1]] if not f.is_router[v]})
            for f, r in zip(b.dom.flats, b.dom.rv)]
    sample = [0, 1, len(b.rows) // 2, len(b.rows) - 1]
    gather = [(j, i, v) for j in sample for i in range(A) for v in nets[i]]
    cells, st, gnh = b.launch(gather=gather)
    planes = [b.host_planes(i) for i in range(A)]
    for j in sample:
        p = [(planes[i][0][b.rows[j, i]], planes[i][1][b.rows[j, i]], planes[i][2][b.rows[j, i]]) for i in range(A)]
        for i in range(A):
            v, n = gather_for(b.dom.flats[i], b.dom.rv[i], p[i])
            got = [int(x) for (jj, ii, _vv), x in zip(gather, gnh) if jj == j and ii == i]
            assert got == [int(x) for x in n]
        same_rib(b.dom.decode(cells[j], p), b.dom.host(p))


def test_refused_jobs_and_rows_out_of_range(ctx, harness):
    b = AbrBatch(ctx, 3, V=30, E=90)
    rows = b.rows.copy()
    rows[1, 0] = b.n_rows[0]                                     # out of range
    b.top[1].status[2] = 1                                        # row 2 of area 1 saturated
    rows[3, 1] = 2
    cells, st, _ = b.launch(rows=rows)
    want, wst = b.harness(harness, rows=rows, status=[t.status.cpu().numpy().view(np.uint32) for t in b.top])
    b.top[1].status[2] = 0
    assert st[1] & capi.JS_INVALID and st[3] & 1
    assert (st == wst).all() and cells.tobytes() == want.tobytes()
    for j in (1, 3):
        assert (cells["winner"][j] == ospf_rib.NO_RECORD).all() and not cells["mpf"][j].any()


def test_argument_errors(ctx):
    import torch
    b = AbrBatch(ctx, 1, n_rows=2, V=30, E=90)
    n, P = len(b.rows), b.rt.n_prefixes
    buf = torch.zeros(n * P * 24, dtype=torch.uint8, device="cuda")
    d_rows = dev_u32(b.rows)
    rs = [t.rs for t in b.top]
    bad = type(rs[0])()
    C.pointer(bad)[0] = rs[0]
    bad.dist = None
    for planes in ([bad] + rs[1:],):
        with pytest.raises(capi.HspfError) as e:
            ospf_rib.abr_rib_cells_device(ctx, b.rt, n, planes, b.n_rows, d_rows.data_ptr(), buf.data_ptr())
        assert e.value.code == capi.HSPF_E_INVAL
    with pytest.raises(capi.HspfError) as e:                      # no rows
        ospf_rib.abr_rib_cells_device(ctx, b.rt, n, rs, b.n_rows, 0, buf.data_ptr())
    assert e.value.code == capi.HSPF_E_INVAL
    fresh = ospf_rib.AbrRibTable(b.rt.router_id, b.dom.flats, b.rt.area_ids, b.dom.summaries, None, b.dom.externals)
    with pytest.raises(capi.HspfError) as e:                      # table not uploaded
        ospf_rib.abr_rib_cells_device(ctx, fresh, n, rs, b.n_rows, d_rows.data_ptr(), buf.data_ptr())
    assert e.value.code == capi.HSPF_E_INVAL
    if torch.cuda.device_count() > 1:                             # a table on another device
        other = capi.Context(device=1)
        fresh.upload(other)
        with pytest.raises(capi.HspfError) as e:
            ospf_rib.abr_rib_cells_device(ctx, fresh, n, rs, b.n_rows, d_rows.data_ptr(), buf.data_ptr())
        assert e.value.code == capi.HSPF_E_INVAL


@pytest.mark.parametrize("narrow", [False, True])
def test_delta_equals_reference(ctx, narrow):
    import torch
    b = AbrBatch(ctx, 4, narrow=narrow, V=30, E=90)
    cells, st, _ = b.launch()
    n, P = cells.shape
    base = cells[:1]
    d_base = torch.from_numpy(base.view(np.uint8).reshape(-1).copy()).cuda()
    d_rows = dev_u32(b.rows)
    for base_of, cap in ((None, None), (np.zeros(n, np.uint32), 5), (None, 0)):
        job_out = torch.zeros(n * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device="cuda")
        cap_ = 4096 if cap is None else cap
        recs = torch.full((cap_ * DELTA_DT.itemsize + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
        total = torch.zeros(1, dtype=torch.int64, device="cuda")
        d_bo = dev_u32(base_of) if base_of is not None else None
        ospf_rib.abr_rib_delta_device(ctx, b.rt, n, [t.rs for t in b.top], b.n_rows, d_rows.data_ptr(), d_base.data_ptr(),
                                      1, d_bo.data_ptr() if d_bo is not None else 0, job_out.data_ptr(),
                                      recs.data_ptr() if cap_ else 0, cap_, total.data_ptr())
        ctx.sync()
        wj, wr, wt = reference(cells, base, base_of, st, cap_)
        assert job_out.cpu().numpy().view(DELTA_JOB_DT).tobytes() == wj.tobytes()
        assert int(total.cpu()[0]) == wt and wt > 0
        h = recs.cpu().numpy()
        assert h[: len(wr) * DELTA_DT.itemsize].view(DELTA_DT).tobytes() == wr.tobytes()
        assert (h[cap_ * DELTA_DT.itemsize:] == SENTINEL).all()


def test_delta_records_tie_to_decoded_tables(ctx):
    """A route-level tie: a job with no records decodes to the base table; a job with records differs from it at
    exactly those prefixes' routes (hspf_ospfv2_rib_diff against the base lists installs there only)."""
    import torch
    b = AbrBatch(ctx, 5)
    A = b.rt.n_areas
    cells, st, _ = b.launch()
    n = len(b.rows)
    d_base = torch.from_numpy(cells[:1].view(np.uint8).reshape(-1).copy()).cuda()
    job_out = torch.zeros(n * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device="cuda")
    recs = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    total = torch.zeros(1, dtype=torch.int64, device="cuda")
    ospf_rib.abr_rib_delta_device(ctx, b.rt, n, [t.rs for t in b.top], b.n_rows, dev_u32(b.rows).data_ptr(),
                                  d_base.data_ptr(), 1, 0, job_out.data_ptr(), recs.data_ptr(), 4096, total.data_ptr())
    ctx.sync()
    records = recs.cpu().numpy()[: int(total.cpu()[0]) * DELTA_DT.itemsize].view(DELTA_DT)
    planes = [b.host_planes(i) for i in range(A)]

    def table(j):
        p = [(planes[i][0][b.rows[j, i]], planes[i][1][b.rows[j, i]], planes[i][2][b.rows[j, i]]) for i in range(A)]
        return b.dom.decode(cells[j], p)

    base_rib = table(0)
    _acts, installed = ospf_rib.rib_diff(None, base_rib)
    base_marked = ospf_rib.Rib(installed, base_rib.nexthops)
    key = lambda r: (int(r["prefix"]), int(r["mask"]))
    pkey = lambda p: (int(b.rt.prefix[p]), (0xFFFFFFFF << (32 - int(b.rt.plen[p]))) & 0xFFFFFFFF if b.rt.plen[p] else 0)
    base_by = {key(r): (r, f) for r, f in zip(base_rib.routes, installed["flags"])}
    n_checked = 0
    for j in range(1, n):
        rib = table(j)
        mine = records[records["job"] == j]
        acts, _ = ospf_rib.rib_diff(base_marked, rib)
        acted = {key((rib.routes if int(a["kind"]) != ospf_rib.RIB_UNINSTALL_OLD else base_rib.routes)[int(a["route"])])
                 for a in acts}
        by = {key(r): r for r in rib.routes}
        # the records are exactly the presence and metric differences of the decoded tables ...
        lost = {pkey(p) for p in mine["prefix"][mine["kind"] & 0x01 != 0]}
        gained = {pkey(p) for p in mine["prefix"][mine["kind"] & 0x02 != 0]}
        metric = {pkey(p) for p in mine["prefix"][mine["kind"] & 0x04 != 0]}
        assert lost == set(base_by) - set(by) and gained == set(by) - set(base_by)
        assert metric == {k for k in set(by) & set(base_by) if by[k]["metric"] != base_by[k][0]["metric"]}
        # ... and rib_diff acts on every one of them that the RIB manager sees: installs for gained and changed
        # metrics of installable routes, uninstalls for lost routes that were installed
        for k in gained | metric:
            if not (by[k]["flags"] & ospf_rib.ROUTE_CONNECTED) and by[k]["n_nh"]:
                assert k in acted
        for k in lost:
            if base_by[k][1] & ospf_rib.ROUTE_INSTALLED:
                assert k in acted
        # a job without records decodes to the base table's routes, metrics and paths (an unchanged cell may still
        # move a next-hop address: the transit networks' atom sets are not in the cell)
        if not len(mine):
            assert [key(r) for r in rib.routes] == [key(r) for r in base_rib.routes]
            assert (rib.routes["metric"] == base_rib.routes["metric"]).all()
        n_checked += int(len(mine) > 0)
    assert n_checked > 0
