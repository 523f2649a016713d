"""GPU: the batched routing-table stage for OSPFv3 area border routers: hspf_ospfv2_abr_rib_cells[16] and
hspf_ospfv2_abr_rib_delta[16] over tables of hspf_ospfv3_abr_ribtable_create.  Each area's SPT planes are written on
the device by one SPT batch per area; a job picks one row per area.  The device cells must equal, byte for byte, the CPU
harness over those planes; sampled jobs decode to update_rib_full_v3; the delta equals the numpy reference over the
stored cells."""
import numpy as np
import pytest

import test_ospf_abr_rib_gpu as g2
from holo_b200 import ospf_rib
from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
from test_isis_route_cells_gpu import DeviceTopology
from test_ospf_abr_rib_cells import harness  # noqa: F401  (the fixture)
from test_ospf_rib_cells import same_rib
from test_ospf_rib_delta import reference
from test_ospfv2_route_cells import gather_for
from test_ospfv3_abr_rib_cells import domain, router_edges

pytestmark = pytest.mark.gpu

dev_u32, SENTINEL, GUARD = g2.dev_u32, g2.SENTINEL, g2.GUARD


class AbrBatch(g2.AbrBatch):
    """test_ospf_abr_rib_gpu.AbrBatch over an ospfv3.abr_view domain."""

    def __init__(self, ctx, seed, n_rows=6, narrow=False, **kw):
        self.ctx, self.narrow = ctx, narrow
        self.dom = domain(seed, **kw)
        self.rt = self.dom.rt
        assert self.rt.v3
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


@pytest.mark.parametrize("narrow", [False, True])
@pytest.mark.parametrize("offset", [0, 8])
def test_device_cells_equal_harness(ctx, harness, narrow, offset):
    b = AbrBatch(ctx, 1, narrow=narrow, V=30, E=90)
    cells, st, _ = b.launch(offset=offset)
    want, wst = b.harness(harness)
    assert (st == wst).all() and not st.any()
    assert cells.tobytes() == want.tobytes()
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
    assert not st.any()
    want, _ = b.harness(harness)
    assert cells.tobytes() == want.tobytes()
    planes = [b.host_planes(i) for i in range(A)]
    for j in sample:
        p = [(planes[i][0][b.rows[j, i]], planes[i][1][b.rows[j, i]], planes[i][2][b.rows[j, i]]) for i in range(A)]
        for i in range(A):
            v, n = gather_for(b.dom.flats[i], b.dom.rv[i], p[i])
            got = [int(x) for (jj, ii, _vv), x in zip(gather, gnh) if jj == j and ii == i]
            assert got == [int(x) for x in n]
        rib = b.dom.decode(cells[j], p)
        same_rib(rib, b.dom.host(p))
        assert set(int(x) for x in rib.routes["path_type"]) == {0, 1, 2, 3}


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
