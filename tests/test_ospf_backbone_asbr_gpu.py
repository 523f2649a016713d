"""GPU: the OSPFv2 backbone-router stage with the borders' type-4 LSAs re-originated per job
(hspf_ospfv2_backbone_asbr_cells[16], _delta[16]).  R's area-0 SPT runs on the device (one row); each border's area
planes sit on the device with one row per job, beside its routing-table cells.  The device cells must equal, byte for
byte, the CPU harness (the kAsbr walk compiled for the host) over the same planes and border cells; every job decodes
to the host chain; the delta equals the reference comparison of the stored cells."""

import numpy as np
import pytest

from holo_b200 import capi, ospf_rib
from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
from test_isis_route_cells_gpu import DeviceTopology
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospf_backbone_asbr_cells import AsbrBackbone, asbr_cells, harness  # noqa: F401  (fixture)
from test_ospf_backbone_cells import SynthBackbone, non_backbone_links, same_rib, synth_jobs
from test_ospf_backbone_cells import harness as bb_harness  # noqa: F401  (fixture)
from test_ospf_rib_delta import reference

pytestmark = pytest.mark.gpu


def dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).to("cuda")


class DevicePlanes:
    """One area's planes of every job as device rows: a capi.ResultStruct / Result16Struct over [J, V] arrays."""

    def __init__(self, rows, narrow_planes):
        import torch
        d = np.stack([r[0] for r in rows])
        h = np.stack([r[1] for r in rows])
        m = np.stack([r[2] for r in rows])
        if narrow_planes:
            d = np.where(d == 0xFFFFFFFF, 0xFFFF, d).astype(np.uint16)
            m = m.astype(np.uint16)
        self.t = [dev(d), dev(h), dev(m), torch.zeros(len(rows), dtype=torch.int32, device="cuda")]
        self.rs = capi.Result16Struct() if narrow_planes else capi.ResultStruct()
        import ctypes as C
        u16p, u32p, u64p = C.POINTER(C.c_uint16), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
        self.rs.dist = C.cast(self.t[0].data_ptr(), u16p if narrow_planes else u32p)
        self.rs.hops = C.cast(self.t[1].data_ptr(), u16p)
        self.rs.nh_mask = C.cast(self.t[2].data_ptr(), u16p if narrow_planes else u64p)
        if not narrow_planes:
            self.rs.nh_words = 1
        self.rs.job_status = C.cast(self.t[3].data_ptr(), u32p)


def setup(ctx, abr, harness, narrow_planes, seed=1):
    bb = AsbrBackbone(seed)
    links = non_backbone_links(bb)
    jobs = [bb.job_overrides((), 0)] + [bb.job_overrides(l, capi.COST_DISABLED) for l in links[:20]]
    jobs += [bb.cut(x) for x in bb.view["area1_asbrs"]] + [bb.cut(x, {2}) for x in bb.view["area1_asbrs"]]
    bp = bb.border_planes(jobs)
    want, st, bcells = bb.cells(abr, harness, bp, narrow_planes)
    assert not st.any()
    bb.table.upload(ctx)
    top = DeviceTopology(ctx, bb.flat.csr, bb.rv, 1, [[]], narrow_planes)
    top.run()
    ctx.sync()
    J = len(jobs)
    dplanes = [[DevicePlanes([bp[b][j][i] for j in range(J)], narrow_planes) for i in range(len(bp[b][0]))]
               for b in range(len(bb.doms))]
    rows = [dev(np.repeat(np.arange(J, dtype=np.uint32)[:, None], len(bp[b][0]), 1)) for b in range(len(bb.doms))]
    return bb, jobs, bp, want, bcells, top, dplanes, rows


def border_args(dplanes, rows, J):
    return ([[p.rs for p in d] for d in dplanes], [[J] * len(d) for d in dplanes], [r.data_ptr() for r in rows])


@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_device_cells_equal_the_harness(ctx, abr_harness, harness, narrow_planes):
    import torch
    bb, jobs, bp, want, bcells, top, dplanes, rows = setup(ctx, abr_harness, harness, narrow_planes)
    J, P = len(jobs), bb.table.n_prefixes
    db = [dev(c) for c in bcells]
    out = torch.zeros(J * P * 24 + 64, dtype=torch.uint8, device="cuda")
    st = torch.full((J,), 7, dtype=torch.int32, device="cuda")
    ospf_rib.backbone_asbr_cells_device(ctx, bb.table, J, top.rs, [x.data_ptr() for x in db], None,
                                        *border_args(dplanes, rows, J), st.data_ptr(), out.data_ptr())
    ctx.sync()
    got = out.cpu().numpy()[: J * P * 24].view(ospf_rib.RIB_CELL_DT).reshape(J, P)
    assert got.tobytes() == want.tobytes()
    assert not st.cpu().numpy().any()
    assert (out.cpu().numpy()[J * P * 24:] == 0).all()
    for j in range(J):
        same_rib(bb.decode(got[j]), bb.host([bp[b][j] for b in range(len(bb.doms))]))
    # the existing call refuses a table with type-4 slots
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.backbone_cells_device(ctx, bb.table, J, top.rs, [x.data_ptr() for x in db], None, 0, out.data_ptr())
    assert e.value.code == capi.HSPF_E_INVAL


@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_delta_equals_the_reference(ctx, abr_harness, harness, narrow_planes):
    import torch
    bb, jobs, bp, want, bcells, top, dplanes, rows = setup(ctx, abr_harness, harness, narrow_planes)
    J = len(jobs)
    db = [dev(c) for c in bcells]
    base = dev(want[0])
    ref_jobs, ref_recs, ref_total = reference(want, want[:1])
    assert ref_total > 0
    for cap in (0, ref_total):
        job_out = torch.zeros(J * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device="cuda")
        recs = torch.zeros(max(cap, 1) * DELTA_DT.itemsize, dtype=torch.uint8, device="cuda")
        n = torch.zeros(1, dtype=torch.int64, device="cuda")
        ospf_rib.backbone_asbr_delta_device(ctx, bb.table, J, top.rs, [x.data_ptr() for x in db], None,
                                            *border_args(dplanes, rows, J), base.data_ptr(), 1, 0, job_out.data_ptr(),
                                            recs.data_ptr() if cap else 0, cap, n.data_ptr())
        ctx.sync()
        assert job_out.cpu().numpy().view(DELTA_JOB_DT).tobytes() == ref_jobs.tobytes()
        assert int(n.cpu().item()) == ref_total
        if cap:
            assert recs.cpu().numpy().view(DELTA_DT)[:ref_total].tobytes() == ref_recs.tobytes()


def test_border_row_out_of_range_refuses_the_job(ctx, abr_harness, harness):
    import torch
    bb, jobs, bp, want, bcells, top, dplanes, rows = setup(ctx, abr_harness, harness, False)
    J, P = len(jobs), bb.table.n_prefixes
    db = [dev(c) for c in bcells]
    r1 = np.repeat(np.arange(J, dtype=np.uint32)[:, None], len(bp[1][0]), 1)
    r1[2, :] = J + 5
    rows[1] = dev(r1)
    out = torch.zeros(J * P * 24, dtype=torch.uint8, device="cuda")
    st = torch.zeros(J, dtype=torch.int32, device="cuda")
    ospf_rib.backbone_asbr_cells_device(ctx, bb.table, J, top.rs, [x.data_ptr() for x in db], None,
                                        *border_args(dplanes, rows, J), st.data_ptr(), out.data_ptr())
    ctx.sync()
    got = out.cpu().numpy().view(ospf_rib.RIB_CELL_DT).reshape(J, P)
    sw = st.cpu().numpy().view(np.uint32)
    assert sw[2] == capi.JS_INVALID and not np.delete(sw, 2).any()
    assert (got["winner"][2] == ospf_rib.NO_RECORD).all() and not got["mpf"][2].any() and not got["nh_mask"][2].any()
    keep = [j for j in range(J) if j != 2]
    assert got[keep].tobytes() == want[keep].tobytes()


def test_zero_jobs_launch_nothing(ctx, abr_harness, harness):
    import torch
    bb, jobs, bp, want, bcells, top, dplanes, rows = setup(ctx, abr_harness, harness, False)
    db = [dev(c) for c in bcells]
    out = torch.zeros(24, dtype=torch.uint8, device="cuda")
    before = ctx.launch_count
    ospf_rib.backbone_asbr_cells_device(ctx, bb.table, 0, top.rs, [x.data_ptr() for x in db], None,
                                        *border_args(dplanes, rows, 0), 0, out.data_ptr())
    ctx.sync()
    assert ctx.launch_count == before


@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_table_without_type4_slots_equals_the_existing_calls(ctx, abr_harness, bb_harness, narrow_planes):
    import torch
    bb = SynthBackbone(1)
    jobs = synth_jobs(bb, 10, 1)
    bp = bb.border_planes(jobs)
    want, st, bcells = bb.cells(abr_harness, bb_harness, bp, narrow_planes)
    t = ospf_rib.BackboneTable(bb.flat, bb.area.router_id, bb.summaries, bb.externals, [d.rt for d in bb.doms],
                               asbr=True)
    assert t.n_asbr_slots == 0
    t.upload(ctx)
    bb.table.upload(ctx)
    top = DeviceTopology(ctx, bb.flat.csr, bb.rv, 1, [[]], narrow_planes)
    top.run()
    ctx.sync()
    J, P = len(jobs), bb.table.n_prefixes
    db = [dev(c) for c in bcells]
    a = torch.zeros(J * P * 24, dtype=torch.uint8, device="cuda")
    b = torch.zeros(J * P * 24, dtype=torch.uint8, device="cuda")
    ospf_rib.backbone_cells_device(ctx, bb.table, J, top.rs, [x.data_ptr() for x in db], None, 0, a.data_ptr())
    ospf_rib.backbone_asbr_cells_device(ctx, t, J, top.rs, [x.data_ptr() for x in db], None, None, None, None, 0,
                                        b.data_ptr())
    ctx.sync()
    assert torch.equal(a, b)
    assert a.cpu().numpy().view(ospf_rib.RIB_CELL_DT).reshape(J, P).tobytes() == want.tobytes()
