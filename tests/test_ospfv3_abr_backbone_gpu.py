"""GPU: the OSPFv3 area-border-router stage over what-if jobs inside another area (hspf_ospfv3_abr_backbone_table_create
through hspf_ospfv2_abr_backbone_cells[16] / _delta[16]).

The full chain runs on the device: each border's SPT batches with the jobs' overrides in its non-backbone areas, its
OSPFv3 ABR cells (hspf_ospfv2_abr_rib_cells[16]) with its job row of area 1 and row 0 of its other areas, R's row 0 of
each of its areas, then R's cells over them, whose Inter-Area-Router slots read the borders' area-1 rows.  The device
cells must equal, byte for byte, the CPU harness (the OSPFv3 walk compiled for the host) over the planes read back, and
every job decodes to the host chain, prefix options included; the delta equals the reference comparison of the stored
cells."""

import numpy as np
import pytest

from holo_b200 import capi, ospf_rib
from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
from test_isis_route_cells_gpu import DeviceTopology
from test_ospf_abr_backbone_cells import abr_backbone_cells
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospf_backbone_asbr_gpu import DevicePlanes, border_args, dev
from test_ospf_rib_cells import same_rib
from test_ospf_rib_delta import reference
from test_ospfv3_abr_backbone_cells import GOLDEN, SynthAbrBackbone, golden, harness  # noqa: F401  (fixture)
from test_ospfv3_backbone_cells import non_backbone_links, synth_jobs

pytestmark = pytest.mark.gpu


def generated_jobs(bb, seed=1):
    last = max(range(len(bb.doms)), key=lambda b: bb.doms[b].areas[0].router_id)
    xs = bb.view["area1_asbrs"]
    return synth_jobs(bb, 10, seed) + [bb.cut(x, {last}) for x in xs] + [bb.cut(x) for x in xs]


def golden_jobs(bb):
    jobs = [bb.job_overrides((), 0)]
    for link in non_backbone_links(bb):
        jobs += [bb.job_overrides(link, capi.COST_DISABLED), bb.job_overrides(link, 35)]
    return jobs


def device_chain(ctx, bb, jobs, narrow_planes):
    """Every border's SPT batches (one row per job in its non-backbone areas, one row in area 0) and ABR cells on the
    device, and R's row 0 of each area.  Returns (border tops [b][i], border rows, border cells, R's tops [i])."""
    import torch
    J = len(jobs)
    tops, rows, cells = [], [], []
    for b, d in enumerate(bb.doms):
        d.rt.upload(ctx)
        tb = []
        r = np.zeros((J, len(d.areas)), np.uint32)
        for i, (a, f, rv) in enumerate(zip(d.areas, d.flats, d.rv)):
            ov = [job[b].get(i, []) for job in jobs] if a.area_id != 0 else [[]]
            t = DeviceTopology(ctx, f.csr, rv, len(ov), ov, narrow_planes)
            t.run()
            tb.append(t)
            if a.area_id != 0:
                r[:, i] = np.arange(J)
        dr = dev(r)
        c = torch.zeros(J * d.rt.n_prefixes * 24, dtype=torch.uint8, device="cuda")
        ospf_rib.abr_rib_cells_device(ctx, d.rt, J, [t.rs for t in tb], [t.n for t in tb], dr.data_ptr(), c.data_ptr())
        tops.append(tb); rows.append(dr); cells.append(c)
    rtops = []
    for f, rv in zip(bb.r.flats, bb.r.rv):
        t = DeviceTopology(ctx, f.csr, rv, 1, [[]], narrow_planes)
        t.run()
        rtops.append(t)
    ctx.sync()
    return tops, rows, cells, rtops


@pytest.mark.parametrize("case", ["generated", "golden"])
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_full_device_chain(ctx, abr_harness, harness, narrow_planes, case):
    import torch
    if case == "golden":
        bb = golden(*GOLDEN[0])[0]
        jobs = golden_jobs(bb)
    else:
        bb = SynthAbrBackbone(1)
        assert bb.table.n_asbr_slots > 0
        jobs = generated_jobs(bb)
    J, P = len(jobs), bb.table.n_prefixes
    tops, rows, bcells_dev, rtops = device_chain(ctx, bb, jobs, narrow_planes)
    bb.table.upload(ctx)
    out = torch.zeros(J * P * 24 + 64, dtype=torch.uint8, device="cuda")
    st = torch.full((J,), 7, dtype=torch.int32, device="cuda")
    bargs = ([[t.rs for t in tb] for tb in tops], [[t.n for t in tb] for tb in tops], [r.data_ptr() for r in rows])
    ospf_rib.abr_backbone_cells_device(ctx, bb.table, J, [t.rs for t in rtops], [c.data_ptr() for c in bcells_dev],
                                       None, *bargs, st.data_ptr(), out.data_ptr())
    ctx.sync()
    got = out.cpu().numpy()[: J * P * 24].view(ospf_rib.RIB_CELL_DT).reshape(J, P)
    assert not st.cpu().numpy().any()
    assert (out.cpu().numpy()[J * P * 24:] == 0).all()
    # the harness over the planes read back
    bp = [[[tb[i].planes(j if tb[i].n > 1 else 0) for i in range(len(tb))] for j in range(J)] for tb in tops]
    bcells = [c.cpu().numpy().view(ospf_rib.RIB_CELL_DT).reshape(J, -1) for c in bcells_dev]
    for b, d in enumerate(bb.doms):
        want_b = np.stack([d.cells(abr_harness, bp[b][j], narrow_planes)[0] for j in range(J)])
        assert bcells[b].tobytes() == want_b.tobytes()
    for t, p in zip(rtops, bb.planes):
        assert t.planes(0)[0].tobytes() == p[0].tobytes()
    want, _ = abr_backbone_cells(harness, bb.table, bb.planes, bcells, bp, narrow_planes)
    assert got.tobytes() == want.tobytes()
    for j in range(J):
        same_rib(bb.decode(got[j]), bb.host([bp[b][j] for b in range(len(bb.doms))]))
    assert (got != got[0]).any()


def harness_setup(ctx, abr, harness, narrow_planes, seed=1):
    """The generated domain's jobs through the harness, with R's row 0 and the borders' job planes on the device."""
    bb = SynthAbrBackbone(seed)
    jobs = generated_jobs(bb, seed)
    bp = bb.border_planes(jobs)
    want, st, bcells = bb.cells(abr, harness, bp, narrow_planes)
    assert not st.any()
    bb.table.upload(ctx)
    rplanes = [DevicePlanes([p], narrow_planes) for p in bb.planes]
    J = len(jobs)
    dplanes = [[DevicePlanes([bp[b][j][i] for j in range(J)], narrow_planes) for i in range(len(bp[b][0]))]
               for b in range(len(bb.doms))]
    rows = [dev(np.repeat(np.arange(J, dtype=np.uint32)[:, None], len(bp[b][0]), 1)) for b in range(len(bb.doms))]
    return bb, jobs, bp, want, bcells, rplanes, dplanes, rows


def cells_device(ctx, bb, J, rplanes, db, status, bargs, st_ptr, out_ptr):
    ospf_rib.abr_backbone_cells_device(ctx, bb.table, J, [p.rs for p in rplanes], [int(x) for x in db], status, *bargs,
                                       st_ptr, out_ptr)


@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_delta_equals_the_reference(ctx, abr_harness, harness, narrow_planes):
    import torch
    bb, jobs, bp, want, bcells, rplanes, dplanes, rows = harness_setup(ctx, abr_harness, harness, narrow_planes, 2)
    J = len(jobs)
    db = [dev(c) for c in bcells]
    base = dev(want[0])
    ref_jobs, ref_recs, ref_total = reference(want, want[:1])
    assert ref_total > 0
    for cap in (0, ref_total):
        job_out = torch.zeros(J * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device="cuda")
        recs = torch.zeros(max(cap, 1) * DELTA_DT.itemsize, dtype=torch.uint8, device="cuda")
        n = torch.zeros(1, dtype=torch.int64, device="cuda")
        ospf_rib.abr_backbone_delta_device(ctx, bb.table, J, [p.rs for p in rplanes], [x.data_ptr() for x in db], None,
                                           *border_args(dplanes, rows, J), base.data_ptr(), 1, 0, job_out.data_ptr(),
                                           recs.data_ptr() if cap else 0, cap, n.data_ptr())
        ctx.sync()
        assert job_out.cpu().numpy().view(DELTA_JOB_DT).tobytes() == ref_jobs.tobytes()
        assert int(n.cpu().item()) == ref_total
        if cap:
            assert recs.cpu().numpy().view(DELTA_DT)[:ref_total].tobytes() == ref_recs.tobytes()


def test_border_status_and_row_out_of_range_refuse_jobs(ctx, abr_harness, harness):
    import torch
    bb, jobs, bp, want, bcells, rplanes, dplanes, rows = harness_setup(ctx, abr_harness, harness, False)
    J, P = len(jobs), bb.table.n_prefixes
    db = [dev(c) for c in bcells]
    r1 = np.repeat(np.arange(J, dtype=np.uint32)[:, None], len(bp[1][0]), 1)
    r1[2, :] = J + 5
    rows[1] = dev(r1)
    bst = np.zeros(J, np.uint32)
    bst[4] = 0x2
    dbst = dev(bst)
    out = torch.zeros(J * P * 24, dtype=torch.uint8, device="cuda")
    st = torch.zeros(J, dtype=torch.int32, device="cuda")
    cells_device(ctx, bb, J, rplanes, [x.data_ptr() for x in db], [0, dbst.data_ptr(), 0],
                 border_args(dplanes, rows, J), st.data_ptr(), out.data_ptr())
    ctx.sync()
    got = out.cpu().numpy().view(ospf_rib.RIB_CELL_DT).reshape(J, P)
    sw = st.cpu().numpy().view(np.uint32)
    assert sw[2] == capi.JS_INVALID and sw[4] == 0x2 and not np.delete(sw, [2, 4]).any()
    for j in (2, 4):
        assert (got["winner"][j] == ospf_rib.NO_RECORD).all() and not got["mpf"][j].any() and not got["nh_mask"][j].any()
    keep = [j for j in range(J) if j not in (2, 4)]
    assert got[keep].tobytes() == want[keep].tobytes()


def test_zero_jobs_launch_nothing(ctx, abr_harness, harness):
    import torch
    bb, jobs, bp, want, bcells, rplanes, dplanes, rows = harness_setup(ctx, abr_harness, harness, False)
    db = [dev(c) for c in bcells]
    out = torch.zeros(24, dtype=torch.uint8, device="cuda")
    before = ctx.launch_count
    cells_device(ctx, bb, 0, rplanes, [x.data_ptr() for x in db], None, border_args(dplanes, rows, 0), 0,
                 out.data_ptr())
    ctx.sync()
    assert ctx.launch_count == before


def test_table_without_inter_area_router_slots_runs_with_null_plane_sets(ctx, abr_harness, harness):
    """A golden domain (no Inter-Area-Router LSA): the three border plane arrays are NULL."""
    import torch
    bb = golden(*GOLDEN[0])[0]
    assert bb.table.n_asbr_slots == 0
    jobs = golden_jobs(bb)
    bp = bb.border_planes(jobs)
    want, st, bcells = bb.cells(abr_harness, harness, bp)
    assert not st.any()
    bb.table.upload(ctx)
    rplanes = [DevicePlanes([p], False) for p in bb.planes]
    J, P = len(jobs), bb.table.n_prefixes
    db = [dev(c) for c in bcells]
    out = torch.zeros(J * P * 24, dtype=torch.uint8, device="cuda")
    cells_device(ctx, bb, J, rplanes, [x.data_ptr() for x in db], None, (None, None, None), 0, out.data_ptr())
    ctx.sync()
    assert out.cpu().numpy().view(ospf_rib.RIB_CELL_DT).reshape(J, P).tobytes() == want.tobytes()


def test_misaligned_border_cells_are_refused_before_any_launch(ctx, abr_harness, harness):
    import torch
    bb, jobs, bp, want, bcells, rplanes, dplanes, rows = harness_setup(ctx, abr_harness, harness, False)
    J, P = len(jobs), bb.table.n_prefixes
    db = [dev(c) for c in bcells]
    out = torch.zeros(J * P * 24, dtype=torch.uint8, device="cuda")
    before = ctx.launch_count
    ptrs = [x.data_ptr() for x in db]
    ptrs[1] += 4
    with pytest.raises(capi.HspfError) as e:
        cells_device(ctx, bb, J, rplanes, ptrs, None, border_args(dplanes, rows, J), 0, out.data_ptr())
    assert e.value.code == capi.HSPF_E_INVAL
    ctx.sync()
    assert ctx.launch_count == before
    assert not out.cpu().numpy().any()
