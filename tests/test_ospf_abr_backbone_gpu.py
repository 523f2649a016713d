"""GPU: the OSPFv2 area-border-router stage over what-if jobs inside another area (hspf_ospfv2_abr_backbone_cells[16],
_delta[16]).  R's row 0 of each area sits on the device; each border's area planes sit on the device with one row per
job, beside its routing-table cells.  The device cells must equal, byte for byte, the CPU harness (the kSlots walk
compiled for the host) over the same planes and border cells; every job decodes to the host chain; the delta equals
the reference comparison of the stored cells."""

import numpy as np
import pytest

from holo_b200 import capi, ospf_rib
from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
from test_ospf_abr_backbone_cells import GOLDEN, SynthAbrBackbone, golden, harness  # noqa: F401  (fixture)
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospf_backbone_asbr_gpu import DevicePlanes, border_args, dev
from test_ospf_backbone_cells import non_backbone_links, same_rib, synth_jobs
from test_ospf_rib_delta import reference

pytestmark = pytest.mark.gpu


def setup(ctx, abr, harness, narrow_planes, bb=None, seed=1):
    if bb is None:
        bb = SynthAbrBackbone(seed)
        jobs = synth_jobs(bb, 10, seed) + [bb.cut(x) for x in bb.view["area1_asbrs"]]
        jobs += [bb.cut(x, {2}) for x in bb.view["area1_asbrs"]]
    else:
        jobs = [bb.job_overrides((), 0)]
        for link in non_backbone_links(bb):
            jobs += [bb.job_overrides(link, capi.COST_DISABLED), bb.job_overrides(link, 35)]
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
    ospf_rib.abr_backbone_cells_device(ctx, bb.table, J, [p.rs for p in rplanes], [x.data_ptr() for x in db], status,
                                       *bargs, st_ptr, out_ptr)


@pytest.mark.parametrize("case", ["generated", "golden"])
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_device_cells_equal_the_harness(ctx, abr_harness, harness, narrow_planes, case):
    import torch
    bb = golden(*GOLDEN[0])[0] if case == "golden" else None
    bb, jobs, bp, want, bcells, rplanes, dplanes, rows = setup(ctx, abr_harness, harness, narrow_planes, bb)
    J, P = len(jobs), bb.table.n_prefixes
    db = [dev(c) for c in bcells]
    out = torch.zeros(J * P * 24 + 64, dtype=torch.uint8, device="cuda")
    st = torch.full((J,), 7, dtype=torch.int32, device="cuda")
    bargs = border_args(dplanes, rows, J) if bb.table.n_asbr_slots else (None, None, None)
    cells_device(ctx, bb, J, rplanes, db, None, bargs, st.data_ptr(), out.data_ptr())
    ctx.sync()
    got = out.cpu().numpy()[: J * P * 24].view(ospf_rib.RIB_CELL_DT).reshape(J, P)
    assert got.tobytes() == want.tobytes()
    assert not st.cpu().numpy().any()
    assert (out.cpu().numpy()[J * P * 24:] == 0).all()
    for j in range(J):
        same_rib(bb.decode(got[j]), bb.host([bp[b][j] for b in range(len(bb.doms))]))


@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_delta_equals_the_reference(ctx, abr_harness, harness, narrow_planes):
    import torch
    bb, jobs, bp, want, bcells, rplanes, dplanes, rows = setup(ctx, abr_harness, harness, narrow_planes)
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


def test_border_status_and_type4_row_out_of_range_refuse_jobs(ctx, abr_harness, harness):
    import torch
    bb, jobs, bp, want, bcells, rplanes, dplanes, rows = setup(ctx, abr_harness, harness, False)
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
    cells_device(ctx, bb, J, rplanes, db, [0, dbst.data_ptr(), 0], border_args(dplanes, rows, J), st.data_ptr(),
                 out.data_ptr())
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
    bb, jobs, bp, want, bcells, rplanes, dplanes, rows = setup(ctx, abr_harness, harness, False)
    db = [dev(c) for c in bcells]
    out = torch.zeros(24, dtype=torch.uint8, device="cuda")
    before = ctx.launch_count
    cells_device(ctx, bb, 0, rplanes, db, None, border_args(dplanes, rows, 0), 0, out.data_ptr())
    ctx.sync()
    assert ctx.launch_count == before


def test_table_without_type4_slots_runs_with_null_plane_sets(ctx, abr_harness, harness):
    """A golden domain (no type-4 LSA): the three border plane arrays are NULL."""
    import torch
    bb = golden(*GOLDEN[4])[0]
    assert bb.table.n_asbr_slots == 0
    bb, jobs, bp, want, bcells, rplanes, dplanes, rows = setup(ctx, abr_harness, harness, False, bb)
    J, P = len(jobs), bb.table.n_prefixes
    db = [dev(c) for c in bcells]
    out = torch.zeros(J * P * 24, dtype=torch.uint8, device="cuda")
    cells_device(ctx, bb, J, rplanes, db, None, (None, None, None), 0, out.data_ptr())
    ctx.sync()
    assert out.cpu().numpy().view(ospf_rib.RIB_CELL_DT).reshape(J, P).tobytes() == want.tobytes()
