"""GPU: the OSPFv3 stage of an internal router of a non-backbone area over what-if jobs on the backbone
(hspf_ospfv3_nonbackbone_table_create through hspf_ospfv2_backbone[_asbr]_cells[16] / _delta[16]).

The full chain runs on the device: each border's area-0 SPT batch with the jobs' overrides, its OSPFv3 ABR cells with
per-job rows, then R's cells over them, whose Inter-Area-Router slots read the borders' area-0 rows.  The device cells
must equal, byte for byte, the CPU harness (the OSPFv3 kNonBackbone walk compiled for the host) over the planes read
back, and every job decodes to the host chain, prefix options included; the delta equals the reference comparison of
the stored cells."""

import numpy as np
import pytest

from holo_b200 import capi, ospf_rib
from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
from test_isis_route_cells_gpu import DeviceTopology
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospf_backbone_asbr_cells import asbr_cells
from test_ospf_backbone_asbr_gpu import dev
from test_ospfv3_nonbackbone_cells import GoldenNonBackbone, SynthNonBackbone, chain_jobs, harness  # noqa: F401
from test_ospf_rib_cells import same_rib
from test_ospf_rib_delta import reference

pytestmark = pytest.mark.gpu


def synth_jobs(bb):
    last = max(range(len(bb.doms)), key=lambda b: bb.doms[b].areas[0].router_id)
    return chain_jobs(bb)[:25] + [bb.cut(bb.view["asbr"], {last}), bb.cut(bb.view["asbr"])]


def device_chain(ctx, bb, jobs, narrow_planes):
    """Every border's SPT batches (one row per job in area 0, one row elsewhere) and ABR cells on the device, and R's
    row 0.  Returns (border tops [b][i], border rows, border cells, R's top)."""
    import torch
    J = len(jobs)
    tops, rows, cells = [], [], []
    for b, d in enumerate(bb.doms):
        d.rt.upload(ctx)
        i0 = d.rt.area_ids.index(0)
        tb = []
        for i, (f, rv) in enumerate(zip(d.flats, d.rv)):
            ov = [job[b].get(i, []) for job in jobs] if i == i0 else [[]]
            t = DeviceTopology(ctx, f.csr, rv, len(ov), ov, narrow_planes)
            t.run()
            tb.append(t)
        r = np.zeros((J, len(d.areas)), np.uint32)
        r[:, i0] = np.arange(J)
        dr = dev(r)
        c = torch.zeros(J * d.rt.n_prefixes * 24, dtype=torch.uint8, device="cuda")
        ospf_rib.abr_rib_cells_device(ctx, d.rt, J, [t.rs for t in tb], [t.n for t in tb], dr.data_ptr(), c.data_ptr())
        tops.append(tb); rows.append(dr); cells.append(c)
    top = DeviceTopology(ctx, bb.flat.csr, bb.rv, 1, [[]], narrow_planes)
    top.run()
    ctx.sync()
    return tops, rows, cells, top


@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_full_device_chain_generated_domain(ctx, abr_harness, harness, narrow_planes):
    import torch
    bb = SynthNonBackbone(1)
    assert bb.table.n_asbr_slots > 0
    jobs = synth_jobs(bb)
    J, P = len(jobs), bb.table.n_prefixes
    tops, rows, bcells_dev, top = device_chain(ctx, bb, jobs, narrow_planes)
    bb.table.upload(ctx)
    out = torch.zeros(J * P * 24 + 64, dtype=torch.uint8, device="cuda")
    st = torch.full((J,), 7, dtype=torch.int32, device="cuda")
    ospf_rib.backbone_asbr_cells_device(ctx, bb.table, J, top.rs, [c.data_ptr() for c in bcells_dev], None,
                                        [[t.rs for t in tb] for tb in tops], [[t.n for t in tb] for tb in tops],
                                        [r.data_ptr() for r in rows], st.data_ptr(), out.data_ptr())
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
    assert top.planes(0)[0].tobytes() == bb.planes[0].tobytes()
    want, _ = asbr_cells(harness, bb.table, bb.planes, bcells, bp, narrow_planes)
    assert got.tobytes() == want.tobytes()
    for j in range(J):
        same_rib(bb.decode(got[j]), bb.host(None, [bp[b][j] for b in range(len(bb.doms))]))
    assert (got != got[0]).any()


def harness_setup(ctx, abr, harness, bb, jobs, narrow_planes=False):
    bp = bb.border_planes(jobs)
    want, st, bcells = bb.cells(abr, harness, bp, narrow_planes)
    assert not st.any()
    bb.table.upload(ctx)
    top = DeviceTopology(ctx, bb.flat.csr, bb.rv, 1, [[]], narrow_planes)
    top.run()
    ctx.sync()
    return bp, want, bcells, top


def border_planes_dev(bp, J, narrow_planes):
    """Per border: its areas' planes of every job as device rows, the row counts and rows [J, n_areas]."""
    from test_ospf_backbone_asbr_gpu import DevicePlanes
    dplanes = [[DevicePlanes([bp[b][j][i] for j in range(J)], narrow_planes) for i in range(len(bp[b][0]))]
               for b in range(len(bp))]
    rows = [dev(np.repeat(np.arange(J, dtype=np.uint32)[:, None], len(bp[b][0]), 1)) for b in range(len(bp))]
    return dplanes, rows


@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_golden_domain_equals_the_harness(ctx, abr_harness, harness, narrow_planes):
    """topo2-2 rt6 (no Inter-Area-Router slot): the borders' harness cells uploaded; the plain call takes the table
    too."""
    import torch
    bb = GoldenNonBackbone("topo2-2", "rt6", ["rt4", "rt5"])
    assert bb.table.n_asbr_slots == 0
    jobs = chain_jobs(bb)
    _bp, want, bcells, top = harness_setup(ctx, abr_harness, harness, bb, jobs, narrow_planes)
    J, P = len(jobs), bb.table.n_prefixes
    db = [dev(c) for c in bcells]
    a = torch.zeros(J * P * 24, dtype=torch.uint8, device="cuda")
    b = torch.zeros(J * P * 24, dtype=torch.uint8, device="cuda")
    ospf_rib.backbone_cells_device(ctx, bb.table, J, top.rs, [x.data_ptr() for x in db], None, 0, a.data_ptr())
    ospf_rib.backbone_asbr_cells_device(ctx, bb.table, J, top.rs, [x.data_ptr() for x in db], None, None, None, None,
                                        0, b.data_ptr())
    ctx.sync()
    assert a.cpu().numpy().view(ospf_rib.RIB_CELL_DT).reshape(J, P).tobytes() == want.tobytes()
    assert torch.equal(a, b)


@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_delta_equals_the_reference(ctx, abr_harness, harness, narrow_planes):
    import torch
    bb = SynthNonBackbone(2)
    jobs = synth_jobs(bb)
    bp, want, bcells, top = harness_setup(ctx, abr_harness, harness, bb, jobs, narrow_planes)
    J = len(jobs)
    dplanes, rows = border_planes_dev(bp, J, narrow_planes)
    db = [dev(c) for c in bcells]
    base = dev(want[0])
    ref_jobs, ref_recs, ref_total = reference(want, want[:1])
    assert ref_total > 0
    for cap in (0, ref_total):
        job_out = torch.zeros(J * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device="cuda")
        recs = torch.zeros(max(cap, 1) * DELTA_DT.itemsize, dtype=torch.uint8, device="cuda")
        n = torch.zeros(1, dtype=torch.int64, device="cuda")
        ospf_rib.backbone_asbr_delta_device(ctx, bb.table, J, top.rs, [x.data_ptr() for x in db], None,
                                            [[p.rs for p in d] for d in dplanes], [[J] * len(d) for d in dplanes],
                                            [r.data_ptr() for r in rows], base.data_ptr(), 1, 0, job_out.data_ptr(),
                                            recs.data_ptr() if cap else 0, cap, n.data_ptr())
        ctx.sync()
        assert job_out.cpu().numpy().view(DELTA_JOB_DT).tobytes() == ref_jobs.tobytes()
        assert int(n.cpu().item()) == ref_total
        if cap:
            assert recs.cpu().numpy().view(DELTA_DT)[:ref_total].tobytes() == ref_recs.tobytes()


def test_refused_jobs(ctx, abr_harness, harness):
    """Border status words and a plane-set row out of range refuse their jobs: empty cells, the job's status word;
    the other jobs are unchanged."""
    import torch
    bb = SynthNonBackbone(1)
    jobs = synth_jobs(bb)[:6]
    bp, want, bcells, top = harness_setup(ctx, abr_harness, harness, bb, jobs)
    J, P = len(jobs), bb.table.n_prefixes
    dplanes, rows = border_planes_dev(bp, J, False)
    i0 = bb.doms[1].rt.area_ids.index(0)
    r1 = np.repeat(np.arange(J, dtype=np.uint32)[:, None], len(bp[1][0]), 1)
    r1[2, i0] = J + 5
    rows[1] = dev(r1)
    bst = [np.zeros(J, np.uint32) for _ in bb.doms]
    bst[0][4] = 0x4
    dst = [dev(s) for s in bst]
    db = [dev(c) for c in bcells]
    out = torch.zeros(J * P * 24, dtype=torch.uint8, device="cuda")
    st = torch.zeros(J, dtype=torch.int32, device="cuda")
    ospf_rib.backbone_asbr_cells_device(ctx, bb.table, J, top.rs, [x.data_ptr() for x in db], [s.data_ptr() for s in dst],
                                        [[p.rs for p in d] for d in dplanes], [[J] * len(d) for d in dplanes],
                                        [r.data_ptr() for r in rows], st.data_ptr(), out.data_ptr())
    ctx.sync()
    got = out.cpu().numpy().view(ospf_rib.RIB_CELL_DT).reshape(J, P)
    sw = st.cpu().numpy().view(np.uint32)
    assert sw[2] == capi.JS_INVALID and sw[4] == 0x4 and not np.delete(sw, [2, 4]).any()
    for j in (2, 4):
        assert (got["winner"][j] == ospf_rib.NO_RECORD).all() and not got["mpf"][j].any() and not got["nh_mask"][j].any()
    keep = [j for j in range(J) if j not in (2, 4)]
    assert got[keep].tobytes() == want[keep].tobytes()


def test_nothing_to_do_launches_nothing(ctx, abr_harness, harness):
    """Zero jobs, and a table without affected prefixes (topo1-1 rt7, a totally stubby area)."""
    import torch
    bb = SynthNonBackbone(0)
    bp, want, bcells, top = harness_setup(ctx, abr_harness, harness, bb, chain_jobs(bb)[:2])
    dplanes, rows = border_planes_dev(bp, 2, False)
    db = [dev(c) for c in bcells]
    out = torch.zeros(24, dtype=torch.uint8, device="cuda")
    before = ctx.launch_count
    ospf_rib.backbone_asbr_cells_device(ctx, bb.table, 0, top.rs, [x.data_ptr() for x in db], None,
                                        [[p.rs for p in d] for d in dplanes], [[2] * len(d) for d in dplanes],
                                        [r.data_ptr() for r in rows], 0, out.data_ptr())
    ctx.sync()
    assert ctx.launch_count == before
    gb = GoldenNonBackbone("topo1-1", "rt7", ["rt6"])
    assert gb.table.n_prefixes == 0
    jobs = chain_jobs(gb)[:3]
    _bp, _want, gcells, gtop = harness_setup(ctx, abr_harness, harness, gb, jobs)
    gd = [dev(c) for c in gcells]
    before = ctx.launch_count
    ospf_rib.backbone_cells_device(ctx, gb.table, len(jobs), gtop.rs, [x.data_ptr() for x in gd], None, 0,
                                   out.data_ptr())
    ospf_rib.backbone_asbr_cells_device(ctx, gb.table, len(jobs), gtop.rs, [x.data_ptr() for x in gd], None, None,
                                        None, None, 0, out.data_ptr())
    ctx.sync()
    assert ctx.launch_count == before
