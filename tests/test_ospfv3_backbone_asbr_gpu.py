"""GPU: the OSPFv3 backbone-router stage with the borders' Inter-Area-Router LSAs re-originated per job
(hspf_ospfv3_backbone_asbr_table_create through hspf_ospfv2_backbone_asbr_cells[16] / _delta[16]).

The full chain runs on the device: each border's SPT batches with the jobs' overrides in its non-backbone areas, its
OSPFv3 ABR cells with per-job rows, then R's cells over them, whose Inter-Area-Router slots read the borders' area-1
rows.  The device cells must equal, byte for byte, the CPU harness (the OSPFv3 kAsbr walk compiled for the host) over
the planes read back, and every job decodes to the host chain, prefix options included; the delta equals the
reference comparison of the stored cells."""

import numpy as np
import pytest

from holo_b200 import capi, ospf_rib
from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
from test_isis_route_cells_gpu import DeviceTopology
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospf_backbone_asbr_cells import asbr_cells
from test_ospf_backbone_asbr_gpu import dev
from test_ospf_rib_cells import same_rib
from test_ospf_rib_delta import reference
from test_ospfv3_backbone_asbr_cells import AsbrBackbone, harness  # noqa: F401  (fixture)
from test_ospfv3_backbone_cells import SynthBackbone, synth_jobs
from test_ospfv3_nonbackbone_gpu import border_planes_dev, harness_setup

pytestmark = pytest.mark.gpu


def asbr_jobs(bb, n=10, seed=1):
    last = max(range(len(bb.doms)), key=lambda b: bb.doms[b].areas[0].router_id)
    xs = bb.view["area1_asbrs"]
    return synth_jobs(bb, n, seed) + [bb.cut(x, {last}) for x in xs] + [bb.cut(x) for x in xs]


def device_chain(ctx, bb, jobs, narrow_planes):
    """Every border's SPT batches (one row per job in its non-backbone areas, one row in area 0) and ABR cells on the
    device, and R's row 0.  Returns (border tops [b][i], border rows, border cells, R's top)."""
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
    top = DeviceTopology(ctx, bb.flat.csr, bb.rv, 1, [[]], narrow_planes)
    top.run()
    ctx.sync()
    return tops, rows, cells, top


@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_full_device_chain_generated_domain(ctx, abr_harness, harness, narrow_planes):
    import torch
    bb = AsbrBackbone(1)
    assert bb.table.n_asbr_slots > 0
    jobs = asbr_jobs(bb)
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


@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_delta_equals_the_reference(ctx, abr_harness, harness, narrow_planes):
    import torch
    bb = AsbrBackbone(2)
    jobs = asbr_jobs(bb, seed=2)
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


def test_border_row_out_of_range_refuses_the_job(ctx, abr_harness, harness):
    """A plane-set row out of range refuses its job (HSPF_JS_INVALID, empty cells); the other jobs are unchanged."""
    import torch
    bb = AsbrBackbone(1)
    jobs = asbr_jobs(bb)[:6]
    bp, want, bcells, top = harness_setup(ctx, abr_harness, harness, bb, jobs)
    J, P = len(jobs), bb.table.n_prefixes
    dplanes, rows = border_planes_dev(bp, J, False)
    i1 = bb.doms[1].rt.area_ids.index(1)
    r1 = np.repeat(np.arange(J, dtype=np.uint32)[:, None], len(bp[1][0]), 1)
    r1[2, i1] = J + 5
    rows[1] = dev(r1)
    db = [dev(c) for c in bcells]
    out = torch.zeros(J * P * 24, dtype=torch.uint8, device="cuda")
    st = torch.zeros(J, dtype=torch.int32, device="cuda")
    ospf_rib.backbone_asbr_cells_device(ctx, bb.table, J, top.rs, [x.data_ptr() for x in db], None,
                                        [[p.rs for p in d] for d in dplanes], [[J] * len(d) for d in dplanes],
                                        [r.data_ptr() for r in rows], st.data_ptr(), out.data_ptr())
    ctx.sync()
    got = out.cpu().numpy().view(ospf_rib.RIB_CELL_DT).reshape(J, P)
    sw = st.cpu().numpy().view(np.uint32)
    assert sw[2] == capi.JS_INVALID and not np.delete(sw, [2]).any()
    assert (got["winner"][2] == ospf_rib.NO_RECORD).all() and not got["mpf"][2].any() and not got["nh_mask"][2].any()
    keep = [j for j in range(J) if j != 2]
    assert got[keep].tobytes() == want[keep].tobytes()


def test_zero_jobs_launch_nothing(ctx, abr_harness, harness):
    import torch
    bb = AsbrBackbone(0)
    bp, _want, bcells, top = harness_setup(ctx, abr_harness, harness, bb, asbr_jobs(bb, 1, 0)[:2])
    dplanes, rows = border_planes_dev(bp, 2, False)
    db = [dev(c) for c in bcells]
    out = torch.zeros(24, dtype=torch.uint8, device="cuda")
    before = ctx.launch_count
    ospf_rib.backbone_asbr_cells_device(ctx, bb.table, 0, top.rs, [x.data_ptr() for x in db], None,
                                        [[p.rs for p in d] for d in dplanes], [[2] * len(d) for d in dplanes],
                                        [r.data_ptr() for r in rows], 0, out.data_ptr())
    ctx.sync()
    assert ctx.launch_count == before


@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_table_without_slots_and_the_old_tables_refusal(ctx, abr_harness, harness, narrow_planes):
    """SynthBackbone (no area-1 ASBR): the asbr create's table, through the asbr calls and the plain calls, gives the
    old create's cells and delta.  The old create's OSPFv3 area-0 table is refused by the asbr calls (HSPF_E_INVAL)
    before any launch."""
    import torch
    bb = SynthBackbone(1)
    jobs = synth_jobs(bb, 6, 1)
    bp = bb.border_planes(jobs)
    J, P = len(jobs), bb.table.n_prefixes
    bcells = [np.stack([d.cells(abr_harness, p, narrow_planes)[0] for p in b]) for d, b in zip(bb.doms, bp)]
    old = bb.table
    new = ospf_rib.BackboneTable(bb.flat, bb.area.router_id, bb.summaries, bb.externals, [d.rt for d in bb.doms],
                                 asbr=True)
    assert new.n_asbr_slots == 0 and new.n_prefixes == P
    old.upload(ctx)
    new.upload(ctx)
    top = DeviceTopology(ctx, bb.flat.csr, bb.rv, 1, [[]], narrow_planes)
    top.run()
    ctx.sync()
    db = [dev(c) for c in bcells]
    ptrs = [x.data_ptr() for x in db]
    outs = [torch.zeros(J * P * 24, dtype=torch.uint8, device="cuda") for _ in range(3)]
    ospf_rib.backbone_cells_device(ctx, old, J, top.rs, ptrs, None, 0, outs[0].data_ptr())
    ospf_rib.backbone_cells_device(ctx, new, J, top.rs, ptrs, None, 0, outs[1].data_ptr())
    ospf_rib.backbone_asbr_cells_device(ctx, new, J, top.rs, ptrs, None, None, None, None, 0, outs[2].data_ptr())
    ctx.sync()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    base = outs[0][: P * 24].clone()
    deltas = []
    for t, asbr in ((old, False), (new, True)):
        job_out = torch.zeros(J * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device="cuda")
        recs = torch.zeros(J * P * DELTA_DT.itemsize, dtype=torch.uint8, device="cuda")
        n = torch.zeros(1, dtype=torch.int64, device="cuda")
        if asbr:
            ospf_rib.backbone_asbr_delta_device(ctx, t, J, top.rs, ptrs, None, None, None, None, base.data_ptr(), 1, 0,
                                                job_out.data_ptr(), recs.data_ptr(), J * P, n.data_ptr())
        else:
            ospf_rib.backbone_delta_device(ctx, t, J, top.rs, ptrs, None, base.data_ptr(), 1, 0, job_out.data_ptr(),
                                           recs.data_ptr(), J * P, n.data_ptr())
        ctx.sync()
        deltas.append((job_out.cpu().numpy().tobytes(), recs.cpu().numpy().tobytes(), int(n.cpu().item())))
    assert deltas[0] == deltas[1] and deltas[0][2] > 0
    # the old create's table: refused by both asbr calls before any launch
    before = ctx.launch_count
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.backbone_asbr_cells_device(ctx, old, J, top.rs, ptrs, None, None, None, None, 0, outs[2].data_ptr())
    assert e.value.code == capi.HSPF_E_INVAL
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.backbone_asbr_delta_device(ctx, old, J, top.rs, ptrs, None, None, None, None, base.data_ptr(), 1, 0,
                                            0, 0, 0, 0)
    assert e.value.code == capi.HSPF_E_INVAL
    ctx.sync()
    assert ctx.launch_count == before
