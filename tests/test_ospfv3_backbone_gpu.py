"""GPU: the routes an OSPFv3 backbone router gets for every what-if job inside other areas (hspf_ospfv2_backbone_cells[16],
_delta[16] over a table of hspf_ospfv3_backbone_table_create).  R's area-0 SPT runs on the device (one row); the
borders' routing-table cells of every job sit on the device and the backbone call reads them in place.  The device
cells must equal, byte for byte, the CPU harness (the same OSPFv3 walk compiled for the host) over the same planes and
border cells; every job decodes to the host chain, prefix options included; the delta equals the reference comparison
of the stored cells."""

import numpy as np
import pytest

from holo_b200 import capi, ospf_rib
from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
from test_isis_route_cells_gpu import DeviceTopology
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospfv3_backbone_cells import Backbone, SynthBackbone, harness, non_backbone_links, same_rib, synth_jobs  # noqa: F401
from test_ospf_rib_delta import reference

pytestmark = pytest.mark.gpu


def dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).to("cuda")


def setup(ctx, abr, harness, narrow_planes, domain="golden"):
    if domain == "golden":
        bb = Backbone("topo2-2", "rt1", ["rt4", "rt5"])
        jobs = [bb.job_overrides((), 0)]
        for link in non_backbone_links(bb):
            jobs += [bb.job_overrides(link, capi.COST_DISABLED), bb.job_overrides(link, 35)]
    else:                          # ospfv3.backbone_view: three borders, an options-flip key, a prefix in two areas
        bb = SynthBackbone(1)
        jobs = synth_jobs(bb, 20, 1)
    bp = bb.border_planes(jobs)
    want, st, bcells = bb.cells(abr, harness, bp, narrow_planes)
    assert not st.any() and bb.table.v3
    bb.table.upload(ctx)
    top = DeviceTopology(ctx, bb.flat.csr, bb.rv, 1, [[]], narrow_planes)
    top.run()
    ctx.sync()
    # the harness over R's device planes read back: R's row 0 must be the oracle's
    d = top.dist.cpu().numpy().view(np.uint16 if narrow_planes else np.uint32)
    want_d = bb.planes[0].astype(np.uint16) if narrow_planes else bb.planes[0]
    if narrow_planes:
        want_d = np.where(bb.planes[0] == 0xFFFFFFFF, 0xFFFF, bb.planes[0]).astype(np.uint16)
    assert (d == want_d).all()
    return bb, jobs, bp, want, bcells, top


@pytest.mark.parametrize("domain", ["golden", "generated"])
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_device_cells_equal_the_harness(ctx, abr_harness, harness, narrow_planes, domain):
    import torch
    bb, jobs, bp, want, bcells, top = setup(ctx, abr_harness, harness, narrow_planes, domain)
    J, P = len(jobs), bb.table.n_prefixes
    db = [dev(c) for c in bcells]
    out = torch.zeros(J * P * 24 + 64, dtype=torch.uint8, device="cuda")
    st = torch.full((J,), 7, dtype=torch.int32, device="cuda")
    ospf_rib.backbone_cells_device(ctx, bb.table, J, top.rs, [x.data_ptr() for x in db], None, st.data_ptr(),
                                   out.data_ptr())
    ctx.sync()
    got = out.cpu().numpy()[: J * P * 24].view(ospf_rib.RIB_CELL_DT).reshape(J, P)
    assert got.tobytes() == want.tobytes()
    assert not st.cpu().numpy().any()
    assert (out.cpu().numpy()[J * P * 24:] == 0).all()
    for j in range(J):
        same_rib(bb.decode(got[j]), bb.host([c[j] for c in bcells], [bp[b][j] for b in range(len(bb.doms))]))


def test_border_status_words_refuse_jobs(ctx, abr_harness, harness):
    import torch
    bb, jobs, bp, want, bcells, top = setup(ctx, abr_harness, harness, False)
    J, P = len(jobs), bb.table.n_prefixes
    db = [dev(c) for c in bcells]
    s0 = np.zeros(J, np.uint32)
    s1 = np.zeros(J, np.uint32)
    s0[1], s1[2] = 0x1, 0x4
    ds = [dev(s0), dev(s1)]
    out = torch.zeros(J * P * 24, dtype=torch.uint8, device="cuda")
    st = torch.zeros(J, dtype=torch.int32, device="cuda")
    ospf_rib.backbone_cells_device(ctx, bb.table, J, top.rs, [x.data_ptr() for x in db], [x.data_ptr() for x in ds],
                                   st.data_ptr(), out.data_ptr())
    ctx.sync()
    got = out.cpu().numpy().view(ospf_rib.RIB_CELL_DT).reshape(J, P)
    sw = st.cpu().numpy().view(np.uint32)
    assert list(sw[:3]) == [0, 0x1, 0x4] and not sw[3:].any()
    for j in (1, 2):
        assert (got["winner"][j] == ospf_rib.NO_RECORD).all() and not got["mpf"][j].any() and not got["nh_mask"][j].any()
    keep = [j for j in range(J) if j not in (1, 2)]
    assert got[keep].tobytes() == want[keep].tobytes()


@pytest.mark.parametrize("domain", ["golden", "generated"])
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_delta_equals_the_reference(ctx, abr_harness, harness, narrow_planes, domain):
    import torch
    bb, jobs, bp, want, bcells, top = setup(ctx, abr_harness, harness, narrow_planes, domain)
    J, P = len(jobs), bb.table.n_prefixes
    db = [dev(c) for c in bcells]
    base = dev(want[0])
    ref_jobs, ref_recs, ref_total = reference(want, want[:1])
    assert ref_total > 0
    for cap in (0, ref_total):
        job_out = torch.zeros(J * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device="cuda")
        recs = torch.zeros(max(cap, 1) * DELTA_DT.itemsize, dtype=torch.uint8, device="cuda")
        n = torch.zeros(1, dtype=torch.int64, device="cuda")
        ospf_rib.backbone_delta_device(ctx, bb.table, J, top.rs, [x.data_ptr() for x in db], None, base.data_ptr(), 1, 0,
                                       job_out.data_ptr(), recs.data_ptr() if cap else 0, cap, n.data_ptr())
        ctx.sync()
        assert job_out.cpu().numpy().view(DELTA_JOB_DT).tobytes() == ref_jobs.tobytes()
        assert int(n.cpu().item()) == ref_total
        if cap:
            assert recs.cpu().numpy().view(DELTA_DT)[:ref_total].tobytes() == ref_recs.tobytes()


def test_zero_jobs_launch_nothing(ctx, abr_harness, harness):
    import torch
    bb, jobs, bp, want, bcells, top = setup(ctx, abr_harness, harness, False)
    db = [dev(c) for c in bcells]
    out = torch.zeros(24, dtype=torch.uint8, device="cuda")
    before = ctx.launch_count
    ospf_rib.backbone_cells_device(ctx, bb.table, 0, top.rs, [x.data_ptr() for x in db], None, 0, out.data_ptr())
    ctx.sync()
    assert ctx.launch_count == before


def test_options_flip_on_the_device_is_other(ctx, abr_harness, harness):
    """A border cell whose winner moves, at its metric, to the other record of the flip key (other options): the
    device delta against job 0 reports exactly one OTHER record, for that key."""
    import torch
    from holo_b200.route_table import DELTA_OTHER
    from test_ospfv3_backbone_cells import flip_cells
    bb = SynthBackbone(0)
    cells, bcells, flipped, bp = flip_cells(bb, abr_harness, harness)
    u = bb.key_index(bb.view["flip"])
    both = [np.concatenate([a, b]) for a, b in zip(bcells, flipped)]
    want, _ = bb.cells_from(harness, both)
    bb.table.upload(ctx)
    top = DeviceTopology(ctx, bb.flat.csr, bb.rv, 1, [[]], False)
    top.run()
    db = [dev(c) for c in both]
    base = dev(want[0])
    job_out = torch.zeros(2 * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device="cuda")
    recs = torch.zeros(4 * DELTA_DT.itemsize, dtype=torch.uint8, device="cuda")
    n = torch.zeros(1, dtype=torch.int64, device="cuda")
    ospf_rib.backbone_delta_device(ctx, bb.table, 2, top.rs, [x.data_ptr() for x in db], None, base.data_ptr(), 1, 0,
                                   job_out.data_ptr(), recs.data_ptr(), 4, n.data_ptr())
    ctx.sync()
    assert int(n.cpu().item()) == 1
    r = recs.cpu().numpy().view(DELTA_DT)[0]
    assert (int(r["job"]), int(r["prefix"]), int(r["kind"])) == (1, u, DELTA_OTHER)
