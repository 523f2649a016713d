"""GPU: the OSPFv3 third-area stage (hspf_ospfv2_third_area_cells[16], _delta[16] over an
hspf_ospfv3_third_area_table_create table) and the ASBR entries of an OSPFv3 area border router
(hspf_ospfv3_abr_backbone_asbr_entries[16]).  The B's cells and area planes sit on the device; each C's OSPFv3
abr_backbone cells and entries are computed on the device from them, and R's cells from those.  One test runs the whole
chain on the device, from the B's SPT batches and ABR cells on.  The device entries and cells must equal, byte for
byte, the CPU harnesses over the same planes; every job decodes to the host chain, prefix options included; the delta
equals the reference comparison of the stored cells."""

import numpy as np
import pytest

from holo_b200 import capi, ospf_rib
from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
from test_isis_route_cells_gpu import DeviceTopology
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospf_backbone_asbr_gpu import DevicePlanes, border_args, dev
from test_ospf_rib_cells import same_rib
from test_ospf_rib_delta import reference
from test_ospf_third_area_cells import harness as entries_harness  # noqa: F401  (fixture)
from test_ospfv3_abr_backbone_cells import harness as abr_backbone_harness  # noqa: F401  (fixture)
from test_ospfv3_third_area_cells import GOLDEN, SynthThirdArea, golden, harness, synth_jobs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


class Pipeline:
    """The device chain of one domain over one batch of jobs, with the CPU harnesses' results beside it."""

    def __init__(self, ctx, abr, abr_backbone, entries_h, harness, t, jobs, narrow_planes):
        import torch
        self.t, self.J = t, len(jobs)
        J = self.J
        self.want, st, self.ccells, self.cents, self.bp = t.run(abr, abr_backbone, entries_h, harness, jobs,
                                                                narrow_planes)
        assert not st.any()
        self.rplanes = DevicePlanes([t.planes], narrow_planes)
        bp = self.bp
        dplanes = [[DevicePlanes([bp[b][j][i] for j in range(J)], narrow_planes) for i in range(len(bp[b][0]))]
                   for b in range(len(t.doms))]
        rows = [dev(np.repeat(np.arange(J, dtype=np.uint32)[:, None], len(bp[b][0]), 1)) for b in range(len(t.doms))]
        self.keep = [dplanes, rows]
        self.bargs = border_args(dplanes, rows, J)
        # the B cells, from the CPU harness, on the device
        bcells = [np.stack([d.cells(abr, p, narrow_planes)[0] for p in bpb]) for d, bpb in zip(t.doms, bp)]
        self.db = [dev(c) for c in bcells]
        self.dc, self.de, self.des = [], [], []
        for c in t.cs:
            c.table.upload(ctx)
            cp = [DevicePlanes([p], narrow_planes) for p in c.planes]
            self.keep.append(cp)
            K, G = c.table.n_prefixes, len(c.table.asbr_ids)
            out = torch.zeros(J * K * 24, dtype=torch.uint8, device="cuda")
            ospf_rib.abr_backbone_cells_device(ctx, c.table, J, [p.rs for p in cp], [x.data_ptr() for x in self.db],
                                               None, *(self.bargs if c.table.n_asbr_slots else (None, None, None)), 0,
                                               out.data_ptr())
            ent = torch.full((max(J * G, 1),), 7, dtype=torch.int32, device="cuda")
            est = torch.full((max(J, 1),), 7, dtype=torch.int32, device="cuda")
            ospf_rib.abr_backbone_asbr_entries_device(ctx, c.table, J, [p.rs for p in cp],
                                                      *(self.bargs if c.table.n_asbr_slots else (None, None, None)),
                                                      est.data_ptr(), ent.data_ptr())
            self.dc.append(out)
            self.de.append(ent)
            self.des.append(est)
        ctx.sync()
        t.table.upload(ctx)

    def check_borders(self):
        J = self.J
        for c, out, ent, est, want_c, want_e in zip(self.t.cs, self.dc, self.de, self.des, self.ccells, self.cents):
            got = out.cpu().numpy().view(ospf_rib.RIB_CELL_DT).reshape(J, c.table.n_prefixes)
            assert got.tobytes() == want_c.tobytes()
            G = len(c.table.asbr_ids)
            assert ent.cpu().numpy().view(np.uint32)[: J * G].reshape(J, G).tobytes() == want_e.tobytes()
            assert not est.cpu().numpy()[:J].any()

    def cells(self, ctx, st_ptr, out_ptr, entries=True, n_jobs=None, cstatus=None):
        J = self.J if n_jobs is None else n_jobs
        ospf_rib.third_area_cells_device(ctx, self.t.table, J, self.rplanes.rs, [x.data_ptr() for x in self.dc],
                                         cstatus, [x.data_ptr() for x in self.de] if entries else None,
                                         [x.data_ptr() for x in self.des], st_ptr, out_ptr)


@pytest.mark.parametrize("n_c,k", [(2, 2), (3, 1)])
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_device_pipeline_equals_the_harness(ctx, abr_harness, abr_backbone_harness, entries_harness, harness,
                                            narrow_planes, n_c, k):
    import torch
    t = SynthThirdArea(1, n_c=n_c, k=k)
    assert t.table.n_asbr_slots > 0
    jobs = synth_jobs(t, 10, 1)
    pl = Pipeline(ctx, abr_harness, abr_backbone_harness, entries_harness, harness, t, jobs, narrow_planes)
    pl.check_borders()
    J, P = pl.J, t.table.n_prefixes
    out = torch.zeros(J * P * 24 + 64, dtype=torch.uint8, device="cuda")
    st = torch.full((J,), 7, dtype=torch.int32, device="cuda")
    pl.cells(ctx, st.data_ptr(), out.data_ptr())
    ctx.sync()
    got = out.cpu().numpy()[: J * P * 24].view(ospf_rib.RIB_CELL_DT).reshape(J, P)
    assert got.tobytes() == pl.want.tobytes()
    assert not st.cpu().numpy().any()
    assert (out.cpu().numpy()[J * P * 24:] == 0).all()
    for j in range(J):
        same_rib(t.decode(got[j]), t.affected(t.host_full([pl.bp[b][j] for b in range(len(t.doms))])))


@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_delta_equals_the_reference(ctx, abr_harness, abr_backbone_harness, entries_harness, harness, narrow_planes):
    import torch
    t = SynthThirdArea(0, n_c=2, k=2)
    pl = Pipeline(ctx, abr_harness, abr_backbone_harness, entries_harness, harness, t, synth_jobs(t, 10, 0),
                  narrow_planes)
    J = pl.J
    base = dev(pl.want[0])
    ref_jobs, ref_recs, ref_total = reference(pl.want, pl.want[:1])
    assert ref_total > 0
    for cap in (0, ref_total):
        job_out = torch.zeros(J * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device="cuda")
        recs = torch.zeros(max(cap, 1) * DELTA_DT.itemsize, dtype=torch.uint8, device="cuda")
        n = torch.zeros(1, dtype=torch.int64, device="cuda")
        ospf_rib.third_area_delta_device(ctx, t.table, J, pl.rplanes.rs, [x.data_ptr() for x in pl.dc], None,
                                         [x.data_ptr() for x in pl.de], [x.data_ptr() for x in pl.des],
                                         base.data_ptr(), 1, 0, job_out.data_ptr(), recs.data_ptr() if cap else 0, cap,
                                         n.data_ptr())
        ctx.sync()
        assert job_out.cpu().numpy().view(DELTA_JOB_DT).tobytes() == ref_jobs.tobytes()
        assert int(n.cpu().item()) == ref_total
        if cap:
            assert recs.cpu().numpy().view(DELTA_DT)[:ref_total].tobytes() == ref_recs.tobytes()


def test_status_words_propagate(ctx, abr_harness, abr_backbone_harness, entries_harness, harness):
    """A B row out of range reaches the C's entries status (HSPF_JS_INVALID), which reaches R's job status; a C cell
    status word too.  Refused jobs get empty cells, the others are unchanged."""
    import torch
    t = SynthThirdArea(1, n_c=2, k=2)
    pl = Pipeline(ctx, abr_harness, abr_backbone_harness, entries_harness, harness, t, synth_jobs(t, 4, 1), False)
    J, P = pl.J, t.table.n_prefixes
    c = t.cs[0]
    assert c.table.n_asbr_slots
    rows = []
    for d in t.doms:
        r1 = np.repeat(np.arange(J, dtype=np.uint32)[:, None], len(d.areas), 1)
        r1[2, :] = J + 5                                                 # every B's row of job 2 out of range
        rows.append(dev(r1))
    bargs = border_args(pl.keep[0], rows, J)
    cp = pl.keep[2]
    ospf_rib.abr_backbone_asbr_entries_device(ctx, c.table, J, [p.rs for p in cp], *bargs, pl.des[0].data_ptr(),
                                              pl.de[0].data_ptr())
    cst = np.zeros(J, np.uint32)
    cst[4] = 0x2
    dcst = dev(cst)
    out = torch.zeros(J * P * 24, dtype=torch.uint8, device="cuda")
    st = torch.zeros(J, dtype=torch.int32, device="cuda")
    pl.cells(ctx, st.data_ptr(), out.data_ptr(), cstatus=[0, dcst.data_ptr()])
    ctx.sync()
    sw = st.cpu().numpy().view(np.uint32)
    est = pl.des[0].cpu().numpy().view(np.uint32)[:J]
    assert est[2] & capi.JS_INVALID and sw[2] & capi.JS_INVALID and sw[4] == 0x2
    G = len(c.table.asbr_ids)
    assert (pl.de[0].cpu().numpy().view(np.uint32)[2 * G: 3 * G] == 0xFFFFFFFF).all()
    got = out.cpu().numpy().view(ospf_rib.RIB_CELL_DT).reshape(J, P)
    bad = [j for j in range(J) if sw[j]]
    assert set(bad) == {2, 4}
    for j in bad:
        assert (got["winner"][j] == ospf_rib.NO_RECORD).all() and not got["mpf"][j].any()
    keep = [j for j in range(J) if j not in bad]
    assert got[keep].tobytes() == pl.want[keep].tobytes()


def test_zero_jobs_launch_nothing(ctx, abr_harness, abr_backbone_harness, entries_harness, harness):
    import torch
    t = SynthThirdArea(0, n_c=2, k=2)
    pl = Pipeline(ctx, abr_harness, abr_backbone_harness, entries_harness, harness, t, synth_jobs(t, 2, 0), False)
    out = torch.zeros(24, dtype=torch.uint8, device="cuda")
    before = ctx.launch_count
    pl.cells(ctx, 0, out.data_ptr(), n_jobs=0)
    c = t.cs[0]
    ospf_rib.abr_backbone_asbr_entries_device(ctx, c.table, 0, [p.rs for p in pl.keep[2]], *pl.bargs, 0,
                                              pl.de[0].data_ptr())
    ctx.sync()
    assert ctx.launch_count == before


def test_backbone_calls_refuse_the_table(ctx, abr_harness, abr_backbone_harness, entries_harness, harness):
    """The plain and asbr backbone calls refuse an OSPFv3 third-area table, with or without chain slots, before any
    launch; the OSPFv2 entries call refuses an OSPFv3 C table.  Without chain slots the third-area call runs with NULL
    entries; with them it needs the entries."""
    import torch
    for k in (0, 2):
        t = SynthThirdArea(2 if k == 0 else 0, n_c=2, k=k)
        assert (t.table.n_asbr_slots > 0) == (k > 0)
        pl = Pipeline(ctx, abr_harness, abr_backbone_harness, entries_harness, harness, t, synth_jobs(t, 3, 0), False)
        J, P = pl.J, t.table.n_prefixes
        out = torch.zeros(J * P * 24, dtype=torch.uint8, device="cuda")
        before = ctx.launch_count
        for call in (lambda: ospf_rib.backbone_cells_device(ctx, t.table, J, pl.rplanes.rs,
                                                            [x.data_ptr() for x in pl.dc], None, 0, out.data_ptr()),
                     lambda: ospf_rib.backbone_asbr_cells_device(ctx, t.table, J, pl.rplanes.rs,
                                                                 [x.data_ptr() for x in pl.dc], None, None, None, None,
                                                                 0, out.data_ptr())):
            with pytest.raises(capi.HspfError) as e:
                call()
            assert e.value.code == capi.HSPF_E_INVAL
        planes = ospf_rib._planes_array([p.rs for p in pl.keep[2]])
        assert ctx.lib.hspf_ospfv2_abr_backbone_asbr_entries(ctx.handle, t.cs[0].table.handle, J, planes, None, None,
                                                             None, None, pl.de[0].data_ptr()) == capi.HSPF_E_INVAL
        if k:
            with pytest.raises(capi.HspfError) as e:                       # chain slots without entries
                pl.cells(ctx, 0, out.data_ptr(), entries=False)
            assert e.value.code == capi.HSPF_E_INVAL
        assert ctx.launch_count == before
        if not k:
            ospf_rib.third_area_cells_device(ctx, t.table, J, pl.rplanes.rs, [x.data_ptr() for x in pl.dc], None,
                                             None, None, 0, out.data_ptr())
            ctx.sync()
            assert out.cpu().numpy().view(ospf_rib.RIB_CELL_DT).reshape(J, P).tobytes() == pl.want.tobytes()


def test_golden_domain_on_the_device(ctx, abr_harness, abr_backbone_harness, entries_harness, harness):
    import torch
    t = golden(*GOLDEN[0])[0]
    jobs = [t.job_overrides((), 0)]
    pl = Pipeline(ctx, abr_harness, abr_backbone_harness, entries_harness, harness, t, jobs, False)
    pl.check_borders()
    J, P = pl.J, t.table.n_prefixes
    out = torch.zeros(max(J * P * 24, 24), dtype=torch.uint8, device="cuda")
    ospf_rib.third_area_cells_device(ctx, t.table, J, pl.rplanes.rs, [x.data_ptr() for x in pl.dc], None, None, None,
                                     0, out.data_ptr())
    ctx.sync()
    got = out.cpu().numpy()[: J * P * 24].view(ospf_rib.RIB_CELL_DT).reshape(J, P)
    assert got.tobytes() == pl.want.tobytes()
    same_rib(t.decode(got[0]), t.affected(t.host_full([pl.bp[0][0]])))


@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_full_device_chain(ctx, abr_harness, abr_backbone_harness, entries_harness, harness, narrow_planes):
    """The B's SPT batches (one row per job in area 1) and ABR cells, each C's row 0, abr_backbone cells and entries,
    and R's row 0 and cells, all on the device; each stage equals its CPU harness over the planes read back."""
    import torch
    t = SynthThirdArea(0, n_c=3, k=2)
    assert t.table.n_asbr_slots > 0
    jobs = synth_jobs(t, 12, 0)
    J, P = len(jobs), t.table.n_prefixes
    tops, rows, bcells = [], [], []
    for b, d in enumerate(t.doms):
        d.rt.upload(ctx)
        i1 = d.rt.area_ids.index(1)
        tb = []
        for i, (f, rv) in enumerate(zip(d.flats, d.rv)):
            ov = [job[b].get(i, []) for job in jobs] if i == i1 else [[]]
            top = DeviceTopology(ctx, f.csr, rv, len(ov), ov, narrow_planes)
            top.run()
            tb.append(top)
        r = np.zeros((J, len(d.areas)), np.uint32)
        r[:, i1] = np.arange(J)
        dr = dev(r)
        c = torch.zeros(J * d.rt.n_prefixes * 24, dtype=torch.uint8, device="cuda")
        ospf_rib.abr_rib_cells_device(ctx, d.rt, J, [x.rs for x in tb], [x.n for x in tb], dr.data_ptr(), c.data_ptr())
        tops.append(tb); rows.append(dr); bcells.append(c)
    bargs = ([[x.rs for x in tb] for tb in tops], [[x.n for x in tb] for tb in tops], [r.data_ptr() for r in rows])
    ctops, dc, de, des = [], [], [], []
    for c in t.cs:
        c.table.upload(ctx)
        ct = [DeviceTopology(ctx, f.csr, rv, 1, [[]], narrow_planes) for f, rv in zip(c.r.flats, c.r.rv)]
        for x in ct:
            x.run()
        G = len(c.table.asbr_ids)
        out = torch.zeros(J * c.table.n_prefixes * 24, dtype=torch.uint8, device="cuda")
        ospf_rib.abr_backbone_cells_device(ctx, c.table, J, [x.rs for x in ct], [x.data_ptr() for x in bcells], None,
                                           *bargs, 0, out.data_ptr())
        ent = torch.zeros(max(J * G, 1), dtype=torch.int32, device="cuda")
        est = torch.full((J,), 7, dtype=torch.int32, device="cuda")
        ospf_rib.abr_backbone_asbr_entries_device(ctx, c.table, J, [x.rs for x in ct], *bargs, est.data_ptr(),
                                                  ent.data_ptr())
        ctops.append(ct); dc.append(out); de.append(ent); des.append(est)
    rtop = DeviceTopology(ctx, t.flat.csr, t.rv, 1, [[]], narrow_planes)
    rtop.run()
    t.table.upload(ctx)
    out = torch.zeros(J * P * 24, dtype=torch.uint8, device="cuda")
    st = torch.full((J,), 7, dtype=torch.int32, device="cuda")
    ospf_rib.third_area_cells_device(ctx, t.table, J, rtop.rs, [x.data_ptr() for x in dc], None,
                                     [x.data_ptr() for x in de], [x.data_ptr() for x in des], st.data_ptr(),
                                     out.data_ptr())
    ctx.sync()
    assert not st.cpu().numpy().any() and not any(x.cpu().numpy().any() for x in des)
    # the planes read back are the oracle's, and each stage equals its harness over them
    bp = [[[tb[i].planes(j if tb[i].n > 1 else 0) for i in range(len(tb))] for j in range(J)] for tb in tops]
    for c, ct in zip(t.cs, ctops):
        assert all(x.planes(0)[0].tobytes() == p[0].tobytes() for x, p in zip(ct, c.planes))
    assert rtop.planes(0)[0].tobytes() == t.planes[0].tobytes()
    for b, d in enumerate(t.doms):
        want_b = np.stack([d.cells(abr_harness, bp[b][j], narrow_planes)[0] for j in range(J)])
        assert bcells[b].cpu().numpy().tobytes() == want_b.tobytes()
    want, wst, ccells, cents, _ = t.run(abr_harness, abr_backbone_harness, entries_harness, harness, jobs,
                                        narrow_planes, bp=bp)
    assert not wst.any()
    for c, x, e, wc, we in zip(t.cs, dc, de, ccells, cents):
        G = len(c.table.asbr_ids)
        assert x.cpu().numpy().tobytes() == wc.tobytes()
        assert e.cpu().numpy().view(np.uint32)[: J * G].tobytes() == we.tobytes()
    got = out.cpu().numpy().view(ospf_rib.RIB_CELL_DT).reshape(J, P)
    assert got.tobytes() == want.tobytes()
    for j in range(J):
        same_rib(t.decode(got[j]), t.affected(t.host_full([bp[b][j] for b in range(len(t.doms))])))
    assert (got != got[0]).any()
