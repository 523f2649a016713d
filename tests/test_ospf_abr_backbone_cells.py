"""CPU: the OSPFv2 area-border-router stage over what-if jobs inside an area the router is not attached to
(hspf_ospfv2_abr_backbone_*, abr_rib_cell_eval with kSlots).

The walk is compiled with kSlots into a test harness and run on the CPU over the oracle's SPT planes: R's row 0 of
each of its areas, each border's routing-table cells of the job and each border's area planes of the job, which the
type-4 slots read.  Every job, decoded by hspf_ospfv2_abr_backbone_from_cells, must equal the host chain: each
border's update_rib_full over its job planes, its net_summaries into area 0 spliced into area 0's type-3/4 LSAs in
place of its own, then R's update_rib_full over its areas' row-0 images, restricted to the affected prefixes."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import golden_util as gu
from holo_b200 import capi, ospf_rib, ospfv2, synth
from test_ospf_abr_rib_cells import Domain, golden_domain, narrow, planes_of
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospf_backbone_cells import Backbone, configs_of, non_backbone_links, snap, summaries_of, synth_jobs
from test_ospf_rib_cells import same_rib
from test_ospf_rib_delta import classify
from test_ospfv2_route_cells import gather_for

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    out = tmp_path_factory.mktemp("harness") / "libospf_abr_backbone_cells_harness.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                    "-o", str(out), str(ROOT / "tests" / "native" / "ospf_abr_backbone_cells_harness.cc")], check=True)
    lib = C.CDLL(str(out))
    for fn in (lib.harness_ospf_abr_backbone_cells, lib.harness_ospf_abr_backbone_cells16):
        fn.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 12
    return lib


def abr_backbone_cells(harness, table, planes, bcells, bplanes, narrow_planes=False, status=None, root_status=None,
                       rows=None, pstatus=None):
    """Cells [J, P] and status words of the kSlots walk.  planes[i]: R's row 0 of area i; bcells[b]: border b's cells
    [J, K_b]; bplanes[b][j][i]: its planes of area i in job j (row j of each area, unless `rows` [b] gives [J, n_areas]
    rows)."""
    J = len(bcells[0])
    pl = [narrow(p) if narrow_planes else p for p in planes]
    keep = [[np.ascontiguousarray(x) for x in p] for p in pl] + list(bcells)
    arr = lambda k: (C.c_void_p * len(pl))(*[keep[i][k].ctypes.data for i in range(len(pl))])
    rs = np.ascontiguousarray(root_status, np.uint32) if root_status is not None else None
    bc = (C.c_void_p * len(bcells))(*[c.ctypes.data for c in bcells])
    st = None
    if status is not None:
        sk = [np.ascontiguousarray(x, np.uint32) for x in status]
        keep += sk
        st = (C.c_void_p * len(sk))(*[x.ctypes.data for x in sk])
    dists, nrs, rws, pss = [], [], [], []
    for b, bp in enumerate(bplanes):
        A = len(bp[0])
        d = [np.ascontiguousarray(np.stack([(narrow(bp[j][i]) if narrow_planes else bp[j][i])[0] for j in range(J)]))
             for i in range(A)]
        keep += d
        dists.append((C.c_void_p * A)(*[x.ctypes.data for x in d]))
        nr = np.full(A, J, np.uint32)
        rw = np.ascontiguousarray(rows[b] if rows is not None else np.repeat(np.arange(J, dtype=np.uint32)[:, None], A, 1),
                                  np.uint32)
        keep += [nr, rw]
        nrs.append(nr.ctypes.data)
        rws.append(rw.ctypes.data)
        if pstatus is not None:
            ps = [np.ascontiguousarray(x, np.uint32) for x in pstatus[b]]
            keep += ps
            pss.append((C.c_void_p * A)(*[x.ctypes.data for x in ps]))
    keep += [dists, pss, rs]
    cells = np.zeros((J, table.n_prefixes), ospf_rib.RIB_CELL_DT)
    out = np.zeros(J, np.uint32)
    fn = harness.harness_ospf_abr_backbone_cells16 if narrow_planes else harness.harness_ospf_abr_backbone_cells
    fn(table.handle, J, arr(0), arr(1), arr(2), rs.ctypes.data if rs is not None else None, bc, st,
       (C.c_void_p * len(dists))(*[C.addressof(x) for x in dists]),
       (C.c_void_p * len(pss))(*[C.addressof(x) for x in pss]) if pstatus is not None else None,
       (C.c_void_p * len(nrs))(*nrs), (C.c_void_p * len(rws))(*rws), cells.ctypes.data, out.ctypes.data)
    return cells, out


class AbrBackbone(Backbone):
    """R's domain (its areas, area 0 first or not, their summaries and active flags), the borders' domains (each
    border's areas in its own order) and the table over them.  cut_border: R's area-0 row 0 with that border's area-0
    links cut (the border is unreachable from R)."""

    def __init__(self, r_dom, doms, cfgs=None, cut_border=None):
        self.r = r_dom
        self.doms = doms
        self.cfgs = cfgs if cfgs is not None else [[ospf_rib.area_config()] * len(d.areas) for d in doms]
        self.externals = r_dom.externals
        self.i0 = [a.area_id for a in r_dom.areas].index(0)
        self.table = ospf_rib.AbrBackboneTable(r_dom.areas[0].router_id, r_dom.flats, [a.area_id for a in r_dom.areas],
                                               r_dom.summaries, r_dom.active, r_dom.externals, [d.rt for d in doms])
        self.planes = r_dom.planes()
        if cut_border is not None:
            f = r_dom.flats[self.i0]
            b, c = f.router_vertex(doms[cut_border].areas[0].router_id), f.csr
            ov = [(e, capi.COST_DISABLED) for e in range(c.n_edges) if c.col[e] == b or c.row_ptr[b] <= e < c.row_ptr[b + 1]]
            self.planes[self.i0] = planes_of(f.csr, r_dom.rv[self.i0], ov)

    def cells(self, abr, harness, bplanes, narrow_planes=False, status=None, root_status=None, rows=None, pstatus=None):
        bcells = [np.stack([d.cells(abr, p, narrow_planes)[0] for p in bp]) for d, bp in zip(self.doms, bplanes)]
        cells, out = abr_backbone_cells(harness, self.table, self.planes, bcells, bplanes, narrow_planes, status,
                                        root_status, rows, pstatus)
        return cells, out, bcells

    def decode(self, cells):
        ga, gv, gn = [], [], []
        for i, (f, r, p) in enumerate(zip(self.r.flats, self.r.rv, self.planes)):
            v, n = gather_for(f, r, p)
            ga += [i] * len(v); gv += list(v); gn += list(n)
        return ospf_rib.abr_backbone_from_cells(self.r.areas, self.table, cells, ga, gv, gn)

    def host(self, job_planes_per_border):
        """The chain: each border's type-3 and type-4 LSAs re-originated into area 0, update_rib_full at R."""
        bid = {d.areas[0].router_id for d in self.doms}
        s0 = self.r.summaries[self.i0]
        new = [s for s in s0 if not (int(s["adv_rtr"]) in bid and s["lsa_type"] in (3, 4))]
        for d, cfg, p in zip(self.doms, self.cfgs, job_planes_per_border):
            new += list(summaries_of(d, cfg, p, [a.area_id for a in d.areas].index(0)))
        s = np.array(new, ospf_rib.SUMMARY_LSA_DT)
        s = s[np.lexsort((s["lsa_id"], s["adv_rtr"], s["lsa_type"]))]
        ra = []
        for i, (a, p) in enumerate(zip(self.r.areas, self.planes)):
            spf = ospfv2.area_from_planes(a, lambda csr, root, nhw, p=p: (p[0], p[1], np.pad(p[2][:, None], ((0, 0), (0, nhw - 1)))))
            ra.append(ospf_rib.RibArea(a.area_id, spf, a.ifaces, s if i == self.i0 else self.r.summaries[i],
                                       self.r.active[i]))
        return self.affected(ospf_rib.update_rib_full(self.r.areas[0].router_id, self.r.areas[0].max_paths, ra,
                                                      self.externals))

    def check(self, abr, harness, jobs, narrow_planes=False):
        bp = self.border_planes(jobs)
        cells, st, _ = self.cells(abr, harness, bp, narrow_planes)
        assert not st.any()
        for j in range(len(jobs)):
            same_rib(self.decode(cells[j]), self.host([bp[b][j] for b in range(len(self.doms))]))
        return cells


class SynthAbrBackbone(AbrBackbone):
    """ospfv2.abr_backbone_view: R an ABR of areas 0 and 2, three borders of area 1 (those in `use`), k area-1 ASBRs."""

    def __init__(self, seed, k=2, n_ext=4, use=(0, 1, 2), cut_border=None, max_paths=16):
        t0 = synth.random_topology(30, 90, synth.SEED_BASE + 950 + 3 * seed, cost_choices=[5, 10, 20])
        t1 = synth.random_topology(25, 70, synth.SEED_BASE + 951 + 3 * seed, cost_choices=[5, 10, 20])
        t2 = synth.random_topology(25, 70, synth.SEED_BASE + 952 + 3 * seed, cost_choices=[5, 10, 20])
        v = ospfv2.abr_backbone_view(t0, t1, t2, seed, max_paths=max_paths, area1_asbrs=k, area1_ext=n_ext)
        self.view = v
        r_dom = Domain(v["r_areas"], v["summaries"], v["externals"])
        doms = [Domain(areas, sums, v["externals"]) for b, (areas, _ids, sums) in enumerate(v["borders"]) if b in use]
        super().__init__(r_dom, doms, cut_border=cut_border)

    def index(self, prefix, mask):
        return int(np.nonzero((self.table.prefix == prefix) & (self.table.plen == bin(mask).count("1")))[0][0])


def present(cells):
    return (ospf_rib.cell_flags(cells) & 1) != 0


# ------------------------------------------------------------------------------------------------ goldens
# topo1-1/1-2/1-3: each ABR among rt2, rt4 and rt6 as R, each other one as the single border of its area
GOLDEN = [(t, r, b) for t in ("topo1-1", "topo1-2", "topo1-3") for r in ("rt2", "rt4", "rt6")
          for b in ("rt2", "rt4", "rt6") if b != r]
GIDS = [f"{t}-{r}-{b}" for t, r, b in GOLDEN]


def golden(topo, r, b):
    rs, bs = snap(topo, r), snap(topo, b)
    r_dom = golden_domain(rs)[0]
    bdom = golden_domain(bs)[0]
    return AbrBackbone(r_dom, [bdom], [configs_of(bs, bdom)]), rs


@pytest.mark.parametrize("g", GOLDEN, ids=GIDS)
def test_base_job_equals_the_recorded_local_rib(abr_harness, harness, g):
    bb, rs = golden(*g)
    assert bb.table.n_prefixes > 0 and bb.table.n_slots > 0
    cells = bb.check(abr_harness, harness, [bb.job_overrides((), 0)])
    got = bb.decode(cells[0])
    keys = gu.global_sort_keys(rs)
    key_name = {v: k for k, v in keys.items()}
    mine = {}
    for r in got.routes:
        nh = sorted(((key_name.get(i, "?"), gu.ipstr(a) if ha else None) for (i, ha, a, _hn, _n, _hl, _l) in got.nh(r)),
                    key=lambda x: (x[0] or "", x[1] or ""))
        mine[f"{gu.ipstr(r['prefix'])}/{bin(int(r['mask'])).count('1')}"] = (int(r["metric"]), ospf_rib.PATH_NAMES[int(r["path_type"])], nh)
    affected = {f"{gu.ipstr(int(p))}/{int(l)}" for p, l in zip(bb.table.prefix, bb.table.plen)}
    want = {k: v for k, v in gu.golden_rib(rs).items() if k in affected}
    norm = lambda d: {k: (v[0], v[1], [(a or "", b or "") for a, b in v[2]]) for k, v in d.items()}
    assert norm(mine) == norm(want)


@pytest.mark.parametrize("g", GOLDEN, ids=GIDS)
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_golden_chain_every_link_failed_and_recosted(abr_harness, harness, g, narrow_planes):
    bb, _ = golden(*g)
    jobs = [bb.job_overrides((), 0)]
    for link in non_backbone_links(bb):
        jobs += [bb.job_overrides(link, capi.COST_DISABLED), bb.job_overrides(link, 35)]
    assert len(jobs) > 1
    bb.check(abr_harness, harness, jobs, narrow_planes)


# ------------------------------------------------------------------------------------------- generated
@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_generated_domains_chain(abr_harness, harness, seed, narrow_planes):
    """Every area-1 link failed and re-costed, one job each, all in one batch."""
    bb = SynthAbrBackbone(seed)
    assert bb.table.n_asbr_slots > 0 and 1 <= bb.table.n_asbr_sets <= 3
    jobs = [bb.job_overrides((), 0)]
    for link in non_backbone_links(bb):
        jobs += [bb.job_overrides(link, capi.COST_DISABLED), bb.job_overrides(link, 37)]
    cells = bb.check(abr_harness, harness, jobs, narrow_planes)
    assert (cells != cells[0]).any()


def test_area2_intra_prefix_never_changes(abr_harness, harness):
    """An area-1 prefix that is also a stub of R's area 2: affected (the borders can advertise it), intra-area at R,
    the same cell in every job."""
    for seed in range(3):
        bb = SynthAbrBackbone(seed)
        u = bb.index(*bb.view["area2_shared"])
        cells = bb.check(abr_harness, harness, synth_jobs(bb, 10, seed))
        assert ospf_rib.cell_path(cells[0][u:u + 1])[0] == ospf_rib.PATH_INTRA and present(cells[0][u:u + 1])[0]
        assert (cells[:, u] == cells[0, u]).all()


def test_tied_borders_merge_atoms(abr_harness, harness):
    """Some inter-area route reaches R through two borders at one metric: its cell ORs their atoms."""
    n = 0
    for seed in range(3):
        bb = SynthAbrBackbone(seed)
        cells = bb.check(abr_harness, harness, synth_jobs(bb, 6, seed))
        inter = present(cells) & (ospf_rib.cell_path(cells) == ospf_rib.PATH_INTER)
        multi = np.vectorize(lambda m: bin(int(m)).count("1") > 1)(cells["nh_mask"])
        n += int((inter & multi & (cells["winner"] >= bb.table.n_records)).sum())
    assert n > 0


def test_lost_then_gained(abr_harness, harness):
    """A link cut that strands area-1 prefixes at every border makes them unreachable at R (LOST); the next job,
    unperturbed, has them back (GAINED)."""
    lost = 0
    for seed in range(3):
        bb = SynthAbrBackbone(seed)
        jobs = [bb.job_overrides((), 0)]
        for link in non_backbone_links(bb):
            jobs += [bb.job_overrides(link, capi.COST_DISABLED), bb.job_overrides((), 0)]
        cells = bb.check(abr_harness, harness, jobs)
        for j in range(1, len(jobs), 2):
            k = classify(cells[j], cells[0])
            if (k == 1).any():
                lost += 1
                assert (classify(cells[j + 1], cells[j])[k == 1] == 2).all()
    assert lost > 0


def test_external_through_area2_asbr_and_area1_asbr(abr_harness, harness):
    """0x0E0A0000/24 is advertised by the area-0 ASBR, each area-1 ASBR and the area-2 ASBR, whose intra-area entry
    in area 2 keeps it routed in every job; the area-2 ASBR's own /24 is not affected.  Cutting an area-1 ASBR off from
    the last border in LsaKey order moves R's entry to an earlier border's slot."""
    moved = 0
    for seed in range(3):
        bb = SynthAbrBackbone(seed)
        assert not ((bb.table.prefix == 0x0E0C0000) & (bb.table.plen == 24)).any()
        u = bb.index(0x0E0A0000, 0xFFFFFF00)
        last = max(range(3), key=lambda b: bb.doms[b].areas[0].router_id)
        jobs = [bb.job_overrides((), 0)] + [bb.cut(x, {last}) for x in bb.view["area1_asbrs"]]
        jobs += synth_jobs(bb, 6, seed)[1:]
        cells = bb.check(abr_harness, harness, jobs)
        assert present(cells[:, u]).all() and (ospf_rib.cell_path(cells[:, u]) >= ospf_rib.PATH_TYPE1).all()
        for j, x in enumerate(bb.view["area1_asbrs"], start=1):
            us = [k for k in bb.ext_prefixes(x) if present(cells[0][k:k + 1])[0]]
            moved += int(cells[j][us].tobytes() != cells[0][us].tobytes())
    assert moved > 0


def test_border_unreachable_from_r(abr_harness, harness):
    """A border R cannot reach in area 0: its slots offer nothing, whatever its cells; the other borders' still do."""
    for seed in range(2):
        bb = SynthAbrBackbone(seed, cut_border=1)
        bb.check(abr_harness, harness, synth_jobs(bb, 6, seed))


# SynthAbrBackbone borrows the asbr test's helpers for cutting ASBRs off and naming their externals
from test_ospf_backbone_asbr_cells import AsbrBackbone  # noqa: E402

SynthAbrBackbone.asbr_links = AsbrBackbone.asbr_links
SynthAbrBackbone.cut = AsbrBackbone.cut
SynthAbrBackbone.ext_prefixes = AsbrBackbone.ext_prefixes


# -------------------------------------------------------------------------------------------- refusals
def test_table_refusals():
    bb = SynthAbrBackbone(0)
    r = bb.r
    ids = [a.area_id for a in r.areas]

    def mk(router_id=r.areas[0].router_id, flats=r.flats, area_ids=ids, sums=r.summaries, active=r.active,
           borders=None):
        return ospf_rib.AbrBackboneTable(router_id, flats, area_ids, sums, active, r.externals,
                                         borders if borders is not None else [d.rt for d in bb.doms])

    def refused(code, **kw):
        with pytest.raises(capi.HspfError) as e:
            mk(**kw)
        assert e.value.code == code

    refused(capi.HSPF_E_INVAL, borders=[])                                    # no border
    refused(capi.HSPF_E_INVAL, borders=[bb.doms[0].rt] * 2)                  # a border twice
    refused(capi.HSPF_E_INVAL, area_ids=[5, 2])                               # no area 0
    refused(capi.HSPF_E_INVAL, active=[False, True])                          # area 0 inactive
    refused(capi.HSPF_E_INVAL, active=[True, False])                          # one active area
    # R without the B flag in its area-0 flat
    a0 = ospfv2.Ospfv2Area(**{k: getattr(r.areas[0], k) for k in r.areas[0].__dataclass_fields__})
    rl = a0.router_lsas.copy()
    rl["flags"][rl["adv_rtr"] == a0.router_id] &= np.uint8(0xFE)
    a0.router_lsas = rl
    refused(capi.HSPF_E_INVAL, flats=[ospfv2.Flat(a0), r.flats[1]])
    # R one of the borders: R's own ABR table given as a border
    refused(capi.HSPF_E_INVAL, borders=[bb.doms[0].rt, r.rt])
    # a border's type-3 LSA for a prefix it cannot advertise, a type-4 LSA for a router it cannot originate for
    b0 = bb.doms[0].areas[0].router_id
    for row in ((b0, 0x09090900, 0xFFFFFF00, 5, 3, 0, (0, 0)), (b0, 0x09090909, 0, 5, 4, 0, (0, 0))):
        s = np.concatenate([r.summaries[0], np.array([row], ospf_rib.SUMMARY_LSA_DT)])
        s = s[np.lexsort((s["lsa_id"], s["adv_rtr"], s["lsa_type"]))]
        refused(capi.HSPF_E_INVAL, sums=[s, r.summaries[1]])
    # a V-flag router in R's area 2 (the transit-area step)
    a2 = ospfv2._set_flags(ospfv2.Ospfv2Area(**{k: getattr(r.areas[1], k) for k in r.areas[1].__dataclass_fields__}),
                           {bb.view["area2_asbr"]: 0x04})
    refused(capi.HSPF_E_UNSUPPORTED, flats=[r.flats[0], ospfv2.Flat(a2)])
    # an E-flag router of a border's area with the B flag
    x = bb.view["area1_asbrs"][0]
    doms = []
    for d in bb.doms:
        areas = [ospfv2._set_flags(ospfv2.Ospfv2Area(**{k: getattr(a, k) for k in a.__dataclass_fields__}), {x: 0x01})
                 if a.area_id != 0 else a for a in d.areas]
        doms.append(Domain(areas, d.summaries, d.externals))
    refused(capi.HSPF_E_UNSUPPORTED, borders=[d.rt for d in doms])


def test_more_than_8_plane_sets_are_refused():
    from test_ospf_backbone_asbr_cells import with_twins
    bb = SynthAbrBackbone(0)
    r = bb.r
    mk = lambda doms: ospf_rib.AbrBackboneTable(r.areas[0].router_id, r.flats, [a.area_id for a in r.areas],
                                                r.summaries, r.active, r.externals, [d.rt for d in doms])
    assert mk([with_twins(bb.doms[0], 1)] + bb.doms[1:]).n_asbr_sets == 4
    with pytest.raises(capi.HspfError) as e:
        mk([with_twins(d, 2) for d in bb.doms])
    assert e.value.code == capi.HSPF_E_UNSUPPORTED


@pytest.mark.parametrize("topo", ["topo3-1", "topo3-3"])
def test_virtual_link_domains_are_refused(topo):
    """R = rt2 of a domain with a virtual link: the transit-area step is out of this stage."""
    r_dom = golden_domain(snap(topo, "rt2"))[0]
    others = [s["rt"] for s in gu.load_ospfv2() if s["topo"] == topo and s["rt"] != "rt2" and len(s["areas"]) > 1]
    assert others
    bdom = golden_domain(snap(topo, others[0]))[0]
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.AbrBackboneTable(r_dom.areas[0].router_id, r_dom.flats, [a.area_id for a in r_dom.areas],
                                  r_dom.summaries, r_dom.active, None, [bdom.rt])
    assert e.value.code == capi.HSPF_E_UNSUPPORTED


def test_job_status_rows(abr_harness, harness):
    """R's row-0 words, the borders' job words and the type-4 rows' words are ORed into a job's word, a type-4 row out
    of range gives HSPF_JS_INVALID, and a refused job gets empty cells; the other jobs are unchanged."""
    bb = SynthAbrBackbone(1)
    jobs = synth_jobs(bb, 3, 1)
    bp = bb.border_planes(jobs)
    want, st, bcells = bb.cells(abr_harness, harness, bp)
    assert not st.any()
    J = len(jobs)
    rows = [np.repeat(np.arange(J, dtype=np.uint32)[:, None], 2, 1) for _ in range(3)]
    rows[1][2, :] = J                                                    # out of range
    ps = [[np.zeros(J, np.uint32) for _ in range(2)] for _ in range(3)]
    ps[0][0][1] = ps[0][1][1] = 0x8
    bst = [np.zeros(J, np.uint32) for _ in range(3)]
    bst[2][3] = 0x2
    got, st = abr_backbone_cells(harness, bb.table, bb.planes, bcells, bp, status=bst, rows=rows, pstatus=ps)
    assert st[2] & capi.JS_INVALID and st[1] == 0x8 and st[3] == 0x2
    for j in (1, 2, 3):
        assert (got["winner"][j] == ospf_rib.NO_RECORD).all() and not got["mpf"][j].any()
    keep = [j for j in range(J) if j not in (1, 2, 3)]
    assert got[keep].tobytes() == want[keep].tobytes()
    got, st = abr_backbone_cells(harness, bb.table, bb.planes, bcells, bp, root_status=[0, 0x4])
    assert (st == 0x4).all() and (got["winner"] == ospf_rib.NO_RECORD).all()
