"""CPU: the OSPFv2 backbone-router stage with the borders' type-4 LSAs re-originated per job
(hspf_ospfv2_backbone_asbr_table_create, ospf_backbone_cell_eval with kAsbr).

The walk is compiled with kAsbr into a test harness and run on the CPU over the oracle's SPT planes: R's area-0 row,
each border's routing-table cells of the job and each border's area planes of the job, which the type-4 slots read.
Every job, decoded by hspf_ospfv2_backbone_from_cells, must equal byte for byte the host chain: each border's
update_rib_full over its job planes, its router tables and net_summaries into area 0, BOTH type-3 and type-4 output
spliced into R's LSDB in LsaKey order in place of the border's own, then update_rib_full at R, restricted to the
affected prefixes.  No recorded conformance data holds a type-4 or type-5 LSA, so that chain is the contract here."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from holo_b200 import capi, ospf_rib, ospfv2, synth
from holo_b200.route_table import DELTA_METRIC, DELTA_NEXTHOPS
from test_ospf_abr_rib_cells import Domain, narrow, planes_of
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospf_backbone_cells import GOLDEN, Backbone, SynthBackbone, non_backbone_links, summaries_of, synth_jobs
from test_ospf_backbone_cells import harness as bb_harness  # noqa: F401  (fixture)
from test_ospf_rib_cells import same_rib
from test_ospf_rib_delta import classify

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    out = tmp_path_factory.mktemp("harness") / "libospf_backbone_asbr_cells_harness.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                    "-o", str(out), str(ROOT / "tests" / "native" / "ospf_backbone_asbr_cells_harness.cc")], check=True)
    lib = C.CDLL(str(out))
    for fn in (lib.harness_ospf_backbone_asbr_cells, lib.harness_ospf_backbone_asbr_cells16):
        fn.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 8
    return lib


def asbr_cells(harness, table, planes, bcells, bplanes, narrow_planes=False, status=None, root_status=0, rows=None,
               pstatus=None):
    """Cells [J, P] and status words of the kAsbr walk.  bcells[b]: border b's cells [J, K_b]; bplanes[b][j][i]: its
    planes of area i in job j (row j of each area, unless `rows` [b] gives [J, n_areas] rows)."""
    J = len(bcells[0])
    pl = narrow(planes) if narrow_planes else planes
    keep = [np.ascontiguousarray(x) for x in pl] + list(bcells)
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
    keep += [dists, pss]
    cells = np.zeros((J, table.n_prefixes), ospf_rib.RIB_CELL_DT)
    out = np.zeros(J, np.uint32)
    fn = harness.harness_ospf_backbone_asbr_cells16 if narrow_planes else harness.harness_ospf_backbone_asbr_cells
    fn(table.handle, J, keep[0].ctypes.data, keep[1].ctypes.data, keep[2].ctypes.data, root_status, bc, st,
       (C.c_void_p * len(dists))(*[C.addressof(x) for x in dists]),
       (C.c_void_p * len(pss))(*[C.addressof(x) for x in pss]) if pstatus is not None else None,
       (C.c_void_p * len(nrs))(*nrs), (C.c_void_p * len(rws))(*rws), cells.ctypes.data, out.ctypes.data)
    return cells, out


class AsbrBackbone(Backbone):
    """ospfv2.backbone_view with area-1 ASBRs: R, three borders of area 1 (those in `use` given to the table; a border
    left out keeps its type-3 / type-4 LSAs as static records), an area-0 ASBR and k area-1 ASBRs."""

    def __init__(self, seed, k=2, n_ext=4, use=(0, 1, 2), V0=30, E0=90, V1=25, E1=70, max_paths=16):
        t0 = synth.random_topology(V0, E0, synth.SEED_BASE + 900 + 2 * seed, cost_choices=[5, 10, 20])
        t1 = synth.random_topology(V1, E1, synth.SEED_BASE + 901 + 2 * seed, cost_choices=[5, 10, 20])
        v = ospfv2.backbone_view(t0, t1, seed, max_paths=max_paths, area1_asbrs=k, area1_ext=n_ext)
        self.view = v
        self.area, self.summaries, self.externals = v["r_area"], v["summaries0"], v["externals"]
        self.flat = ospfv2.Flat(self.area)
        self.rv = self.flat.router_vertex(self.area.router_id)
        self.doms = [Domain(areas, sums, self.externals) for b, (areas, _ids, sums) in enumerate(v["borders"]) if b in use]
        self.cfgs = [[ospf_rib.area_config()] * 2 for _ in self.doms]
        self.table = ospf_rib.BackboneTable(self.flat, self.area.router_id, self.summaries, self.externals,
                                            [d.rt for d in self.doms], asbr=True)
        self.planes = planes_of(self.flat.csr, self.rv)

    def cells(self, abr, harness, bplanes, narrow_planes=False, status=None, root_status=0):
        bcells = [np.stack([d.cells(abr, p, narrow_planes)[0] for p in bp]) for d, bp in zip(self.doms, bplanes)]
        cells, out = asbr_cells(harness, self.table, self.planes, bcells, bplanes, narrow_planes, status, root_status)
        return cells, out, bcells

    def host(self, job_planes_per_border):
        """The chain with each border's type-3 and type-4 LSAs re-originated."""
        bid = {d.areas[0].router_id for d in self.doms}
        new = [s for s in self.summaries if not (int(s["adv_rtr"]) in bid and s["lsa_type"] in (3, 4))]
        for d, cfg, p in zip(self.doms, self.cfgs, job_planes_per_border):
            i0 = next(i for i, a in enumerate(d.areas) if a.area_id == 0)
            new += list(summaries_of(d, cfg, p, i0))
        s = np.array(new, ospf_rib.SUMMARY_LSA_DT)
        s = s[np.lexsort((s["lsa_id"], s["adv_rtr"], s["lsa_type"]))]
        p = self.planes
        spf = ospfv2.area_from_planes(self.area, lambda csr, root, nhw: (p[0], p[1], np.pad(p[2][:, None], ((0, 0), (0, nhw - 1)))))
        ra = [ospf_rib.RibArea(0, spf, self.area.ifaces, s, True)]
        return self.affected(ospf_rib.update_rib_full(self.area.router_id, self.area.max_paths, ra, self.externals))

    def asbr_links(self, x):
        return [l for l in non_backbone_links(self) if x in l]

    def cut(self, x, borders=None):
        """A job: every area-1 link of router x disabled in the area planes of the borders in `borders` (all: None)."""
        ovs = [self.job_overrides(l, capi.COST_DISABLED) for l in self.asbr_links(x)]
        out = []
        for b in range(len(self.doms)):
            m = {} if borders is not None and b not in borders else \
                {i: e for i in range(2) if (e := sum((o[b].get(i, []) for o in ovs), []))}
            out.append(m)
        return out

    def ext_prefixes(self, x):
        """Table indices of the prefixes router x advertises as type-5."""
        e = self.externals[self.externals["adv_rtr"] == x]
        return [u for u, (p, l) in enumerate(zip(self.table.prefix, self.table.plen))
                if any(int(y["lsa_id"]) == int(p) and bin(int(y["mask"])).count("1") == int(l) for y in e)]


def ext_path(cells):
    return (ospf_rib.cell_path(cells) >= ospf_rib.PATH_TYPE1) & ((ospf_rib.cell_flags(cells) & 1) != 0)


# ------------------------------------------------------------------------------------------- the chain
@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_generated_domains_chain(abr_harness, harness, seed, narrow_planes):
    """Every area-1 link failed and re-costed, one job each, all in one batch; the externals of the area-1 ASBRs
    are affected prefixes and route through the borders' type-4 slots."""
    bb = AsbrBackbone(seed)
    assert bb.table.n_asbr_slots > 0 and 1 <= bb.table.n_asbr_sets <= 3
    links = non_backbone_links(bb)
    jobs = [bb.job_overrides((), 0)]
    for link in links:
        jobs += [bb.job_overrides(link, capi.COST_DISABLED), bb.job_overrides(link, 37)]
    cells = bb.check(abr_harness, harness, jobs, narrow_planes)
    for x in bb.view["area1_asbrs"]:
        u = bb.ext_prefixes(x)
        assert u and ext_path(cells[0][u]).any()
    assert (cells != cells[0]).any()


def test_asbr_cut_off_from_the_last_border_moves_to_an_earlier_one(abr_harness, harness):
    """Only the last border in LsaKey order loses the ASBR: R's entry is the previous border's slot (walked from the
    end), which need not be the cheapest; every external of the ASBR still routes, through the other borders."""
    n = 0
    for seed in range(3):
        bb = AsbrBackbone(seed)
        last = max(range(3), key=lambda b: bb.doms[b].areas[0].router_id)
        for x in bb.view["area1_asbrs"]:
            cells = bb.check(abr_harness, harness, [bb.job_overrides((), 0), bb.cut(x, {last})])
            u = [k for k in bb.ext_prefixes(x) if ext_path(cells[0][k:k + 1])[0]]
            assert ext_path(cells[1][u]).all()
            n += int(cells[1][u].tobytes() != cells[0][u].tobytes())
    assert n > 0


def test_asbr_cut_off_from_every_border_is_lost_then_gained(abr_harness, harness):
    bb = AsbrBackbone(0)
    x = bb.view["area1_asbrs"][0]
    jobs = [bb.job_overrides((), 0), bb.cut(x), bb.job_overrides((), 0)]
    cells = bb.check(abr_harness, harness, jobs)
    k = classify(cells[1], cells[0])
    assert (k == 1).any()                                              # LOST
    assert (classify(cells[2], cells[1])[k == 1] == 2).all()           # GAINED
    assert cells[2].tobytes() == cells[0].tobytes()


def test_shared_external_flips_between_area0_and_area1_asbr(abr_harness, harness):
    """0x0E0A0000/24 is type-2 at metric 12 from the area-0 ASBR and from each area-1 ASBR: the forwarding metric
    decides, and cutting the area-1 ASBRs hands the route to the area-0 one (or back)."""
    flips = 0
    for seed in range(3):
        bb = AsbrBackbone(seed)
        u = int(np.nonzero((bb.table.prefix == 0x0E0A0000) & (bb.table.plen == 24))[0][0])
        cut_all = [{i: e for i in range(2) if (e := sum((bb.cut(x)[b].get(i, []) for x in bb.view["area1_asbrs"]), []))}
                   for b in range(3)]
        jobs = [bb.job_overrides((), 0), cut_all] + synth_jobs(bb, 8, seed)[1:]
        cells = bb.check(abr_harness, harness, jobs)
        flips += len({int(c["nh_mask"]) for c in cells[:, u]}) > 1
    assert flips > 0


def test_type1_and_type2_moves_show_as_metric_and_nexthops(abr_harness, harness):
    """A moved forwarding metric changes a type-1 external's metric (METRIC) and a type-2's next hops only; an entry
    that moves to another border at the same distance changes next hops (NEXTHOPS)."""
    kinds, types = 0, set()
    for seed in range(3):
        bb = AsbrBackbone(seed)
        cells = bb.check(abr_harness, harness, synth_jobs(bb, 12, seed))
        for x in bb.view["area1_asbrs"]:
            u = bb.ext_prefixes(x)
            types |= {int(p) for p in ospf_rib.cell_path(cells[0][u])}
            k = np.stack([classify(cells[j][u], cells[0][u]) for j in range(1, len(cells))])
            kinds |= int(np.bitwise_or.reduce(k, axis=None))
    assert {ospf_rib.PATH_TYPE1, ospf_rib.PATH_TYPE2} <= types
    assert kinds & DELTA_METRIC and kinds & DELTA_NEXTHOPS


def test_static_type4_of_another_abr_sits_at_its_lsakey_position(abr_harness, harness):
    """The middle border left out of the table: its type-4 LSAs stay static records between the two borders' slots,
    and the walk from the end reaches it after the last border's slot."""
    for seed in range(3):
        bb = AsbrBackbone(seed, use=(0, 2))
        mid = bb.view["borders"][1][0][0].router_id
        assert ((bb.summaries["adv_rtr"] == mid) & (bb.summaries["lsa_type"] == 4)).any()
        jobs = [bb.job_overrides((), 0)] + [bb.cut(x, {1}) for x in bb.view["area1_asbrs"]] + synth_jobs(bb, 6, seed)[1:]
        bb.check(abr_harness, harness, jobs)


# ------------------------------------------------------------------------------------------- refusals
def test_table_refusals():
    bb = AsbrBackbone(0)
    mk = lambda sums=bb.summaries, borders=None, ext=bb.externals: ospf_rib.BackboneTable(
        bb.flat, bb.area.router_id, sums, ext, borders or [d.rt for d in bb.doms], asbr=True)
    # the existing create still refuses the borders' type-4 LSAs
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.BackboneTable(bb.flat, bb.area.router_id, bb.summaries, bb.externals, [d.rt for d in bb.doms])
    assert e.value.code == capi.HSPF_E_UNSUPPORTED
    # a border's type-4 LSA for a router its table cannot originate for
    b0 = bb.doms[0].areas[0].router_id
    bad = np.concatenate([bb.summaries, np.array([(b0, 0x09090909, 0, 5, 4, 0, (0, 0))], ospf_rib.SUMMARY_LSA_DT)])
    bad = bad[np.lexsort((bad["lsa_id"], bad["adv_rtr"], bad["lsa_type"]))]
    with pytest.raises(capi.HspfError) as e:
        mk(sums=bad)
    assert e.value.code == capi.HSPF_E_INVAL
    dead = bad.copy()
    dead["maxage"][dead["lsa_id"] == 0x09090909] = 1
    mk(sums=dead)
    # an E-flag router of a border's area with the B flag
    x = bb.view["area1_asbrs"][0]
    doms = []
    for d in bb.doms:
        areas = [ospfv2._set_flags(ospfv2.Ospfv2Area(**{k: getattr(a, k) for k in a.__dataclass_fields__}), {x: 0x01})
                 if a.area_id != 0 else a for a in d.areas]
        doms.append(Domain(areas, d.summaries, d.externals))
    with pytest.raises(capi.HspfError) as e:
        mk(borders=[d.rt for d in doms])
    assert e.value.code == capi.HSPF_E_UNSUPPORTED


def with_twins(d, n):
    """Border domain d with n copies of its non-backbone area added as areas 2, 3, ...: the area-1 ASBRs are E-flag
    routers in each, one (border, area) plane set apiece."""
    i1 = [i for i, a in enumerate(d.areas) if a.area_id != 0][0]
    twins = []
    for k in range(n):
        t = ospfv2.Ospfv2Area(**{f: getattr(d.areas[i1], f) for f in d.areas[i1].__dataclass_fields__})
        t.area_id = 2 + k
        twins.append(t)
    return Domain(d.areas + twins, list(d.summaries) + [np.zeros(0, ospf_rib.SUMMARY_LSA_DT)] * n, d.externals)


def test_more_than_8_plane_sets_are_refused():
    """Every slot of a border reads the plane set of its (border, area); three borders with three non-backbone areas
    each would read nine."""
    bb = AsbrBackbone(0)
    mk = lambda doms: ospf_rib.BackboneTable(bb.flat, bb.area.router_id, bb.summaries, bb.externals,
                                             [d.rt for d in doms], asbr=True)
    t = mk([with_twins(bb.doms[0], 1)] + bb.doms[1:])
    assert t.n_asbr_sets == 4 and t.n_asbr_slots > 0
    with pytest.raises(capi.HspfError) as e:
        mk([with_twins(d, 2) for d in bb.doms])
    assert e.value.code == capi.HSPF_E_UNSUPPORTED


def test_existing_walk_on_a_table_without_type4_slots(abr_harness, harness, bb_harness):
    """On the golden Backbone cases and SynthBackbone, the asbr create gives the table of the existing create and the
    kAsbr walk gives the existing harness's cells byte for byte."""
    for g in GOLDEN[:4]:
        bb = Backbone(*g)
        t = ospf_rib.BackboneTable(bb.flat, bb.area.router_id, bb.summaries, bb.externals, [d.rt for d in bb.doms],
                                   asbr=True)
        assert (t.n_asbr_slots, t.n_asbr_sets, t.n_prefixes, t.n_records) == (0, 0, bb.table.n_prefixes, bb.table.n_records)
        bp = bb.border_planes([bb.job_overrides((), 0)] + [bb.job_overrides(l, capi.COST_DISABLED)
                                                            for l in non_backbone_links(bb)[:4]])
        want, _, bcells = Backbone.cells(bb, abr_harness, bb_harness, bp)
        got, _ = asbr_cells(harness, t, bb.planes, bcells, bp)
        assert got.tobytes() == want.tobytes()
    bb = SynthBackbone(1)
    bp = bb.border_planes(synth_jobs(bb, 6, 1))
    for narrow_planes in (False, True):
        want, _, bcells = bb.cells(abr_harness, bb_harness, bp, narrow_planes)
        t = ospf_rib.BackboneTable(bb.flat, bb.area.router_id, bb.summaries, bb.externals, [d.rt for d in bb.doms],
                                   asbr=True)
        got, _ = asbr_cells(harness, t, bb.planes, bcells, bp, narrow_planes)
        assert got.tobytes() == want.tobytes()


def test_job_status_rows(abr_harness, harness):
    """A border row out of range refuses the job (HSPF_JS_INVALID, empty cells); a read row's status word is ORed in;
    the other jobs are unchanged."""
    bb = AsbrBackbone(1)
    jobs = synth_jobs(bb, 3, 1)
    bp = bb.border_planes(jobs)
    want, st, bcells = bb.cells(abr_harness, harness, bp)
    assert not st.any()
    J = len(jobs)
    rows = [np.repeat(np.arange(J, dtype=np.uint32)[:, None], 2, 1) for _ in range(3)]
    rows[1][2, :] = J                                                  # out of range
    ps = [[np.zeros(J, np.uint32) for _ in range(2)] for _ in range(3)]
    ps[0][0][1] = ps[0][1][1] = 0x8
    got, st = asbr_cells(harness, bb.table, bb.planes, bcells, bp, rows=rows, pstatus=ps)
    assert st[2] & capi.JS_INVALID and st[1] == 0x8
    for j in (1, 2):
        assert (got["winner"][j] == ospf_rib.NO_RECORD).all() and not got["mpf"][j].any()
    keep = [j for j in range(J) if j not in (1, 2)]
    assert got[keep].tobytes() == want[keep].tobytes()
