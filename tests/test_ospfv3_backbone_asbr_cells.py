"""CPU: the OSPFv3 backbone-router stage with the borders' Inter-Area-Router LSAs re-originated per job
(hspf_ospfv3_backbone_asbr_table_create, ospf_backbone_cell_eval with kV3 and kAsbr).

The walk is compiled into a test harness and run on the CPU over the oracle's SPT planes: R's area-0 row, each border's
routing-table cells of the job and each border's area planes of the job, which the Inter-Area-Router slots read.  Every
job, decoded by hspf_ospfv3_backbone_from_cells, must equal byte for byte, prefix options included, the host chain:
each border's update_rib_full_v3 over its job planes, its net_summaries_v3 and rtr_summaries_v3 into area 0 spliced
into R's LSDB in LsaKey order in place of the border's own, then update_rib_full_v3 at R, restricted to the affected
prefixes.  No recorded conformance data holds an Inter-Area-Router LSA, so that chain is the contract here."""
import ctypes as C
import subprocess
import types
from pathlib import Path

import numpy as np
import pytest
from numpy.lib.recfunctions import repack_fields

import test_ospfv3_abr_rib_cells as v3abr
from holo_b200 import capi, ospf_rib, ospfv3, synth
from holo_b200.route_table import DELTA_METRIC, DELTA_NEXTHOPS, DELTA_OTHER
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospf_abr_rib_cells import planes_of
from test_ospf_backbone_asbr_cells import asbr_cells, ext_path
from test_ospf_rib_cells import same_rib
from test_ospf_rib_delta import classify, reference
from test_ospfv3_backbone_cells import GOLDEN, Backbone, SynthBackbone, non_backbone_links, synth_jobs
from test_ospfv3_backbone_cells import harness as bb_harness  # noqa: F401  (fixture)
from test_ospfv3_nonbackbone_cells import job_rib_areas, spf_of, srt

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    """The OSPFv3 kAsbr walk over area 0, under the names asbr_cells calls (its arguments are the asbr harness's)."""
    out = tmp_path_factory.mktemp("harness") / "libospfv3_backbone_asbr_cells_harness.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                    "-o", str(out), str(ROOT / "tests" / "native" / "ospfv3_backbone_asbr_cells_harness.cc")],
                   check=True)
    lib = C.CDLL(str(out))
    for fn in (lib.harness_ospfv3_backbone_asbr_cells, lib.harness_ospfv3_backbone_asbr_cells16):
        fn.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 8
        fn.restype = C.c_int
    return types.SimpleNamespace(lib=lib, harness_ospf_backbone_asbr_cells=lib.harness_ospfv3_backbone_asbr_cells,
                                 harness_ospf_backbone_asbr_cells16=lib.harness_ospfv3_backbone_asbr_cells16)


class AsbrBackbone(Backbone):
    """ospfv3.backbone_view with area-1 ASBRs: R, three borders of area 1 (the first also in area 2; those in `use`
    given to the table, a border left out keeping its LSAs as static records), an area-0 ASBR and k area-1 ASBRs."""

    def __init__(self, seed, k=2, n_ext=4, use=(0, 1, 2), V0=30, E0=90, V1=25, E1=70, max_paths=16):
        t0 = synth.random_topology(V0, E0, synth.SEED_BASE + 950 + 2 * seed, cost_choices=[5, 10, 20])
        t1 = synth.random_topology(V1, E1, synth.SEED_BASE + 951 + 2 * seed, cost_choices=[5, 10, 20])
        v = ospfv3.backbone_view(t0, t1, seed, max_paths=max_paths, area1_asbrs=k, area1_ext=n_ext)
        self.view = v
        self.area, self.summaries, self.externals = v["r_area"], v["summaries0"], v["externals"]
        self.flat = ospfv3.Flat(self.area)
        self.rv = self.flat.router_vertex(self.area.router_id)
        self.doms = [v3abr.Domain(areas, sums, self.externals) for b, (areas, _ids, sums) in enumerate(v["borders"])
                     if b in use]
        self.cfgs = [[ospf_rib.area_config()] * len(d.areas) for d in self.doms]
        self.make_table()
        self.planes = planes_of(self.flat.csr, self.rv)

    def make_table(self, doms=None, summaries=None):
        self.table = self.table_of(doms, summaries)

    def table_of(self, doms=None, summaries=None):
        return ospf_rib.BackboneTable(self.flat, self.area.router_id,
                                      self.summaries if summaries is None else summaries, self.externals,
                                      [d.rt for d in (doms or self.doms)], asbr=True)

    def cells(self, abr, harness, bplanes, narrow_planes=False, status=None, root_status=0):
        bcells = [np.stack([d.cells(abr, p, narrow_planes)[0] for p in bp]) for d, bp in zip(self.doms, bplanes)]
        cells, out = asbr_cells(harness, self.table, self.planes, bcells, bplanes, narrow_planes, status, root_status)
        return cells, out, bcells

    def border_lsas(self, d, cfg, job_planes):
        """What border d originates into area 0 in the job: net_summaries_v3 and rtr_summaries_v3 over its
        update_rib_full_v3."""
        i0 = next(i for i, a in enumerate(d.areas) if a.area_id == 0)
        return ospfv3.nonbackbone_lsas(d.areas[0].router_id, d.areas[0].max_paths, job_rib_areas(d, job_planes),
                                       self.externals, i0, cfg)

    def lsdb(self, bplanes_of_job):
        """Area 0's LSDB of the job: each border's Inter-Area-Prefix / Inter-Area-Router LSAs re-originated."""
        bid = {d.areas[0].router_id for d in self.doms}
        new = [tuple(s) for s in self.summaries.tolist() if int(s[0]) not in bid]
        for d, cfg, p in zip(self.doms, self.cfgs, bplanes_of_job):
            new += self.border_lsas(d, cfg, p)
        return srt(np.array(new, ospf_rib.INTER_AREA_LSA_DT))

    def host(self, bcells_of_job, bplanes_of_job):
        ra = [ospf_rib.RibArea(0, ospfv3.area_from_planes(self.area, spf_of(self.planes)), self.area.ifaces,
                               self.lsdb(bplanes_of_job), True)]
        return self.affected(ospf_rib.update_rib_full_v3(self.area.router_id, self.area.max_paths, ra, self.externals))

    def key_index(self, key):
        return SynthBackbone.key_index(self, key)

    def cut(self, x, borders=None):
        """A job: every non-backbone link of router x disabled in the area planes of the borders in `borders` (all:
        None)."""
        ovs = [self.job_overrides(l, capi.COST_DISABLED) for l in non_backbone_links(self)
               if any(y[0] == x and y[2] for y in l)]
        return [{} if borders is not None and b not in borders else
                {i: e for i in range(len(d.areas)) if (e := sum((o[b].get(i, []) for o in ovs), []))}
                for b, d in enumerate(self.doms)]

    def ext_keys(self, x):
        """Table indices of the prefixes router x advertises as AS-external."""
        e = self.externals[self.externals["adv_rtr"] == x]
        want = {(y["prefix"]["bytes"].tobytes(), int(y["len"])) for y in e}
        return [u for u in range(self.table.n_prefixes)
                if (self.table.prefixes6[u]["bytes"].tobytes(), int(self.table.plen[u])) in want]


def check_jobs(bb, abr, harness, jobs, narrow_planes=False):
    cells, _ = bb.check(abr, harness, jobs, narrow_planes)
    return cells


# ------------------------------------------------------------------------------------------- the chain
@pytest.mark.parametrize("seed", range(3))
def test_base_job_lsas_and_decode(abr_harness, harness, seed):
    """The generator's Inter-Area-Router LSAs are each border's rtr_summaries_v3 into area 0, and job 0 decodes to R's
    update_rib_full_v3 over the generated LSDB."""
    bb = AsbrBackbone(seed)
    assert bb.table.n_asbr_slots > 0 and 1 <= bb.table.n_asbr_sets <= 3
    keep = [n for n in ospf_rib.INTER_AREA_LSA_DT.names if n != "lsa_id"]
    n4 = 0
    for d in bb.doms:
        rid = d.areas[0].router_id
        i0 = next(i for i, a in enumerate(d.areas) if a.area_id == 0)
        got = ospf_rib.rtr_summaries_v3(rid, job_rib_areas(d, d.planes()), [ospf_rib.area_config()] * len(d.areas), i0)
        rec = bb.summaries[(bb.summaries["adv_rtr"] == rid) & (bb.summaries["lsa_type"] == 4)]
        assert repack_fields(got[keep]).tobytes() == repack_fields(rec[keep]).tobytes()
        assert set(rec["router_id"].tolist()) <= set(bb.view["area1_asbrs"])
        n4 += len(rec)
    assert n4 > 0
    cells = check_jobs(bb, abr_harness, harness, [bb.job_overrides((), 0)])
    ra = [ospf_rib.RibArea(0, ospfv3.area_from_planes(bb.area, spf_of(bb.planes)), bb.area.ifaces, bb.summaries, True)]
    same_rib(bb.decode(cells[0]),
             bb.affected(ospf_rib.update_rib_full_v3(bb.area.router_id, bb.area.max_paths, ra, bb.externals)))
    for x in bb.view["area1_asbrs"]:
        u = bb.ext_keys(x)
        assert u and ext_path(cells[0][u]).any()


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_generated_domains_chain(abr_harness, harness, seed, narrow_planes):
    """Every non-backbone link failed and re-costed, one job each, all in one batch; the externals of the area-1
    ASBRs are affected prefixes and route through the borders' Inter-Area-Router slots."""
    bb = AsbrBackbone(seed)
    jobs = [bb.job_overrides((), 0)]
    for link in non_backbone_links(bb):
        jobs += [bb.job_overrides(link, capi.COST_DISABLED), bb.job_overrides(link, 37)]
    cells = check_jobs(bb, abr_harness, harness, jobs, narrow_planes)
    assert (cells != cells[0]).any()
    u = sorted({k for x in bb.view["area1_asbrs"] for k in bb.ext_keys(x)})
    assert (cells[:, u] != cells[0][u]).any()


# ------------------------------------------------------------------------------------------- hand cases
def test_asbr_cut_off_from_the_last_border_moves_to_an_earlier_one(abr_harness, harness):
    """Only the last border in LsaKey order loses the ASBR: R's entry is the previous border's slot (walked from the
    end), which need not be the cheapest; every external of the ASBR still routes, through the other borders."""
    n = 0
    for seed in range(3):
        bb = AsbrBackbone(seed)
        last = max(range(3), key=lambda b: bb.doms[b].areas[0].router_id)
        for x in bb.view["area1_asbrs"]:
            cells = check_jobs(bb, abr_harness, harness, [bb.job_overrides((), 0), bb.cut(x, {last})])
            u = [k for k in bb.ext_keys(x) if ext_path(cells[0][k:k + 1])[0]]
            assert ext_path(cells[1][u]).all()
            n += int(cells[1][u].tobytes() != cells[0][u].tobytes())
    assert n > 0


def test_asbr_cut_off_from_every_border_is_lost_then_gained(abr_harness, harness):
    bb = AsbrBackbone(0)
    x = bb.view["area1_asbrs"][0]
    cells = check_jobs(bb, abr_harness, harness, [bb.job_overrides((), 0), bb.cut(x), bb.job_overrides((), 0)])
    k = classify(cells[1], cells[0])
    assert (k == 1).any()                                              # LOST
    assert (classify(cells[2], cells[1])[k == 1] == 2).all()           # GAINED
    assert cells[2].tobytes() == cells[0].tobytes()


def test_shared_external_flips_between_area0_and_area1_asbr(abr_harness, harness):
    """The area-0 ASBR's /64 is type-2 at metric 12 from it and at 11 from each area-1 ASBR: an area-1 ASBR's LSA
    wins while R reaches one, and cutting the area-1 ASBRs off hands the route to the area-0 one."""
    for seed in range(3):
        bb = AsbrBackbone(seed)
        a0 = bb.externals[(bb.externals["adv_rtr"] == bb.view["asbr"]) & (bb.externals["len"] == 64)][0]
        u = bb.key_index((a0["prefix"]["bytes"].tobytes(), 64))
        cuts = [bb.cut(x) for x in bb.view["area1_asbrs"]]
        cut_all = [{i: e for i in range(len(d.areas)) if (e := sum((c[b].get(i, []) for c in cuts), []))}
                   for b, d in enumerate(bb.doms)]
        cells = check_jobs(bb, abr_harness, harness, [bb.job_overrides((), 0), cut_all] + synth_jobs(bb, 8, seed)[1:])
        w = cells[:, u]
        assert (ospf_rib.cell_path(w) == ospf_rib.PATH_TYPE2).all()
        assert (int(w[0]["aux"]), int(w[1]["aux"])) == (11, 12) and w[0]["winner"] != w[1]["winner"]


def test_type1_and_type2_moves_show_as_metric_and_nexthops(abr_harness, harness):
    """A moved forwarding metric changes a type-1 external's metric (METRIC) and a type-2's next hops only; an entry
    that moves to another border at the same distance changes next hops (NEXTHOPS)."""
    kinds, types_ = 0, set()
    for seed in range(3):
        bb = AsbrBackbone(seed)
        last = max(range(3), key=lambda b: bb.doms[b].areas[0].router_id)
        jobs = synth_jobs(bb, 12, seed) + [bb.cut(x, {last}) for x in bb.view["area1_asbrs"]]
        cells = check_jobs(bb, abr_harness, harness, jobs)
        for x in bb.view["area1_asbrs"]:
            u = bb.ext_keys(x)
            types_ |= {int(p) for p in ospf_rib.cell_path(cells[0][u])}
            k = np.stack([classify(cells[j][u], cells[0][u]) for j in range(1, len(cells))])
            kinds |= int(np.bitwise_or.reduce(k, axis=None))
    assert {ospf_rib.PATH_TYPE1, ospf_rib.PATH_TYPE2} <= types_
    assert kinds & DELTA_METRIC and kinds & DELTA_NEXTHOPS


def test_static_inter_area_router_lsa_of_another_abr_sits_at_its_lsakey_position(abr_harness, harness):
    """The middle border left out of the table: its Inter-Area-Router LSAs stay static records between the two
    borders' slots, and the walk from the end reaches it after the last border's slot."""
    for seed in range(3):
        bb = AsbrBackbone(seed, use=(0, 2))
        mid = bb.view["borders"][1][0][0].router_id
        assert ((bb.summaries["adv_rtr"] == mid) & (bb.summaries["lsa_type"] == 4)).any()
        jobs = [bb.job_overrides((), 0)] + [bb.cut(x, {1}) for x in bb.view["area1_asbrs"]] + \
            [bb.cut(x) for x in bb.view["area1_asbrs"]] + synth_jobs(bb, 6, seed)[1:]
        check_jobs(bb, abr_harness, harness, jobs)


def test_winning_external_lsa_changes_options_at_an_equal_metric(abr_harness, harness):
    """backbone_view's flip_ext /64: the first two area-1 ASBRs advertise it as type-1 (LA, P) at costs that tie
    through the last border, so R's route takes the first's LSA.  Cutting that ASBR off hands the route to the other's
    LSA; where its metric and next hops stay, only the winner changes, the delta reports OTHER and the decode gives
    the other options."""
    n = 0
    for seed in range(3):
        bb = AsbrBackbone(seed)
        fx = bb.view["flip_ext"]
        assert fx is not None
        u = bb.key_index((fx[0], fx[1]))
        cells = check_jobs(bb, abr_harness, harness, [bb.job_overrides((), 0), bb.cut(fx[2])])
        a, b = cells[0][u], cells[1][u]
        assert ospf_rib.cell_path(a) == ospf_rib.PATH_TYPE1
        if int(a["mpf"]) == int(b["mpf"]) and int(a["nh_mask"]) == int(b["nh_mask"]) and a["winner"] != b["winner"]:
            _, recs, _ = reference(cells, cells[:1])
            assert [int(r["kind"]) for r in recs if int(r["job"]) == 1 and int(r["prefix"]) == u] == [DELTA_OTHER]
            o = lambda rib: {(x["prefix"]["bytes"].tobytes(), int(x["len"])): int(x["prefix_options"])
                             for x in rib.routes}
            k = (fx[0], fx[1])
            assert (o(bb.decode(cells[0]))[k], o(bb.decode(cells[1]))[k]) == (ospfv3.PFX_LA, ospfv3.PFX_P)
            n += 1
    assert n > 0


# ------------------------------------------------------------------------------------------- refusals
def iar_row(adv, rid, opts=0):
    return np.array([(adv, 0x777, 5, rid, ospfv3.ip_rec("::"), 0, opts, 4, 0)], ospf_rib.INTER_AREA_LSA_DT)


def refused(code, fn):
    with pytest.raises(capi.HspfError) as e:
        fn()
    assert e.value.code == code


def test_table_refusals():
    bb = AsbrBackbone(0)
    # the existing create still refuses the borders' Inter-Area-Router LSAs
    refused(capi.HSPF_E_UNSUPPORTED, lambda: ospf_rib.BackboneTable(bb.flat, bb.area.router_id, bb.summaries,
                                                                     bb.externals, [d.rt for d in bb.doms]))
    # the existing create's own refusals
    for doms in ([bb.doms[0]] * 2, [bb.doms[0]] * 9):
        refused(capi.HSPF_E_INVAL, lambda: bb.table_of(doms))
    import test_ospf_abr_rib_cells as v2abr
    d2 = v2abr.domain(0)
    refused(capi.HSPF_E_INVAL, lambda: bb.table_of([bb.doms[0], d2]))
    # a border's Inter-Area-Router LSA for a router its table cannot originate for, with or without NU (NU leaves
    # out prefixes only)
    b0 = bb.doms[0].areas[0].router_id
    for opts in (0, ospfv3.PFX_NU):
        bad = srt(np.concatenate([bb.summaries, iar_row(b0, 0x09090909, opts)]))
        refused(capi.HSPF_E_INVAL, lambda: bb.table_of(summaries=bad))
    dead = bad.copy()
    dead["maxage"][dead["router_id"] == 0x09090909] = 1
    bb.table_of(summaries=dead)
    # ... and from an ABR outside the table it is a static record
    other = AsbrBackbone(0, use=(0, 2))
    mid = other.view["borders"][1][0][0].router_id
    other.table_of(summaries=srt(np.concatenate([other.summaries, iar_row(mid, 0x09090909)])))
    # an E-flag router of a border's non-backbone area with the B flag
    x = bb.view["area1_asbrs"][0]
    doms = []
    for d in bb.doms:
        areas = []
        for a in d.areas:
            if a.area_id != 0:
                a = ospfv3.Ospfv3Area(**{k: getattr(a, k) for k in a.__dataclass_fields__})
                rl = a.router_lsas.copy()
                rl["flags"][rl["adv_rtr"] == x] |= 0x01
                a.router_lsas = rl
            areas.append(a)
        doms.append(v3abr.Domain(areas, d.summaries, d.externals))
    refused(capi.HSPF_E_UNSUPPORTED, lambda: bb.table_of(doms))


def test_asbr_flag_takes_area0_flats_only():
    """asbr=True with a config, or with a flat of another area, raises before any call."""
    bb = AsbrBackbone(0)
    with pytest.raises(ValueError):
        ospf_rib.BackboneTable(bb.flat, bb.area.router_id, bb.summaries, bb.externals, [d.rt for d in bb.doms],
                               asbr=True, config=ospf_rib.area_config())
    a1 = next(a for a in bb.doms[1].areas if a.area_id == 1)
    with pytest.raises(ValueError):
        ospf_rib.BackboneTable(ospfv3.Flat(a1), a1.router_id, None, None, [d.rt for d in bb.doms], asbr=True)


def with_twins(d, n):
    """Border domain d with n copies of its area 1 added as areas 3, 4, ...: the area-1 ASBRs are E-flag routers in
    each, one (border, area) plane set apiece."""
    i1 = [i for i, a in enumerate(d.areas) if a.area_id == 1][0]
    twins = []
    for k in range(n):
        t = ospfv3.Ospfv3Area(**{f: getattr(d.areas[i1], f) for f in d.areas[i1].__dataclass_fields__})
        t.area_id = 3 + k
        twins.append(t)
    return v3abr.Domain(d.areas + twins, list(d.summaries) + [np.zeros(0, ospf_rib.INTER_AREA_LSA_DT)] * n, d.externals)


def test_more_than_8_plane_sets_are_refused():
    """Every slot of a border reads the plane set of its (border, area): 4 + 2 + 2 sets build, 4 + 2 + 3 are refused."""
    bb = AsbrBackbone(0)
    d0, d1, d2 = bb.doms
    t = bb.table_of([with_twins(d0, 3), with_twins(d1, 1), with_twins(d2, 1)])
    assert t.n_asbr_sets == 8 and t.n_asbr_slots > bb.table.n_asbr_slots
    refused(capi.HSPF_E_UNSUPPORTED, lambda: bb.table_of([with_twins(d0, 3), with_twins(d1, 1), with_twins(d2, 2)]))


# ------------------------------------------------------------------------------------------- tables without slots
def test_existing_walk_on_a_table_without_slots(abr_harness, harness, bb_harness):
    """On the golden Backbone cases and SynthBackbone, the asbr create gives the table of the existing create and the
    kAsbr walk gives the existing OSPFv3 harness's cells byte for byte."""
    cases = [Backbone(*g) for g in GOLDEN[:3]] + [SynthBackbone(1)]
    for bb in cases:
        t = ospf_rib.BackboneTable(bb.flat, bb.area.router_id, bb.summaries, bb.externals, [d.rt for d in bb.doms],
                                   asbr=True)
        assert (t.n_asbr_slots, t.n_asbr_sets, t.n_prefixes, t.n_records, t.n_slots) == \
            (0, 0, bb.table.n_prefixes, bb.table.n_records, bb.table.n_slots)
        assert t.prefixes6.tobytes() == bb.table.prefixes6.tobytes()
        jobs = [bb.job_overrides((), 0)] + [bb.job_overrides(l, capi.COST_DISABLED) for l in non_backbone_links(bb)[:4]]
        bp = bb.border_planes(jobs)
        for narrow_planes in (False, True):
            want, _, bcells = Backbone.cells(bb, abr_harness, bb_harness, bp, narrow_planes)
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
    rows = [np.repeat(np.arange(J, dtype=np.uint32)[:, None], len(d.areas), 1) for d in bb.doms]
    rows[1][2, :] = J                                                  # out of range
    ps = [[np.zeros(J, np.uint32) for _ in d.areas] for d in bb.doms]
    for i in range(len(bb.doms[0].areas)):
        ps[0][i][1] = 0x8
    got, st = asbr_cells(harness, bb.table, bb.planes, bcells, bp, rows=rows, pstatus=ps)
    assert st[2] & capi.JS_INVALID and st[1] == 0x8
    for j in (1, 2):
        assert (got["winner"][j] == ospf_rib.NO_RECORD).all() and not got["mpf"][j].any()
    keep = [j for j in range(J) if j not in (1, 2)]
    assert got[keep].tobytes() == want[keep].tobytes()
