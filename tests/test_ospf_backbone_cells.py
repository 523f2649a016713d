"""CPU: Summary-LSA origination (hspf_ospfv2_net_summaries) and the backbone-router stage over what-if jobs inside
other areas (hspf_ospfv2_backbone_*).

The device kernel's body (ospf_backbone_cell_eval, holo_b200/csrc/ospf_backbone_cells.h) is compiled into a test
harness and run on the CPU over the oracle's SPT planes.  Each job perturbs one link of a non-backbone area at every
border that has it.  The cells, decoded by hspf_ospfv2_backbone_from_cells, must equal byte for byte the host chain:
each border's update_rib_full over its job's planes, its net_summaries into area 0 spliced into R's LSDB in place of
its type-3 LSAs, and update_rib_full at R, restricted to the affected prefixes."""
import ctypes as C
import json
import subprocess
from pathlib import Path

import numpy as np
import pytest

import golden_util as gu
from holo_b200 import capi, ospf_rib, ospfv2, synth
from test_ospf_abr_rib_cells import Domain, golden_domain, narrow, planes_of
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospf_rib_cells import same_rib
from test_ospfv2_route_cells import gather_for

ROOT = Path(__file__).resolve().parent.parent
SNAPS = gu.load_ospfv2()
MULTI = [s for s in SNAPS if len(s["areas"]) > 1]
SUMS = {(s["topo"], s["rt"]): s for s in json.loads((ROOT / "tests" / "golden" / "ospfv2_summaries.json").read_text())}
AREA_TYPE = {"normal": ospf_rib.AREA_NORMAL, "stub": ospf_rib.AREA_STUB, "nssa": ospf_rib.AREA_NSSA}


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    out = tmp_path_factory.mktemp("harness") / "libospf_backbone_cells_harness.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                    "-o", str(out), str(ROOT / "tests" / "native" / "ospf_backbone_cells_harness.cc")], check=True)
    lib = C.CDLL(str(out))
    for fn in (lib.harness_ospf_backbone_cells, lib.harness_ospf_backbone_cells16):
        fn.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 4
    return lib


def snap(topo, rt):
    return next(s for s in SNAPS if s["topo"] == topo and s["rt"] == rt)


def configs_of(s, dom):
    by_id = {a["area_id"]: a for a in SUMS[(s["topo"], s["rt"])]["areas"]}
    return [ospf_rib.area_config(AREA_TYPE[by_id[gu.ipstr(a.area_id)]["area_type"]], by_id[gu.ipstr(a.area_id)]["summary"],
                                 by_id[gu.ipstr(a.area_id)]["default_cost"]) for a in dom.areas]


def rib_areas(dom, job_planes):
    ra = []
    for i, (a, p) in enumerate(zip(dom.areas, job_planes)):
        spf = ospfv2.area_from_planes(a, lambda csr, root, nhw, p=p: (p[0], p[1], np.pad(p[2][:, None], ((0, 0), (0, nhw - 1)))))
        ra.append(ospf_rib.RibArea(a.area_id, spf, a.ifaces, dom.summaries[i], dom.active[i]))
    return ra


def summaries_of(dom, configs, job_planes, target):
    ra = rib_areas(dom, job_planes)
    rid = dom.areas[0].router_id
    rib = ospf_rib.update_rib_full(rid, dom.areas[0].max_paths, ra, dom.externals)
    return ospf_rib.net_summaries(rid, rib, ospf_rib.router_tables(rid, ra), ra, configs, target)


# ------------------------------------------------------------------------------------------ summary pin
@pytest.mark.parametrize("s", MULTI, ids=[f"{s['topo']}-{s['rt']}" for s in MULTI])
def test_net_summaries_equal_the_recorded_lsas(s):
    """The type-3 / type-4 LSAs the router originated into each attached area, as the reference recorded them."""
    dom, _ = golden_domain(s)
    cfg = configs_of(s, dom)
    rec = {a["area_id"]: a for a in SUMS[(s["topo"], s["rt"])]["areas"]}
    assert not any(a["ranges"] for a in rec.values())
    p = dom.planes()
    for i, a in enumerate(dom.areas):
        got = summaries_of(dom, cfg, p, i)
        t3 = sorted([gu.ipstr(int(x["lsa_id"])), gu.ipstr(int(x["mask"])), int(x["metric"])] for x in got if x["lsa_type"] == 3)
        t4 = sorted([gu.ipstr(int(x["lsa_id"])), int(x["metric"])] for x in got if x["lsa_type"] == 4)
        want = rec[gu.ipstr(a.area_id)]
        assert (t3, t4) == (want["type3"], want["type4"]), (s["topo"], s["rt"], gu.ipstr(a.area_id))


def test_summary_fixture_covers_every_multi_area_snapshot():
    assert len(MULTI) == 17 and len(SUMS) == 17
    kinds = {a["area_type"] for s in SUMS.values() for a in s["areas"]}
    assert kinds == {"normal", "stub"}
    assert any(not a["summary"] for s in SUMS.values() for a in s["areas"])     # a totally stubby area (topo1 rt6)


# -------------------------------------------------------------------------------------- backbone domains
class Backbone:
    """R's area-0 image and the borders' ABR domains (from their own snapshots), the table over them."""

    def __init__(self, topo, r, borders, externals=None):
        sr = snap(topo, r)
        keys = gu.global_sort_keys(sr)
        a0 = next(a for a in sr["areas"] if a["area_id"] == "0.0.0.0")
        self.area = gu.ospfv2_area_image(sr, a0, keys)
        self.keys, self.snap = keys, sr
        self.flat = ospfv2.Flat(self.area)
        self.rv = self.flat.router_vertex(self.area.router_id)
        self.summaries = gu.ospfv2_summaries(a0)
        self.externals = externals
        self.bsnaps = [snap(topo, b) for b in borders]
        self.doms = [golden_domain(b)[0] for b in self.bsnaps]
        self.cfgs = [configs_of(b, d) for b, d in zip(self.bsnaps, self.doms)]
        self.table = ospf_rib.BackboneTable(self.flat, self.area.router_id, self.summaries, externals,
                                            [d.rt for d in self.doms])
        self.planes = planes_of(self.flat.csr, self.rv)

    def job_overrides(self, link, cost):
        """Per border, per area: the overrides of link (router id pair) at `cost` in the borders' non-backbone areas."""
        out = []
        for d in self.doms:
            ov = {}
            for i, (a, f) in enumerate(zip(d.areas, d.flats)):
                if a.area_id == 0:
                    continue
                ids = [int(x) for x in f.ids]
                src = np.repeat(np.arange(f.csr.n_vertices), np.diff(f.csr.row_ptr))
                e = [(int(k), cost) for k in range(f.csr.n_edges) if {ids[src[k]], ids[f.csr.col[k]]} == set(link)]
                if e:
                    ov[i] = e
            out.append(ov)
        return out

    def border_planes(self, jobs):
        return [[d.planes(ov[b]) for ov in jobs] for b, d in enumerate(self.doms)]

    def cells(self, abr, harness, bplanes, narrow_planes=False, status=None, root_status=0):
        """Backbone cells [J, P] over each border's cells of the J jobs."""
        bcells = [np.stack([d.cells(abr, p, narrow_planes)[0] for p in bp]) for d, bp in zip(self.doms, bplanes)]
        cells, out = self.cells_from(harness, bcells, narrow_planes, status, root_status)
        return cells, out, bcells

    def cells_from(self, harness, bcells, narrow_planes=False, status=None, root_status=0):
        """Backbone cells [J, P] and status words over the borders' cells [J, K_b]."""
        J = len(bcells[0])
        pl = narrow(self.planes) if narrow_planes else self.planes
        keep = [np.ascontiguousarray(x) for x in pl] + bcells
        bc = (C.c_void_p * len(bcells))(*[c.ctypes.data for c in bcells])
        st = None
        if status is not None:
            sk = [np.ascontiguousarray(x, np.uint32) for x in status]
            keep += sk
            st = (C.c_void_p * len(sk))(*[x.ctypes.data for x in sk])
        cells = np.zeros((J, self.table.n_prefixes), ospf_rib.RIB_CELL_DT)
        out = np.zeros(J, np.uint32)
        fn = harness.harness_ospf_backbone_cells16 if narrow_planes else harness.harness_ospf_backbone_cells
        fn(self.table.handle, J, keep[0].ctypes.data, keep[1].ctypes.data, keep[2].ctypes.data, root_status, bc, st,
           cells.ctypes.data, out.ctypes.data)
        return cells, out

    def decode(self, cells):
        v, n = gather_for(self.flat, self.rv, self.planes)
        return ospf_rib.backbone_from_cells(self.area, self.table, cells, v, n)

    def affected(self, rib):
        keep = {(int(p), int(l)) for p, l in zip(self.table.prefix, self.table.plen)}
        sel = [k for k, r in enumerate(rib.routes) if (int(r["prefix"]), bin(int(r["mask"])).count("1")) in keep]
        routes, hops = [], []
        for k in sel:
            r = rib.routes[k].copy()
            h = rib.nexthops[int(r["nh_off"]): int(r["nh_off"]) + int(r["n_nh"])]
            r["nh_off"] = sum(len(x) for x in hops)
            routes.append(r)
            hops.append(h)
        return ospf_rib.Rib(np.array(routes, ospf_rib.RIB_ROUTE_DT), np.concatenate(hops) if hops else
                            np.zeros(0, ospfv2.NEXTHOP_DT))

    def host(self, job_planes_per_border):
        """The chain: each border's net_summaries into area 0 in place of its type-3 LSAs, update_rib_full at R."""
        bid = {d.areas[0].router_id for d in self.doms}
        new = [s for s in self.summaries if not (int(s["adv_rtr"]) in bid and s["lsa_type"] == 3)]
        for d, cfg, p in zip(self.doms, self.cfgs, job_planes_per_border):
            i0 = next(i for i, a in enumerate(d.areas) if a.area_id == 0)
            got = summaries_of(d, cfg, p, i0)
            new += [x for x in got if x["lsa_type"] == 3]
        s = np.array(new, ospf_rib.SUMMARY_LSA_DT)
        s = s[np.lexsort((s["lsa_id"], s["adv_rtr"], s["lsa_type"]))]
        p = self.planes
        spf = ospfv2.area_from_planes(self.area, lambda csr, root, nhw: (p[0], p[1], np.pad(p[2][:, None], ((0, 0), (0, nhw - 1)))))
        ra = [ospf_rib.RibArea(0, spf, self.area.ifaces, s, True)]
        return self.affected(ospf_rib.update_rib_full(self.area.router_id, self.area.max_paths, ra, self.externals))

    def check(self, abr, harness, jobs, narrow_planes=False):
        bp = self.border_planes(jobs)
        cells, st, _ = self.cells(abr, harness, bp, narrow_planes)
        assert not st.any()
        for j in range(len(jobs)):
            same_rib(self.decode(cells[j]), self.host([bp[b][j] for b in range(len(self.doms))]))
        return cells


GOLDEN = [("topo1-1", "rt3", ["rt2", "rt4", "rt6"]), ("topo1-2", "rt3", ["rt2", "rt4", "rt6"]),
          ("topo1-3", "rt3", ["rt2", "rt4", "rt6"]), ("topo2-2", "rt1", ["rt4", "rt5"]),
          ("topo2-2", "rt2", ["rt4", "rt5"]), ("topo2-2", "rt3", ["rt4", "rt5"])]
GIDS = [f"{t}-{r}" for t, r, _ in GOLDEN]


def non_backbone_links(bb):
    """Vertex-id pairs of the links of the borders' non-backbone areas: router to router, router to network."""
    out = set()
    for d in bb.doms:
        for a, f in zip(d.areas, d.flats):
            if a.area_id == 0:
                continue
            ids = [int(x) for x in f.ids]
            src = np.repeat(np.arange(f.csr.n_vertices), np.diff(f.csr.row_ptr))
            for e in range(f.csr.n_edges):
                if f.is_router[src[e]]:
                    out.add(tuple(sorted((ids[src[e]], ids[f.csr.col[e]]))))
    return sorted(out)


@pytest.mark.parametrize("g", GOLDEN, ids=GIDS)
def test_base_job_equals_the_recorded_local_rib(abr_harness, harness, g):
    bb = Backbone(*g)
    cells = bb.check(abr_harness, harness, [bb.job_overrides((), 0)])
    got = bb.decode(cells[0])
    key_name = {v: k for k, v in bb.keys.items()}
    mine = {}
    for r in got.routes:
        nh = sorted(((key_name.get(i, "?"), gu.ipstr(a) if ha else None) for (i, ha, a, _hn, _n, _hl, _l) in got.nh(r)),
                    key=lambda x: (x[0] or "", x[1] or ""))
        mine[f"{gu.ipstr(r['prefix'])}/{bin(int(r['mask'])).count('1')}"] = (int(r["metric"]), ospf_rib.PATH_NAMES[int(r["path_type"])], nh)
    want = {k: v for k, v in gu.golden_rib(bb.snap).items() if k in mine or
            any(k == f"{gu.ipstr(int(p))}/{int(l)}" for p, l in zip(bb.table.prefix, bb.table.plen))}
    norm = lambda d: {k: (v[0], v[1], [(a or "", b or "") for a, b in v[2]]) for k, v in d.items()}
    assert norm(mine) == norm(want)
    assert bb.table.n_prefixes > 0


@pytest.mark.parametrize("g", GOLDEN, ids=GIDS)
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_chain_one_link_failed_or_recosted(abr_harness, harness, g, narrow_planes):
    """Every non-backbone link failed, then re-costed, one job each, all jobs in one batch."""
    bb = Backbone(*g)
    links = non_backbone_links(bb)
    assert links
    jobs = [bb.job_overrides((), 0)]
    for link in links:
        jobs.append(bb.job_overrides(link, capi.COST_DISABLED))
        jobs.append(bb.job_overrides(link, 35))
    cells = bb.check(abr_harness, harness, jobs, narrow_planes)
    assert (cells != cells[0]).any()


def test_lost_then_gained(abr_harness, harness):
    """topo1-1: cutting a stub area's only link to its border makes its prefixes unreachable at R (LOST), and the
    next job, unperturbed, has them back (GAINED)."""
    bb = Backbone("topo1-1", "rt3", ["rt2", "rt4", "rt6"])
    jobs = [bb.job_overrides((), 0)]
    n_lost = 0
    for link in non_backbone_links(bb):
        jobs += [bb.job_overrides(link, capi.COST_DISABLED), bb.job_overrides((), 0)]
    cells = bb.check(abr_harness, harness, jobs)
    present = (ospf_rib.cell_flags(cells) & 1) != 0
    for j in range(1, len(jobs), 2):
        lost = present[0] & ~present[j]
        n_lost += int(lost.any())
        assert (present[j + 1] == present[0]).all()
    assert n_lost > 0


def test_equal_metric_borders_merge_atoms(abr_harness, harness):
    """topo2-2: rt4 and rt5 border one area; R's routes to that area tie across both, so ORed atoms."""
    n = 0
    for r in ("rt1", "rt2", "rt3"):
        bb = Backbone("topo2-2", r, ["rt4", "rt5"])
        cells = bb.check(abr_harness, harness, [bb.job_overrides((), 0)])
        inter = cells[0][ospf_rib.cell_path(cells[0]) == ospf_rib.PATH_INTER]
        n += sum(1 for c in inter if bin(int(c["nh_mask"])).count("1") > 1)
    assert n > 0


def test_slot_sits_at_its_border_lsakey_position(abr_harness, harness):
    """topo2-2 with rt4 alone as the border: rt5's type-3 LSAs stay static records.  Where the two tie, the winner is
    the first in LsaKey order: rt4's slot (4.4.4.4 < 5.5.5.5), whose winner lies past the table's records."""
    bb = Backbone("topo2-2", "rt1", ["rt4"])
    cells, st, _ = bb.cells(abr_harness, harness, bb.border_planes([bb.job_overrides((), 0)]))
    n_recs = bb.table.n_records
    inter = [c for c in cells[0] if ospf_rib.cell_path(c) == ospf_rib.PATH_INTER and ospf_rib.cell_flags(c) & 1]
    ties = [c for c in inter if bin(int(c["nh_mask"])).count("1") > 1]
    assert ties
    assert all(n_recs <= int(c["winner"]) < n_recs + bb.table.n_slots for c in ties)
    same_rib(bb.decode(cells[0]), bb.host([bp[0] for bp in bb.border_planes([bb.job_overrides((), 0)])]))


# ------------------------------------------------------------------------------------------- refusals
def test_table_refusals():
    bb = Backbone("topo2-2", "rt1", ["rt4", "rt5"])
    d4, d5 = bb.doms
    mk = lambda borders, flat=bb.flat, rid=bb.area.router_id, sums=bb.summaries: ospf_rib.BackboneTable(flat, rid, sums, None, borders)
    for borders in ([], [d4.rt] * 2, [d4.rt] * 9):
        with pytest.raises(capi.HspfError) as e:
            mk(borders)
        assert e.value.code == capi.HSPF_E_INVAL
    # R with the B flag, or R one of the borders: rt4 as R
    s4 = snap("topo2-2", "rt4")
    k4 = gu.global_sort_keys(s4)
    a4 = gu.ospfv2_area_image(s4, next(a for a in s4["areas"] if a["area_id"] == "0.0.0.0"), k4)
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.BackboneTable(ospfv2.Flat(a4), a4.router_id, None, None, [d5.rt])
    assert e.value.code == capi.HSPF_E_INVAL
    # a border table without area 0
    no0 = ospf_rib.AbrRibTable(d4.areas[1].router_id, [d4.flats[1]], [d4.areas[1].area_id], [d4.summaries[1]])
    with pytest.raises(capi.HspfError) as e:
        mk([no0])
    assert e.value.code == capi.HSPF_E_INVAL
    # a border that is not a B-flag router of R's flat: R's LSDB without rt5's B flag
    a = ospfv2.Ospfv2Area(**{k: getattr(bb.area, k) for k in bb.area.__dataclass_fields__})
    rl = a.router_lsas.copy()
    rl["flags"][rl["adv_rtr"] == d5.areas[0].router_id] &= ~np.uint8(1)
    a.router_lsas = rl
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.BackboneTable(ospfv2.Flat(a), a.router_id, bb.summaries, None, [d4.rt, d5.rt])
    assert e.value.code == capi.HSPF_E_INVAL
    # a border type-3 LSA for a prefix that is not one of its keys
    bad = np.concatenate([bb.summaries, np.array([(d4.areas[0].router_id, 0xC0A80000, 0xFFFFFF00, 5, 3, 0, (0, 0))],
                                                 ospf_rib.SUMMARY_LSA_DT)])
    bad = bad[np.lexsort((bad["lsa_id"], bad["adv_rtr"], bad["lsa_type"]))]
    with pytest.raises(capi.HspfError) as e:
        mk([d4.rt, d5.rt], sums=bad)
    assert e.value.code == capi.HSPF_E_INVAL
    # ... which is fine from another ABR, and so is a dead one from a border
    dead = bad.copy()
    dead["maxage"][(dead["lsa_id"] == 0xC0A80000)] = 1
    mk([d4.rt, d5.rt], sums=dead)
    # an OSPFv3 border table
    from holo_b200 import ospfv3
    v3 = ospfv3.abr_view([synth.random_topology(20, 50, synth.SEED_BASE + 990 + k, cost_choices=[10]) for k in range(2)], 3,
                         roots=[0, 0])
    fl3 = [ospfv3.Flat(a) for a in v3[0]]
    t3 = ospf_rib.AbrRibTable(v3[0][0].router_id, fl3, [a.area_id for a in v3[0]], v3[1], None, v3[2])
    assert t3.v3
    with pytest.raises(capi.HspfError) as e:
        mk([d4.rt, t3])
    assert e.value.code == capi.HSPF_E_INVAL
    # a usable type-4 LSA from a border
    t4 = np.concatenate([bb.summaries, np.array([(d4.areas[0].router_id, 0x09090909, 0, 5, 4, 0, (0, 0))],
                                                ospf_rib.SUMMARY_LSA_DT)])
    with pytest.raises(capi.HspfError) as e:
        mk([d4.rt, d5.rt], sums=t4)
    assert e.value.code == capi.HSPF_E_UNSUPPORTED


def test_virtual_link_transit_area(abr_harness, harness):
    """topo3-1: area 1 is the transit area of a virtual link between the borders rt2 and rt5, and rt5's area 2 reaches
    the backbone through it.  The borders' cells carry the transit-area step; the chain still holds."""
    bb = Backbone("topo3-1", "rt1", ["rt2", "rt5"])
    jobs = [bb.job_overrides((), 0)] + [bb.job_overrides(link, capi.COST_DISABLED) for link in non_backbone_links(bb)]
    bb.check(abr_harness, harness, jobs)


def test_virtual_link_in_area_0_is_refused():
    """A V-flag router in R's area 0: hspf_ospfv2_ribtable_create's rule (the transit-area step could rewrite R's
    intra-area routes)."""
    bb = Backbone("topo2-2", "rt1", ["rt4", "rt5"])
    a = ospfv2.Ospfv2Area(**{k: getattr(bb.area, k) for k in bb.area.__dataclass_fields__})
    rl = a.router_lsas.copy()
    rl["flags"][rl["adv_rtr"] == bb.doms[0].areas[0].router_id] |= np.uint8(0x04)
    a.router_lsas = rl
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.BackboneTable(ospfv2.Flat(a), a.router_id, bb.summaries, None, [d.rt for d in bb.doms])
    assert e.value.code == capi.HSPF_E_UNSUPPORTED


def test_job_refusals(abr_harness, harness):
    bb = Backbone("topo2-2", "rt1", ["rt4", "rt5"])
    bp = bb.border_planes([bb.job_overrides((), 0)] * 3)
    cells, st, _ = bb.cells(abr_harness, harness, bp, status=[np.array([0, 0x1, 0], np.uint32), np.array([0, 0, 0x4], np.uint32)])
    assert list(st) == [0, 0x1, 0x4]
    assert (cells["winner"][0] != ospf_rib.NO_RECORD).any()
    for j in (1, 2):
        assert (cells["winner"][j] == ospf_rib.NO_RECORD).all() and not cells["mpf"][j].any()
    cells, st, _ = bb.cells(abr_harness, harness, bp, root_status=0x2)
    assert list(st) == [0x2] * 3 and (cells["winner"] == ospf_rib.NO_RECORD).all()


def test_decode_refusals(abr_harness, harness):
    bb = Backbone("topo2-2", "rt1", ["rt4", "rt5"])
    cells, _, _ = bb.cells(abr_harness, harness, bb.border_planes([bb.job_overrides((), 0)]))
    bad = cells[0].copy()
    k = int(np.nonzero(ospf_rib.cell_path(bad) == ospf_rib.PATH_INTER)[0][0])
    bad["winner"][k] = 0xFFFFFFF0                                       # past every slot
    with pytest.raises(capi.HspfError):
        bb.decode(bad)


# ------------------------------------------------------------------------------------------- generated domains
class SynthBackbone(Backbone):
    """ospfv2.backbone_view: R and three borders of one area, with an ASBR in area 0 and a shared prefix.
    cut_border: R's row 0 with that border's area-0 links cut (the border is unreachable from R)."""

    def __init__(self, seed, V0=30, E0=90, V1=25, E1=70, cut_border=None, max_paths=16):
        t0 = synth.random_topology(V0, E0, synth.SEED_BASE + 900 + 2 * seed, cost_choices=[5, 10, 20])
        t1 = synth.random_topology(V1, E1, synth.SEED_BASE + 901 + 2 * seed, cost_choices=[5, 10, 20])
        v = ospfv2.backbone_view(t0, t1, seed, max_paths=max_paths)
        self.view = v
        self.area, self.summaries, self.externals = v["r_area"], v["summaries0"], v["externals"]
        self.flat = ospfv2.Flat(self.area)
        self.rv = self.flat.router_vertex(self.area.router_id)
        self.doms = [Domain(areas, sums, self.externals) for areas, _ids, sums in v["borders"]]
        self.cfgs = [[ospf_rib.area_config()] * 2 for _ in self.doms]
        self.table = ospf_rib.BackboneTable(self.flat, self.area.router_id, self.summaries, self.externals,
                                            [d.rt for d in self.doms])
        ov = ()
        if cut_border is not None:
            b = self.flat.router_vertex(self.doms[cut_border].areas[0].router_id)
            c = self.flat.csr
            ov = [(e, capi.COST_DISABLED) for e in range(c.n_edges)
                  if c.col[e] == b or c.row_ptr[b] <= e < c.row_ptr[b + 1]]
        self.planes = planes_of(self.flat.csr, self.rv, ov)


def synth_jobs(bb, n, seed):
    links = non_backbone_links(bb)
    rng = np.random.default_rng(seed)
    jobs = [bb.job_overrides((), 0)]
    for k in rng.choice(len(links), min(n, len(links)), replace=False):
        jobs.append(bb.job_overrides(links[int(k)], capi.COST_DISABLED))
        jobs.append(bb.job_overrides(links[int(k)], int(rng.choice([1, 40]))))
    return jobs


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_generated_domains_chain(abr_harness, harness, seed, narrow_planes):
    """Every job's decode equals the host chain on backbone_view domains; externals whose prefixes are keys take
    over a key some job makes unreachable from area 1."""
    bb = SynthBackbone(seed)
    jobs = synth_jobs(bb, 12, seed)
    cells = bb.check(abr_harness, harness, jobs, narrow_planes)
    path = ospf_rib.cell_path(cells)
    present = (ospf_rib.cell_flags(cells) & 1) != 0
    keys = {(int(p), int(l)) for p, l in zip(bb.table.prefix, bb.table.plen)}
    ext_keys = [i for i, (p, l) in enumerate(zip(bb.table.prefix, bb.table.plen))
                if any(int(x["lsa_id"]) == int(p) and bin(int(x["mask"])).count("1") == int(l) for x in bb.externals)]
    assert ext_keys and all((int(bb.table.prefix[u]), int(bb.table.plen[u])) in keys for u in ext_keys)
    assert (path[0, ext_keys] == ospf_rib.PATH_INTER).all()
    assert (present & (path == ospf_rib.PATH_INTER)).any()


def test_generated_domain_key_falls_back_to_its_external(abr_harness, harness):
    """Cutting an area-1 loopback that is also an external's prefix: R's route for the key becomes the external."""
    n = 0
    for seed in range(3):
        bb = SynthBackbone(seed)
        for x in bb.externals:
            u = np.nonzero((bb.table.prefix == x["lsa_id"]) & (bb.table.plen == 32))[0]
            if not len(u):
                continue
            # every link of the router whose loopback it is
            links = [l for l in non_backbone_links(bb) if int(x["lsa_id"]) in l]
            ovs = [bb.job_overrides(l, capi.COST_DISABLED) for l in links]
            merged = [{i: sum((o[b].get(i, []) for o in ovs), []) for i in range(2)} for b in range(len(bb.doms))]
            merged = [{i: e for i, e in m.items() if e} for m in merged]
            cells = bb.check(abr_harness, harness, [bb.job_overrides((), 0), merged])
            assert ospf_rib.cell_path(cells[0][u[0]]) == ospf_rib.PATH_INTER
            assert ospf_rib.cell_path(cells[1][u[0]]) in (ospf_rib.PATH_TYPE1, ospf_rib.PATH_TYPE2)
            n += 1
    assert n > 0


@pytest.mark.parametrize("cut", [0, 2])
def test_border_unreachable_from_r(abr_harness, harness, cut):
    """R's row 0 does not reach one border: its slots never contribute, the other borders' still do."""
    bb = SynthBackbone(1, cut_border=cut)
    assert bb.planes[0][bb.flat.router_vertex(bb.doms[cut].areas[0].router_id)] == 0xFFFFFFFF
    cells = bb.check(abr_harness, harness, synth_jobs(bb, 6, 1))
    assert ((ospf_rib.cell_flags(cells) & 1) != 0).any()


def test_shared_prefix_is_intra_area_in_both_areas_at_the_first_border(abr_harness, harness):
    """backbone_view's shared /24 ties at the first border (area 1 listed first): the border's cell is won by an
    area-1 record and carries area-0 atoms, so the border does not advertise it; R routes it intra-area."""
    bb = SynthBackbone(0)
    d = bb.doms[0]
    p, m = bb.view["shared"]
    pl = d.planes()
    c, _ = d.cells(abr_harness, pl)
    u = int(np.nonzero((d.rt.prefix == p) & (d.rt.plen == bin(m).count("1")))[0][0])
    i0 = d.rt.area_ids.index(0)
    a0 = ((1 << d.rt.n_atoms[i0]) - 1) << d.rt.atom_base[i0]
    assert ospf_rib.cell_path(c[u]) == ospf_rib.PATH_INTRA and int(c[u]["nh_mask"]) & a0 and int(c[u]["nh_mask"]) & ~a0
    assert int(c[u]["winner"]) < d.rt.off[0, -1]                    # an area-1 record (area 1 is the table's first)
    got = summaries_of(d, bb.cfgs[0], pl, i0)
    assert not ((got["lsa_id"] == p) & (got["mask"] == m)).any()
    bb.check(abr_harness, harness, [bb.job_overrides((), 0)])


def test_split_horizon_in_the_walk(abr_harness, harness):
    """A border cell won by a non-backbone record that carries an area-0 atom is not advertised.  In a consistent
    LSDB such a prefix is intra-area in area 0, so R's intra-area route hides the slot; here the border cells of an
    inter-area key at R get an area-0 atom directly, and the walk must treat the border as not advertising it."""
    bb = SynthBackbone(2)
    jobs = [bb.job_overrides((), 0)]
    cells, _, bcells = bb.cells(abr_harness, harness, bb.border_planes(jobs))
    n = 0
    for b, d in enumerate(bb.doms):
        i0 = d.rt.area_ids.index(0)
        if d.rt.n_atoms[i0] == 0:
            continue
        for u in np.nonzero(ospf_rib.cell_path(cells[0]) == ospf_rib.PATH_INTER)[0]:
            k = np.nonzero((d.rt.prefix == bb.table.prefix[u]) & (d.rt.plen == bb.table.plen[u]))[0]
            if not len(k) or not ospf_rib.cell_flags(bcells[b][0][k[0]]) & 1:
                continue
            with_atom = [c.copy() for c in bcells]
            with_atom[b][0][k[0]]["nh_mask"] |= np.uint64(1 << d.rt.atom_base[i0])
            absent = [c.copy() for c in bcells]
            absent[b][0][k[0]]["mpf"] = 0
            absent[b][0][k[0]]["winner"] = ospf_rib.NO_RECORD
            got, _ = bb.cells_from(harness, with_atom)
            want, _ = bb.cells_from(harness, absent)
            assert got.tobytes() == want.tobytes()
            n += int(got[0][u].tobytes() != cells[0][u].tobytes())
    assert n > 0
