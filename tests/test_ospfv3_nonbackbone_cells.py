"""CPU: Inter-Area-Router origination (hspf_ospfv3_rtr_summaries) and the OSPFv3 stage of an internal router of a
non-backbone area over what-if jobs on the backbone (hspf_ospfv3_nonbackbone_table_create, ospf_backbone_cell_eval
with kV3, kAsbr and kNonBackbone).

The walk is compiled into a test harness and run on the CPU over the oracle's SPT planes: R's row of its area A, each
border's routing-table cells of the job and each border's area planes of the job, which the Inter-Area-Router slots
read.  Each job perturbs area 0 only.  Every job, decoded by hspf_ospfv3_backbone_from_cells over R's image of A, must
equal byte for byte, prefix options included, the host chain: each border's update_rib_full over its job planes, its
net_summaries_v3 and rtr_summaries_v3 into A spliced into A's LSDB in LsaKey order in place of the border's own, then
update_rib_full_v3 at R, restricted to the affected prefixes."""
import ctypes as C
import subprocess
import types
from pathlib import Path

import numpy as np
import pytest

import golden_util as gu
import test_ospfv3_abr_rib_cells as v3abr
from holo_b200 import capi, ospf_rib, ospfv3, synth
from holo_b200.route_table import DELTA_OTHER
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospf_abr_rib_cells import planes_of
from test_ospf_backbone_asbr_cells import asbr_cells, ext_path
from test_ospf_rib_cells import same_rib
from test_ospf_rib_delta import reference
from test_ospfv2_route_cells import gather_for
from test_ospfv3_backbone_cells import (MULTI, Backbone, configs_of, full_image, full_inter_area_lsas, golden_domain,
                                        snap, vertex_names)
from test_ospfv3_rib_cells import rib_dict

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    """The OSPFv3 kNonBackbone walk, under the names asbr_cells calls (its arguments are the asbr harness's)."""
    out = tmp_path_factory.mktemp("harness") / "libospfv3_nonbackbone_cells_harness.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                    "-o", str(out), str(ROOT / "tests" / "native" / "ospfv3_nonbackbone_cells_harness.cc")], check=True)
    lib = C.CDLL(str(out))
    for fn in (lib.harness_ospfv3_nonbackbone_cells, lib.harness_ospfv3_nonbackbone_cells16):
        fn.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 8
        fn.restype = C.c_int
    lib.harness_backbone_winners_fit.argtypes = [C.c_uint64, C.c_uint64, C.c_int]
    return types.SimpleNamespace(lib=lib, harness_ospf_backbone_asbr_cells=lib.harness_ospfv3_nonbackbone_cells,
                                 harness_ospf_backbone_asbr_cells16=lib.harness_ospfv3_nonbackbone_cells16)


def oracle_spf(csr, root, nhw):
    d, h, m = planes_of(csr, root)
    return d, h, np.pad(m[:, None], ((0, 0), (0, nhw - 1)))


def spf_of(p):
    return lambda csr, root, nhw: (p[0], p[1], np.pad(p[2][:, None], ((0, 0), (0, nhw - 1))))


def job_rib_areas(d, job_planes):
    """A border's RibArea list over its job planes (results included), as update_rib_full_v3 takes it."""
    return [ospf_rib.RibArea(a.area_id, ospfv3.area_from_planes(a, spf_of(p)), a.ifaces, d.summaries[i], d.active[i])
            for i, (a, p) in enumerate(zip(d.areas, job_planes))]


def area0_links(doms):
    """Vertex-name pairs of the router links of the borders' area 0."""
    out = set()
    for d in doms:
        for a, f in zip(d.areas, d.flats):
            if a.area_id != 0:
                continue
            names = vertex_names(f)
            src = np.repeat(np.arange(f.csr.n_vertices), np.diff(f.csr.row_ptr))
            for e in range(f.csr.n_edges):
                if f.is_router[src[e]]:
                    out.add(tuple(sorted((names[src[e]], names[f.csr.col[e]]))))
    return sorted(out)


def srt(x):
    return x[np.lexsort((x["lsa_id"], x["adv_rtr"], x["lsa_type"]))] if len(x) else x


class NonBackbone(Backbone):
    """R of area A, its borders' OSPFv3 ABR domains and the table.  Subclasses set area, summaries, externals, doms,
    cfgs and config, then call _finish."""

    def _finish(self):
        self.flat = ospfv3.Flat(self.area)
        self.rv = self.flat.router_vertex(self.area.router_id)
        self.make_table()
        self.planes = planes_of(self.flat.csr, self.rv)

    def make_table(self):
        self.table = ospf_rib.BackboneTable(self.flat, self.area.router_id, self.summaries, self.externals,
                                            [d.rt for d in self.doms], config=self.config)

    def job_overrides(self, link, cost):
        """Per border, per area: the overrides of link (vertex-name pair) at `cost` in the borders' area 0."""
        out = []
        for d in self.doms:
            ov = {}
            for i, (a, f) in enumerate(zip(d.areas, d.flats)):
                if a.area_id != 0:
                    continue
                names = vertex_names(f)
                src = np.repeat(np.arange(f.csr.n_vertices), np.diff(f.csr.row_ptr))
                e = [(int(k), cost) for k in range(f.csr.n_edges) if {names[src[k]], names[f.csr.col[k]]} == set(link)]
                if e:
                    ov[i] = e
            out.append(ov)
        return out

    def cut(self, rid, borders=None):
        """A job: every area-0 link of router `rid` disabled in the area planes of the borders in `borders` (all:
        None)."""
        ovs = [self.job_overrides(l, capi.COST_DISABLED) for l in area0_links(self.doms)
               if any(x[0] == rid and x[2] for x in l)]
        return [{} if borders is not None and b not in borders else
                {i: e for i in range(len(d.areas)) if (e := sum((o[b].get(i, []) for o in ovs), []))}
                for b, d in enumerate(self.doms)]

    def cells(self, abr, harness, bplanes, narrow_planes=False, status=None, root_status=0):
        bcells = [np.stack([d.cells(abr, p, narrow_planes)[0] for p in bp]) for d, bp in zip(self.doms, bplanes)]
        cells, out = asbr_cells(harness, self.table, self.planes, bcells, bplanes, narrow_planes, status, root_status)
        return cells, out, bcells

    def lsdb(self, bplanes_of_job):
        """A's LSDB of the job: each border's Inter-Area-Prefix / Inter-Area-Router LSAs re-originated."""
        bid = {d.areas[0].router_id for d in self.doms}
        new = [tuple(s) for s in self.summaries.tolist() if int(s[0]) not in bid]
        for d, cfg, p in zip(self.doms, self.cfgs, bplanes_of_job):
            ia = next(i for i, a in enumerate(d.areas) if a.area_id == self.area.area_id)
            new += ospfv3.nonbackbone_lsas(d.areas[0].router_id, d.areas[0].max_paths, job_rib_areas(d, p),
                                           d.externals, ia, cfg)
        return srt(np.array(new, ospf_rib.INTER_AREA_LSA_DT))

    def host(self, bcells_of_job, bplanes_of_job):
        ra = [ospf_rib.RibArea(self.area.area_id, ospfv3.area_from_planes(self.area, spf_of(self.planes)),
                               self.area.ifaces, self.lsdb(bplanes_of_job), True)]
        return self.affected(ospf_rib.update_rib_full_v3(self.area.router_id, self.area.max_paths, ra, self.externals))


class GoldenNonBackbone(NonBackbone):
    """R's recorded area image and LSDB; the borders from their own snapshots; A's configuration as the borders
    recorded it."""

    def __init__(self, topo, r, borders):
        sr = snap(topo, r)
        self.keys, self.snap = gu.global_sort_keys(sr), sr
        assert len(sr["areas"]) == 1
        a = sr["areas"][0]
        self.area = full_image(sr, a, self.keys)
        self.summaries, self.externals = full_inter_area_lsas(a), None
        self.bsnaps = [snap(topo, b) for b in borders]
        self.doms = [golden_domain(b)[0] for b in self.bsnaps]
        self.cfgs = [configs_of(b, d) for b, d in zip(self.bsnaps, self.doms)]
        d0 = self.doms[0]
        self.config = self.cfgs[0][[x.area_id for x in d0.areas].index(self.area.area_id)]
        self._finish()


class SynthNonBackbone(NonBackbone):
    """ospfv3.nonbackbone_view: R of area 1, three borders (the first also in area 2), an area-0 ASBR with
    AS-external LSAs, the inter-area flip."""

    def __init__(self, seed, V0=30, E0=90, V1=25, E1=70, n_ext=4, max_paths=16):
        t0 = synth.random_topology(V0, E0, synth.SEED_BASE + 960 + 2 * seed, cost_choices=[5, 10, 20])
        t1 = synth.random_topology(V1, E1, synth.SEED_BASE + 961 + 2 * seed, cost_choices=[5, 10, 20])
        v = ospfv3.nonbackbone_view(t0, t1, seed, oracle_spf, max_paths=max_paths, n_ext=n_ext)
        self.view = v
        self.area, self.summaries, self.externals = v["r_area"], v["summaries1"], v["externals"]
        self.doms = [v3abr.Domain(areas, sums, self.externals) for areas, _ids, sums in v["borders"]]
        self.cfgs = [[ospf_rib.area_config()] * len(d.areas) for d in self.doms]
        self.config = ospf_rib.area_config()
        self._finish()

    def key_index(self, key):
        b = np.frombuffer(key[0], np.uint8)
        u = [i for i in range(self.table.n_prefixes)
             if (self.table.prefixes6[i]["bytes"] == b).all() and int(self.table.plen[i]) == key[1]]
        return u[0] if u else None


def chain_jobs(bb, costs=(capi.COST_DISABLED, 35)):
    jobs = [bb.job_overrides((), 0)]
    for link in area0_links(bb.doms):
        jobs += [bb.job_overrides(link, c) for c in costs]
    return jobs


# ------------------------------------------------------------------------------------- Inter-Area-Router origination
@pytest.mark.parametrize("s", MULTI, ids=[f"{s['topo']}-{s['rt']}" for s in MULTI])
def test_rtr_summaries_empty_on_the_snapshots(s):
    """The fixture records no Inter-Area-Router LSA in any area of the 14 multi-area snapshots: no ASBR there."""
    dom, _ = golden_domain(s)
    cfg = configs_of(s, dom)
    ra = job_rib_areas(dom, dom.planes())
    for i in range(len(dom.areas)):
        assert len(ospf_rib.rtr_summaries_v3(dom.areas[0].router_id, ra, cfg, i)) == 0


def restated(rid, ra, cfgs, target):
    """compute_rtr_summaries restated over the areas' SPF routers and area 0's Inter-Area-Router LSAs."""
    act = sum(bool(a.active) for a in ra)
    if act <= 1 or cfgs[target][1] != ospf_rib.AREA_NORMAL:
        return {}
    ta = ra[target]
    ifs = {int(x["sort_key"]) for x in ta.ifaces}
    tabs = []
    for a in ra:
        t = {}
        for r in a.result.routers:
            hops = a.result.nexthops[int(r["nh_off"]): int(r["nh_off"]) + int(r["n_nh"])]
            t[int(r["router_id"])] = (a.area_id, int(r["metric"]), ospf_rib.PATH_INTRA, int(r["flags"]),
                                      {int(a.ifaces[int(h["iface"])]["sort_key"]) for h in hops})
        tabs.append(t)
    for a, t in zip(ra, tabs):
        if a.area_id != 0:
            continue
        for l in a.summaries:
            if int(l["lsa_type"]) != 4 or l["maxage"] or int(l["metric"]) >= 0xFFFFFF or int(l["adv_rtr"]) == rid:
                continue
            br = t.get(int(l["adv_rtr"]))
            if br and br[3] & 0x01:
                t[int(l["router_id"])] = (0, br[1] + int(l["metric"]), ospf_rib.PATH_INTER, 0x02, br[4])
    out = {}
    for t in tabs:
        for x, (aid, m, path, fl, sk) in sorted(t.items()):
            if aid == ta.area_id or not fl & 0x02 or m >= 0xFFFFFF:
                continue
            if ta.area_id == 0 and path != ospf_rib.PATH_INTRA:
                continue
            if sk & ifs:
                continue
            out[x] = m
    return out


@pytest.mark.parametrize("seed", range(3))
def test_rtr_summaries_equal_a_restatement(seed):
    """Every border of the generated domains, into each of its areas."""
    bb = SynthNonBackbone(seed)
    n = 0
    for d in bb.doms:
        ra = job_rib_areas(d, d.planes())
        for i in range(len(d.areas)):
            cfg = [ospf_rib.area_config()] * len(d.areas)
            got = ospf_rib.rtr_summaries_v3(d.areas[0].router_id, ra, cfg, i)
            assert (got["lsa_type"] == 4).all() and (got["adv_rtr"] == d.areas[0].router_id).all()
            assert list(got["router_id"]) == sorted(got["router_id"])
            assert {int(x["router_id"]): int(x["metric"]) for x in got} == restated(d.areas[0].router_id, ra, cfg, i)
            n += len(got)
    assert n > 0


def test_rtr_summaries_on_a_large_domain():
    """A border of a 4 000-router area 0: the output buffer (one entry per router, 160 kB) is allocated outside the
    small heap, so its pointer must cross the C ABI whole (the call's signature is declared)."""
    assert capi.load_library().hspf_ospfv3_rtr_summaries.argtypes is not None
    t0 = synth.random_topology(4000, 12000, synth.SEED_BASE + 970, cost_choices=[5, 10, 20])
    t1 = synth.random_topology(25, 70, synth.SEED_BASE + 971, cost_choices=[5, 10, 20])
    v = ospfv3.nonbackbone_view(t0, t1, 0, oracle_spf)
    areas, ids, sums = v["borders"][1]
    d = v3abr.Domain(areas, sums, v["externals"])
    ra = job_rib_areas(d, d.planes())
    cfg = [ospf_rib.area_config()] * len(areas)
    got = ospf_rib.rtr_summaries_v3(areas[0].router_id, ra, cfg, ids.index(1))
    assert v["asbr"] in set(got["router_id"].tolist())
    assert {int(x["router_id"]): int(x["metric"]) for x in got} == restated(areas[0].router_id, ra, cfg, ids.index(1))


def test_rtr_summaries_hand_cases():
    """A stub target takes none; an entry with a next hop on a target interface is left out; an inter-area entry goes
    into a non-backbone area only; an id in two areas keeps the later area's."""
    bb = SynthNonBackbone(0)
    d = bb.doms[1]                                       # areas 0, 1
    ra = job_rib_areas(d, d.planes())
    rid, asbr = d.areas[0].router_id, bb.view["asbr"]
    cfg = [ospf_rib.area_config()] * 2
    i0, i1 = d.rt.area_ids.index(0), d.rt.area_ids.index(1)
    base = ospf_rib.rtr_summaries_v3(rid, ra, cfg, i1)
    assert asbr in set(base["router_id"].tolist())
    assert len(ospf_rib.rtr_summaries_v3(rid, ra, cfg, i0)) == 0          # area 0's ASBR is area 0's own
    stub = list(cfg)
    stub[i1] = ospf_rib.area_config(ospf_rib.AREA_STUB)
    assert len(ospf_rib.rtr_summaries_v3(rid, ra, stub, i1)) == 0
    # the next-hop rule: the ASBR's next hops named as the target area's interfaces
    r1 = ra[i1]
    hops = [int(x["sort_key"]) for x in ra[i0].ifaces]
    ifs = r1.ifaces.copy()
    ifs0 = np.concatenate([ifs, ra[i0].ifaces])
    on = [ospf_rib.RibArea(a.area_id, a.result, ifs0 if k == i1 else a.ifaces, a.summaries, a.active)
          for k, a in enumerate(ra)]
    assert hops and asbr not in set(ospf_rib.rtr_summaries_v3(rid, on, cfg, i1)["router_id"].tolist())
    # an inter-area entry (an Inter-Area-Router LSA in area 0 from another ABR) into area 1, not into area 0
    other = next(dd for dd in bb.doms if dd is not d).areas[0].router_id
    iar = np.array([(other, 0x55, 3, 0x0C000001, ospfv3.ip_rec("::"), 0, 0, 4, 0)], ospf_rib.INTER_AREA_LSA_DT)
    with4 = [ospf_rib.RibArea(a.area_id, a.result, a.ifaces, srt(np.concatenate([a.summaries, iar])) if k == i0 else
                              a.summaries, a.active) for k, a in enumerate(ra)]
    got = ospf_rib.rtr_summaries_v3(rid, with4, cfg, i1)
    assert 0x0C000001 in set(got["router_id"].tolist())
    assert 0x0C000001 not in set(ospf_rib.rtr_summaries_v3(rid, with4, cfg, i0)["router_id"].tolist())
    # an id in two areas: area 0's ASBR also an E-flag router of area 2, a copy of area 0 at three times its link
    # costs; the entry of whichever area comes later in the call is the one originated
    twin = ospfv3.Ospfv3Area(**{k: getattr(d.areas[i0], k) for k in d.areas[i0].__dataclass_fields__})
    twin.area_id = 2
    ifs2 = twin.ifaces.copy()
    ifs2["sort_key"] += 50000
    twin.ifaces = ifs2
    lk = twin.links.copy()
    lk["metric"] *= 3
    twin.links = lk
    p2 = planes_of(ospfv3.Flat(twin).csr, ospfv3.Flat(twin).router_vertex(rid))
    r2 = ospf_rib.RibArea(2, ospfv3.area_from_planes(twin, spf_of(p2)), twin.ifaces, np.zeros(0, ospf_rib.INTER_AREA_LSA_DT))
    m0 = int(base[base["router_id"] == asbr]["metric"][0])
    c3 = cfg + [ospf_rib.area_config()]
    for areas, target, want in ((ra + [r2], i1, 3 * m0), ([r2] + ra, i1 + 1, m0)):
        got = ospf_rib.rtr_summaries_v3(rid, areas, c3, target)
        assert int(got[got["router_id"] == asbr]["metric"][0]) == want
        assert restated(rid, areas, c3, target) == {int(x["router_id"]): int(x["metric"]) for x in got}


# ------------------------------------------------------------------------------------------ recorded data
GOLDEN = [(f"topo1-{k}", r, [b]) for k in (1, 2) for r, b in (("rt1", "rt2"), ("rt5", "rt4"), ("rt7", "rt6"))] + \
         [("topo2-2", "rt6", ["rt4", "rt5"]), ("topo3-1", "rt6", ["rt5"]), ("topo3-3", "rt6", ["rt5"])]
GIDS = [f"{t}-{r}" for t, r, _ in GOLDEN]


@pytest.mark.parametrize("g", GOLDEN, ids=GIDS)
def test_base_job_equals_the_recorded_local_rib(abr_harness, harness, g):
    """Job 0 equals R's recorded local-rib over the affected prefixes: metric, route type, next hops, and the prefix
    options the host chain gives."""
    bb = GoldenNonBackbone(*g)
    cells, _ = bb.check(abr_harness, harness, [bb.job_overrides((), 0)])
    got = bb.decode(cells[0])
    mine = rib_dict(got, {v: k for k, v in bb.keys.items()})
    keys = {f"{ospfv3.ip_str(p)}/{int(l)}" for p, l in zip(bb.table.prefixes6, bb.table.plen)}
    want = {k: v for k, v in gu.golden_rib(bb.snap).items() if k in keys}
    norm = lambda d: {k: (v[0], v[1], [(a or "", b or "") for a, b in v[2]]) for k, v in d.items()}
    assert norm(mine) == norm(want)
    assert bb.table.v3 and bb.table.area_id == bb.area.area_id
    if bb.config[2] == 0:                                              # totally stubby: only the static default
        assert bb.table.n_prefixes == 0 and bb.table.n_slots == 0
    else:
        assert bb.table.n_prefixes > 0 and bb.table.n_slots > 0
    if bb.config[1] == ospf_rib.AREA_STUB:
        assert not any(int(l) == 0 and not p["bytes"].any() for p, l in zip(bb.table.prefixes6, bb.table.plen))
        assert bb.table.n_asbr_slots == 0


@pytest.mark.parametrize("g", GOLDEN, ids=GIDS)
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_chain_area0_link_failed_or_recosted(abr_harness, harness, g, narrow_planes):
    """Every area-0 link failed, then re-costed to 35, at every border that has it, all jobs in one batch."""
    bb = GoldenNonBackbone(*g)
    jobs = chain_jobs(bb)
    assert len(jobs) > 1
    bb.check(abr_harness, harness, jobs, narrow_planes)


def test_stub_default_stays_static(abr_harness, harness):
    """topo1 rt5 (stub area): the border's ::/0 is a static record at default_cost, in every job."""
    bb = GoldenNonBackbone("topo1-1", "rt5", ["rt4"])
    assert bb.config[1] == ospf_rib.AREA_STUB
    bb.check(abr_harness, harness, chain_jobs(bb))
    dflt = [x for x in bb.summaries if int(x["lsa_type"]) == 3 and int(x["len"]) == 0]
    assert dflt and int(dflt[0]["metric"]) == bb.config[0]


@pytest.mark.parametrize("topo", ["topo3-1", "topo3-3"])
@pytest.mark.parametrize("r", ["rt3", "rt4"])
def test_transit_area_routers_are_refused(topo, r):
    sr = snap(topo, r)
    a = sr["areas"][0]
    area = full_image(sr, a, gu.global_sort_keys(sr))
    dom = golden_domain(snap(topo, "rt5"))[0]
    cfg = configs_of(snap(topo, "rt5"), dom)[[x.area_id for x in dom.areas].index(area.area_id)]
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.BackboneTable(ospfv3.Flat(area), area.router_id, full_inter_area_lsas(a), None, [dom.rt], config=cfg)
    assert e.value.code == capi.HSPF_E_UNSUPPORTED


# ------------------------------------------------------------------------------------------ generated domains
@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_generated_domains_chain(abr_harness, harness, seed, narrow_planes):
    """Every area-0 link failed and re-costed, one job each; the area-0 ASBR's externals route through the borders'
    Inter-Area-Router slots, which read the borders' area-0 plane sets."""
    bb = SynthNonBackbone(seed)
    assert bb.table.n_asbr_slots > 0 and bb.table.n_asbr_sets == 3
    cells, _ = bb.check(abr_harness, harness, chain_jobs(bb, (capi.COST_DISABLED, 37)), narrow_planes)
    assert ext_path(cells[0]).any()
    assert (cells != cells[0]).any()
    assert bb.key_index(bb.view["flip"][:2]) is not None


def test_asbr_unreachable_from_one_border_moves_to_another(abr_harness, harness):
    """The area-0 ASBR cut off at the last border in LsaKey order only: its externals at R move to an earlier border's
    slot; every one still routes."""
    n = 0
    for seed in range(3):
        bb = SynthNonBackbone(seed)
        last = max(range(3), key=lambda b: bb.doms[b].areas[0].router_id)
        cells, _ = bb.check(abr_harness, harness, [bb.job_overrides((), 0), bb.cut(bb.view["asbr"], {last})])
        u = np.nonzero(ext_path(cells[0]))[0]
        assert len(u) and ext_path(cells[1][u]).all()
        n += int(cells[1][u].tobytes() != cells[0][u].tobytes())
    assert n > 0


def test_inter_area_flip_at_an_equal_metric_is_other(abr_harness, harness):
    """The flip /128 is inter-area at the first border, from two area-0 LSAs that tie there with other options.  A job
    that cuts the first advertiser off at the first border alone hands the border's route to the other LSA at the same
    metric: where R's route goes through that border, R's winner changes at the same metric and next hops, the delta
    reports OTHER, and the decode gives the other options."""
    n = 0
    for seed in range(3):
        bb = SynthNonBackbone(seed)
        key, _ln, x, _y = bb.view["flip"]
        cut = bb.cut(x, {0})
        cells, _ = bb.check(abr_harness, harness, [bb.job_overrides((), 0), cut])
        u = bb.key_index(bb.view["flip"][:2])
        a, b = cells[0][u], cells[1][u]
        assert ospf_rib.cell_path(a) == ospf_rib.PATH_INTER
        if int(a["mpf"]) == int(b["mpf"]) and int(a["nh_mask"]) == int(b["nh_mask"]) and a["winner"] != b["winner"]:
            _jobs, recs, _ = reference(cells, cells[:1])
            assert any(int(r["prefix"]) == u and int(r["kind"]) == DELTA_OTHER for r in recs if int(r["job"]) == 1)
            o = lambda rib: {(z["prefix"].tobytes()[:16], int(z["len"])): int(z["prefix_options"]) for z in rib.routes}
            assert {o(bb.decode(cells[0]))[(key, 128)], o(bb.decode(cells[1]))[(key, 128)]} == \
                {ospfv3.PFX_LA, ospfv3.PFX_P}
            n += 1
    assert n > 0


# ------------------------------------------------------------------------------------------- refusals
def test_table_refusals():
    bb = SynthNonBackbone(0)
    rts = [d.rt for d in bb.doms]
    cfg = ospf_rib.area_config()

    def refused(code, flat=None, rid=None, sums=None, borders=None, config=cfg, ext=bb.externals):
        with pytest.raises(capi.HspfError) as e:
            ospf_rib.BackboneTable(flat or bb.flat, rid or bb.area.router_id, bb.summaries if sums is None else sums,
                                   ext, rts if borders is None else borders, config=config)
        assert e.value.code == code

    # a flat of area 0: a border's area-0 image, R there being the border's neighbour
    a0 = next(a for a in bb.doms[1].areas if a.area_id == 0)
    refused(capi.HSPF_E_INVAL, flat=ospfv3.Flat(a0), rid=a0.router_id)
    # a NULL config: the create called directly
    h = C.c_void_p()
    arr = (C.c_void_p * 3)(*[r.handle.value for r in rts])
    lib = capi.load_library()
    assert lib.hspf_ospfv3_nonbackbone_table_create(bb.flat.handle, bb.area.router_id, None,
                                                    bb.summaries.ctypes.data, len(bb.summaries), None, 0, arr, 3,
                                                    C.byref(h)) == capi.HSPF_E_INVAL
    # R missing, R with the B flag (a border as R)
    refused(capi.HSPF_E_INVAL, rid=0x0909FFFF)
    a1 = next(a for a in bb.doms[1].areas if a.area_id == 1)
    refused(capi.HSPF_E_INVAL, flat=ospfv3.Flat(a1), rid=a1.router_id, borders=[rts[0], rts[2]])
    # a border table without area 0, or without A
    d = bb.doms[1]
    for keep in (0, 1):
        i = d.rt.area_ids.index(keep)
        only = ospf_rib.AbrRibTable(d.areas[i].router_id, [d.flats[i]], [keep], [d.summaries[i]], None, bb.externals)
        refused(capi.HSPF_E_INVAL, borders=[rts[0], only, rts[2]])
    # a border given twice, an OSPFv2 border table
    refused(capi.HSPF_E_INVAL, borders=[rts[0], rts[0], rts[1]])
    import test_ospf_abr_rib_cells as v2abr
    refused(capi.HSPF_E_INVAL, borders=[rts[0], v2abr.domain(0).rt])
    # a border's Inter-Area-Prefix LSA for a prefix it cannot advertise, an Inter-Area-Router LSA for a router it
    # cannot originate for; dead ones are fine
    b0 = bb.doms[0].areas[0].router_id
    for extra in ((b0, 0x777, 5, 0, ospfv3.ip_rec("2001:db8:9999::"), 64, 0, 3, 0),
                  (b0, 0x778, 5, 0x09090909, ospfv3.ip_rec("::"), 0, 0, 4, 0)):
        bad = srt(np.concatenate([bb.summaries, np.array([extra], ospf_rib.INTER_AREA_LSA_DT)]))
        refused(capi.HSPF_E_INVAL, sums=bad)
        dead = bad.copy()
        dead["maxage"][(dead["lsa_id"] == extra[1]) & (dead["adv_rtr"] == b0)] = 1
        ospf_rib.BackboneTable(bb.flat, bb.area.router_id, dead, bb.externals, rts, config=cfg)
    # NSSA
    refused(capi.HSPF_E_UNSUPPORTED, config=ospf_rib.area_config(ospf_rib.AREA_NSSA))
    # a V-flag router in A
    a = ospfv3.Ospfv3Area(**{k: getattr(bb.area, k) for k in bb.area.__dataclass_fields__})
    rl = a.router_lsas.copy()
    rl["flags"][rl["adv_rtr"] == b0] |= np.uint8(0x04)
    a.router_lsas = rl
    refused(capi.HSPF_E_UNSUPPORTED, flat=ospfv3.Flat(a))
    # a usable Inter-Area-Router LSA of another ABR in a border's area-0 LSAs
    b1 = bb.doms[1].areas[0].router_id
    doms = []
    for dm in bb.doms:
        s = list(dm.summaries)
        i0 = dm.rt.area_ids.index(0)
        if dm.areas[0].router_id != b1:
            s[i0] = srt(np.concatenate([s[i0], np.array([(b1, 0x779, 5, 0x0A0B0C0D, ospfv3.ip_rec("::"), 0, 0, 4, 0)],
                                                         ospf_rib.INTER_AREA_LSA_DT)]))
        doms.append(v3abr.Domain(dm.areas, s, dm.externals))
    refused(capi.HSPF_E_UNSUPPORTED, borders=[x.rt for x in doms])
    # an E+B router in a border's area other than A: the area-0 ASBR given the B flag there
    doms = []
    for dm in bb.doms:
        areas = []
        for ar in dm.areas:
            if ar.area_id == 0:
                ar = ospfv3.Ospfv3Area(**{k: getattr(ar, k) for k in ar.__dataclass_fields__})
                rl = ar.router_lsas.copy()
                rl["flags"][rl["adv_rtr"] == bb.view["asbr"]] |= np.uint8(0x01)
                ar.router_lsas = rl
            areas.append(ar)
        doms.append(v3abr.Domain(areas, dm.summaries, dm.externals))
    refused(capi.HSPF_E_UNSUPPORTED, borders=[x.rt for x in doms])
    # 0 or more than 8 borders
    refused(capi.HSPF_E_UNSUPPORTED, borders=[])
    refused(capi.HSPF_E_UNSUPPORTED, borders=[rts[0]] * 9)


def test_slot_winners_must_fit_32_bits(harness):
    """The create refuses a table whose slot winners would not fit 32 bits (HSPF_E_UNSUPPORTED).  A real table there
    needs about 2^24 OSPFv3 slots, millions of prefixes per border, so the rule the builder applies
    (backbone_winners_fit) is checked at its boundary: n_recs + (slots << 8) must stay below 0xFFFFFFFF."""
    fit = harness.lib.harness_backbone_winners_fit
    S = 0xFFFFFF
    assert fit(0xFE, S, 1) == 1 and fit(0xFF, S, 1) == 0 and fit(0, S + 1, 1) == 0
    assert fit(0xFF, S, 0) == 1 and fit(0xFFFFFFFE - S, S, 0) == 1 and fit(0xFFFFFFFF - S, S, 0) == 0
    bb = SynthNonBackbone(0)
    assert fit(bb.table.n_records, bb.table.n_slots, 1) == 1


def test_more_than_8_plane_sets_are_refused():
    """The area-0 ASBR is also an E-flag router of copies of area 0 added to the borders: each (border, area) pair is a
    plane set, and three borders with three such areas read nine."""
    bb = SynthNonBackbone(0)

    def with_twins(d, n):
        i0 = d.rt.area_ids.index(0)
        twins = []
        for k in range(n):
            t = ospfv3.Ospfv3Area(**{f: getattr(d.areas[i0], f) for f in d.areas[i0].__dataclass_fields__})
            t.area_id = 3 + k
            twins.append(t)
        return v3abr.Domain(d.areas + twins, list(d.summaries) + [np.zeros(0, ospf_rib.INTER_AREA_LSA_DT)] * n,
                            d.externals)

    mk = lambda doms: ospf_rib.BackboneTable(bb.flat, bb.area.router_id, bb.summaries, bb.externals,
                                             [d.rt for d in doms], config=ospf_rib.area_config())
    t = mk([with_twins(bb.doms[0], 1)] + bb.doms[1:])
    assert t.n_asbr_sets == 4
    with pytest.raises(capi.HspfError) as e:
        mk([with_twins(d, 2) for d in bb.doms])
    assert e.value.code == capi.HSPF_E_UNSUPPORTED


def test_asbr_flag_and_other_area_decode_are_refused(abr_harness, harness):
    """asbr=True with an OSPFv3 flat still raises (the area-0 create's own refusals are test_ospfv3_backbone_cells'),
    and the decode of a non-backbone table refuses R's image of another area."""
    bb = SynthNonBackbone(1)
    with pytest.raises(ValueError):
        ospf_rib.BackboneTable(bb.flat, bb.area.router_id, bb.summaries, bb.externals, [d.rt for d in bb.doms],
                               asbr=True)
    cells, _, _ = bb.cells(abr_harness, harness, bb.border_planes([bb.job_overrides((), 0)]))
    other = ospfv3.Ospfv3Area(**{k: getattr(bb.area, k) for k in bb.area.__dataclass_fields__})
    other.area_id = 0
    v, n = gather_for(bb.flat, bb.rv, bb.planes)
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.backbone_from_cells_v3(other, bb.table, cells[0], v, n)
    assert e.value.code == capi.HSPF_E_INVAL
    bb.decode(cells[0])


def test_job_status_rows(abr_harness, harness):
    """A border row out of range refuses the job (HSPF_JS_INVALID, empty cells); a read row's status word is ORed in;
    the other jobs are unchanged."""
    bb = SynthNonBackbone(1)
    jobs = chain_jobs(bb)[:5]
    bp = bb.border_planes(jobs)
    want, st, bcells = bb.cells(abr_harness, harness, bp)
    assert not st.any()
    J = len(jobs)
    rows = [np.repeat(np.arange(J, dtype=np.uint32)[:, None], len(d.areas), 1) for d in bb.doms]
    rows[1][2, :] = J
    ps = [[np.zeros(J, np.uint32) for _ in d.areas] for d in bb.doms]
    for i in range(len(bb.doms[0].areas)):
        ps[0][i][1] = 0x8
    got, st = asbr_cells(harness, bb.table, bb.planes, bcells, bp, rows=rows, pstatus=ps)
    assert st[2] & capi.JS_INVALID and st[1] == 0x8
    for j in (1, 2):
        assert (got["winner"][j] == ospf_rib.NO_RECORD).all() and not got["mpf"][j].any()
    keep = [j for j in range(J) if j not in (1, 2)]
    assert got[keep].tobytes() == want[keep].tobytes()
