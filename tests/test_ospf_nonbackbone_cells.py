"""CPU: the OSPFv2 stage of an internal router of a non-backbone area over what-if jobs on the backbone
(hspf_ospfv2_nonbackbone_table_create, ospf_backbone_cell_eval with kAsbr and kNonBackbone).

The walk is compiled into a test harness and run on the CPU over the oracle's SPT planes: R's row of its area A, each
border's routing-table cells of the job and each border's area planes of the job, which the type-4 slots read.  Each
job perturbs area 0 only.  Every job, decoded by hspf_ospfv2_backbone_from_cells over R's image of A, must equal byte
for byte the host chain: each border's update_rib_full over its job planes, its router tables and net_summaries into
A, type 3 and type 4 spliced into A's LSDB in LsaKey order in place of the border's own, then update_rib_full at R,
restricted to the affected prefixes."""
import ctypes as C
import subprocess
import types
from pathlib import Path

import numpy as np
import pytest

import golden_util as gu
from holo_b200 import capi, ospf_rib, ospfv2, synth
from test_ospf_abr_rib_cells import Domain, golden_domain, planes_of
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospf_backbone_asbr_cells import asbr_cells, ext_path
from test_ospf_backbone_cells import Backbone, configs_of, snap, summaries_of
from test_ospf_rib_cells import harness as rib_harness  # noqa: F401  (fixture)
from test_ospf_rib_cells import harness_cells as rib_cells
from test_ospf_rib_cells import same_rib
from test_ospfv2_route_cells import gather_for

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    """The kNonBackbone walk, under the names asbr_cells calls (its arguments are the asbr harness's)."""
    out = tmp_path_factory.mktemp("harness") / "libospf_nonbackbone_cells_harness.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                    "-o", str(out), str(ROOT / "tests" / "native" / "ospf_nonbackbone_cells_harness.cc")], check=True)
    lib = C.CDLL(str(out))
    for fn in (lib.harness_ospf_nonbackbone_cells, lib.harness_ospf_nonbackbone_cells16):
        fn.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 8
    return types.SimpleNamespace(lib=lib, harness_ospf_backbone_asbr_cells=lib.harness_ospf_nonbackbone_cells,
                                 harness_ospf_backbone_asbr_cells16=lib.harness_ospf_nonbackbone_cells16)


def oracle_spf(csr, root, nhw):
    d, h, m = planes_of(csr, root)
    return d, h, np.pad(m[:, None], ((0, 0), (0, nhw - 1)))


def area0_links(doms):
    """Vertex-id pairs of the router links of the borders' area 0."""
    out = set()
    for d in doms:
        for a, f in zip(d.areas, d.flats):
            if a.area_id != 0:
                continue
            ids = [int(x) for x in f.ids]
            src = np.repeat(np.arange(f.csr.n_vertices), np.diff(f.csr.row_ptr))
            for e in range(f.csr.n_edges):
                if f.is_router[src[e]]:
                    out.add(tuple(sorted((ids[src[e]], ids[f.csr.col[e]]))))
    return sorted(out)


class NonBackbone(Backbone):
    """R of area A, its borders' ABR domains and the table.  Subclasses set area, summaries, externals, doms, cfgs
    and config, then call _finish."""

    def _finish(self):
        self.flat = ospfv2.Flat(self.area)
        self.rv = self.flat.router_vertex(self.area.router_id)
        self.table = ospf_rib.BackboneTable(self.flat, self.area.router_id, self.summaries, self.externals,
                                            [d.rt for d in self.doms], config=self.config)
        self.planes = planes_of(self.flat.csr, self.rv)

    def job_overrides(self, link, cost):
        """Per border, per area: the overrides of link (router id pair) at `cost` in the borders' area 0."""
        out = []
        for d in self.doms:
            ov = {}
            for i, (a, f) in enumerate(zip(d.areas, d.flats)):
                if a.area_id != 0:
                    continue
                ids = [int(x) for x in f.ids]
                src = np.repeat(np.arange(f.csr.n_vertices), np.diff(f.csr.row_ptr))
                e = [(int(k), cost) for k in range(f.csr.n_edges) if {ids[src[k]], ids[f.csr.col[k]]} == set(link)]
                if e:
                    ov[i] = e
            out.append(ov)
        return out

    def cut(self, x, borders=None):
        """A job: every area-0 link of router x disabled in the area planes of the borders in `borders` (all: None)."""
        ovs = [self.job_overrides(l, capi.COST_DISABLED) for l in area0_links(self.doms) if x in l]
        return [{} if borders is not None and b not in borders else
                {i: e for i in range(len(d.areas)) if (e := sum((o[b].get(i, []) for o in ovs), []))}
                for b, d in enumerate(self.doms)]

    def cells(self, abr, harness, bplanes, narrow_planes=False, status=None, root_status=0):
        bcells = [np.stack([d.cells(abr, p, narrow_planes)[0] for p in bp]) for d, bp in zip(self.doms, bplanes)]
        cells, out = asbr_cells(harness, self.table, self.planes, bcells, bplanes, narrow_planes, status, root_status)
        return cells, out, bcells

    def host(self, job_planes_per_border):
        """The chain with each border's type-3 and type-4 LSAs into A re-originated."""
        bid = {d.areas[0].router_id for d in self.doms}
        new = [s for s in self.summaries if int(s["adv_rtr"]) not in bid]
        for d, cfg, p in zip(self.doms, self.cfgs, job_planes_per_border):
            ia = next(i for i, a in enumerate(d.areas) if a.area_id == self.area.area_id)
            new += list(summaries_of(d, cfg, p, ia))
        s = np.array(new, ospf_rib.SUMMARY_LSA_DT)
        if len(s):
            s = s[np.lexsort((s["lsa_id"], s["adv_rtr"], s["lsa_type"]))]
        p = self.planes
        spf = ospfv2.area_from_planes(self.area, lambda csr, root, nhw: (p[0], p[1], np.pad(p[2][:, None], ((0, 0), (0, nhw - 1)))))
        ra = [ospf_rib.RibArea(self.area.area_id, spf, self.area.ifaces, s, True)]
        return self.affected(ospf_rib.update_rib_full(self.area.router_id, self.area.max_paths, ra, self.externals))


class GoldenNonBackbone(NonBackbone):
    """R's recorded area image and LSDB; the borders from their own snapshots; A's configuration as the borders
    recorded it."""

    def __init__(self, topo, r, borders):
        sr = snap(topo, r)
        self.keys, self.snap = gu.global_sort_keys(sr), sr
        assert len(sr["areas"]) == 1
        a = sr["areas"][0]
        self.area = gu.ospfv2_area_image(sr, a, self.keys)
        self.summaries, self.externals = gu.ospfv2_summaries(a), None
        self.bsnaps = [snap(topo, b) for b in borders]
        self.doms = [golden_domain(b)[0] for b in self.bsnaps]
        self.cfgs = [configs_of(b, d) for b, d in zip(self.bsnaps, self.doms)]
        d0 = self.doms[0]
        self.config = self.cfgs[0][[x.area_id for x in d0.areas].index(self.area.area_id)]
        self._finish()


class SynthNonBackbone(NonBackbone):
    """ospfv2.nonbackbone_view: R of area 1, three borders, an area-0 ASBR with type-5 LSAs, the shared /24."""

    def __init__(self, seed, V0=30, E0=90, V1=25, E1=70, n_ext=4, max_paths=16):
        t0 = synth.random_topology(V0, E0, synth.SEED_BASE + 900 + 2 * seed, cost_choices=[5, 10, 20])
        t1 = synth.random_topology(V1, E1, synth.SEED_BASE + 901 + 2 * seed, cost_choices=[5, 10, 20])
        v = ospfv2.nonbackbone_view(t0, t1, seed, oracle_spf, max_paths=max_paths, n_ext=n_ext)
        self.view = v
        self.area, self.summaries, self.externals = v["r_area"], v["summaries1"], v["externals"]
        self.doms = [Domain(areas, sums, self.externals) for areas, _ids, sums in v["borders"]]
        self.cfgs = [[ospf_rib.area_config()] * 2 for _ in self.doms]
        self.config = ospf_rib.area_config()
        self._finish()


def chain_jobs(bb, costs=(capi.COST_DISABLED, 35)):
    jobs = [bb.job_overrides((), 0)]
    for link in area0_links(bb.doms):
        jobs += [bb.job_overrides(link, c) for c in costs]
    return jobs


# ------------------------------------------------------------------------------------------ recorded data
GOLDEN = [("topo2-2", "rt6", ["rt4", "rt5"])] + [(f"topo1-{k}", r, [b]) for k in (1, 2, 3)
                                                 for r, b in (("rt1", "rt2"), ("rt5", "rt4"), ("rt7", "rt6"))]
GIDS = [f"{t}-{r}" for t, r, _ in GOLDEN]


@pytest.mark.parametrize("g", GOLDEN, ids=GIDS)
def test_base_job_equals_the_recorded_local_rib(abr_harness, harness, g):
    bb = GoldenNonBackbone(*g)
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
    if bb.config[2] == 0:                                              # totally stubby: only the static default
        assert bb.table.n_prefixes == 0 and bb.table.n_slots == 0
    else:
        assert bb.table.n_prefixes > 0 and bb.table.n_slots > 0
    if bb.config[1] == ospf_rib.AREA_STUB:
        assert not ((bb.table.prefix == 0) & (bb.table.plen == 0)).any()
        assert bb.table.n_asbr_slots == 0


@pytest.mark.parametrize("g", GOLDEN, ids=GIDS)
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_chain_area0_link_failed_or_recosted(abr_harness, harness, g, narrow_planes):
    """Every area-0 link failed, then re-costed to 35, at every border that has it, all jobs in one batch."""
    bb = GoldenNonBackbone(*g)
    jobs = chain_jobs(bb)
    assert len(jobs) > 1
    cells = bb.check(abr_harness, harness, jobs, narrow_planes)
    if bb.table.n_prefixes and g[0] == "topo2-2":
        assert (cells != cells[0]).any()


def test_stub_default_stays_static(abr_harness, harness):
    """topo1 rt5 (stub area 2): the border's default route is a static record at default_cost, in every job."""
    bb = GoldenNonBackbone("topo1-1", "rt5", ["rt4"])
    assert bb.config[1] == ospf_rib.AREA_STUB
    cells = bb.check(abr_harness, harness, chain_jobs(bb))
    assert cells.shape[1] == bb.table.n_prefixes
    dflt = [x for x in bb.summaries if int(x["lsa_id"]) == 0 and int(x["mask"]) == 0]
    assert dflt and int(dflt[0]["metric"]) == 10


# ------------------------------------------------------------------------------------------ generated domains
@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_generated_domains_chain(abr_harness, harness, seed, narrow_planes):
    """Every area-0 link failed and re-costed, one job each; the area-0 ASBR's externals route through the borders'
    type-4 slots, which read the borders' area-0 plane sets."""
    bb = SynthNonBackbone(seed)
    assert bb.table.n_asbr_slots > 0 and bb.table.n_asbr_sets == 3
    cells = bb.check(abr_harness, harness, chain_jobs(bb, (capi.COST_DISABLED, 37)), narrow_planes)
    e = bb.externals[bb.externals["adv_rtr"] == bb.view["asbr"]]
    u = [k for k, (p, l) in enumerate(zip(bb.table.prefix, bb.table.plen))
         if any(int(y["lsa_id"]) == int(p) and bin(int(y["mask"])).count("1") == int(l) for y in e)]
    assert u and ext_path(cells[0][u]).any()
    assert (cells != cells[0]).any()


def test_asbr_unreachable_from_one_border_moves_to_another(abr_harness, harness):
    """The area-0 ASBR cut off at the last border in LsaKey order only: its externals at R move to an earlier border's
    type-4 slot; every one still routes."""
    n = 0
    for seed in range(3):
        bb = SynthNonBackbone(seed)
        last = max(range(3), key=lambda b: bb.doms[b].areas[0].router_id)
        cells = bb.check(abr_harness, harness, [bb.job_overrides((), 0), bb.cut(bb.view["asbr"], {last})])
        e = bb.externals[bb.externals["adv_rtr"] == bb.view["asbr"]]
        u = [k for k, (p, l) in enumerate(zip(bb.table.prefix, bb.table.plen))
             if any(int(y["lsa_id"]) == int(p) and bin(int(y["mask"])).count("1") == int(l) for y in e)
             and ext_path(cells[0][k:k + 1])[0]]
        assert u and ext_path(cells[1][u]).all()
        n += int(cells[1][u].tobytes() != cells[0][u].tobytes())
    assert n > 0


def test_shared_prefix_ties_at_the_first_border(abr_harness, harness):
    """The shared /24 ties at the first border between area 0 and area 1: its cell carries A atoms, so the border does
    not advertise it into A; R routes it intra-area."""
    bb = SynthNonBackbone(0)
    d = bb.doms[0]
    p, m = bb.view["shared"]
    c, _ = d.cells(abr_harness, d.planes())
    u = int(np.nonzero((d.rt.prefix == p) & (d.rt.plen == bin(m).count("1")))[0][0])
    i1 = d.rt.area_ids.index(1)
    a1 = ((1 << d.rt.n_atoms[i1]) - 1) << d.rt.atom_base[i1]
    assert int(c[u]["nh_mask"]) & a1 and int(c[u]["nh_mask"]) & ~a1
    cells = bb.check(abr_harness, harness, chain_jobs(bb))
    k = int(np.nonzero((bb.table.prefix == p) & (bb.table.plen == bin(m).count("1")))[0][0])
    assert (ospf_rib.cell_path(cells[:, k]) == ospf_rib.PATH_INTRA).all()


def test_a_atom_filter_in_the_walk(abr_harness, harness):
    """A border cell of an affected prefix that gains an A atom is not advertised: the walk treats it as absent."""
    bb = SynthNonBackbone(2)
    cells, _, bcells = bb.cells(abr_harness, harness, bb.border_planes([bb.job_overrides((), 0)]))
    n = 0
    for b, d in enumerate(bb.doms):
        i1 = d.rt.area_ids.index(1)
        for u in np.nonzero(ospf_rib.cell_path(cells[0]) == ospf_rib.PATH_INTER)[0]:
            k = np.nonzero((d.rt.prefix == bb.table.prefix[u]) & (d.rt.plen == bb.table.plen[u]))[0]
            if not len(k) or not ospf_rib.cell_flags(bcells[b][0][k[0]]) & 1:
                continue
            bp = bb.border_planes([bb.job_overrides((), 0)])
            with_atom = [c.copy() for c in bcells]
            with_atom[b][0][k[0]]["nh_mask"] |= np.uint64(1 << d.rt.atom_base[i1])
            absent = [c.copy() for c in bcells]
            absent[b][0][k[0]]["mpf"] = 0
            absent[b][0][k[0]]["winner"] = ospf_rib.NO_RECORD
            got, _ = asbr_cells(harness, bb.table, bb.planes, with_atom, bp)
            want, _ = asbr_cells(harness, bb.table, bb.planes, absent, bp)
            assert got.tobytes() == want.tobytes()
            n += int(got[0][u].tobytes() != cells[0][u].tobytes())
    assert n > 0


def test_area0_router_needs_no_new_stage(rib_harness):
    """topo2-2 rt1, an area-0 internal router, over the same area-0 jobs: the ordinary one-area walk
    (hspf_ospfv2_rib_cells' body, the job's area-0 row) decodes to its host chain, update_rib_full over its job planes
    with its recorded LSDB.  The type-3/4 LSAs in area 0 come from the ABRs' non-backbone SPTs, which these jobs do not
    move."""
    sr = snap("topo2-2", "rt1")
    a = gu.ospfv2_area_image(sr, sr["areas"][0], gu.global_sort_keys(sr))
    sums = gu.ospfv2_summaries(sr["areas"][0])
    flat = ospfv2.Flat(a)
    rv = flat.router_vertex(a.router_id)
    rt = ospf_rib.RibTable(flat, 0, sums, None)
    ids = [int(x) for x in flat.ids]
    src = np.repeat(np.arange(flat.csr.n_vertices), np.diff(flat.csr.row_ptr))
    links = area0_links([golden_domain(snap("topo2-2", b))[0] for b in ("rt4", "rt5")])
    assert links
    for link in links:
        for cost in (capi.COST_DISABLED, 35):
            ov = [(int(k), cost) for k in range(flat.csr.n_edges) if {ids[src[k]], ids[flat.csr.col[k]]} == set(link)]
            p = planes_of(flat.csr, rv, ov)
            cells, st = rib_cells(rib_harness, rt, [rv], tuple(x[None] for x in p))
            assert st[0] == 0
            v, nh = gather_for(flat, rv, p)
            got = ospf_rib.rib_from_cells(a, rt, cells[0], v, nh)
            spf = ospfv2.area_from_planes(a, lambda csr, root, nhw, p=p: (p[0], p[1], np.pad(p[2][:, None], ((0, 0), (0, nhw - 1)))))
            same_rib(got, ospf_rib.update_rib_full(a.router_id, a.max_paths, [ospf_rib.RibArea(0, spf, a.ifaces, sums)]))


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
    a0 = next(a for a in bb.doms[0].areas if a.area_id == 0)
    refused(capi.HSPF_E_INVAL, flat=ospfv2.Flat(a0), rid=a0.router_id)
    # R with the B flag: a border as R
    a1 = next(a for a in bb.doms[1].areas if a.area_id == 1)
    refused(capi.HSPF_E_INVAL, flat=ospfv2.Flat(a1), rid=a1.router_id, borders=[rts[0], rts[2]])
    # a border table without area 0, or without A
    d = bb.doms[0]
    for keep in (0, 1):
        i = d.rt.area_ids.index(keep)
        only = ospf_rib.AbrRibTable(d.areas[i].router_id, [d.flats[i]], [keep], [d.summaries[i]], None, bb.externals)
        refused(capi.HSPF_E_INVAL, borders=[only] + rts[1:])
    # a border given twice
    refused(capi.HSPF_E_INVAL, borders=[rts[0], rts[0], rts[1]])
    # a border's type-3 LSA for a prefix it cannot advertise, a type-4 for a router it cannot originate for
    b0 = bb.doms[0].areas[0].router_id
    for extra in ((b0, 0xC0A80000, 0xFFFFFF00, 5, 3, 0, (0, 0)), (b0, 0x09090909, 0, 5, 4, 0, (0, 0))):
        bad = np.concatenate([bb.summaries, np.array([extra], ospf_rib.SUMMARY_LSA_DT)])
        bad = bad[np.lexsort((bad["lsa_id"], bad["adv_rtr"], bad["lsa_type"]))]
        refused(capi.HSPF_E_INVAL, sums=bad)
        dead = bad.copy()
        dead["maxage"][(dead["lsa_id"] == extra[1]) & (dead["adv_rtr"] == b0)] = 1
        ospf_rib.BackboneTable(bb.flat, bb.area.router_id, dead, bb.externals, rts, config=cfg)
    # NSSA
    refused(capi.HSPF_E_UNSUPPORTED, config=ospf_rib.area_config(ospf_rib.AREA_NSSA))
    # a V-flag router in A
    a = ospfv2.Ospfv2Area(**{k: getattr(bb.area, k) for k in bb.area.__dataclass_fields__})
    rl = a.router_lsas.copy()
    rl["flags"][rl["adv_rtr"] == b0] |= np.uint8(0x04)
    a.router_lsas = rl
    refused(capi.HSPF_E_UNSUPPORTED, flat=ospfv2.Flat(a))
    # a usable type-4 LSA of another ABR in a border's area-0 summaries (an inter-area router entry at the border)
    b1 = bb.doms[1].areas[0].router_id
    doms = []
    for dm in bb.doms:
        s = list(dm.summaries)
        i0 = dm.rt.area_ids.index(0)
        if dm.areas[0].router_id != b1:
            s[i0] = np.concatenate([s[i0], np.array([(b1, 0x0A0B0C0D, 0, 5, 4, 0, (0, 0))], ospf_rib.SUMMARY_LSA_DT)])
            s[i0] = s[i0][np.lexsort((s[i0]["lsa_id"], s[i0]["adv_rtr"], s[i0]["lsa_type"]))]
        doms.append(Domain(dm.areas, s, dm.externals))
    refused(capi.HSPF_E_UNSUPPORTED, borders=[x.rt for x in doms])
    # 0 or more than 8 borders
    refused(capi.HSPF_E_UNSUPPORTED, borders=[])
    refused(capi.HSPF_E_UNSUPPORTED, borders=[rts[0]] * 9)


def test_more_than_8_plane_sets_are_refused():
    """The area-0 ASBR is also an E-flag router of copies of area 0 added to the borders as areas 2, 3: each
    (border, area) pair is a plane set, and three borders with three such areas read nine."""
    bb = SynthNonBackbone(0)

    def with_twins(d, n):
        i0 = d.rt.area_ids.index(0)
        twins = []
        for k in range(n):
            t = ospfv2.Ospfv2Area(**{f: getattr(d.areas[i0], f) for f in d.areas[i0].__dataclass_fields__})
            t.area_id = 2 + k
            twins.append(t)
        return Domain(d.areas + twins, list(d.summaries) + [np.zeros(0, ospf_rib.SUMMARY_LSA_DT)] * n, d.externals)

    mk = lambda doms: ospf_rib.BackboneTable(bb.flat, bb.area.router_id, bb.summaries, bb.externals,
                                             [d.rt for d in doms], config=ospf_rib.area_config())
    t = mk([with_twins(bb.doms[0], 1)] + bb.doms[1:])
    assert t.n_asbr_sets == 4
    with pytest.raises(capi.HspfError) as e:
        mk([with_twins(d, 2) for d in bb.doms])
    assert e.value.code == capi.HSPF_E_UNSUPPORTED


def test_decode_refuses_an_image_of_another_area(abr_harness, harness):
    bb = SynthNonBackbone(1)
    cells, _, _ = bb.cells(abr_harness, harness, bb.border_planes([bb.job_overrides((), 0)]))
    other = ospfv2.Ospfv2Area(**{k: getattr(bb.area, k) for k in bb.area.__dataclass_fields__})
    other.area_id = 0
    v, n = gather_for(bb.flat, bb.rv, bb.planes)
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.backbone_from_cells(other, bb.table, cells[0], v, n)
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
    rows = [np.repeat(np.arange(J, dtype=np.uint32)[:, None], 2, 1) for _ in range(3)]
    rows[1][2, :] = J
    ps = [[np.zeros(J, np.uint32) for _ in range(2)] for _ in range(3)]
    ps[0][0][1] = ps[0][1][1] = 0x8
    got, st = asbr_cells(harness, bb.table, bb.planes, bcells, bp, rows=rows, pstatus=ps)
    assert st[2] & capi.JS_INVALID and st[1] == 0x8
    for j in (1, 2):
        assert (got["winner"][j] == ospf_rib.NO_RECORD).all() and not got["mpf"][j].any()
    keep = [j for j in range(J) if j not in (1, 2)]
    assert got[keep].tobytes() == want[keep].tobytes()
