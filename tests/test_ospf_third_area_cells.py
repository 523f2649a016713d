"""CPU: the OSPFv2 stage of an internal router R of a non-backbone area over what-if jobs inside another non-backbone
area (hspf_ospfv2_third_area_table_create, ospf_backbone_cell_eval with kAsbr and kNonBackbone and chain slots), and
the ASBR entries of its area's border routers (hspf_ospfv2_abr_backbone_asbr_entries, abr_asbr_entry).

The walks are compiled into test harnesses and run on the CPU over the oracle's SPT planes.  Area 1 is perturbed; its
ABRs (B) compute their cells per job, R's area's ABRs (C) their abr_backbone cells and ASBR entries over the B's, and
R its cells over the C's.  Every job, decoded by hspf_ospfv2_backbone_from_cells over R's image of its area, must equal
byte for byte the host chain: each B's update_rib_full and net_summaries into area 0, spliced into area 0's LSAs; each
C's update_rib_full over those, and its net_summaries into R's area, spliced into that area's LSAs; then
update_rib_full at R, restricted to the affected prefixes.  No OSPFv2 conformance snapshot holds a type-4 LSA, so the
chain slots rest on that host restatement."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import golden_util as gu
from holo_b200 import capi, ospf_rib, ospfv2, synth
from test_ospf_abr_backbone_cells import AbrBackbone
from test_ospf_abr_backbone_cells import harness as abr_backbone_harness  # noqa: F401  (fixture)
from test_ospf_abr_rib_cells import Domain, golden_domain, narrow, planes_of
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospf_backbone_cells import Backbone, configs_of, non_backbone_links, snap, summaries_of
from test_ospf_nonbackbone_cells import oracle_spf
from test_ospf_rib_cells import same_rib
from test_ospfv2_route_cells import gather_for

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    out = tmp_path_factory.mktemp("harness") / "libospf_third_area_cells_harness.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                    "-o", str(out), str(ROOT / "tests" / "native" / "ospf_third_area_cells_harness.cc")], check=True)
    lib = C.CDLL(str(out))
    for fn in (lib.harness_ospf_third_area_cells, lib.harness_ospf_third_area_cells16):
        fn.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 6
    for fn in (lib.harness_ospf_abr_asbr_entries, lib.harness_ospf_abr_asbr_entries16):
        fn.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 10
    lib.harness_third_area_winners_fit.argtypes = [C.c_uint64, C.c_uint64]
    return lib


def asbr_entries(harness, ct, planes, bplanes, narrow_planes=False, root_status=None, rows=None, pstatus=None):
    """Entries [J, G] and status words of C's table ct.  planes[i]: C's row 0 of area i; bplanes[b][j][i]: B b's
    planes of area i in job j (row j, unless rows[b] gives [J, n_areas] rows)."""
    J = len(bplanes[0])
    pl = [narrow(p) if narrow_planes else p for p in planes]
    keep = [[np.ascontiguousarray(x) for x in p] for p in pl]
    arr = lambda k: (C.c_void_p * len(pl))(*[keep[i][k].ctypes.data for i in range(len(pl))])
    rs = np.ascontiguousarray(root_status, np.uint32) if root_status is not None else None
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
    G = len(ct.asbr_ids)
    ent = np.zeros((J, G), np.uint32)
    out = np.zeros(J, np.uint32)
    fn = harness.harness_ospf_abr_asbr_entries16 if narrow_planes else harness.harness_ospf_abr_asbr_entries
    fn(ct.handle, J, arr(0), arr(1), arr(2), rs.ctypes.data if rs is not None else None,
       (C.c_void_p * len(dists))(*[C.addressof(x) for x in dists]),
       (C.c_void_p * len(pss))(*[C.addressof(x) for x in pss]) if pstatus is not None else None,
       (C.c_void_p * len(nrs))(*nrs), (C.c_void_p * len(rws))(*rws), ent.ctypes.data if G else None, out.ctypes.data)
    return ent, out


def third_area_cells(harness, table, planes, ccells, entries, narrow_planes=False, status=None, entry_status=None,
                     root_status=0):
    """R's cells [J, P] and status words over the C's cells [J, K_c] and entries [J, G_c]."""
    J = len(ccells[0])
    pl = narrow(planes) if narrow_planes else planes
    keep = [np.ascontiguousarray(x) for x in pl] + list(ccells) + [np.ascontiguousarray(e) for e in entries]
    bc = (C.c_void_p * len(ccells))(*[c.ctypes.data for c in ccells])
    en = (C.c_void_p * len(entries))(*[keep[3 + len(ccells) + b].ctypes.data if entries[b].size else None
                                       for b in range(len(entries))])
    st = es = None
    if status is not None:
        keep += [np.ascontiguousarray(x, np.uint32) for x in status]
        st = (C.c_void_p * len(status))(*[x.ctypes.data for x in keep[-len(status):]])
    if entry_status is not None:
        keep += [np.ascontiguousarray(x, np.uint32) for x in entry_status]
        es = (C.c_void_p * len(entry_status))(*[x.ctypes.data for x in keep[-len(entry_status):]])
    cells = np.zeros((J, table.n_prefixes), ospf_rib.RIB_CELL_DT)
    out = np.zeros(J, np.uint32)
    fn = harness.harness_ospf_third_area_cells16 if narrow_planes else harness.harness_ospf_third_area_cells
    fn(table.handle, J, keep[0].ctypes.data, keep[1].ctypes.data, keep[2].ctypes.data, root_status, bc, st, en, es,
       cells.ctypes.data, out.ctypes.data)
    return cells, out


class ThirdArea(Backbone):
    """R's area image, its summaries and configuration; the C's (AbrBackbone over the B domains) and R's table.
    `doms` are the B domains (their area-1 links are the jobs' links, as Backbone.job_overrides reads them)."""

    def __init__(self, area, summaries, externals, config, cs, bdoms, bcfgs, ccfgs):
        self.area, self.summaries, self.externals, self.config = area, summaries, externals, config
        self.cs, self.doms, self.cfgs, self.ccfgs = cs, bdoms, bcfgs, ccfgs
        self.flat = ospfv2.Flat(area)
        self.rv = self.flat.router_vertex(area.router_id)
        self.table = ospf_rib.BackboneTable(self.flat, area.router_id, summaries, externals, [c.table for c in cs],
                                            config=config)
        self.planes = planes_of(self.flat.csr, self.rv)

    def run(self, abr, abr_backbone, harness, jobs, narrow_planes=False, bp=None):
        """R's cells and status words, the C's cells and entries, the B planes per job (bp: those planes given)."""
        bp = self.border_planes(jobs) if bp is None else bp
        ccells, cents = [], []
        for c in self.cs:
            cc, st, _ = c.cells(abr, abr_backbone, bp, narrow_planes)
            assert not st.any()
            ent, est = asbr_entries(harness, c.table, c.planes, bp, narrow_planes)
            assert not est.any()
            ccells.append(cc)
            cents.append(ent)
        cells, st = third_area_cells(harness, self.table, self.planes, ccells, cents, narrow_planes)
        return cells, st, ccells, cents, bp

    def c_rib(self, c, job_bplanes):
        """C's area ribs' inputs and its routing table of the job (area 0 with the B's LSAs re-originated)."""
        bid = {d.areas[0].router_id for d in self.doms}
        s0 = c.r.summaries[c.i0]
        new = [s for s in s0 if not (int(s["adv_rtr"]) in bid and s["lsa_type"] in (3, 4))]
        for d, cfg, p in zip(self.doms, self.cfgs, job_bplanes):
            new += list(summaries_of(d, cfg, p, [a.area_id for a in d.areas].index(0)))
        s = np.array(new, ospf_rib.SUMMARY_LSA_DT)
        s = s[np.lexsort((s["lsa_id"], s["adv_rtr"], s["lsa_type"]))]
        ra = []
        for i, (a, p) in enumerate(zip(c.r.areas, c.planes)):
            spf = ospfv2.area_from_planes(a, lambda csr, root, nhw, p=p: (p[0], p[1], np.pad(p[2][:, None], ((0, 0), (0, nhw - 1)))))
            ra.append(ospf_rib.RibArea(a.area_id, spf, a.ifaces, s if i == c.i0 else c.r.summaries[i], c.r.active[i]))
        rid = c.r.areas[0].router_id
        return ra, ospf_rib.update_rib_full(rid, c.r.areas[0].max_paths, ra, c.externals)

    def c_summaries(self, c, cfg, job_bplanes):
        ra, rib = self.c_rib(c, job_bplanes)
        rid = c.r.areas[0].router_id
        target = [a.area_id for a in c.r.areas].index(self.area.area_id)
        return ospf_rib.net_summaries(rid, rib, ospf_rib.router_tables(rid, ra), ra, cfg, target)

    def host(self, job_bplanes):
        """The three-step chain, R's whole table."""
        cid = {c.r.areas[0].router_id for c in self.cs}
        new = [s for s in self.summaries if int(s["adv_rtr"]) not in cid]
        for c, cfg in zip(self.cs, self.ccfgs):
            new += list(self.c_summaries(c, cfg, job_bplanes))
        s = np.array(new, ospf_rib.SUMMARY_LSA_DT)
        if len(s):
            s = s[np.lexsort((s["lsa_id"], s["adv_rtr"], s["lsa_type"]))]
        p = self.planes
        spf = ospfv2.area_from_planes(self.area, lambda csr, root, nhw: (p[0], p[1], np.pad(p[2][:, None], ((0, 0), (0, nhw - 1)))))
        ra = [ospf_rib.RibArea(self.area.area_id, spf, self.area.ifaces, s, True)]
        return ospf_rib.update_rib_full(self.area.router_id, self.area.max_paths, ra, self.externals)

    def decode(self, cells):
        v, n = gather_for(self.flat, self.rv, self.planes)
        return ospf_rib.backbone_from_cells(self.area, self.table, cells, v, n)

    def check(self, abr, abr_backbone, harness, jobs, narrow_planes=False):
        cells, st, ccells, cents, bp = self.run(abr, abr_backbone, harness, jobs, narrow_planes)
        assert not st.any()
        keep = {(int(p), int(l)) for p, l in zip(self.table.prefix, self.table.plen)}
        key = lambda r: (int(r["prefix"]), bin(int(r["mask"])).count("1"))
        base = None
        for j in range(len(jobs)):
            jb = [bp[b][j] for b in range(len(self.doms))]
            full = self.host(jb)
            same_rib(self.decode(cells[j]), self.affected(full))
            # every prefix outside the table keeps R's base route
            rest = {key(r): (tuple(int(r[f]) for f in ("metric", "path_type", "area_id", "type2_metric", "tag")), repr(full.nh(r))) for r in full.routes
                    if key(r) not in keep}
            base = rest if base is None else base
            assert rest == base
            # the entries are the type-4 rows of each C's net_summaries into R's area
            for c, cfg, ent in zip(self.cs, self.ccfgs, cents):
                t4 = {int(x["lsa_id"]): int(x["metric"]) for x in self.c_summaries(c, cfg, jb) if x["lsa_type"] == 4}
                want = [t4.get(int(a), 0xFFFFFFFF) for a in c.table.asbr_ids]
                assert list(ent[j]) == want
        return cells, ccells, cents


# ------------------------------------------------------------------------------------------ recorded data
# topo1-1/2/3: R an internal router of area 1 (rt1, border rt2), a stub area 2 (rt5, rt4) or a totally stubby area 3
# (rt7, rt6), and either other area perturbed (its ABR the single B)
AREA_OF = {"rt1": "rt2", "rt5": "rt4", "rt7": "rt6"}
GOLDEN = [(t, r, b) for t in ("topo1-1", "topo1-2", "topo1-3") for r in AREA_OF for b in AREA_OF.values()
          if b != AREA_OF[r]]
GIDS = [f"{t}-{r}-{b}" for t, r, b in GOLDEN]


def golden(topo, r, b):
    sr = snap(topo, r)
    keys = gu.global_sort_keys(sr)
    a = sr["areas"][0]
    area = gu.ospfv2_area_image(sr, a, keys)
    bs, cs_ = snap(topo, b), snap(topo, AREA_OF[r])
    bdom, cdom = golden_domain(bs)[0], golden_domain(cs_)[0]
    bcfg, ccfg = configs_of(bs, bdom), configs_of(cs_, cdom)
    c = AbrBackbone(cdom, [bdom], [bcfg])
    config = ccfg[[x.area_id for x in cdom.areas].index(area.area_id)]
    t = ThirdArea(area, gu.ospfv2_summaries(a), None, config, [c], [bdom], [bcfg], [ccfg])
    return t, sr, keys


@pytest.mark.parametrize("g", GOLDEN, ids=GIDS)
def test_base_job_equals_the_recorded_local_rib(abr_harness, abr_backbone_harness, harness, g):
    t, sr, keys = golden(*g)
    jobs = [t.job_overrides((), 0)]
    for link in non_backbone_links(t)[:4]:
        jobs.append(t.job_overrides(link, capi.COST_DISABLED))
    cells, _, _ = t.check(abr_harness, abr_backbone_harness, harness, jobs)
    got = t.decode(cells[0])
    key_name = {v: k for k, v in keys.items()}
    mine = {}
    for r in got.routes:
        nh = sorted(((key_name.get(i, "?"), gu.ipstr(a) if ha else None) for (i, ha, a, _hn, _n, _hl, _l) in got.nh(r)),
                    key=lambda x: (x[0] or "", x[1] or ""))
        mine[f"{gu.ipstr(r['prefix'])}/{bin(int(r['mask'])).count('1')}"] = (int(r["metric"]), ospf_rib.PATH_NAMES[int(r["path_type"])], nh)
    affected = {f"{gu.ipstr(int(p))}/{int(l)}" for p, l in zip(t.table.prefix, t.table.plen)}
    want = {k: v for k, v in gu.golden_rib(sr).items() if k in affected}
    norm = lambda d: {k: (v[0], v[1], [(a or "", b or "") for a, b in v[2]]) for k, v in d.items()}
    assert norm(mine) == norm(want)
    if t.config[2] == 0:                                               # totally stubby: nothing moves
        assert t.table.n_slots == 0
    else:
        assert t.table.n_prefixes > 0 and t.table.n_slots > 0
    assert t.table.n_asbr_slots == 0 and t.table.n_asbr_sets == 0     # no type-4 LSA in the recorded data


# ------------------------------------------------------------------------------------------- generated
class SynthThirdArea(ThirdArea):
    """ospfv2.third_area_view: R of area 2, n_c C's, the three B's of area 1, k area-1 ASBRs."""

    def __init__(self, seed, n_c=2, k=2, max_paths=16):
        t0 = synth.random_topology(30, 90, synth.SEED_BASE + 950 + 3 * seed, cost_choices=[5, 10, 20])
        t1 = synth.random_topology(25, 70, synth.SEED_BASE + 951 + 3 * seed, cost_choices=[5, 10, 20])
        t2 = synth.random_topology(25, 70, synth.SEED_BASE + 952 + 3 * seed, cost_choices=[5, 10, 20])
        v = ospfv2.third_area_view(t0, t1, t2, seed, oracle_spf, n_c=n_c, max_paths=max_paths, area1_asbrs=k)
        self.view = v
        ext = v["externals"]
        bdoms = [Domain(areas, sums, ext) for areas, _ids, sums in v["borders"]]
        bcfgs = [[ospf_rib.area_config()] * 2 for _ in bdoms]
        cs = [AbrBackbone(Domain(areas, sums, ext), bdoms, bcfgs) for areas, _ids, sums in v["c_areas"]]
        super().__init__(v["r_area"], v["summaries2"], ext, ospf_rib.area_config(), cs, bdoms, bcfgs,
                         [[ospf_rib.area_config()] * 2 for _ in cs])


def synth_jobs(t, n, seed):
    links = non_backbone_links(t)
    rng = np.random.default_rng(seed)
    jobs = [t.job_overrides((), 0)]
    for k in rng.choice(len(links), min(n, len(links)), replace=False):
        jobs.append(t.job_overrides(links[int(k)], capi.COST_DISABLED))
        jobs.append(t.job_overrides(links[int(k)], int(rng.choice([1, 40]))))
    return jobs


@pytest.mark.parametrize("seed,n_c,k", [(0, 2, 2), (1, 3, 2), (2, 2, 0), (3, 3, 1)])
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_generated_domains_chain(abr_harness, abr_backbone_harness, harness, seed, n_c, k, narrow_planes):
    t = SynthThirdArea(seed, n_c=n_c, k=k)
    assert t.table.n_slots > 0
    assert (t.table.n_asbr_slots > 0) == (k > 0) and t.table.n_asbr_sets == 0
    cells, _, cents = t.check(abr_harness, abr_backbone_harness, harness, synth_jobs(t, 8, seed), narrow_planes)
    assert (cells != cells[0]).any()
    if k:
        assert all(e.shape[1] > 0 for e in cents)


def test_chain_moves_external_routes(abr_harness, abr_backbone_harness, harness):
    """Cutting an area-1 ASBR off from every B changes the C's entries for it, and R's routes to its externals."""
    moved = 0
    for seed in range(3):
        t = SynthThirdArea(seed, n_c=2, k=2)
        jobs = [t.job_overrides((), 0)]
        for x in t.view["area1_asbrs"]:
            ov = [t.job_overrides(l, capi.COST_DISABLED) for l in non_backbone_links(t) if x in l]
            jobs.append([{i: sum((o[b].get(i, []) for o in ov), []) for i in range(len(d.areas))}
                         for b, d in enumerate(t.doms)])
        cells, _, cents = t.check(abr_harness, abr_backbone_harness, harness, jobs)
        for j in range(1, len(jobs)):
            moved += int(any((e[j] != e[0]).any() for e in cents)) + int(cells[j].tobytes() != cells[0].tobytes())
    assert moved > 0


def test_ties_between_cs_merge_atoms(abr_harness, abr_backbone_harness, harness):
    """Some inter-area route reaches R through two C's at one metric: its cell ORs their atoms."""
    n = 0
    for seed in range(4):
        t = SynthThirdArea(seed, n_c=3, k=1)
        cells, _, _ = t.check(abr_harness, abr_backbone_harness, harness, synth_jobs(t, 4, seed))
        inter = ((ospf_rib.cell_flags(cells) & 1) != 0) & (ospf_rib.cell_path(cells) == ospf_rib.PATH_INTER)
        multi = np.vectorize(lambda m: bin(int(m)).count("1") > 1)(cells["nh_mask"])
        n += int((inter & multi).sum())
    assert n > 0


# -------------------------------------------------------------------------------------------- refusals
def test_table_refusals():
    t = SynthThirdArea(0)
    cts = [c.table for c in t.cs]

    def mk(flat=t.flat, rid=t.area.router_id, config=t.config, sums=t.summaries, borders=cts):
        return ospf_rib.BackboneTable(flat, rid, sums, t.externals, borders, config=config)

    def refused(code, **kw):
        with pytest.raises(capi.HspfError) as e:
            mk(**kw)
        assert e.value.code == code

    refused(capi.HSPF_E_INVAL, config=None)
    # no border: the create itself (the Python table picks the third-area create from its borders)
    h = C.c_void_p()
    cfg = np.array([t.config], ospf_rib.AREA_CONFIG_DT)
    lib = capi.load_library()
    assert lib.hspf_ospfv2_third_area_table_create(t.flat.handle, t.area.router_id, cfg.ctypes.data,
                                                   t.summaries.ctypes.data, len(t.summaries), None, 0,
                                                   (C.c_void_p * 1)(cts[0].handle.value), 0, C.byref(h)) == \
        capi.HSPF_E_INVAL
    # an OSPFv3 border table
    from test_ospfv3_abr_backbone_cells import SynthAbrBackbone as SynthAbrBackboneV3
    v3 = SynthAbrBackboneV3(0)
    assert v3.table.v3
    refused(capi.HSPF_E_INVAL, borders=[cts[0], v3.table])
    # a border that is not a B-flag router of R's area
    c1 = t.cs[1].r.areas[0].router_id
    nb = ospfv2.Ospfv2Area(**{k: getattr(t.area, k) for k in t.area.__dataclass_fields__})
    rl = nb.router_lsas.copy()
    rl["flags"][rl["adv_rtr"] == c1] &= np.uint8(0xFE)
    nb.router_lsas = rl
    refused(capi.HSPF_E_INVAL, flat=ospfv2.Flat(nb))
    with pytest.raises(ValueError):                                        # borders of both kinds
        mk(borders=[cts[0], t.doms[0].rt])
    refused(capi.HSPF_E_INVAL, borders=[cts[0]] * 2)                                  # a border twice
    refused(capi.HSPF_E_INVAL, borders=cts * 5)                                       # more than 8
    refused(capi.HSPF_E_INVAL, rid=t.cs[0].r.areas[0].router_id)                     # R is an ABR, among the borders
    refused(capi.HSPF_E_UNSUPPORTED, config=ospf_rib.area_config(ospf_rib.AREA_NSSA))
    # a C's type-3 LSA for a prefix of its table it cannot advertise: an area-1 ASBR's external /24
    c0 = t.cs[0].r.areas[0].router_id
    p = next(int(x) for x in cts[0].prefix if int(x) >> 24 == 0x0F)
    row = (c0, p, 0xFFFFFF00, 5, 3, 0, (0, 0))
    s = np.concatenate([t.summaries, np.array([row], ospf_rib.SUMMARY_LSA_DT)])
    s = s[np.lexsort((s["lsa_id"], s["adv_rtr"], s["lsa_type"]))]
    refused(capi.HSPF_E_INVAL, sums=s)
    # a V-flag router in R's area
    a = ospfv2._set_flags(ospfv2.Ospfv2Area(**{k: getattr(t.area, k) for k in t.area.__dataclass_fields__}),
                          {t.view["area2_asbr"]: 0x04})
    refused(capi.HSPF_E_UNSUPPORTED, flat=ospfv2.Flat(a))
    # a B that is a router of R's area: B 0's id given to an area-2 router
    rl = t.area.router_lsas.copy()
    x = int(t.view["area2_asbr"])
    bid = t.doms[0].areas[0].router_id
    for f in ("adv_rtr", "lsa_id"):
        rl[f][rl[f] == x] = bid
    rl = rl[np.lexsort((rl["lsa_id"], rl["adv_rtr"]))]
    a2 = ospfv2.Ospfv2Area(**{k: getattr(t.area, k) for k in t.area.__dataclass_fields__})
    a2.router_lsas = rl
    links = a2.links.copy()
    links["link_id"][links["link_id"] == x] = bid
    a2.links = links
    refused(capi.HSPF_E_UNSUPPORTED, flat=ospfv2.Flat(a2))


def test_slot_winners_must_fit_32_bits(harness):
    """A table whose slot winners would not fit 32 bits is refused (HSPF_E_UNSUPPORTED).  A real one needs about 2^32
    records, so the rule the create applies (backbone_winners_fit, OSPFv2 encoding: n_records + slot index; chain slots
    are no winners) is checked at its boundary, and a generated table is checked to pass it."""
    fit = harness.harness_third_area_winners_fit
    assert fit(0xFFFFFFFF - 5, 5) == 0 and fit(0xFFFFFFFE - 5, 5) == 1 and fit(0, 0xFFFFFFFF) == 0
    t = SynthThirdArea(0)
    assert fit(t.table.n_records, t.table.n_slots) == 1


def test_job_status(abr_harness, abr_backbone_harness, harness):
    """A B status word or a B row out of range reaches C's entries status, which reaches R's job status; R's row-0
    word and C's cell status too.  A refused job gets empty cells; the others are unchanged."""
    t = SynthThirdArea(1, n_c=2, k=2)
    jobs = synth_jobs(t, 3, 1)
    J = len(jobs)
    want, st, ccells, cents, bp = t.run(abr_harness, abr_backbone_harness, harness, jobs)
    assert not st.any()
    c = t.cs[0]
    assert c.table.n_asbr_sets > 0 and len(c.table.asbr_ids) > 0
    rows = [np.repeat(np.arange(J, dtype=np.uint32)[:, None], 2, 1) for _ in range(3)]
    for r in rows:
        r[2, :] = J                                                       # every B's row of job 2 out of range
    ps = [[np.zeros(J, np.uint32) for _ in range(2)] for _ in range(3)]
    for b in range(3):
        ps[b][0][1] = ps[b][1][1] = 0x8                                   # every B's words of job 1
    ent, est = asbr_entries(harness, c.table, c.planes, bp, rows=rows, pstatus=ps)
    assert est[2] & capi.JS_INVALID and est[1] == 0x8
    assert (ent[1] == 0xFFFFFFFF).all() and (ent[2] == 0xFFFFFFFF).all()
    assert not np.delete(est, [1, 2]).any() and np.delete(ent, [1, 2], 0).tobytes() == np.delete(cents[0], [1, 2], 0).tobytes()
    cst = [np.zeros(J, np.uint32) for _ in t.cs]
    cst[1][3] = 0x2
    got, st = third_area_cells(harness, t.table, t.planes, ccells, cents, status=cst, entry_status=[est, np.zeros(J)])
    assert st[1] == 0x8 and st[2] & capi.JS_INVALID and st[3] == 0x2
    bad = [j for j in range(J) if st[j]]
    assert bad == [1, 2, 3]
    for j in bad:
        assert (got["winner"][j] == ospf_rib.NO_RECORD).all() and not got["mpf"][j].any()
    keep = [j for j in range(J) if j not in bad]
    assert got[keep].tobytes() == want[keep].tobytes()
    got, st = third_area_cells(harness, t.table, t.planes, ccells, cents, root_status=0x4)
    assert (st == 0x4).all() and (got["winner"] == ospf_rib.NO_RECORD).all()
