"""CPU: the OSPFv3 stage of an internal router R of a non-backbone area over what-if jobs inside another non-backbone
area (hspf_ospfv3_third_area_table_create, ospf_backbone_cell_eval with kV3, kAsbr, kNonBackbone and kSlotWinners),
and the ASBR entries of its area's border routers (hspf_ospfv3_abr_backbone_asbr_entries, abr_asbr_entry).

The walk is compiled into a test harness and run on the CPU over the oracle's SPT planes.  Area 1 is perturbed; its
ABRs (B) compute their cells per job, R's area's ABRs (C) their OSPFv3 abr_backbone cells and ASBR entries over the
B's, and R its cells over the C's.  Every job, decoded by hspf_ospfv3_backbone_from_cells over R's image of its area,
must equal byte for byte, prefix options included, the host chain: each B's update_rib_full_v3, net_summaries_v3 and
rtr_summaries_v3 into area 0, spliced into area 0's LSAs; each C's same chain over those, into R's area, spliced into
that area's LSAs; then update_rib_full_v3 at R, restricted to the affected prefixes.  The options of a C's route
through a B's slot reach R through two hops: the B copies them into its LSA, C's cell winner carries them, and C
copies them into its own."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import golden_util as gu
from holo_b200 import capi, ospf_rib, ospfv3, synth
from holo_b200.route_table import DELTA_OTHER
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospf_abr_rib_cells import narrow, planes_of
from test_ospf_rib_cells import same_rib
from test_ospf_rib_delta import reference
from test_ospf_third_area_cells import asbr_entries
from test_ospf_third_area_cells import harness as entries_harness  # noqa: F401  (fixture)
from test_ospfv3_abr_backbone_cells import AbrBackbone
from test_ospfv3_abr_backbone_cells import harness as abr_backbone_harness  # noqa: F401  (fixture)
from test_ospfv3_backbone_cells import (Backbone, configs_of, full_image, full_inter_area_lsas, golden_domain,
                                        non_backbone_links, snap)
from test_ospfv3_nonbackbone_cells import oracle_spf, spf_of, srt
import test_ospfv3_abr_rib_cells as v3abr

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    out = tmp_path_factory.mktemp("harness") / "libospfv3_third_area_cells_harness.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                    "-o", str(out), str(ROOT / "tests" / "native" / "ospfv3_third_area_cells_harness.cc")], check=True)
    lib = C.CDLL(str(out))
    for fn in (lib.harness_ospfv3_third_area_cells, lib.harness_ospfv3_third_area_cells16):
        fn.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 6
        fn.restype = C.c_int
    lib.harness_third_area_v3_winners_fit.argtypes = [C.c_uint64, C.c_uint64]
    return lib


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
    fn = harness.harness_ospfv3_third_area_cells16 if narrow_planes else harness.harness_ospfv3_third_area_cells
    assert fn(table.handle, J, keep[0].ctypes.data, keep[1].ctypes.data, keep[2].ctypes.data, root_status, bc, st, en,
              es, cells.ctypes.data, out.ctypes.data) == 0
    return cells, out


class ThirdArea(Backbone):
    """R's area image, its LSAs and configuration; the C's (OSPFv3 AbrBackbone over the B domains) and R's table.
    `doms` are the B domains (their area-1 links are the jobs' links, as Backbone.job_overrides reads them)."""

    def __init__(self, area, summaries, externals, config, cs, bdoms, bcfgs, ccfgs, keys=None):
        self.area, self.summaries, self.externals, self.config = area, summaries, externals, config
        self.cs, self.doms, self.cfgs, self.ccfgs, self.keys = cs, bdoms, bcfgs, ccfgs, keys
        self.flat = ospfv3.Flat(area)
        self.rv = self.flat.router_vertex(area.router_id)
        self.table = ospf_rib.BackboneTable(self.flat, area.router_id, summaries, externals, [c.table for c in cs],
                                            config=config)
        self.planes = planes_of(self.flat.csr, self.rv)

    def run(self, abr, abr_backbone, entries_h, harness, jobs, narrow_planes=False, bp=None):
        """R's cells and status words, the C's cells and entries, the B planes per job (bp: those planes given)."""
        bp = self.border_planes(jobs) if bp is None else bp
        ccells, cents = [], []
        for c in self.cs:
            cc, st, _ = c.cells(abr, abr_backbone, bp, narrow_planes)
            assert not st.any()
            ent, est = asbr_entries(entries_h, c.table, c.planes, bp, narrow_planes)
            assert not est.any()
            ccells.append(cc)
            cents.append(ent)
        cells, st = third_area_cells(harness, self.table, self.planes, ccells, cents, narrow_planes)
        return cells, st, ccells, cents, bp

    def c_rib_areas(self, c, job_bplanes):
        """C's RibArea list of the job: area 0 with the B's LSAs re-originated (AbrBackbone.lsdb)."""
        s0 = c.lsdb(job_bplanes)
        return [ospf_rib.RibArea(a.area_id, ospfv3.area_from_planes(a, spf_of(p)), a.ifaces,
                                 s0 if i == c.i0 else c.r.summaries[i], c.r.active[i])
                for i, (a, p) in enumerate(zip(c.r.areas, c.planes))]

    def c_lsas(self, c, cfg, job_bplanes):
        """C's Inter-Area-Prefix / Inter-Area-Router LSAs into R's area in the job."""
        target = [a.area_id for a in c.r.areas].index(self.area.area_id)
        r0 = c.r.areas[0]
        return ospfv3.nonbackbone_lsas(r0.router_id, r0.max_paths, self.c_rib_areas(c, job_bplanes), self.externals,
                                       target, cfg)

    def host_full(self, job_bplanes):
        """The three-step chain, R's whole table."""
        cid = {c.r.areas[0].router_id for c in self.cs}
        new = [tuple(s) for s in self.summaries.tolist() if int(s[0]) not in cid]
        for c, cfg in zip(self.cs, self.ccfgs):
            new += self.c_lsas(c, cfg, job_bplanes)
        s = srt(np.array(new, ospf_rib.INTER_AREA_LSA_DT))
        ra = [ospf_rib.RibArea(self.area.area_id, ospfv3.area_from_planes(self.area, spf_of(self.planes)),
                               self.area.ifaces, s, True)]
        return ospf_rib.update_rib_full_v3(self.area.router_id, self.area.max_paths, ra, self.externals)

    def check(self, abr, abr_backbone, entries_h, harness, jobs, narrow_planes=False):
        cells, st, ccells, cents, bp = self.run(abr, abr_backbone, entries_h, harness, jobs, narrow_planes)
        assert not st.any()
        keep = {(p.tobytes(), int(l)) for p, l in zip(self.table.prefixes6, self.table.plen)}
        base = None
        for j in range(len(jobs)):
            jb = [bp[b][j] for b in range(len(self.doms))]
            full = self.host_full(jb)
            same_rib(self.decode(cells[j]), self.affected(full))
            # every prefix outside the table keeps R's base route
            rest = {}
            for r in full.routes:
                if (r["prefix"].tobytes(), int(r["len"])) in keep:
                    continue
                x = r.copy()
                x["nh_off"] = 0
                hops = full.nexthops[int(r["nh_off"]): int(r["nh_off"]) + int(r["n_nh"])]
                rest[(r["prefix"].tobytes(), int(r["len"]))] = (x.tobytes(), hops.tobytes())
            base = rest if base is None else base
            assert rest == base
            # the entries are the Inter-Area-Router rows of each C's rtr_summaries_v3 into R's area
            for c, cfg, ent in zip(self.cs, self.ccfgs, cents):
                target = [a.area_id for a in c.r.areas].index(self.area.area_id)
                iar = ospf_rib.rtr_summaries_v3(c.r.areas[0].router_id, self.c_rib_areas(c, jb), cfg, target)
                t4 = {int(x["router_id"]): int(x["metric"]) for x in iar}
                assert list(ent[j]) == [t4.get(int(a), 0xFFFFFFFF) for a in c.table.asbr_ids]
        return cells, ccells, cents


# ------------------------------------------------------------------------------------------ recorded data
# topo1-1/1-2: R an internal router of area 1 (rt1, border rt2), area 2 (rt5, rt4) or area 3 (rt7, rt6), and either
# other area perturbed (its ABR the single B)
AREA_OF = {"rt1": "rt2", "rt5": "rt4", "rt7": "rt6"}
GOLDEN = [(t, r, b) for t in ("topo1-1", "topo1-2") for r in AREA_OF for b in AREA_OF.values() if b != AREA_OF[r]]
GIDS = [f"{t}-{r}-{b}" for t, r, b in GOLDEN]


def golden(topo, r, b):
    sr = snap(topo, r)
    keys = gu.global_sort_keys(sr)
    a = sr["areas"][0]
    area = full_image(sr, a, keys)
    bs, cs_ = snap(topo, b), snap(topo, AREA_OF[r])
    bdom, cdom = golden_domain(bs)[0], golden_domain(cs_)[0]
    bcfg, ccfg = configs_of(bs, bdom), configs_of(cs_, cdom)
    c = AbrBackbone(cdom, [bdom], [bcfg])
    config = ccfg[[x.area_id for x in cdom.areas].index(area.area_id)]
    t = ThirdArea(area, full_inter_area_lsas(a), None, config, [c], [bdom], [bcfg], [ccfg], keys)
    return t, sr


def rib_map(rib, key_name):
    out = {}
    for r in rib.routes:
        hops = rib.nexthops[int(r["nh_off"]): int(r["nh_off"]) + int(r["n_nh"])]
        nh = sorted(((key_name.get(int(x["iface"]), "?"), ospfv3.ip_str(x["addr"]) if x["has_addr"] else None) for x in hops),
                    key=lambda x: (x[0] or "", x[1] or ""))
        out[f"{ospfv3.ip_str(r['prefix'])}/{int(r['len'])}"] = (int(r["metric"]), ospf_rib.PATH_NAMES[int(r["path_type"])],
                                                                nh, int(r["prefix_options"]))
    return out


@pytest.mark.parametrize("g", GOLDEN, ids=GIDS)
def test_base_job_equals_the_recorded_local_rib(abr_harness, abr_backbone_harness, entries_harness, harness, g):
    """Job 0 equals R's recorded local-rib over the affected prefixes (metric, route type, next hops); an inter-area
    route's prefix options are those of its recorded Inter-Area-Prefix LSA.  A totally stubby area gets no slots."""
    t, sr = golden(*g)
    jobs = [t.job_overrides((), 0)]
    for link in non_backbone_links(t)[:4]:
        jobs.append(t.job_overrides(link, capi.COST_DISABLED))
    cells, _, _ = t.check(abr_harness, abr_backbone_harness, entries_harness, harness, jobs)
    mine = rib_map(t.decode(cells[0]), {v: k for k, v in t.keys.items()})
    affected = {f"{ospfv3.ip_str(p)}/{int(l)}" for p, l in zip(t.table.prefixes6, t.table.plen)}
    want = {k: v for k, v in gu.golden_rib(sr).items() if k in affected}
    norm = lambda d: {k: (v[0], v[1], [(a or "", b or "") for a, b in v[2]]) for k, v in d.items()}
    assert norm(mine) == norm(want)
    recorded = {}
    for s in t.summaries[t.summaries["lsa_type"] == 3]:
        recorded.setdefault(f"{ospfv3.ip_str(s['prefix'])}/{int(s['len'])}", set()).add(int(s["prefix_options"]))
    for k, v in mine.items():
        if v[1] == "inter-area":
            assert v[3] in recorded[k]
    if t.config[2] == 0:                                               # totally stubby: nothing moves
        assert t.table.n_slots == 0
    else:
        assert t.table.n_prefixes > 0 and t.table.n_slots > 0
    assert t.table.v3 and t.table.third_area and t.table.n_asbr_slots == 0 and t.table.n_asbr_sets == 0


# ------------------------------------------------------------------------------------------- generated
class SynthThirdArea(ThirdArea):
    """ospfv3.third_area_view: R of area 3, n_c C's, the three B's of area 1, k area-1 ASBRs."""

    def __init__(self, seed, n_c=2, k=2, max_paths=16):
        t0 = synth.random_topology(30, 90, synth.SEED_BASE + 950 + 3 * seed, cost_choices=[5, 10, 20])
        t1 = synth.random_topology(25, 70, synth.SEED_BASE + 951 + 3 * seed, cost_choices=[5, 10, 20])
        t3 = synth.random_topology(25, 70, synth.SEED_BASE + 952 + 3 * seed, cost_choices=[5, 10, 20])
        v = ospfv3.third_area_view(t0, t1, t3, seed, oracle_spf, n_c=n_c, max_paths=max_paths, area1_asbrs=k)
        self.view = v
        ext = v["externals"]
        bdoms = [v3abr.Domain(areas, sums, ext) for areas, _ids, sums in v["borders"]]
        bcfgs = [[ospf_rib.area_config()] * len(d.areas) for d in bdoms]
        cs = [AbrBackbone(v3abr.Domain(areas, sums, ext), bdoms, bcfgs) for areas, _ids, sums in v["c_areas"]]
        super().__init__(v["r_area"], v["summaries3"], ext, ospf_rib.area_config(), cs, bdoms, bcfgs,
                         [[ospf_rib.area_config()] * 2 for _ in cs])

    def key_index(self, key):
        b = np.frombuffer(key[0], np.uint8)
        u = [i for i in range(self.table.n_prefixes)
             if (self.table.prefixes6[i]["bytes"] == b).all() and int(self.table.plen[i]) == key[1]]
        return u[0] if u else None

    def cut(self, x):
        """A job: every area-1 link of router x disabled in every B's area planes."""
        ovs = [self.job_overrides(l, capi.COST_DISABLED) for l in non_backbone_links(self)
               if any(y[0] == x and y[2] for y in l)]
        return [{i: e for i in range(len(d.areas)) if (e := sum((o[b].get(i, []) for o in ovs), []))}
                for b, d in enumerate(self.doms)]


def synth_jobs(t, n, seed):
    links = [l for l in non_backbone_links(t)]
    rng = np.random.default_rng(seed)
    jobs = [t.job_overrides((), 0)]
    for k in rng.choice(len(links), min(n, len(links)), replace=False):
        jobs.append(t.job_overrides(links[int(k)], capi.COST_DISABLED))
        jobs.append(t.job_overrides(links[int(k)], int(rng.choice([1, 40]))))
    return jobs


@pytest.mark.parametrize("seed,n_c,k", [(0, 2, 2), (1, 3, 2), (2, 2, 0), (3, 3, 1)])
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_generated_domains_chain(abr_harness, abr_backbone_harness, entries_harness, harness, seed, n_c, k,
                                 narrow_planes):
    t = SynthThirdArea(seed, n_c=n_c, k=k)
    assert t.table.n_slots > 0 and t.table.v3
    assert (t.table.n_asbr_slots > 0) == (k > 0) and t.table.n_asbr_sets == 0
    cells, _, cents = t.check(abr_harness, abr_backbone_harness, entries_harness, harness, synth_jobs(t, 8, seed),
                              narrow_planes)
    assert (cells != cells[0]).any()
    if k:
        assert all(e.shape[1] > 0 for e in cents)


def test_chain_moves_external_routes(abr_harness, abr_backbone_harness, entries_harness, harness):
    """Cutting an area-1 ASBR off from every B changes the C's entries for it, and R's routes to its externals."""
    moved = 0
    for seed in range(3):
        t = SynthThirdArea(seed, n_c=2, k=2)
        jobs = [t.job_overrides((), 0)] + [t.cut(x) for x in t.view["area1_asbrs"]]
        cells, _, cents = t.check(abr_harness, abr_backbone_harness, entries_harness, harness, jobs)
        for j in range(1, len(jobs)):
            moved += int(any((e[j] != e[0]).any() for e in cents)) + int(cells[j].tobytes() != cells[0].tobytes())
    assert moved > 0


def test_option_flip_through_two_hops_is_other(abr_harness, abr_backbone_harness, entries_harness, harness):
    """third_area_view's flip /128: cutting the links of its lower-id advertiser hands the first B's route to the other
    advertiser's record at the same metric, with the other option (LA / P).  Where C's route goes through that B's
    slot and R's route keeps its metric and next hops, R's winner changes, the delta reports OTHER and the decode gives
    the other option."""
    n = 0
    for seed in range(4):
        t = SynthThirdArea(seed, n_c=2, k=0)
        key = t.view["flip"]
        a1 = next(a for a in t.doms[0].areas if a.area_id == 1)
        advs = sorted(int(l["adv_rtr"]) for l in a1.iap_lsas
                      for p in a1.prefixes[int(l["prefix_off"]): int(l["prefix_off"]) + int(l["n_prefixes"])]
                      if bytes(int(b) for b in p["addr"]["bytes"]) == key[0])
        cells, ccells, _ = t.check(abr_harness, abr_backbone_harness, entries_harness, harness,
                                   [t.job_overrides((), 0), t.cut(advs[0])])
        u = t.key_index(key)
        assert u is not None
        a, b = cells[0][u], cells[1][u]
        assert ospf_rib.cell_path(a) == ospf_rib.PATH_INTER and int(a["winner"]) >= t.table.n_records
        if int(a["mpf"]) == int(b["mpf"]) and int(a["nh_mask"]) == int(b["nh_mask"]) and a["winner"] != b["winner"]:
            assert (int(a["winner"]) ^ int(b["winner"])) & 0xFF                   # the options byte moved
            _, recs, _ = reference(cells, cells[:1])
            assert [int(r["kind"]) for r in recs if int(r["job"]) == 1 and int(r["prefix"]) == u] == [DELTA_OTHER]
            o = lambda rib: {(x["prefix"].tobytes()[:16], int(x["len"])): int(x["prefix_options"]) for x in rib.routes}
            assert {o(t.decode(cells[0]))[key], o(t.decode(cells[1]))[key]} == {ospfv3.PFX_LA, ospfv3.PFX_P}
            n += 1
    assert n > 0


def test_ties_between_cs_merge_atoms(abr_harness, abr_backbone_harness, entries_harness, harness):
    """Some inter-area route reaches R through two C's at one metric: its cell ORs their atoms."""
    n = 0
    for seed in range(4):
        t = SynthThirdArea(seed, n_c=3, k=1)
        cells, _, _ = t.check(abr_harness, abr_backbone_harness, entries_harness, harness, synth_jobs(t, 4, seed))
        inter = ((ospf_rib.cell_flags(cells) & 1) != 0) & (ospf_rib.cell_path(cells) == ospf_rib.PATH_INTER)
        multi = np.vectorize(lambda m: bin(int(m)).count("1") > 1)(cells["nh_mask"])
        n += int((inter & multi & (cells["winner"] >= t.table.n_records)).sum())
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
    lib = capi.load_library()
    h = C.c_void_p()
    cfg = np.array([t.config], ospf_rib.AREA_CONFIG_DT)
    arr = (C.c_void_p * 1)(cts[0].handle.value)
    # no border, and a NULL border array
    assert lib.hspf_ospfv3_third_area_table_create(t.flat.handle, t.area.router_id, cfg.ctypes.data,
                                                   t.summaries.ctypes.data, len(t.summaries), None, 0, arr, 0,
                                                   C.byref(h)) == capi.HSPF_E_INVAL
    assert lib.hspf_ospfv3_third_area_table_create(t.flat.handle, t.area.router_id, cfg.ctypes.data,
                                                   t.summaries.ctypes.data, len(t.summaries), None, 0, None, 1,
                                                   C.byref(h)) == capi.HSPF_E_INVAL
    # versions: an OSPFv2 C table to the OSPFv3 create, an OSPFv3 one to the OSPFv2 create, and the Python table
    # refusing a flat and borders of different versions
    import test_ospf_third_area_cells as v2t
    v2 = v2t.SynthThirdArea(0)
    v2c = v2.cs[0].table
    assert lib.hspf_ospfv3_third_area_table_create(t.flat.handle, t.area.router_id, cfg.ctypes.data,
                                                   t.summaries.ctypes.data, len(t.summaries), None, 0,
                                                   (C.c_void_p * 2)(cts[0].handle.value, v2c.handle.value), 2,
                                                   C.byref(h)) == capi.HSPF_E_INVAL
    cfg2 = np.array([v2.config], ospf_rib.AREA_CONFIG_DT)
    assert lib.hspf_ospfv2_third_area_table_create(v2.flat.handle, v2.area.router_id, cfg2.ctypes.data,
                                                   v2.summaries.ctypes.data, len(v2.summaries), None, 0,
                                                   (C.c_void_p * 1)(cts[0].handle.value), 1,
                                                   C.byref(h)) == capi.HSPF_E_INVAL
    with pytest.raises(ValueError):
        mk(borders=[v2c])
    with pytest.raises(ValueError):
        ospf_rib.BackboneTable(v2.flat, v2.area.router_id, v2.summaries, v2.externals, cts, config=v2.config)
    with pytest.raises(ValueError):                                        # borders of both kinds
        mk(borders=[cts[0], t.doms[0].rt])
    # a border that is not a B-flag router of R's area
    from test_ospfv3_abr_backbone_cells import with_b_cleared, with_flags
    c1 = t.cs[1].r.areas[0].router_id
    refused(capi.HSPF_E_INVAL, flat=ospfv3.Flat(with_b_cleared(t.area, c1)))
    refused(capi.HSPF_E_INVAL, borders=[cts[0]] * 2)                                  # a border twice
    refused(capi.HSPF_E_INVAL, borders=cts * 5)                                       # more than 8
    refused(capi.HSPF_E_INVAL, rid=t.cs[0].r.areas[0].router_id)                     # R is an ABR, among the borders
    refused(capi.HSPF_E_UNSUPPORTED, config=ospf_rib.area_config(ospf_rib.AREA_NSSA))
    # a C's Inter-Area-Prefix LSA for a prefix of its table it cannot advertise: a B-advertised prefix that C's table
    # holds only through an external
    c0 = t.cs[0].r.areas[0].router_id
    from test_ospfv3_abr_backbone_cells import iap_row
    ext_keys = {(e["prefix"]["bytes"].tobytes(), int(e["len"])) for e in t.externals
                if int(e["adv_rtr"]) in set(t.view["area1_asbrs"])}
    key = next((p["bytes"].tobytes(), int(l)) for p, l in zip(cts[0].prefixes6, cts[0].plen)
               if (p["bytes"].tobytes(), int(l)) in ext_keys)
    s = srt(np.concatenate([t.summaries, iap_row(c0, key)]))
    refused(capi.HSPF_E_INVAL, sums=s)
    # a V-flag router in R's area
    refused(capi.HSPF_E_UNSUPPORTED, flat=ospfv3.Flat(with_flags(t.area, t.view["area3_asbr"], 0x04)))


def test_slot_winners_must_fit_32_bits(harness):
    """A table whose slot winners would not fit 32 bits is refused (HSPF_E_UNSUPPORTED).  A real one needs about 2^24
    OSPFv3 slots, so the rule the create applies with the OSPFv3 encoding (n_records + (slots << 8) below 0xFFFFFFFF;
    chain slots are no winners) is checked at its exact edge, and a generated table is checked to pass it."""
    fit = harness.harness_third_area_v3_winners_fit
    S = 0xFFFFFF
    assert fit(0xFE, S) == 1 and fit(0xFF, S) == 0 and fit(0, S + 1) == 0
    assert fit(0xFFFFFFFE, 0) == 1 and fit(0xFFFFFFFF, 0) == 0
    t = SynthThirdArea(0)
    assert fit(t.table.n_records, t.table.n_slots) == 1


def test_versions_do_not_mix(abr_harness, abr_backbone_harness, entries_harness, harness):
    """The OSPFv3 walk's harness refuses a table that is not an OSPFv3 third-area one; the OSPFv2 decode refuses the
    OSPFv3 table."""
    import test_ospf_third_area_cells as v2t
    v2 = v2t.SynthThirdArea(0)
    assert harness.harness_ospfv3_third_area_cells(v2.table.handle, 0, *([None] * 3), 0, *([None] * 6)) == -1
    t = SynthThirdArea(0)
    cells, _, _, _, _ = t.run(abr_harness, abr_backbone_harness, entries_harness, harness, [t.job_overrides((), 0)])
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.backbone_from_cells(v2.area, t.table, cells[0], [], [])
    assert e.value.code == capi.HSPF_E_INVAL


def test_job_status(abr_harness, abr_backbone_harness, entries_harness, harness):
    """A B status word or a B row out of range reaches C's entries status, which reaches R's job status; R's row-0
    word and C's cell status too.  A refused job gets empty cells; the others are unchanged."""
    t = SynthThirdArea(1, n_c=2, k=2)
    jobs = synth_jobs(t, 3, 1)
    J = len(jobs)
    want, st, ccells, cents, bp = t.run(abr_harness, abr_backbone_harness, entries_harness, harness, jobs)
    assert not st.any()
    c = t.cs[0]
    assert c.table.n_asbr_sets > 0 and len(c.table.asbr_ids) > 0
    rows = [np.repeat(np.arange(J, dtype=np.uint32)[:, None], len(d.areas), 1) for d in t.doms]
    for r in rows:
        r[2, :] = J                                                       # every B's row of job 2 out of range
    ps = [[np.zeros(J, np.uint32) for _ in d.areas] for d in t.doms]
    for b in range(len(t.doms)):
        for x in ps[b]:
            x[1] = 0x8                                                    # every B's words of job 1
    ent, est = asbr_entries(entries_harness, c.table, c.planes, bp, rows=rows, pstatus=ps)
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
