"""CPU: the batched routing-table stage for area border routers (update_rib_full over every attached area, for
every job of a what-if batch).

The device kernel's body (abr_rib_cell_eval, holo_b200/csrc/ospf_abr_rib_cells.h) is compiled into a test harness and
run on the CPU over the oracle's SPT planes, one row per area and job.  The cells, decoded by
hspf_ospfv2_abr_rib_from_cells, must equal byte for byte what hspf_ospfv2_update_rib_full gives over
hspf_ospfv2_area_from_planes of each area's row, with the areas' Summary-LSAs and the AS-external LSAs."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import golden_util as gu
from holo_b200 import capi, ospf_rib, ospfv2, synth
from oracle import pyoracle
from test_ospf_rib_cells import same_rib
from test_ospf_rib_delta import link_pairs
from test_ospfv2_route_cells import gather_for

ROOT = Path(__file__).resolve().parent.parent
SNAPS = [s for s in gu.load_ospfv2() if len(s["areas"]) > 1]


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    out = tmp_path_factory.mktemp("harness") / "libospf_abr_rib_cells_harness.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                    "-o", str(out), str(ROOT / "tests" / "native" / "ospf_abr_rib_cells_harness.cc")], check=True)
    lib = C.CDLL(str(out))
    for fn in (lib.harness_abr_rib_cells, lib.harness_abr_rib_cells16):
        fn.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 8
    return lib


def planes_of(csr, root, overrides=()):
    c = pyoracle.csr_spf(csr, root, overrides=overrides, nh_words=1)
    assert c["status"] == 0
    return (np.ascontiguousarray(c["dist"], np.uint32), np.ascontiguousarray(c["hops"], np.uint16),
            np.ascontiguousarray(c["nh_mask"], np.uint64).reshape(-1))


def narrow(p):
    d = np.where(p[0] == 0xFFFFFFFF, 0xFFFF, p[0]).astype(np.uint16)
    return d, p[1], p[2].astype(np.uint16)


def harness_cells(harness, rt, area_rows, rows, status=None, narrow_planes=False):
    """Cells [n_jobs, P] and status words: area_rows[i] = (d [R_i, V_i], h, m) stacked rows of area i; rows [J, A]."""
    rows = np.ascontiguousarray(rows, np.uint32)
    J = rows.shape[0]
    keep = [np.ascontiguousarray(x) for ar in area_rows for x in ar]
    ptr = lambda k: (C.c_void_p * len(area_rows))(*[keep[3 * i + k].ctypes.data for i in range(len(area_rows))])
    n_rows = np.asarray([ar[0].shape[0] for ar in area_rows], np.uint32)
    st = None
    if status is not None:
        sk = [np.ascontiguousarray(s, np.uint32) for s in status]
        keep += sk
        st = (C.c_void_p * len(sk))(*[s.ctypes.data for s in sk])
    cells = np.zeros((J, rt.n_prefixes), ospf_rib.RIB_CELL_DT)
    out = np.zeros(J, np.uint32)
    fn = harness.harness_abr_rib_cells16 if narrow_planes else harness.harness_abr_rib_cells
    fn(rt.handle, J, rows.ctypes.data, ptr(0), ptr(1), ptr(2), st, n_rows.ctypes.data, cells.ctypes.data, out.ctypes.data)
    return cells, out


class Domain:
    """One ABR's attached areas (images in instance order), their flats, summaries, externals and the table."""

    def __init__(self, areas, summaries, externals, active=None):
        self.areas, self.summaries, self.externals = areas, summaries, externals
        self.active = active if active is not None else [True] * len(areas)
        self.flats = [ospfv2.Flat(a) for a in areas]
        self.rv = [f.router_vertex(a.router_id) for f, a in zip(self.flats, areas)]
        self.rt = ospf_rib.AbrRibTable(areas[0].router_id, self.flats, [a.area_id for a in areas], summaries,
                                       self.active, externals)

    def planes(self, overrides=None):
        """Each area's planes (overrides: {area index: [(edge, cost)]})."""
        overrides = overrides or {}
        return [planes_of(f.csr, r, overrides.get(i, ())) for i, (f, r) in enumerate(zip(self.flats, self.rv))]

    def cells(self, harness, job_planes, narrow_planes=False):
        ps = [narrow(p) if narrow_planes else p for p in job_planes]
        area_rows = [tuple(x[None] for x in p) for p in ps]
        cells, st = harness_cells(harness, self.rt, area_rows, [[0] * len(ps)], narrow_planes=narrow_planes)
        return cells[0], int(st[0])

    def decode(self, cells, job_planes):
        ga, gv, gn = [], [], []
        for i, (f, r, p) in enumerate(zip(self.flats, self.rv, job_planes)):
            v, n = gather_for(f, r, p)
            ga += [i] * len(v); gv += list(v); gn += list(n)
        return ospf_rib.abr_rib_from_cells(self.areas, self.rt, cells, ga, gv, gn)

    def host(self, job_planes, lsdb_areas=None):
        """The contract: update_rib_full over area_from_planes of each area's planes."""
        areas = lsdb_areas or self.areas
        ra = []
        for i, (a, p) in enumerate(zip(areas, job_planes)):
            spf = ospfv2.area_from_planes(a, lambda csr, root, nhw, p=p: (p[0], p[1], np.pad(p[2][:, None], ((0, 0), (0, nhw - 1)))))
            ra.append(ospf_rib.RibArea(a.area_id, spf, a.ifaces, self.summaries[i], self.active[i]))
        return ospf_rib.update_rib_full(areas[0].router_id, areas[0].max_paths, ra, self.externals)

    def check(self, harness, overrides=None, narrow_planes=False):
        p = self.planes(overrides)
        cells, st = self.cells(harness, p, narrow_planes)
        assert st == 0
        got = self.decode(cells, p)
        want = self.host(p)
        same_rib(got, want)
        return cells, got


def golden_domain(snap):
    keys = gu.global_sort_keys(snap)
    areas, sums, active = [], [], []
    for area in snap["areas"]:
        img = gu.ospfv2_area_image(snap, area, keys)
        if ospfv2.Flat(img).router_vertex(img.router_id) == 0xFFFFFFFF:
            continue
        areas.append(img)
        sums.append(gu.ospfv2_summaries(area))
        active.append(any((i.get("state") or "down") != "down" for i in area["interfaces"]))
    return Domain(areas, sums, None, active), keys


# ---------------------------------------------------------------------------------------------- goldens
@pytest.mark.parametrize("snap", SNAPS, ids=[f"{s['topo']}-{s['rt']}" for s in SNAPS])
def test_golden_snapshots(harness, snap):
    """Every multi-area golden snapshot (ABRs): the decoded cells equal update_rib_full, and the reference's local-rib."""
    dom, keys = golden_domain(snap)
    cells, got = dom.check(harness)
    key_name = {v: k for k, v in keys.items()}
    mine = {}
    for r in got.routes:
        nh = sorted(((key_name.get(i, "?"), gu.ipstr(a) if ha else None) for (i, ha, a, _hn, _n, _hl, _l) in got.nh(r)),
                    key=lambda x: (x[0] or "", x[1] or ""))
        mine[f"{gu.ipstr(r['prefix'])}/{bin(int(r['mask'])).count('1')}"] = (int(r["metric"]), ospf_rib.PATH_NAMES[int(r["path_type"])], nh)
    want = gu.golden_rib(snap)
    norm = lambda d: {k: (v[0], v[1], [(a or "", b or "") for a, b in v[2]]) for k, v in d.items()}
    assert norm(mine) == norm(want)


def test_golden_snapshots_cover_abrs_and_transit_areas(harness):
    assert len(SNAPS) == 17
    n_transit = 0
    for snap in SNAPS:
        dom, _ = golden_domain(snap)
        vl = dom.rt.off  # noqa: F841
        p = dom.planes()
        # a transit area: some area with a reached V-flag router, which the walk's step 3 reads
        for a, f, pl in zip(dom.areas, dom.flats, p):
            vs = [v for v in range(len(f.ids)) if f.is_router[v] and int(a.router_lsas["flags"][[int(x) for x in a.router_lsas["adv_rtr"]].index(int(f.ids[v]))]) & 0x04]
            if any(pl[0][v] != 0xFFFFFFFF for v in vs):
                n_transit += 1
                break
    assert n_transit == 6


# ------------------------------------------------------------------------------------------- synthetic
def topo(V, E, seed, **kw):
    return synth.random_topology(V, E, synth.SEED_BASE + 700 + seed, **kw)


def domain(seed, n_areas=3, V=40, E=150, area_ids=None, active=None, max_paths=16, v_flag_area=1, lan=0.15):
    ts = [topo(V + 7 * k, E + 20 * k, seed * 10 + k, cost_choices=[5, 10, 20], lan_fraction=lan) for k in range(n_areas)]
    areas, sums, ext = ospfv2.abr_view(ts, 1000 + seed, area_ids=area_ids, roots=[k for k in range(n_areas)],
                                       max_paths=max_paths, v_flag_area=v_flag_area)
    return Domain(areas, sums, ext, active)


def router_edges(dom, i, rng, n=1):
    """Overrides disabling n router-to-router links of area i, both directions."""
    pairs = link_pairs(dom.flats[i])
    return [(int(e), capi.COST_DISABLED) for k in rng.choice(len(pairs), n, replace=False) for e in pairs[int(k)]]


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("mp", [1, 2, 16])
def test_synthetic_domains(harness, seed, mp):
    dom = domain(seed, max_paths=mp)
    cells, got = dom.check(harness)
    kinds = set(int(x) for x in got.routes["path_type"])
    assert kinds == {0, 1, 2, 3}


@pytest.mark.parametrize("seed", range(3))
def test_what_if_rows(harness, seed):
    """Jobs whose rows perturb the backbone, one other area, or both: each job against the host pipeline over the
    same planes."""
    dom = domain(seed)
    rng = np.random.default_rng(seed)
    for which in ({0}, {1}, {0, 1}, {2}, {0, 2}):
        for _ in range(3):
            ov = {i: router_edges(dom, i, rng, 2) for i in which}
            dom.check(harness, ov)


def test_what_if_rows_in_one_batch(harness):
    """Several jobs over stacked rows of each area: rows select per area; cells equal the one-job runs."""
    dom = domain(1)
    rng = np.random.default_rng(5)
    base = dom.planes()
    alt = [dom.planes({i: router_edges(dom, i, rng, 2)})[i] for i in range(3)]
    area_rows = [tuple(np.stack([b[k], a[k]]) for k in range(3)) for b, a in zip(base, alt)]
    rows = [[0, 0, 0], [1, 0, 0], [0, 1, 1], [1, 1, 1]]
    cells, st = harness_cells(harness, dom.rt, area_rows, rows)
    assert not st.any()
    for j, r in enumerate(rows):
        p = [alt[i] if r[i] else base[i] for i in range(3)]
        one, _ = dom.cells(harness, p)
        assert cells[j].tobytes() == one.tobytes()
        same_rib(dom.decode(cells[j], p), dom.host(p))


def v_flag_vertices(dom, i):
    a, f = dom.areas[i], dom.flats[i]
    fl = {int(r): int(x) for r, x in zip(a.router_lsas["adv_rtr"], a.router_lsas["flags"])}
    return [v for v in range(len(f.ids)) if f.is_router[v] and fl.get(int(f.ids[v]), 0) & 0x04]


def test_cutting_the_v_flag_router_turns_the_transit_step_off(harness):
    """A job that cuts the only reached V-flag router of the transit area: step 3 is off for that job only."""
    n_diff = 0
    for seed in range(6):
        dom = domain(seed)
        vs = v_flag_vertices(dom, 1)
        assert len(vs) == 1
        f = dom.flats[1]
        ov = {1: [(e, capi.COST_DISABLED) for e in range(f.csr.n_edges)
                  if f.csr.col[e] == vs[0] or f.csr.row_ptr[vs[0]] <= e < f.csr.row_ptr[vs[0] + 1]]}
        p = dom.planes(ov)
        assert p[1][0][vs[0]] == 0xFFFFFFFF
        c_cut, _ = dom.check(harness, ov)
        c_base, _ = dom.check(harness)
        n_diff += int((c_cut != c_base).any())
    assert n_diff > 0


def test_cutting_another_abr(harness):
    dom = domain(2)
    a0, f0 = dom.areas[0], dom.flats[0]
    abr = next(f0.router_vertex(int(r)) for r, x in zip(a0.router_lsas["adv_rtr"], a0.router_lsas["flags"])
               if x & 0x01 and int(r) != a0.router_id and f0.router_vertex(int(r)) != 0xFFFFFFFF
               and dom.planes()[0][0][f0.router_vertex(int(r))] != 0xFFFFFFFF)
    ov = {0: [(e, capi.COST_DISABLED) for e in range(f0.csr.n_edges)
              if f0.csr.col[e] == abr or f0.csr.row_ptr[abr] <= e < f0.csr.row_ptr[abr + 1]]}
    dom.check(harness, ov)


def test_one_active_area(harness):
    """With one active area every area's summaries are read (and type-4 entries of non-backbone areas count)."""
    for seed in range(3):
        d_all = domain(seed)
        d_one = domain(seed, active=[True, False, False])
        d_one.check(harness)
        d_two = domain(seed, active=[False, True, False])
        d_two.check(harness)
        assert d_one.rt.n_contributors >= d_all.rt.n_contributors


def test_abr_without_backbone(harness):
    for seed in range(3):
        dom = domain(seed, n_areas=2, area_ids=[1, 2], v_flag_area=None)
        dom.check(harness)


def test_narrow_planes_equal_wide(harness):
    n = 0
    for seed in range(4):
        dom = domain(seed, V=30, E=90)
        p = dom.planes()
        if any(int(np.bitwise_or.reduce(x[2])) >> 16 for x in p):
            continue
        wide, _ = dom.cells(harness, p)
        nar, _ = dom.cells(harness, p, narrow_planes=True)
        assert wide.tobytes() == nar.tobytes()
        n += 1
    assert n >= 1


def atom_masks(rt):
    return [(((1 << rt.n_atoms[i]) - 1) << rt.atom_base[i]) if rt.n_atoms[i] else 0 for i in range(rt.n_areas)]


def test_equal_cost_intra_routes_merge_across_areas(harness):
    """Shared prefixes at tying metrics, no transit area (step 3 never runs): some intra-area cell's atoms come from
    two areas, which only the step-1 merge across areas gives."""
    n = 0
    for seed in range(4):
        dom = domain(seed, v_flag_area=None)
        cells, _ = dom.check(harness)
        masks = atom_masks(dom.rt)
        for c in cells:
            if ospf_rib.cell_flags(c) & 1 and ospf_rib.cell_path(c) == ospf_rib.PATH_INTRA:
                n += int(sum(1 for m in masks if int(c["nh_mask"]) & m) > 1)
    assert n > 0


def ext_cells(dom, cells, prefixes):
    u = [int(np.nonzero(dom.rt.prefix == p)[0][0]) for p in prefixes if (dom.rt.prefix == p).any()]
    return cells[u]


def test_step4_prefers_a_non_backbone_intra_area_entry(harness):
    """Each non-backbone area's ASBR is also named by a backbone type-4 LSA at a lower forwarding metric: the externals
    still go through the intra-area entry of the non-backbone area."""
    n = 0
    for seed in range(3):
        dom = domain(seed)
        cells, _ = dom.check(harness)
        p = dom.planes()
        masks = atom_masks(dom.rt)
        f0, s0 = dom.flats[0], dom.summaries[0]
        for k in (1, 2):
            a, f = dom.areas[k], dom.flats[k]
            asbr = next(int(r) for r, x in zip(a.router_lsas["adv_rtr"], a.router_lsas["flags"]) if x & 0x02)
            t4 = s0[(s0["lsa_type"] == 4) & (s0["lsa_id"] == asbr)]
            assert len(t4) == 1
            via_bb = int(p[0][0][f0.router_vertex(int(t4["adv_rtr"][0]))]) + 1
            if via_bb >= int(p[k][0][f.router_vertex(asbr)]):
                continue
            ec = ext_cells(dom, cells, [0x0E000000 + (k << 16) + (i << 8) for i in range(3)])
            assert len(ec) and all(int(c["nh_mask"]) & ~masks[k] == 0 and int(c["nh_mask"]) for c in ec)
            n += 1
    assert n > 0


def test_step4_ties_across_areas_go_to_the_higher_area_id(harness):
    """With one active area every area's type-4 LSAs count: the ASBR every non-backbone area names at one forwarding
    metric is reached through the area with the higher id."""
    for seed in range(3):
        dom = domain(seed, active=[True, False, False])
        cells, _ = dom.check(harness)
        masks = atom_masks(dom.rt)
        ec = ext_cells(dom, cells, [0x0E0F0000, 0x0E0F0100])
        assert len(ec) == 2
        assert all(int(c["nh_mask"]) and int(c["nh_mask"]) & ~masks[2] == 0 for c in ec)


def test_transit_step_rechecks_the_area_after_every_lsa(harness):
    """Two transit-area type-3 LSAs for an area-0 route: the first lowers it (the route leaves area 0), so the second,
    at the same metric through another ABR, must not merge its atoms."""
    INF = 0xFFFFFFFF
    n = 0
    for seed in range(6):
        dom = domain(seed)
        p = dom.planes()
        base = dom.host(p)
        f1, a1 = dom.flats[1], dom.areas[1]
        d1, m1 = p[1][0], p[1][2]
        abrs = sorted(int(r) for r, x in zip(a1.router_lsas["adv_rtr"], a1.router_lsas["flags"])
                      if x & 0x01 and int(r) != a1.router_id and d1[f1.router_vertex(int(r))] != INF)
        pairs = [(x, y) for x in abrs for y in abrs if x < y and m1[f1.router_vertex(x)] & ~m1[f1.router_vertex(y)]
                 and m1[f1.router_vertex(y)] & ~m1[f1.router_vertex(x)]]
        if not pairs:
            continue
        x, y = pairs[0]
        dx, dy = int(d1[f1.router_vertex(x)]), int(d1[f1.router_vertex(y)])
        T = max(dx, dy) + 1
        cand = [r for r in base.routes if r["path_type"] == ospf_rib.PATH_INTRA and r["area_id"] == 0 and r["metric"] > T
                and not (dom.summaries[1]["lsa_id"] == r["prefix"]).any()]
        if not cand:
            continue
        r = cand[0]
        add = np.array([(x, r["prefix"], r["mask"], T - dx, 3, 0, (0, 0)), (y, r["prefix"], r["mask"], T - dy, 3, 0, (0, 0))],
                       ospf_rib.SUMMARY_LSA_DT)
        s1 = np.concatenate([dom.summaries[1], add])
        s1 = s1[np.lexsort((s1["lsa_id"], s1["adv_rtr"], s1["lsa_type"]))]
        d2 = Domain(dom.areas, [dom.summaries[0], s1] + dom.summaries[2:], dom.externals)
        cells, got = d2.check(harness)
        u = int(np.nonzero((d2.rt.prefix == r["prefix"]) & (d2.rt.plen == bin(int(r["mask"])).count("1")))[0][0])
        assert ospf_rib.cell_path(cells[u]) == ospf_rib.PATH_INTER
        assert int(cells[u]["nh_mask"]) == int(m1[f1.router_vertex(x)]) << d2.rt.atom_base[1]
        n += 1
    assert n > 0


# ------------------------------------------------------------------------------------------- refusals
def test_table_refusals():
    dom = domain(0)
    flats, ids = dom.flats, [a.area_id for a in dom.areas]
    rid = dom.areas[0].router_id
    with pytest.raises(capi.HspfError) as e:                     # more areas than the kernels' bound
        ospf_rib.AbrRibTable(rid, flats * 3, ids * 3, dom.summaries * 3)
    assert e.value.code == capi.HSPF_E_UNSUPPORTED
    with pytest.raises(capi.HspfError) as e:                     # the root missing from one flat
        ospf_rib.AbrRibTable(rid + 1, flats, ids, dom.summaries)
    assert e.value.code == capi.HSPF_E_INVAL
    # a usable backbone type-4 LSA naming an ABR
    a0 = dom.areas[0]
    abrs = [int(r) for r, x in zip(a0.router_lsas["adv_rtr"], a0.router_lsas["flags"]) if x & 0x01 and int(r) != rid]
    bad = np.concatenate([dom.summaries[0], np.array([(abrs[1], abrs[0], 0, 10, 4, 0, (0, 0))], ospf_rib.SUMMARY_LSA_DT)])
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.AbrRibTable(rid, flats, ids, [bad] + dom.summaries[1:])
    assert e.value.code == capi.HSPF_E_UNSUPPORTED
    # ... not in an area step 2 does not read
    a1 = dom.areas[1]
    abrs1 = [int(r) for r, x in zip(a1.router_lsas["adv_rtr"], a1.router_lsas["flags"]) if x & 0x01 and int(r) != rid]
    ok = np.concatenate([dom.summaries[1], np.array([(abrs1[0], abrs1[1], 0, 10, 4, 0, (0, 0))], ospf_rib.SUMMARY_LSA_DT)])
    ospf_rib.AbrRibTable(rid, flats, ids, [dom.summaries[0], ok, dom.summaries[2]])
    # more than 64 atoms
    big = [synth.random_topology(40, 900, synth.SEED_BASE + 790 + k, cost_choices=[10]) for k in range(3)]
    areas, sums, ext = ospfv2.abr_view(big, 5, roots=[0, 0, 0])
    fl = [ospfv2.Flat(a) for a in areas]
    n_atoms = sum(capi.atom_count(f.csr, f.router_vertex(areas[0].router_id)) for f in fl)
    assert n_atoms > 64 and all(capi.atom_count(f.csr, f.router_vertex(areas[0].router_id)) <= 64 for f in fl)
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.AbrRibTable(areas[0].router_id, fl, [a.area_id for a in areas], sums)
    assert e.value.code == capi.HSPF_E_UNSUPPORTED
    # areas whose max_paths differ
    a2 = ospfv2.Ospfv2Area(**{k: getattr(dom.areas[1], k) for k in dom.areas[1].__dataclass_fields__})
    a2.max_paths = 2
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.AbrRibTable(rid, [flats[0], ospfv2.Flat(a2)], ids[:2], dom.summaries[:2])
    assert e.value.code == capi.HSPF_E_INVAL


def test_job_refusals(harness):
    dom = domain(1)
    p = dom.planes()
    area_rows = [tuple(np.stack([x, x]) for x in q) for q in p]
    rows = [[0, 0, 0], [0, 2, 0], [1, 1, 1], [0, 0, 1]]
    status = [np.array([0, 0], np.uint32), np.array([0, 0x1], np.uint32), np.array([0, 0x4], np.uint32)]
    cells, st = harness_cells(harness, dom.rt, area_rows, rows, status=status)
    assert list(st) == [0, capi.JS_INVALID, 0x1 | 0x4, 0x4]
    assert (cells["winner"][0] != ospf_rib.NO_RECORD).any()
    for j in (1, 2, 3):
        assert (cells["winner"][j] == ospf_rib.NO_RECORD).all() and not cells["mpf"][j].any() and not cells["nh_mask"][j].any()


def test_decode_refusals(harness):
    dom = domain(0)
    p = dom.planes()
    cells, _ = dom.cells(harness, p)
    with pytest.raises(capi.HspfError):                           # areas out of the table's order
        ospf_rib.abr_rib_from_cells(dom.areas[::-1], dom.rt, cells, [], [], [])
    bad = cells.copy()
    k = int(np.nonzero((ospf_rib.cell_flags(bad) & 1) & (ospf_rib.cell_path(bad) == ospf_rib.PATH_INTRA))[0][0])
    bad["mpf"][k] |= np.uint32(0x4 << 28)                          # HL_CELL_MIXED_SID
    assert ospf_rib.abr_rib_from_cells(dom.areas, dom.rt, bad, [], [], []).rc == capi.HSPF_E_UNSUPPORTED
