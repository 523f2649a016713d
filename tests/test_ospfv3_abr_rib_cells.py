"""CPU: the batched routing-table stage for OSPFv3 area border routers (update_rib_full<Ospfv3> over every attached
area, for every job of a what-if batch).

The device kernel's body (abr_rib_cell_eval, holo_b200/csrc/ospf_abr_rib_cells.h) runs in the CPU harness over the
oracle's SPT planes, one row per area and job, and the table of hspf_ospfv3_abr_ribtable_create.  The cells, decoded by
hspf_ospfv3_abr_rib_from_cells, must equal byte for byte what hspf_ospfv3_update_rib_full gives over
hspf_ospfv3_area_from_planes of each area's row, with the areas' Inter-Area-Prefix / Inter-Area-Router LSAs and the
AS-external LSAs — routes, prefix options and next hops."""
import ctypes as C

import numpy as np
import pytest

import golden_util as gu
import test_ospf_abr_rib_cells as v2
from holo_b200 import capi, ospf_rib, ospfv3, synth
from test_ospf_abr_rib_cells import harness, harness_cells  # noqa: F401  (harness: the fixture)
from test_ospf_rib_cells import same_rib
from test_ospfv2_route_cells import gather_for
from test_ospfv3_rib_cells import rib_dict

SNAPS = [s for s in gu.load_ospfv3() if len(s["areas"]) > 1]
INF = 0xFFFFFFFF


class Domain(v2.Domain):
    """One OSPFv3 ABR's attached areas (images in instance order), flats, inter-area LSAs, externals and the table."""

    def __init__(self, areas, summaries, externals, active=None):
        self.areas, self.summaries, self.externals = areas, summaries, externals
        self.active = active if active is not None else [True] * len(areas)
        self.flats = [ospfv3.Flat(a) for a in areas]
        self.rv = [f.router_vertex(a.router_id) for f, a in zip(self.flats, areas)]
        self.rt = ospf_rib.AbrRibTable(areas[0].router_id, self.flats, [a.area_id for a in areas], summaries,
                                       self.active, externals)

    def gathers(self, job_planes):
        ga, gv, gn = [], [], []
        for i, (f, r, p) in enumerate(zip(self.flats, self.rv, job_planes)):
            v, n = gather_for(f, r, p)
            ga += [i] * len(v); gv += list(v); gn += list(n)
        return ga, gv, gn

    def decode(self, cells, job_planes):
        return ospf_rib.abr_rib_from_cells_v3(self.areas, self.rt, cells, *self.gathers(job_planes))

    def host(self, job_planes, lsdb_areas=None):
        areas = lsdb_areas or self.areas
        ra = []
        for i, (a, p) in enumerate(zip(areas, job_planes)):
            spf = ospfv3.area_from_planes(a, lambda csr, root, nhw, p=p: (p[0], p[1], np.pad(p[2][:, None], ((0, 0), (0, nhw - 1)))))
            ra.append(ospf_rib.RibArea(a.area_id, spf, a.ifaces, self.summaries[i], self.active[i]))
        return ospf_rib.update_rib_full_v3(areas[0].router_id, areas[0].max_paths, ra, self.externals)


def golden_domain(snap):
    keys = gu.global_sort_keys(snap)
    areas, sums, active = [], [], []
    for area in snap["areas"]:
        img = gu.ospfv3_area_image(snap, area, keys)
        if ospfv3.Flat(img).router_vertex(img.router_id) == INF:
            continue
        areas.append(img)
        sums.append(gu.ospfv3_inter_area_lsas(area))
        active.append(any((i.get("state") or "down") != "down" for i in area["interfaces"]))
    return Domain(areas, sums, None, active), keys


def router_edges(dom, i, rng, n=1):
    """Overrides disabling n router-to-router links of area i, both directions."""
    csr, isr = dom.flats[i].csr, dom.flats[i].is_router
    src = np.repeat(np.arange(csr.n_vertices), np.diff(csr.row_ptr))
    pairs, seen = [], set()
    for e in range(csr.n_edges):
        a, b = int(src[e]), int(csr.col[e])
        if e in seen or not (isr[a] and isr[b]):
            continue
        back = [f for f in range(int(csr.row_ptr[b]), int(csr.row_ptr[b + 1])) if int(csr.col[f]) == a and f not in seen]
        if back:
            seen |= {e, back[0]}
            pairs.append((e, back[0]))
    return [(int(e), capi.COST_DISABLED) for k in rng.choice(len(pairs), n, replace=False) for e in pairs[int(k)]]


def first_flags(area):
    out = {}
    for r, f in zip(area.router_lsas["adv_rtr"], area.router_lsas["flags"]):
        out.setdefault(int(r), int(f))                 # the first fragment's, as the table reads them
    return out


def v_flag_vertices(dom, i):
    fl, f = first_flags(dom.areas[i]), dom.flats[i]
    return [v for v in range(len(f.router_ids)) if f.is_router[v] and fl.get(int(f.router_ids[v]), 0) & 0x04]


# ---------------------------------------------------------------------------------------------- goldens
@pytest.mark.parametrize("snap", SNAPS, ids=[f"{s['topo']}-{s['rt']}" for s in SNAPS])
def test_golden_snapshots(harness, snap):
    """Every multi-area OSPFv3 golden snapshot (ABRs): the decoded cells equal update_rib_full_v3, and the reference's
    local-rib."""
    dom, keys = golden_domain(snap)
    assert dom.rt.v3 and len(dom.areas) > 1
    cells, got = dom.check(harness)
    mine = rib_dict(got, {v: k for k, v in keys.items()})
    norm = lambda d: {k: (v[0], v[1], [(a or "", b or "") for a, b in v[2]]) for k, v in d.items()}
    assert norm(mine) == norm(gu.golden_rib(snap))


def test_golden_snapshots_cover_abrs_and_transit_areas():
    """14 ABR snapshots, of which N_TRANSIT have a transit area: an area with a V-flag router the root reaches, which
    the walk's transit-area step reads."""
    assert len(SNAPS) == 14
    n_transit = 0
    for snap in SNAPS:
        dom, _ = golden_domain(snap)
        p = dom.planes()
        n_transit += int(any(p[i][0][v] != INF for i in range(len(dom.areas)) for v in v_flag_vertices(dom, i)))
    assert n_transit == N_TRANSIT


N_TRANSIT = 6


# ------------------------------------------------------------------------------------------- synthetic
def domain(seed, n_areas=3, V=40, E=150, area_ids=None, active=None, max_paths=16, v_flag_area=1, lan=0.15, roots=None,
           order=None):
    ts = [v2.topo(V + 7 * k, E + 20 * k, 50 + seed * 10 + k, cost_choices=[5, 10, 20], lan_fraction=lan)
          for k in range(n_areas)]
    areas, sums, ext = ospfv3.abr_view(ts, 3000 + seed, area_ids=area_ids,
                                       roots=roots if roots is not None else list(range(n_areas)),
                                       max_paths=max_paths, v_flag_area=v_flag_area)
    if order is not None:
        areas, sums = [areas[i] for i in order], [sums[i] for i in order]
        active = None if active is None else [active[i] for i in order]
    return Domain(areas, sums, ext, active)


@pytest.mark.parametrize("roots", [(0, 1, 2), (3, 0, 5), (7, 7, 7)])
@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("mp", [1, 2, 16])
def test_synthetic_domains(harness, roots, seed, mp):
    dom = domain(seed, max_paths=mp, roots=list(roots))
    cells, got = dom.check(harness)
    assert set(int(x) for x in got.routes["path_type"]) == {0, 1, 2, 3}
    assert (got.routes["prefix_options"] != 0).any()


@pytest.mark.parametrize("seed", range(3))
def test_what_if_rows(harness, seed):
    """Jobs whose rows perturb the backbone, one other area, or both: each job against the host pipeline."""
    dom = domain(seed)
    rng = np.random.default_rng(seed)
    for which in ({0}, {1}, {0, 1}, {2}, {0, 2}):
        for _ in range(2):
            dom.check(harness, {i: router_edges(dom, i, rng, 2) for i in which})


def test_what_if_rows_in_one_batch(harness):
    dom = domain(1)
    rng = np.random.default_rng(5)
    base = dom.planes()
    alt = [dom.planes({i: router_edges(dom, i, rng, 2)})[i] for i in range(3)]
    area_rows = [tuple(np.stack([b[k], a[k]]) for k in range(3)) for b, a in zip(base, alt)]
    rows = [[0, 0, 0], [1, 0, 0], [0, 1, 1], [1, 1, 1], [0, 0, 1]]
    cells, st = harness_cells(harness, dom.rt, area_rows, rows)
    assert not st.any()
    for j, r in enumerate(rows):
        p = [alt[i] if r[i] else base[i] for i in range(3)]
        one, _ = dom.cells(harness, p)
        assert cells[j].tobytes() == one.tobytes()
        same_rib(dom.decode(cells[j], p), dom.host(p))


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
        same_rib(dom.decode(nar, p), dom.host(p))
        n += 1
    assert n >= 1


def test_cutting_the_v_flag_router_turns_the_transit_step_off(harness):
    n_diff = 0
    for seed in range(6):
        dom = domain(seed)
        vs = v_flag_vertices(dom, 1)
        assert len(vs) == 1
        f = dom.flats[1]
        ov = {1: [(e, capi.COST_DISABLED) for e in range(f.csr.n_edges)
                  if f.csr.col[e] == vs[0] or f.csr.row_ptr[vs[0]] <= e < f.csr.row_ptr[vs[0] + 1]]}
        assert dom.planes(ov)[1][0][vs[0]] == INF
        c_cut, _ = dom.check(harness, ov)
        c_base, _ = dom.check(harness)
        n_diff += int((c_cut != c_base).any())
    assert n_diff > 0


def test_cutting_another_abr(harness):
    for seed in range(2):
        dom = domain(seed)
        a0, f0 = dom.areas[0], dom.flats[0]
        p0 = dom.planes()[0][0]
        abr = next(f0.router_vertex(r) for r, x in first_flags(a0).items()
                   if x & 0x01 and r != a0.router_id and f0.router_vertex(r) != INF and p0[f0.router_vertex(r)] != INF)
        ov = {0: [(e, capi.COST_DISABLED) for e in range(f0.csr.n_edges)
                  if f0.csr.col[e] == abr or f0.csr.row_ptr[abr] <= e < f0.csr.row_ptr[abr + 1]]}
        dom.check(harness, ov)


def test_one_active_area(harness):
    for seed in range(3):
        d_all = domain(seed)
        d_one = domain(seed, active=[True, False, False])
        d_one.check(harness)
        domain(seed, active=[False, True, False]).check(harness)
        assert d_one.rt.n_contributors >= d_all.rt.n_contributors


def test_abr_without_backbone(harness):
    for seed in range(3):
        domain(seed, n_areas=2, area_ids=[1, 2], v_flag_area=None).check(harness)


# ------------------------------------------------------------------------------------------- walk rules
def intra_ties(dom, cells):
    """Prefix indices of intra-area cells whose atoms come from more than one area."""
    masks = v2.atom_masks(dom.rt)
    return [u for u, c in enumerate(cells) if ospf_rib.cell_flags(c) & 1 and ospf_rib.cell_path(c) == ospf_rib.PATH_INTRA
            and sum(1 for m in masks if int(c["nh_mask"]) & m) > 1]


def test_cross_area_tie_keeps_the_first_areas_prefix_options(harness):
    """Intra-area routes of two areas at one metric, whose prefix options differ (abr_view gives area 0's prefix no
    option and the other area's the LA bit): the route keeps the options of the first area in the caller's order, as
    update_rib_full does, whichever that area is."""
    n = 0
    for seed in range(4):
        for order in ([0, 1, 2], [1, 0, 2], [2, 1, 0]):
            dom = domain(seed, v_flag_area=None, order=order)
            cells, got = dom.check(harness)
            masks = v2.atom_masks(dom.rt)
            by_prefix = {(x["prefix"].tobytes(), int(x["len"])): x for x in got.routes}
            for u in intra_ties(dom, cells):
                r = by_prefix[(dom.rt.prefixes6[u].tobytes(), int(dom.rt.plen[u]))]
                # the first area, in the caller's order, of those whose routes tie
                first = next(dom.areas[i].area_id for i in range(3) if int(cells[u]["nh_mask"]) & masks[i])
                assert int(r["area_id"]) == first
                want = 0 if first == 0 else ospfv3.PFX_LA
                assert int(r["prefix_options"]) == want, (order, u)
                n += 1
    assert n > 0


def test_step4_prefers_a_non_backbone_intra_area_entry(harness):
    """Each non-backbone area's ASBR is also named by a backbone Inter-Area-Router LSA at a lower forwarding metric: its
    externals still go through the intra-area entry of the non-backbone area."""
    n = 0
    for seed in range(3):
        dom = domain(seed)
        cells, _ = dom.check(harness)
        p = dom.planes()
        masks = v2.atom_masks(dom.rt)
        f0, s0 = dom.flats[0], dom.summaries[0]
        for k in (1, 2):
            a, f = dom.areas[k], dom.flats[k]
            asbr = next(r for r, x in first_flags(a).items() if x & 0x02)
            t4 = s0[(s0["lsa_type"] == 4) & (s0["router_id"] == asbr)]
            assert len(t4) == 1 and int(t4["lsa_id"][0]) != asbr
            via_bb = int(p[0][0][f0.router_vertex(int(t4["adv_rtr"][0]))]) + 1
            if via_bb >= int(p[k][0][f.router_vertex(asbr)]):
                continue
            own = ipv6_rows(dom, [(0xE0_0000 + (k << 8) + i) for i in (0, 2)])
            assert len(own) == 2
            for u in own:
                c = cells[u]
                assert int(c["nh_mask"]) and int(c["nh_mask"]) & ~masks[k] == 0
            n += 1
    assert n > 0


def ipv6_rows(dom, his):
    """Prefix indices of the table's 2001:db8:<hi>::/64 prefixes, for each hi present."""
    out = []
    for hi in his:
        b = np.frombuffer(((0x20010DB8 << 96) | (hi << 64)).to_bytes(16, "big"), np.uint8)
        k = [u for u in range(dom.rt.n_prefixes) if (dom.rt.prefixes6[u]["bytes"] == b).all() and dom.rt.plen[u] == 64]
        out += k
    return out


def test_step4_ties_across_areas_go_to_the_higher_area_id(harness):
    for seed in range(3):
        dom = domain(seed, active=[True, False, False])
        cells, _ = dom.check(harness)
        masks = v2.atom_masks(dom.rt)
        ec = ipv6_rows(dom, [0xEF_0000, 0xEF_0001])
        assert len(ec) == 2
        assert all(int(cells[u]["nh_mask"]) and int(cells[u]["nh_mask"]) & ~masks[2] == 0 for u in ec)


def test_transit_step_rechecks_the_area_after_every_lsa(harness):
    """Two transit-area Inter-Area-Prefix LSAs for an area-0 route: the first lowers it (the route leaves area 0), so
    the second, at the same metric through another ABR, must not merge its atoms."""
    n = 0
    for seed in range(6):
        dom = domain(seed)
        p = dom.planes()
        base = dom.host(p)
        f1, a1 = dom.flats[1], dom.areas[1]
        d1, m1 = p[1][0], p[1][2]
        abrs = sorted(r for r, x in first_flags(a1).items()
                      if x & 0x01 and r != a1.router_id and d1[f1.router_vertex(r)] != INF)
        pairs = [(x, y) for x in abrs for y in abrs if x < y and m1[f1.router_vertex(x)] & ~m1[f1.router_vertex(y)]
                 and m1[f1.router_vertex(y)] & ~m1[f1.router_vertex(x)]]
        if not pairs:
            continue
        x, y = pairs[0]
        dx, dy = int(d1[f1.router_vertex(x)]), int(d1[f1.router_vertex(y)])
        T = max(dx, dy) + 1
        s1 = dom.summaries[1]
        named = {s["prefix"].tobytes() for s in s1}
        cand = [r for r in base.routes if r["path_type"] == ospf_rib.PATH_INTRA and r["area_id"] == 0 and r["metric"] > T
                and r["prefix"].tobytes() not in named]
        if not cand:
            continue
        r = cand[0]
        add = np.zeros(2, ospf_rib.INTER_AREA_LSA_DT)
        add[0] = (x, 0x900, T - dx, 0, r["prefix"], r["len"], 0, 3, 0)
        add[1] = (y, 0x900, T - dy, 0, r["prefix"], r["len"], 0, 3, 0)
        s1 = np.concatenate([s1, add])
        s1 = s1[np.lexsort((s1["lsa_id"], s1["adv_rtr"], s1["lsa_type"]))]
        d2 = Domain(dom.areas, [dom.summaries[0], s1] + dom.summaries[2:], dom.externals)
        cells, got = d2.check(harness)
        u = next(u for u in range(d2.rt.n_prefixes)
                 if d2.rt.prefixes6[u].tobytes() == r["prefix"].tobytes() and d2.rt.plen[u] == r["len"])
        assert ospf_rib.cell_path(cells[u]) == ospf_rib.PATH_INTER
        assert int(cells[u]["nh_mask"]) == int(m1[f1.router_vertex(x)]) << d2.rt.atom_base[1]
        n += 1
    assert n > 0


def table_arrays(rt):
    return (rt.n_prefixes, rt.off.tobytes(), rt.contribs.tobytes(), rt.prefixes6.tobytes(), rt.plen.tobytes())


def test_nu_option_lsas_are_left_out(harness):
    """An Inter-Area-Prefix or AS-external LSA with the NU option builds the same table as no LSA at all, while an
    Inter-Area-Router LSA with it still counts."""
    dom = domain(2)
    s0, ext = dom.summaries[0], dom.externals
    nu3 = (s0["lsa_type"] == 3) & (s0["prefix_options"] & ospfv3.PFX_NU != 0)
    nu5 = ext["prefix_options"] & ospfv3.PFX_NU != 0
    assert nu3.any() and nu5.any()
    for summaries, externals in (([s0[~nu3]] + dom.summaries[1:], ext), (dom.summaries, ext[~nu5])):
        d2 = Domain(dom.areas, summaries, externals)
        assert table_arrays(d2.rt) == table_arrays(dom.rt)
    nu4 = (s0["lsa_type"] == 4) & (s0["prefix_options"] & ospfv3.PFX_NU != 0)
    if nu4.any():
        d3 = Domain(dom.areas, [s0[~nu4]] + dom.summaries[1:], ext)
        assert table_arrays(d3.rt) != table_arrays(dom.rt)
    dom.check(harness)


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
    # a usable backbone Inter-Area-Router LSA naming an ABR (in router_id; its lsa_id names nothing)
    fl0 = first_flags(dom.areas[0])
    abrs = [r for r, x in fl0.items() if x & 0x01 and r != rid]
    bad = np.zeros(1, ospf_rib.INTER_AREA_LSA_DT)
    bad[0] = (abrs[1], 0x999, 10, abrs[0], dom.summaries[0]["prefix"][0], 0, 0, 4, 0)
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.AbrRibTable(rid, flats, ids, [np.concatenate([dom.summaries[0], bad])] + dom.summaries[1:])
    assert e.value.code == capi.HSPF_E_UNSUPPORTED
    # the same LSA with the ABR in lsa_id only is no refusal
    ok0 = bad.copy()
    ok0[0]["lsa_id"], ok0[0]["router_id"] = abrs[0], 0x0B0000AA
    ospf_rib.AbrRibTable(rid, flats, ids, [np.concatenate([dom.summaries[0], ok0])] + dom.summaries[1:])
    # ... nor in an area step 2 does not read
    fl1 = first_flags(dom.areas[1])
    abrs1 = [r for r, x in fl1.items() if x & 0x01 and r != rid]
    ok = bad.copy()
    ok[0]["adv_rtr"], ok[0]["router_id"] = abrs1[0], abrs1[1]
    ospf_rib.AbrRibTable(rid, flats, ids, [dom.summaries[0], np.concatenate([dom.summaries[1], ok]), dom.summaries[2]])
    # more than 64 atoms
    big = [synth.random_topology(40, 900, synth.SEED_BASE + 790 + k, cost_choices=[10]) for k in range(3)]
    areas, sums, ext = ospfv3.abr_view(big, 5, roots=[0, 0, 0])
    fl = [ospfv3.Flat(a) for a in areas]
    counts = [capi.atom_count(f.csr, f.router_vertex(ospfv3.ABR_ROUTER_ID)) for f in fl]
    assert sum(counts) > 64 and max(counts) <= 64
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.AbrRibTable(ospfv3.ABR_ROUTER_ID, fl, [a.area_id for a in areas], sums)
    assert e.value.code == capi.HSPF_E_UNSUPPORTED
    # areas whose max_paths differ
    a2 = ospfv3.Ospfv3Area(**{k: getattr(dom.areas[1], k) for k in dom.areas[1].__dataclass_fields__})
    a2.max_paths = 2
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.AbrRibTable(rid, [flats[0], ospfv3.Flat(a2)], ids[:2], dom.summaries[:2])
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


def raw_decode(fn, area_struct, areas, rt, cells, ga, gv, gn, route_dt, nh_dt, caps):
    arr = (area_struct * len(areas))(*[a.as_struct() for a in areas])
    ga, gv = np.asarray(ga, np.uint32), np.asarray(gv, np.uint32)
    gn = np.asarray(gn, np.uint64)
    routes, nhs = np.zeros(max(caps[0], 1), route_dt), np.zeros(max(caps[1], 1), nh_dt)
    r = ospf_rib.RibStruct(caps[0], 0, routes.ctypes.data, caps[1], 0, nhs.ctypes.data)
    rc = fn(rt.handle, arr, len(areas), np.ascontiguousarray(cells).ctypes.data, ga.ctypes.data, gv.ctypes.data,
            gn.ctypes.data, len(gv), C.byref(r))
    return rc, r.n_routes, r.n_nexthops


def test_decode_refusals(harness):
    lib = capi.load_library()
    dom = domain(0)
    p = dom.planes()
    cells, _ = dom.cells(harness, p)
    ga, gv, gn = dom.gathers(p)
    got = dom.decode(cells, p)
    v3 = lambda areas, rt=dom.rt, c=cells, g=(ga, gv, gn), caps=(4096, 65536): raw_decode(
        lib.hspf_ospfv3_abr_rib_from_cells, ospfv3.AreaStruct, areas, rt, c, *g, ospf_rib.RIB_ROUTE6_DT,
        ospfv3.NEXTHOP6_DT, caps)
    assert v3(dom.areas)[0] == capi.HSPF_OK
    # the whole table does not fit: HSPF_E_NOMEM with the counts
    assert v3(dom.areas, caps=(1, 65536)) == (capi.HSPF_E_NOMEM, len(got.routes), len(got.nexthops))
    assert v3(dom.areas, caps=(4096, 1)) == (capi.HSPF_E_NOMEM, len(got.routes), len(got.nexthops))
    assert v3(dom.areas[::-1])[0] == capi.HSPF_E_INVAL                      # areas out of the table's order
    wrong_rid = [ospfv3.Ospfv3Area(**{k: getattr(a, k) for k in a.__dataclass_fields__}) for a in dom.areas]
    wrong_rid[1].router_id += 1
    assert v3(wrong_rid)[0] == capi.HSPF_E_INVAL
    wrong_area = [ospfv3.Ospfv3Area(**{k: getattr(a, k) for k in a.__dataclass_fields__}) for a in dom.areas]
    wrong_area[2].area_id += 7
    assert v3(wrong_area)[0] == capi.HSPF_E_INVAL
    assert v3(dom.areas, g=([3] + ga[1:], gv, gn))[0] == capi.HSPF_E_INVAL   # gather_area out of range
    bad = cells.copy()
    k = int(np.nonzero((ospf_rib.cell_flags(bad) & 1) & (ospf_rib.cell_path(bad) == ospf_rib.PATH_INTRA))[0][0])
    bad["mpf"][k] |= np.uint32(0x4 << 28)                                    # HL_CELL_MIXED_SID
    assert v3(dom.areas, c=bad)[0] == capi.HSPF_E_UNSUPPORTED
    # the versions' tables and decodes do not mix
    d2 = v2.domain(0)
    c2, _ = d2.cells(harness, d2.planes())
    assert not d2.rt.__dict__.get("v3")
    assert raw_decode(lib.hspf_ospfv3_abr_rib_from_cells, ospfv3.AreaStruct, dom.areas, d2.rt, c2, [], [], [],
                      ospf_rib.RIB_ROUTE6_DT, ospfv3.NEXTHOP6_DT, (4096, 65536))[0] == capi.HSPF_E_INVAL
    assert raw_decode(lib.hspf_ospfv2_abr_rib_from_cells, ospf_rib.ospfv2.AreaStruct, d2.areas, dom.rt, cells, [], [], [],
                      ospf_rib.RIB_ROUTE_DT, ospf_rib.ospfv2.NEXTHOP_DT, (4096, 65536))[0] == capi.HSPF_E_INVAL
    assert lib.hspf_ospfv3_abr_ribtable_prefixes6(d2.rt.handle, None, None) == capi.HSPF_E_INVAL
