"""CPU: the batched routing-table stage over OSPFv3 areas (update_rib_full<Ospfv3>, holo-ospf/src/route.rs:146-193, for
every job of a batch).

The device kernel's body (ospf_rib_cell_eval, holo_b200/csrc/ospf_rib_cells.h) runs in the CPU harness over the oracle's
SPT planes and the table of hspf_ospfv3_ribtable_create.  The cells, decoded by hspf_ospfv3_rib_from_cells, must equal
byte for byte what hspf_ospfv3_update_rib_full gives over hspf_ospfv3_area_from_planes of the same planes, with the
area's Inter-Area-Prefix / Inter-Area-Router LSAs and the AS-external LSAs — routes, prefix options and next hops."""
import ctypes as C

import numpy as np
import pytest

import golden_util as gu
from holo_b200 import capi, ospf_rib, ospfv2, ospfv3, synth
from oracle import pyoracle
from test_ospf_rib_cells import harness, harness_cells, planes_of, same_rib  # noqa: F401  (harness: the fixture)
from test_ospfv2_route_cells import gather_for

SNAPS = [s for s in gu.load_ospfv3() if len(s["areas"]) == 1]
INFINITY = ospf_rib.LSA_INFINITY


def host_rib(area, summaries, externals, csr_planes):
    """The contract: update_rib_full_v3 over area_from_planes of the job's planes, one active area."""
    spf = ospfv3.area_from_planes(area, csr_planes)
    return ospf_rib.update_rib_full_v3(area.router_id, area.max_paths,
                                       [ospf_rib.RibArea(area.area_id, spf, area.ifaces, summaries)], externals)


def job_cells(harness, area, rt, overrides=(), narrow=False):
    """(cells, status, gather) of area.router_id's job over the planes of the area's CSR with `overrides`."""
    flat = rt.flat
    rv = flat.router_vertex(area.router_id)
    pl = planes_of(flat.csr, rv, overrides=overrides)
    p = pl
    if narrow:
        d = np.where(pl[0] == 0xFFFFFFFF, 0xFFFF, pl[0]).astype(np.uint16)
        p = (d, pl[1], pl[2].astype(np.uint16))
    cells, st = harness_cells(harness, rt, [rv], tuple(x.reshape(1, -1) for x in p), narrow=narrow)
    return cells[0], int(st[0]), gather_for(flat, rv, (pl[0], pl[1], pl[2].reshape(-1)))


def check_job(harness, area, summaries, externals, overrides=(), lsdb_area=None, narrow=False, rt=None):
    """Cells of area.router_id's job decoded, and the host pipeline over `lsdb_area` (the LSDB with the overridden
    metrics; default: `area`).  Returns (rt, cells, status, got, want)."""
    rt = rt or ospf_rib.RibTable(ospfv3.Flat(area), area.area_id, summaries, externals)
    cells, st, (gv, gn) = job_cells(harness, area, rt, overrides, narrow)
    if st:
        return rt, cells, st, None, None
    got = ospf_rib.rib_from_cells_v3(area, rt, cells, gv, gn)
    base = lsdb_area if lsdb_area is not None else area
    want = host_rib(base, summaries, externals, lambda csr, root, nhw: planes_of(csr, root, nhw))
    return rt, cells, 0, got, want


def copy_area(area, **kw):
    a = ospfv3.Ospfv3Area(**{k: getattr(area, k) for k in area.__dataclass_fields__})
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def rib_dict(rib, key_name):
    out = {}
    for r in rib.routes:
        hops = rib.nexthops[int(r["nh_off"]): int(r["nh_off"]) + int(r["n_nh"])]
        nh = sorted(((key_name.get(int(x["iface"]), "?"), ospfv3.ip_str(x["addr"]) if x["has_addr"] else None) for x in hops),
                    key=lambda x: (x[0] or "", x[1] or ""))
        out[f"{ospfv3.ip_str(r['prefix'])}/{int(r['len'])}"] = (int(r["metric"]), ospf_rib.PATH_NAMES[int(r["path_type"])], nh)
    return out


# ---------------------------------------------------------------------------------------------- goldens
@pytest.mark.parametrize("snap", SNAPS, ids=[f"{s['topo']}-{s['rt']}" for s in SNAPS])
def test_golden_snapshots(harness, snap):
    """Every single-area OSPFv3 golden snapshot: the decoded cells equal update_rib_full_v3, and the reference's
    local-rib."""
    keys = gu.global_sort_keys(snap)
    area_j = snap["areas"][0]
    img = gu.ospfv3_area_image(snap, area_j, keys)
    sums = gu.ospfv3_inter_area_lsas(area_j)
    rt, cells, st, got, want = check_job(harness, img, sums, None)
    assert st == 0
    same_rib(got, want)
    mine = rib_dict(got, {v: k for k, v in keys.items()})
    ref = gu.golden_rib(snap)
    assert set(mine) == set(ref)
    for prefix, (metric, rtype, nh) in ref.items():
        assert mine[prefix][:2] == (metric, rtype), (prefix, mine[prefix])
        assert [(a or "", b or "") for a, b in mine[prefix][2]] == [(a or "", b or "") for a, b in nh], prefix


def test_golden_snapshots_cover_inter_area_routes():
    n_inter = sum(1 for s in SNAPS if any(r["type"] == "inter-area" for r in s["local_rib"]))
    assert len(SNAPS) == 30 and n_inter == 24


# ------------------------------------------------------------------------------------------- synthetic
def view(t, root, seed, max_paths=16, frag=0, **kw):
    """Router `root`'s image of area 0.0.0.1 of topology `t`, with the generator's ABRs, ASBRs and LSAs."""
    a = ospfv3.synth_area(t, root=root, max_paths=max_paths, max_links_per_fragment=frag, area_id=1)
    return ospfv3.inter_area_view(a, seed, **kw)


def flags_of(area):
    out = {}
    for r, f in zip(area.router_lsas["adv_rtr"], area.router_lsas["flags"]):
        out.setdefault(int(r), int(f))                 # the first fragment's, as the table reads them
    return out


@pytest.mark.parametrize("V,E,seed,kw,frag,mp", [
    (40, 160, 1, dict(cost_choices=[10]), 0, 16),
    (60, 240, 2, dict(cost_choices=[10, 20], lan_fraction=0.15), 0, 16),
    (60, 240, 3, dict(cost_choices=[10, 20], lan_fraction=0.15), 3, 2),
    (50, 220, 4, dict(cost_choices=[10], lan_fraction=0.1), 2, 1),
    (80, 300, 5, dict(cost_choices=[5, 10], lan_fraction=0.2), 0, 16),
])
def test_every_root_of_synthetic_areas(harness, V, E, seed, kw, frag, mp):
    t = synth.random_topology(V, E, synth.SEED_BASE + 500 + seed, **kw)
    kinds, n_refused, n_multi, n_options = set(), 0, 0, 0
    for root in range(V):
        area, sums, ext = view(t, root, 1900 + seed, mp, frag)
        rt, cells, st, got, want = check_job(harness, area, sums, ext)
        if st:
            assert st == ospf_rib.JS_NOT_INTERNAL and flags_of(area)[area.router_id] & 0x01
            assert (cells["winner"] == ospf_rib.NO_RECORD).all() and not cells["mpf"].any()
            n_refused += 1
            continue
        same_rib(got, want)
        kinds |= set(int(x) for x in got.routes["path_type"])
        n_multi += int((got.routes["n_nh"] > 1).sum())
        n_options += int((got.routes["prefix_options"] != 0).sum())
    assert kinds == {0, 1, 2, 3} and n_refused == 4
    if mp > 1 and kw.get("lan_fraction"):
        assert n_multi > 0
    if frag:
        assert len(np.unique(area.router_lsas["adv_rtr"])) < len(area.router_lsas)


def test_generated_lsas_exercise_every_rule(harness):
    """The generator's LSAs meet every rule of the walk: intra over inter over external, an ABR no job reaches, NU-bit
    LSAs, Inter-Area-Router LSAs whose lsa_id is not the ASBR, maxage and infinity."""
    t = synth.random_topology(60, 240, synth.SEED_BASE + 502, cost_choices=[10, 20], lan_fraction=0.15)
    area, sums, ext = view(t, 0, 1902)
    flat = ospfv3.Flat(area)
    rt = ospf_rib.RibTable(flat, area.area_id, sums, ext)
    assert rt.v3 and not rt.prefix.dtype == np.uint32 and (rt.prefix["is_v6"] == 1).all()
    P = rt.n_prefixes
    n_intra, n3, n5 = (np.diff(rt.off[i]) > 0 for i in range(3))
    assert (n_intra & n3).any() and (n3 & n5).any() and (n_intra & n5).any() and (~n_intra & ~n3 & n5).any()
    key = [(bytes(int(b) for b in p["bytes"]), int(l)) for p, l in zip(rt.prefix, rt.plen)]
    assert key == sorted(set(key))                                       # 16 address bytes, then the length
    nu = ospfv3.PFX_NU
    t3 = sums[sums["lsa_type"] == 3]
    assert (t3["prefix_options"] & nu).any() and (ext["prefix_options"] & nu).any()
    usable5 = int(((ext["maxage"] == 0) & (ext["metric"] < INFINITY) & ((ext["prefix_options"] & nu) == 0)).sum())
    assert rt.off[2][P] - rt.off[2][0] == usable5
    iar = sums[sums["lsa_type"] == 4]
    assert (iar["lsa_id"] != iar["router_id"]).all()
    e_rtr = {r for r, f in flags_of(area).items() if f & 0x02}
    assert e_rtr & {int(x) for x in iar["router_id"]}
    # self-originated: a job rooted at an in-area ASBR drops its own externals
    asbr = next(r for r in sorted(e_rtr) if r in {int(x) for x in ext["adv_rtr"]})
    a2, s2, e2 = view(t, asbr - ospfv3.RID_BASE, 1902)
    _, _, st, got, want = check_job(harness, a2, s2, e2)
    assert st == 0
    same_rib(got, want)


def test_narrow_planes_equal_wide(harness):
    t = synth.random_topology(60, 240, synth.SEED_BASE + 502, cost_choices=[10, 20], lan_fraction=0.15)
    n = 0
    for root in range(0, 60, 7):
        area, sums, ext = view(t, root, 1902)
        flat = ospfv3.Flat(area)
        if capi.atom_count(flat.csr, flat.router_vertex(area.router_id)) > 16:
            continue
        rt, wide, st, _, _ = check_job(harness, area, sums, ext)
        _, narrow, st16, _, _ = check_job(harness, area, sums, ext, narrow=True, rt=rt)
        assert st == st16
        assert wide.tobytes() == narrow.tobytes()
        n += 1
    assert n >= 4


# -------------------------------------------------------------------------------------------- what-if
@pytest.mark.parametrize("seed", range(3))
def test_what_if_overrides(harness, seed):
    """A job with edge overrides over the base table equals update_rib_full_v3 on the LSDB with those metrics; a cut
    ABR equals the host stages over the same overridden planes."""
    rng = np.random.default_rng(60 + seed)
    t = synth.random_topology(50, 200, synth.SEED_BASE + 520 + seed, cost_choices=[10, 20], lan_fraction=0.1)
    area, sums, ext = view(t, 3, 1950 + seed, frag=2 if seed == 1 else 0)
    flat = ospfv3.Flat(area)
    rt = ospf_rib.RibTable(flat, area.area_id, sums, ext)
    csr = flat.csr
    n = 0
    for _ in range(6):
        # new metrics on three router links of the LSDB: the edges whose cost moves are the job's overrides
        links = area.links.copy()
        for i in rng.choice(np.nonzero(links["link_type"] != ospfv2.LINK_TRANSIT)[0], 3, replace=False):
            links["metric"][i] = int(rng.choice([1, 5, 30, 200]))
        changed = copy_area(area, links=links)
        ncsr = ospfv3.Flat(changed).csr
        assert np.array_equal(ncsr.col, csr.col)
        es = np.nonzero(ncsr.cost != csr.cost)[0]
        _, _, st, got, want = check_job(harness, area, sums, ext, overrides=[(int(e), int(ncsr.cost[e])) for e in es],
                                        lsdb_area=changed, rt=rt)
        assert st == 0
        same_rib(got, want)
        n += len(es) > 0
    assert n >= 4
    abr = next(flat.router_vertex(r) for r, f in flags_of(area).items() if f & 0x01 and r != area.router_id
               and flat.router_vertex(r) != 0xFFFFFFFF and csr.row_ptr[flat.router_vertex(r) + 1] > csr.row_ptr[flat.router_vertex(r)])
    ov = [(e, capi.COST_DISABLED) for e in range(csr.n_edges) if csr.col[e] == abr or csr.row_ptr[abr] <= e < csr.row_ptr[abr + 1]]
    cells, st, (gv, gn) = job_cells(harness, area, rt, ov)
    got = ospf_rib.rib_from_cells_v3(area, rt, cells, gv, gn)
    want = host_rib(area, sums, ext, lambda c, r, nhw: planes_of(c, r, nhw, overrides=ov))
    same_rib(got, want)


# ------------------------------------------------------------------------------------ hand-made LSAs
def small_view(root=0):
    t = synth.random_topology(30, 120, synth.SEED_BASE + 530, cost_choices=[10])
    area, sums, ext = view(t, root, 1960, n_inter=0, n_ext=0, unreachable_abr=False)
    fl = flags_of(area)
    abrs = sorted(r for r, f in fl.items() if f & 0x01)
    plain = sorted(r for r, f in fl.items() if not f & 0x03 and r != area.router_id)
    return area, abrs, plain


def ia_lsa(adv, lsa_id, metric, prefix="2001:db8:77::", plen=64, options=0, lsa_type=3, router_id=0, maxage=0):
    return (adv, lsa_id, metric, router_id, ospfv3.ip_rec(prefix), plen, options, lsa_type, maxage)


def ext_lsa(adv, lsa_id, metric, prefix="2001:db8:99::", plen=64, options=0, e_bit=0, tag=7, maxage=0):
    return (adv, lsa_id, metric, tag, ospfv3.ip_rec(prefix), plen, options, e_bit, maxage)


def lsas(rows, dt):
    out = np.zeros(len(rows), dt)
    for i, r in enumerate(rows):
        out[i] = r
    return out


def decode(harness, area, sums, ext):
    rt, cells, st, got, want = check_job(harness, area, lsas(sums, ospf_rib.INTER_AREA_LSA_DT),
                                         lsas(ext, ospf_rib.EXTERNAL6_LSA_DT))
    assert st == 0
    same_rib(got, want)
    return {f"{ospfv3.ip_str(r['prefix'])}/{int(r['len'])}": r for r in got.routes}


def test_nu_bit_lsas(harness):
    """Inter-Area-Prefix and AS-external LSAs with the NU option give no route; an Inter-Area-Router LSA with it is
    used; the options of the winning LSA are the route's."""
    area, abrs, plain = small_view()
    asbr_out = 0x0B000001
    sums = [ia_lsa(abrs[0], 1, 10, "2001:db8:77::", options=ospfv3.PFX_NU),
            ia_lsa(abrs[0], 2, 10, "2001:db8:78::", options=0x02),
            ia_lsa(abrs[1], 3, 20, "2001:db8:78::", options=0x04),
            ia_lsa(abrs[0], 4, 5, lsa_type=4, router_id=asbr_out, options=ospfv3.PFX_NU)]
    sums.sort(key=lambda x: (x[7], x[0], x[1]))
    ext = [ext_lsa(asbr_out, 1, 3, "2001:db8:99::", options=ospfv3.PFX_NU),
           ext_lsa(asbr_out, 2, 3, "2001:db8:9a::", options=0x08, e_bit=1, tag=11)]
    got = decode(harness, area, sums, ext)
    assert "2001:db8:77::/64" not in got and "2001:db8:99::/64" not in got
    r = got["2001:db8:78::/64"]
    assert int(r["path_type"]) == ospf_rib.PATH_INTER and int(r["prefix_options"]) == 0x02
    r = got["2001:db8:9a::/64"]
    assert int(r["path_type"]) == ospf_rib.PATH_TYPE2 and int(r["prefix_options"]) == 0x08 and int(r["tag"]) == 11
    # the same LSAs without NU are used
    sums[0] = ia_lsa(abrs[0], 1, 10, "2001:db8:77::")
    ext[0] = ext_lsa(asbr_out, 1, 3, "2001:db8:99::")
    got = decode(harness, area, sums, ext)
    assert "2001:db8:77::/64" in got and "2001:db8:99::/64" in got


def test_last_usable_inter_area_router_lsa_wins(harness):
    """An ASBR's entry is the last usable Inter-Area-Router LSA naming it in router_id (lsa_id names nothing):
    maxage, infinity and an LSA from a router that is not an ABR do not count."""
    area, abrs, plain = small_view()
    asbr = 0x0B000005
    flat = ospfv3.Flat(area)
    d = pyoracle.csr_spf(flat.csr, flat.router_vertex(area.router_id))["dist"]
    dist = {r: int(d[flat.router_vertex(r)]) for r in abrs}
    a0, a1 = abrs[0], abrs[1]

    def metric_of(iars):
        sums = sorted(iars + [ia_lsa(a0, 50, 1, "2001:db8:70::")], key=lambda x: (x[7], x[0], x[1]))
        got = decode(harness, area, sums, [ext_lsa(asbr, 1, 3)])
        return int(got["2001:db8:99::/64"]["metric"]) if "2001:db8:99::/64" in got else None

    first, last = ia_lsa(a0, 1, 100, lsa_type=4, router_id=asbr), ia_lsa(a1, 2, 40, lsa_type=4, router_id=asbr)
    assert metric_of([first, last]) == dist[a1] + 40 + 3
    assert metric_of([first]) == dist[a0] + 100 + 3
    for dead in (ia_lsa(a1, 2, 40, lsa_type=4, router_id=asbr, maxage=1), ia_lsa(a1, 2, INFINITY, lsa_type=4, router_id=asbr),
                 ia_lsa(plain[0], 2, 1, lsa_type=4, router_id=asbr)):
        assert metric_of([first, dead]) == dist[a0] + 100 + 3
    # an lsa_id equal to the ASBR's id with another router_id names that other router
    assert metric_of([ia_lsa(a0, asbr, 100, lsa_type=4, router_id=asbr + 1)]) is None


# ------------------------------------------------------------------------------------------- refusals
def test_table_refusals():
    area, abrs, plain = small_view()
    flat = ospfv3.Flat(area)
    ospf_rib.RibTable(flat, 1)
    rl = area.router_lsas.copy()
    rl["flags"][rl["adv_rtr"] == plain[0]] |= 0x04
    vl = copy_area(area, router_lsas=rl)
    ospf_rib.RibTable(ospfv3.Flat(vl), 1)                              # area 1: V flags are not looked at
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.RibTable(ospfv3.Flat(vl), 0)                          # backbone with a virtual-link endpoint
    assert e.value.code == capi.HSPF_E_UNSUPPORTED
    # a usable Inter-Area-Router LSA naming an ABR in router_id
    bad = lsas([ia_lsa(abrs[1], 1, 10, lsa_type=4, router_id=abrs[0])], ospf_rib.INTER_AREA_LSA_DT)
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.RibTable(flat, 1, bad)
    assert e.value.code == capi.HSPF_E_UNSUPPORTED
    for kw in (dict(maxage=1), dict(metric=INFINITY), dict(adv=plain[0])):    # not usable: no refusal
        row = dict(adv=abrs[1], lsa_id=1, metric=10, lsa_type=4, router_id=abrs[0])
        row.update(kw)
        ospf_rib.RibTable(flat, 1, lsas([ia_lsa(**row)], ospf_rib.INTER_AREA_LSA_DT))
    # an ABR's id in lsa_id is not a refusal: router_id names the ASBR
    ospf_rib.RibTable(flat, 1, lsas([ia_lsa(abrs[1], abrs[0], 10, lsa_type=4, router_id=0x0B000001)],
                                    ospf_rib.INTER_AREA_LSA_DT))


def test_job_refusals(harness):
    area, abrs, plain = small_view()
    flat = ospfv3.Flat(area)
    sums = lsas([ia_lsa(abrs[0], 1, 10)], ospf_rib.INTER_AREA_LSA_DT)
    rt = ospf_rib.RibTable(flat, area.area_id, sums)
    V = flat.csr.n_vertices
    abr_v, ok_v = flat.router_vertex(abrs[0]), flat.router_vertex(plain[0])
    jobs = [ok_v, abr_v, V, ok_v]
    planes = [planes_of(flat.csr, v if v < V else ok_v) for v in jobs]
    stack = tuple(np.stack([p[i].reshape(-1) for p in planes]) for i in range(3))
    cells, st = harness_cells(harness, rt, jobs, stack, status=np.array([0, 0, 0, 0x1], np.uint32))
    assert list(st) == [0, ospf_rib.JS_NOT_INTERNAL, 0x8, 0x1]
    assert (cells["winner"][0] != ospf_rib.NO_RECORD).any()
    for j in (1, 2, 3):
        assert (cells["winner"][j] == ospf_rib.NO_RECORD).all() and not cells["mpf"][j].any() and not cells["nh_mask"][j].any()


def test_tables_of_one_version_are_refused_by_the_other(harness):
    area, abrs, plain = small_view()
    rt3 = ospf_rib.RibTable(ospfv3.Flat(area), area.area_id)
    t2 = synth.random_topology(30, 120, synth.SEED_BASE + 530, cost_choices=[10])
    a2 = ospfv2.synth_area(t2, root=0)
    a2.area_id = 1
    rt2 = ospf_rib.RibTable(ospfv2.Flat(a2), 1)
    assert not rt2.v3 and rt3.v3
    lib = capi.load_library()
    for fn, a, rt in ((lib.hspf_ospfv2_rib_from_cells, a2, rt3), (lib.hspf_ospfv3_rib_from_cells, area, rt2)):
        cells = np.zeros(rt.n_prefixes, ospf_rib.RIB_CELL_DT)
        out = ospf_rib.RibStruct()
        s = a.as_struct()
        assert fn(C.byref(s), rt.handle, cells.ctypes.data, None, None, 0, C.byref(out)) == capi.HSPF_E_INVAL
    assert lib.hspf_ospfv3_ribtable_prefixes6(rt2.handle, None, None) == capi.HSPF_E_INVAL
    # the OSPFv3 table's common arrays: prefix[] zero, plen the lengths
    pp, pl = C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint32)()
    lib.hspf_ospfv2_ribtable_arrays(rt3.handle, C.byref(pp), C.byref(pl), None, None)
    assert not np.ctypeslib.as_array(pp, (rt3.n_prefixes,)).any()
    assert np.array_equal(np.ctypeslib.as_array(pl, (rt3.n_prefixes,)), rt3.plen)
    # an area root that is not a router of the area
    cells = np.zeros(rt3.n_prefixes, ospf_rib.RIB_CELL_DT)
    with pytest.raises(capi.HspfError):
        ospf_rib.rib_from_cells_v3(copy_area(area, router_id=0x7F000009), rt3, cells, [], [])
