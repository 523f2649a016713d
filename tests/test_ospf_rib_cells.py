"""CPU: the batched routing-table stage for roots attached to one area (update_rib_full, holo-ospf/src/route.rs:146-193,
for every job of a batch).

The device kernel's body (ospf_rib_cell_eval, holo_b200/csrc/ospf_rib_cells.h) is compiled into a test harness and
run on the CPU over the oracle's SPT planes.  The cells, decoded by hspf_ospfv2_rib_from_cells, must equal byte for
byte what hspf_ospfv2_update_rib_full gives over hspf_ospfv2_area_from_planes of the same planes, with the area's
Summary-LSAs and the AS-external LSAs — routes and next hops."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import golden_util as gu
from holo_b200 import capi, ospf_rib, ospfv2, synth
from oracle import pyoracle
from test_ospfv2_route_cells import gather_for

ROOT = Path(__file__).resolve().parent.parent
SNAPS = [s for s in gu.load_ospfv2() if len(s["areas"]) == 1]


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    out = tmp_path_factory.mktemp("harness") / "libospf_rib_cells_harness.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                    "-o", str(out), str(ROOT / "tests" / "native" / "ospf_rib_cells_harness.cc")], check=True)
    lib = C.CDLL(str(out))
    lib.harness_rib_cells.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 7
    lib.harness_rib_cells16.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 7
    return lib


def planes_of(csr, root, nh_words=1, overrides=()):
    c = pyoracle.csr_spf(csr, root, overrides=overrides, nh_words=nh_words)
    assert c["status"] == 0
    return (np.ascontiguousarray(c["dist"], np.uint32), np.ascontiguousarray(c["hops"], np.uint16),
            np.ascontiguousarray(c["nh_mask"], np.uint64).reshape(len(c["dist"]), nh_words))


def harness_cells(harness, rt, roots, planes, status=None, narrow=False):
    """Cells [n_jobs, P] and status words of jobs rooted at `roots` over stacked planes (d [J, V], h [J, V], m [J, V])."""
    d, h, m = planes
    J = len(roots)
    roots = np.ascontiguousarray(roots, np.uint32)
    st = None if status is None else np.ascontiguousarray(status, np.uint32)
    cells = np.zeros((J, rt.n_prefixes), ospf_rib.RIB_CELL_DT)
    out = np.zeros(J, np.uint32)
    fn = harness.harness_rib_cells16 if narrow else harness.harness_rib_cells
    fn(rt.handle, J, roots.ctypes.data, None if st is None else st.ctypes.data, np.ascontiguousarray(d).ctypes.data,
       np.ascontiguousarray(h).ctypes.data, np.ascontiguousarray(m).ctypes.data, cells.ctypes.data, out.ctypes.data)
    return cells, out


def host_rib(area, summaries, externals, csr_planes):
    """The contract: update_rib_full over area_from_planes of the job's planes, one active area."""
    spf = ospfv2.area_from_planes(area, csr_planes)
    return ospf_rib.update_rib_full(area.router_id, area.max_paths,
                                    [ospf_rib.RibArea(area.area_id, spf, area.ifaces, summaries)], externals)


def same_rib(got, want):
    assert got.rc == capi.HSPF_OK
    assert len(got.routes) == len(want.routes), (len(got.routes), len(want.routes))
    for a, b in zip(got.routes, want.routes):
        assert a.tobytes() == b.tobytes(), (a, b)
    assert got.nexthops.tobytes() == want.nexthops.tobytes()


def check_job(harness, area, summaries, externals, overrides=(), lsdb_area=None, narrow=False, rt=None):
    """Cells of area.router_id's job (planes of the area's CSR with `overrides`) decoded, and the host pipeline over
    `lsdb_area` (the LSDB with the overridden metrics; default: `area`).  Returns (rt, cells, status, got, want)."""
    flat = ospfv2.Flat(area)
    rt = rt or ospf_rib.RibTable(flat, area.area_id, summaries, externals)
    rv = flat.router_vertex(area.router_id)
    pl = planes_of(flat.csr, rv, overrides=overrides)
    p = pl
    if narrow:
        d = np.where(pl[0] == 0xFFFFFFFF, 0xFFFF, pl[0]).astype(np.uint16)
        p = (d, pl[1], pl[2].astype(np.uint16))
    cells, st = harness_cells(harness, rt, [rv], tuple(x[None] if x.ndim == 1 else x.reshape(1, -1) for x in p),
                              narrow=narrow)
    if st[0]:
        return rt, cells[0], int(st[0]), None, None
    gv, gn = gather_for(flat, rv, (pl[0], pl[1], pl[2].reshape(-1)))
    got = ospf_rib.rib_from_cells(area, rt, cells[0], gv, gn)
    base = lsdb_area if lsdb_area is not None else area
    want = host_rib(base, summaries, externals, lambda csr, root, nhw: planes_of(csr, root, nhw))
    return rt, cells[0], 0, got, want


# ---------------------------------------------------------------------------------------------- goldens
@pytest.mark.parametrize("snap", SNAPS, ids=[f"{s['topo']}-{s['rt']}" for s in SNAPS])
def test_golden_snapshots(harness, snap):
    """Every single-area golden snapshot: the decoded cells equal update_rib_full, and the reference's local-rib."""
    keys = gu.global_sort_keys(snap)
    area_j = snap["areas"][0]
    img = gu.ospfv2_area_image(snap, area_j, keys)
    sums = gu.ospfv2_summaries(area_j)
    rt, cells, st, got, want = check_job(harness, img, sums, None)
    assert st == 0
    same_rib(got, want)
    key_name = {v: k for k, v in keys.items()}
    mine = {}
    for r in got.routes:
        nh = sorted(((key_name.get(i, "?"), gu.ipstr(a) if ha else None) for (i, ha, a, _hn, _n, _hl, _l) in got.nh(r)),
                    key=lambda x: (x[0] or "", x[1] or ""))
        mine[f"{gu.ipstr(r['prefix'])}/{bin(int(r['mask'])).count('1')}"] = (int(r["metric"]), ospf_rib.PATH_NAMES[int(r["path_type"])], nh)
    assert mine == gu.golden_rib(snap)


def test_golden_snapshots_cover_inter_area_routes():
    n_inter = sum(1 for s in SNAPS if any(r["type"] == "inter-area" for r in s["local_rib"]))
    assert len(SNAPS) == 46 and n_inter == 28
    assert any(any(l["flags"] & 0x04 for l in s["areas"][0]["router_lsas"]) and s["areas"][0]["area_id"] != "0.0.0.0"
               for s in SNAPS)                                   # a transit area with virtual-link endpoints


# ------------------------------------------------------------------------------------------- synthetic
def view(t, root, seed, max_paths=16, **kw):
    """Router `root`'s image of area 0.0.0.1 of topology `t`, with the generator's ABRs, ASBRs and LSAs."""
    a = ospfv2.synth_area(t, root=root, max_paths=max_paths)
    a.area_id = 1
    return ospfv2.inter_area_view(a, seed, **kw)


def flags_of(area):
    return {int(r): int(f) for r, f in zip(area.router_lsas["adv_rtr"], area.router_lsas["flags"])}


@pytest.mark.parametrize("V,E,seed,kw,mp", [
    (40, 160, 1, dict(cost_choices=[10]), 16),
    (60, 240, 2, dict(cost_choices=[10, 20], lan_fraction=0.15), 16),
    (60, 240, 3, dict(cost_choices=[10, 20], lan_fraction=0.15), 2),
    (50, 220, 4, dict(cost_choices=[10], lan_fraction=0.1), 1),
    (80, 300, 5, dict(cost_choices=[5, 10], lan_fraction=0.2), 16),
])
def test_every_root_of_synthetic_areas(harness, V, E, seed, kw, mp):
    t = synth.random_topology(V, E, synth.SEED_BASE + 300 + seed, **kw)
    kinds, n_refused, n_multi = set(), 0, 0
    for root in range(V):
        area, sums, ext = view(t, root, 900 + seed, mp)
        rt, cells, st, got, want = check_job(harness, area, sums, ext)
        if st:
            assert st == ospf_rib.JS_NOT_INTERNAL and int(area.router_lsas["flags"][root]) & 0x01
            assert (cells["winner"] == ospf_rib.NO_RECORD).all() and not cells["mpf"].any()
            n_refused += 1
            continue
        same_rib(got, want)
        kinds |= set(int(x) for x in got.routes["path_type"])
        n_multi += int((got.routes["n_nh"] > 1).sum())
    assert kinds == {0, 1, 2, 3} and n_refused == 4
    if mp > 1 and kw.get("lan_fraction"):
        assert n_multi > 0


def test_generated_lsas_exercise_every_rule(harness):
    """The generator's LSAs meet every rule of the walk for some root: intra over inter over external, an ABR no job
    reaches, a type-4 entry replacing an ASBR's intra-area entry, self-originated externals, equal type-2 metrics."""
    t = synth.random_topology(60, 240, synth.SEED_BASE + 302, cost_choices=[10, 20], lan_fraction=0.15)
    area, sums, ext = view(t, 0, 902)
    flat = ospfv2.Flat(area)
    rt = ospf_rib.RibTable(flat, area.area_id, sums, ext)
    P = rt.n_prefixes
    n_intra = np.diff(rt.off[0]) > 0
    n3 = np.diff(rt.off[1]) > 0
    n5 = np.diff(rt.off[2]) > 0
    assert (n_intra & n3).any() and (n3 & n5).any() and (n_intra & n5).any() and (~n_intra & ~n3 & n5).any()
    # host bits kept: a type-3 / type-5 prefix that is not a network address
    masks = np.where(rt.plen == 0, 0, (0xFFFFFFFF << (32 - rt.plen.astype(np.uint64))) & 0xFFFFFFFF).astype(np.uint64)
    assert ((rt.prefix.astype(np.uint64) & ~masks & 0xFFFFFFFF) != 0).any()
    lost = int(area.router_lsas["adv_rtr"][-1])
    assert flat.router_vertex(lost) != 0xFFFFFFFF and pyoracle.csr_spf(flat.csr, 0)["dist"][flat.router_vertex(lost)] == 0xFFFFFFFF
    # in-area ASBRs named by type-4 LSAs; externals with e_bit both ways; maxage and infinity are left out
    e_rtr = {r for r, f in flags_of(area).items() if f & 0x02}
    assert e_rtr & {int(x) for x in sums[sums["lsa_type"] == 4]["lsa_id"]}
    assert set(ext["e_bit"]) == {0, 1} and sums["maxage"].any() and (ext["metric"] == ospf_rib.LSA_INFINITY).any()
    usable5 = int(((ext["maxage"] == 0) & (ext["metric"] < ospf_rib.LSA_INFINITY)).sum())
    assert rt.off[2][P] - rt.off[2][0] == usable5
    # self-originated: a job rooted at an ASBR drops its own externals
    asbr = next(r for r in e_rtr if r in {int(x) for x in ext["adv_rtr"]})
    root = int(np.nonzero(area.router_lsas["adv_rtr"] == asbr)[0][0])
    a2, s2, e2 = view(t, root, 902)
    rt2, cells, st, got, want = check_job(harness, a2, s2, e2)
    assert st == 0
    same_rib(got, want)


def test_narrow_planes_equal_wide(harness):
    t = synth.random_topology(60, 240, synth.SEED_BASE + 302, cost_choices=[10, 20], lan_fraction=0.15)
    n = 0
    for root in range(0, 60, 7):
        area, sums, ext = view(t, root, 902)
        flat = ospfv2.Flat(area)
        rv = flat.router_vertex(area.router_id)
        if capi.atom_count(flat.csr, rv) > 16:
            continue
        rt, wide, st, _, _ = check_job(harness, area, sums, ext)
        _, narrow, st16, _, _ = check_job(harness, area, sums, ext, narrow=True, rt=rt)
        assert st == st16
        assert wide.tobytes() == narrow.tobytes()
        n += 1
    assert n >= 4


# -------------------------------------------------------------------------------------------- what-if
@pytest.mark.parametrize("seed", range(4))
def test_what_if_overrides(harness, seed):
    """A job with edge overrides (metrics changed, links cut): its cells over the base table equal update_rib_full on
    the LSDB with those metrics — including ABRs and ASBRs that a cut leaves unreachable."""
    rng = np.random.default_rng(40 + seed)
    t = synth.random_topology(50, 200, synth.SEED_BASE + 320 + seed, cost_choices=[10, 20], lan_fraction=0.1)
    area, sums, ext = view(t, 3, 950 + seed)
    flat = ospfv2.Flat(area)
    rt = ospf_rib.RibTable(flat, area.area_id, sums, ext)
    csr = flat.csr
    for _ in range(6):
        # router-to-router edges only (a network's edges have no link of their own to change)
        cand = [e for e in range(csr.n_edges) if flat.link_index[e] != 0xFFFFFFFF]
        es = [int(x) for x in rng.choice(cand, 3, replace=False)]
        costs = [int(rng.choice([1, 5, 30, 200, capi.COST_DISABLED])) for _ in es]
        changed = ospfv2.Ospfv2Area(**{k: getattr(area, k) for k in area.__dataclass_fields__})
        changed.links = area.links.copy()
        cut = False
        for e, c in zip(es, costs):
            if c == capi.COST_DISABLED:
                cut = True
            else:
                changed.links["metric"][flat.link_index[e]] = c
        if cut:
            continue                                   # a cut has no LSDB twin with the same vertices; see below
        rt_, cells, st, got, want = check_job(harness, area, sums, ext, overrides=list(zip(es, costs)), lsdb_area=changed,
                                              rt=rt)
        if st:
            continue
        same_rib(got, want)
    # a cut: every edge into and out of an ABR, against the host stages over the same (overridden) planes
    abr = next(flat.router_vertex(r) for r, f in flags_of(area).items() if f & 0x01 and r != area.router_id)
    ov = [(e, capi.COST_DISABLED) for e in range(csr.n_edges)
          if csr.col[e] == abr or csr.row_ptr[abr] <= e < csr.row_ptr[abr + 1]]
    rv = flat.router_vertex(area.router_id)
    pl = planes_of(csr, rv, overrides=ov)
    cells, st = harness_cells(harness, rt, [rv], (pl[0][None], pl[1][None], pl[2].reshape(1, -1)))
    gv, gn = gather_for(flat, rv, (pl[0], pl[1], pl[2].reshape(-1)))
    got = ospf_rib.rib_from_cells(area, rt, cells[0], gv, gn)
    want = host_rib(area, sums, ext, lambda c, r, nhw: planes_of(c, r, nhw, overrides=ov))
    same_rib(got, want)


# ------------------------------------------------------------------------------------------- refusals
def test_table_refusals():
    t = synth.random_topology(30, 120, synth.SEED_BASE + 330, cost_choices=[10])
    area, sums, ext = view(t, 0, 960)
    flat = ospfv2.Flat(area)
    ospf_rib.RibTable(flat, 1, sums, ext)                       # area 1: V flags are not looked at
    vl = area.router_lsas.copy()
    vl["flags"][5] |= 0x04
    a2 = ospfv2.Ospfv2Area(**{k: getattr(area, k) for k in area.__dataclass_fields__})
    a2.router_lsas = vl
    ospf_rib.RibTable(ospfv2.Flat(a2), 1, sums, ext)
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.RibTable(ospfv2.Flat(a2), 0, sums, ext)        # backbone with a virtual-link endpoint
    assert e.value.code == capi.HSPF_E_UNSUPPORTED
    # a usable type-4 LSA naming an ABR
    abr, abr2 = [r for r, f in flags_of(area).items() if f & 0x01][:2]
    bad = np.concatenate([sums, np.array([(abr2, abr, 0, 10, 4, 0, (0, 0))], ospf_rib.SUMMARY_LSA_DT)])
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.RibTable(flat, 1, bad, ext)
    assert e.value.code == capi.HSPF_E_UNSUPPORTED
    for maxage, metric in ((1, 10), (0, ospf_rib.LSA_INFINITY)):    # not usable: no refusal
        ok = np.concatenate([sums, np.array([(abr2, abr, 0, metric, 4, maxage, (0, 0))], ospf_rib.SUMMARY_LSA_DT)])
        ospf_rib.RibTable(flat, 1, ok, ext)


def test_job_refusals(harness):
    t = synth.random_topology(30, 120, synth.SEED_BASE + 330, cost_choices=[10])
    area, sums, ext = view(t, 0, 960)
    flat = ospfv2.Flat(area)
    rt = ospf_rib.RibTable(flat, area.area_id, sums, ext)
    V = flat.csr.n_vertices
    fl = flags_of(area)
    abr_v = flat.router_vertex(next(r for r, f in fl.items() if f & 0x01))
    ok_v = flat.router_vertex(next(r for r, f in fl.items() if not f & 0x01))
    jobs = [ok_v, abr_v, V, ok_v]
    planes = [planes_of(flat.csr, v if v < V else ok_v) for v in jobs]
    stack = tuple(np.stack([p[i].reshape(-1) for p in planes]) for i in range(3))
    status = np.array([0, 0, 0, 0x1], np.uint32)                  # job 3: HSPF_JS_SATURATED
    cells, st = harness_cells(harness, rt, jobs, stack, status=status)
    assert list(st) == [0, ospf_rib.JS_NOT_INTERNAL, 0x8, int(status[3])]
    assert (cells["winner"][0] != ospf_rib.NO_RECORD).any()
    for j in (1, 2, 3):
        assert (cells["winner"][j] == ospf_rib.NO_RECORD).all() and not cells["mpf"][j].any() and not cells["nh_mask"][j].any()
