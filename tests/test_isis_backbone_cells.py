"""CPU: the routes a backbone router R gets from an IS-IS area's L1/L2 routers ("borders") for every L1 what-if job
(include/holo_spf_lsdb.h, hspf_isis_backbone_*).

The device kernels' bodies (isis_l1_to_l2_cell_eval for the borders, isis_backbone_cell_eval for R) are compiled
into test harnesses and run on the CPU over the oracle's SPT planes.  For job j the reference chain builds R's L2
image from its base image: the borders' derived entries dropped, each border's hspf_isis_l1_to_l2 output for the job
appended to its zeroth fragment; then hspf_isis_routes_from_planes and the oracle's compute_routes run on it.  The
product's hspf_isis_backbone_from_cells over R's cells must give the chain's routes of the affected prefixes, byte for
byte, and every other prefix of the chain must be R's base route."""
import copy
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from holo_b200 import capi, isis, ospfv3
from holo_b200.route_table import DELTA_NEXTHOPS, DELTA_OTHER
from oracle import pyoracle
from test_isis_l1_to_l2_cells import adjacencies, failure, view_jobs
from test_isis_l1l2_rib_cells import (TOPOS, golden_pair, level_routes, oracle_planes, own_derived, same_rib,
                                      topology_flat, without)
from test_route_delta import reference

import golden_util as gu

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "holo_b200" / "csrc"


def _harness(name, hdrs):
    out = ROOT / "tests" / "_build" / f"lib{name}_harness.so"
    src = ROOT / "tests" / "native" / f"{name}_harness.cc"
    deps = [src] + [CSRC / n for n in hdrs]
    if not out.exists() or out.stat().st_mtime < max(p.stat().st_mtime for p in deps):
        out.parent.mkdir(parents=True, exist_ok=True)
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                        "-o", str(out), str(src)], check=True)
    return C.CDLL(str(out))


WALK_HDRS = ("isis_l1_to_l2_cells.h", "isis_l1l2_rib_cells.h", "isis_route_cells.h", "route_cells.h")


@pytest.fixture(scope="module")
def harness(built):
    l1 = _harness("isis_l1_to_l2_cells", WALK_HDRS)
    l1.harness_isis_l1_to_l2_cells.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 6
    bb = _harness("isis_backbone_cells", WALK_HDRS + ("isis_backbone_cells.h",))
    bb.harness_isis_backbone_cells.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 5
    return l1, bb


# ---- the borders ------------------------------------------------------------------------------------------------
class Border:
    """One L1/L2 router: its images, tables and, per job, its L1 planes, L1 -> L2 cells and entries."""

    def __init__(self, l1, l2, cfg, mask):
        self.l1, self.l2, self.cfg = l1, l2, cfg
        self.rib = isis.L1L2RibTable(l1, l2, cfg, mask)
        self.t = isis.L1ToL2Table(l1, l2, self.rib)
        self.lid = l1["system_id"] << 8

    def run(self, l1h, jobs):
        """jobs: per job the [std, mt6] L1 overrides of this border's area, or None (its base row)."""
        self.planes = [oracle_planes(self.l1, self.rib.root[0], self.rib.n_vertices[0],
                                     {0: o[0], 1: o[1]} if o is not None else None) for o in jobs]
        n = len(jobs)
        arrs = []
        for k in range(2):
            have = [p[k] for p in self.planes if p[k] is not None]
            arrs.append(None if not have else tuple(np.ascontiguousarray(np.concatenate([h[i] for h in have])) for i in range(3)))
        ptr = lambda i: (C.c_void_p * 2)(*[a[i].ctypes.data if a is not None else None for a in arrs])
        rows = np.arange(n, dtype=np.uint32)
        words = np.zeros((n, max(self.t.n_summaries, 1)), np.uint64)
        cells = np.zeros((n, max(self.t.n_keys, 1)), isis.CELL_DT)
        l1h.harness_isis_l1_to_l2_cells(self.t.handle, n, ptr(0), ptr(1), ptr(2), rows.ctypes.data, words.ctypes.data,
                                        cells.ctypes.data)
        self.cells = np.ascontiguousarray(cells[:, : self.t.n_keys])
        self.words = words[:, : self.t.n_summaries]
        self.entries = [isis.l1_to_l2_from_cells(self.l1, self.t, self.cells[j], self.words[j]) for j in range(n)]


def r_planes(r):
    """R's unperturbed (dist, hops, nh) per topology, None without a root."""
    roots, nv = [], []
    for t, mt in TOPOS:
        f = topology_flat(r, mt) if t == isis.TOPO_STD or r["mt_ipv6"] else None
        roots.append(f.vertex(r["system_id"] << 8) if f is not None else isis.NO_ROOT)
        nv.append(f.csr.n_vertices if f is not None else 0)
    return oracle_planes(r, roots, nv)


def backbone_cells(bbh, bt, borders, planes, n_jobs):
    ptr = lambda i: (C.c_void_p * 2)(*[p[i].ctypes.data if p is not None else None for p in planes])
    bc = (C.c_void_p * len(borders))(*[b.cells.ctypes.data for b in borders])
    cells = np.zeros((n_jobs, max(bt.n_prefixes, 1)), isis.CELL_DT)
    bbh.harness_isis_backbone_cells(bt.handle, n_jobs, ptr(0), ptr(1), ptr(2), bc, cells.ctypes.data)
    return cells[:, : bt.n_prefixes].copy()


# ---- the reference chain --------------------------------------------------------------------------------------
def rkey(r):
    return (int(r["prefix"]["is_v6"]), bytes(r["prefix"]["bytes"]), int(r["len"]))


def restrict(rib, keep):
    """The routes of `rib` whose prefix `keep` says to keep, with their next hops."""
    sel = [i for i, r in enumerate(rib.routes) if keep(rkey(r))]
    routes, nhs, off = rib.routes[sel].copy(), [], 0
    for k, i in enumerate(sel):
        a, n = int(rib.routes[i]["nh_off"]), int(rib.routes[i]["n_nh"])
        nhs.append(rib.nexthops[a:a + n])
        routes[k]["nh_off"] = off
        off += n
    return isis.IsisRib(routes, np.concatenate(nhs) if nhs else rib.nexthops[:0].copy())


def spliced(r, derived, borders, j):
    base = without(r, derived) if derived is not None else r
    entries = {b.lid: [tuple(x.tolist()) for x in b.entries[j]] for b in borders}
    return dict(base, level=isis._with_ipreach(base["level"], entries))


def check(harness, r, derived, borders, jobs, mixed_ok=False):
    """Every job: decoded cells == the chain over the spliced image, restricted to the affected prefixes; the chain ==
    the oracle; every other prefix of the chain == R's base route.  jobs: per job {border index: overrides}."""
    l1h, bbh = harness
    for k, b in enumerate(borders):
        b.run(l1h, [o.get(k) for o in jobs])
    bt = isis.BackboneTable(r, [b.t for b in borders], derived)
    planes = r_planes(r)
    cells = backbone_cells(bbh, bt, borders, planes, len(jobs))
    affected = {(int(p["is_v6"]), bytes(p["bytes"]), int(n)) for p, n in zip(bt.prefix, bt.len)}
    base_routes = None
    n_mixed = 0
    for j in range(len(jobs)):
        x = spliced(r, derived, borders, j)
        want = level_routes(x)
        same_rib(want, pyoracle.isis_compute_routes(x))
        entries = [b.entries[j] for b in borders]
        c = cells[j]
        mixed = (c["flags"] & isis.CELL_MIXED_SID) != 0
        if mixed.any():
            assert mixed_ok, j
            n_mixed += 1
            assert isis.backbone_from_cells(r, bt, c, [p[:2] if p is not None else None for p in planes],
                                            entries).rc == capi.HSPF_E_UNSUPPORTED
            c = c.copy()
            c["flags"][mixed] = 0
            skip = {k for k, m in zip(sorted(affected), mixed) if m}
        else:
            skip = set()
        got = isis.backbone_from_cells(r, bt, c, [p[:2] if p is not None else None for p in planes], entries)
        same_rib(got, restrict(want, lambda k: k in affected and k not in skip))
        if j == 0:
            base_routes = restrict(want, lambda k: k not in affected)
        elif j % 3 == 1:        # sampled: what the table leaves out is R's base table
            same_rib(restrict(want, lambda k: k not in affected), base_routes)
    return bt, cells, n_mixed


def kinds(cells):
    jw, rw, tw = reference(cells, cells[:1])
    return rw["kind"] if len(rw) else np.zeros(0, np.uint8)


# ---- reference goldens -------------------------------------------------------------------------------------------
def golden(topo, rt):
    return next(s for s in gu.load_isis() if s["topo"] == topo and s["rt"] == rt)


def golden_border(topo, rt):
    l1, l2 = golden_pair(golden(topo, rt))
    return Border(l1, l2, isis.summary_cfg([]), own_derived(l1, l2))


def golden_derived(r, borders):
    """The entries of each border's LSP in R's image that are keys of its table and not in its own L1 LSP."""
    lv = r["level"]
    mask = np.zeros(len(lv.ipreaches), np.uint8)
    ek = lambda e: (int(e["kind"]), int(e["prefix"]["is_v6"]), bytes(e["prefix"]["bytes"]), int(e["len"]))
    for b in borders:
        keys = {(int(k), int(p["is_v6"]), bytes(p["bytes"]), int(n)) for k, p, n in zip(b.t.kind, b.t.prefix, b.t.len)}
        l1v = b.l1["level"]
        own = {ek(e) for i in range(len(l1v.lsps)) if int(l1v.lsps["lan_id"][i]) == b.lid
               for e in l1v.ipreaches[int(l1v.lsps["ipreach_off"][i]): int(l1v.lsps["ipreach_off"][i]) + int(l1v.lsps["n_ipreach"][i])]}
        for i in range(len(lv.lsps)):
            if int(lv.lsps["lan_id"][i]) != b.lid:
                continue
            a = int(lv.lsps["ipreach_off"][i])
            for k in range(a, a + int(lv.lsps["n_ipreach"][i])):
                mask[k] = ek(lv.ipreaches[k]) in keys and ek(lv.ipreaches[k]) not in own
    return mask


def l1_jobs(borders, area):
    """The base job, then every adjacency failure of the L1 area of the borders listed in `area`."""
    b0 = borders[area[0]]
    return [{}] + [{k: failure(borders[k].l1, a, b) for k in area} for a, b in adjacencies(b0.l1)]


# Snapshot pairs that were not converged: R's recorded L2 LSDB (and local-rib) lacks entries the borders' own L1
# snapshots propagate, so the decode has routes the recording does not.
NOT_CONVERGED = {("topo2-4", "rt2"): {"2001:db8:1000::6/128", "fc00:0:0:8::/64"}}


def local_rib_check(snap, bt, got):
    """R's recorded local-rib, restricted to the affected prefixes, equals the decode of the base job: the same
    prefixes, and per prefix the metric and the next-hop addresses."""
    from holo_b200 import ospfv3
    skip = NOT_CONVERGED.get((snap["topo"], snap["rt"]), set())
    affected = {f"{ospfv3.ip_str(p)}/{int(n)}" for p, n in zip(bt.prefix, bt.len)}
    want = {r["prefix"]: (r["metric"], sorted(h[1] for h in r["nexthops"])) for r in snap["local_rib"]
            if r["prefix"] in affected}
    have = {}
    for r in got.routes:
        p = f"{ospfv3.ip_str(r['prefix'])}/{int(r['len'])}"
        have[p] = (int(r["metric"]), sorted(h[1] for h in got.nh(r)))
    assert not (skip & set(want))
    assert {p: x for p, x in have.items() if p not in skip} == want


@pytest.mark.parametrize("topo", ["topo2-2", "topo2-4"])
@pytest.mark.parametrize("rt", ["rt1", "rt2", "rt3"])
def test_goldens_two_borders_of_one_area(harness, topo, rt):
    borders = [golden_border(topo, "rt4"), golden_border(topo, "rt5")]
    snap = golden(topo, rt)
    r = gu.isis_instance_image(snap, snap["levels"][0])
    derived = golden_derived(r, borders)
    assert derived.any()
    bt, cells, _ = check(harness, r, derived, borders, l1_jobs(borders, [0, 1]))
    assert bt.n_prefixes > 0 and (cells[0]["flags"] & isis.CELL_PRESENT).any()
    planes = r_planes(r)
    got = isis.backbone_from_cells(r, bt, cells[0], [p[:2] if p is not None else None for p in planes],
                                   [b.entries[0] for b in borders])
    local_rib_check(snap, bt, got)


def test_golden_borders_of_different_areas(harness):
    """topo1-2: rt3 is a level-2 router behind the L1/L2 routers rt2, rt4 and rt6.  A failure in one area leaves the
    borders of the other areas on their base row."""
    names = ["rt2", "rt4", "rt6"]
    borders = [golden_border("topo1-2", n) for n in names]
    snap = golden("topo1-2", "rt3")
    r = gu.isis_instance_image(snap, snap["levels"][0])
    derived = golden_derived(r, borders)
    areas = {}
    for k, b in enumerate(borders):
        f = topology_flat(b.l1, isis.MT_STANDARD)
        areas.setdefault(tuple(sorted(int(x) for x in f.ids)), []).append(k)
    jobs = [{}]
    for area in areas.values():
        jobs += l1_jobs(borders, area)[1:]
    bt, cells, _ = check(harness, r, derived, borders, jobs)
    planes = r_planes(r)
    got = isis.backbone_from_cells(r, bt, cells[0], [p[:2] if p is not None else None for p in planes],
                                   [b.entries[0] for b in borders])
    local_rib_check(snap, bt, got)


# ---- synthetic domains -----------------------------------------------------------------------------------------
def view_borders(seed, **kw):
    vs = [isis.l1l2_view(seed, root=b, **kw) for b in range(3)]
    return vs[0], [Border(v["l1"], v["l2"], v["cfg"], v["l2_derived"]) for v in vs]


def synth(harness, seed, n_fail=16, backbone=(5, 17), mixed_ok=False, **kw):
    kw = dict(dict(n_l1=40, n_l2=30), **kw)
    v, borders = view_borders(seed, **kw)
    jobs = [{k: o for k in range(3)} if o is not None else {} for o in
            [None] + [j for j in view_jobs(v, n_fail)[1:]]]
    out = []
    for i in backbone:
        out.append(check(harness, isis.l1l2_backbone(v, i), v["derived_all"], borders, jobs, mixed_ok))
    return v, borders, out


@pytest.mark.parametrize("mtype", [isis.METRIC_WIDE, isis.METRIC_STANDARD, isis.METRIC_BOTH])
def test_synthetic_metric_types(harness, mtype):
    v, borders, out = synth(harness, 21, metric_type=mtype, summaries=[("10.2.0.0/16", None), ("10.1.0.3/32", 9)],
                            cost_choices=[5, 10])
    for bt, cells, _ in out:
        assert (cells["flags"] & isis.CELL_PRESENT).any()


def test_synthetic_mt_ipv6(harness):
    v, borders, out = synth(harness, 22, mt6=True, summaries=[("10.2.0.0/16", None), ("2001:db8::/32", None)],
                            cost_choices=[5, 10])
    bt = out[0][0]
    assert bt.prefix["is_v6"].any()


def test_synthetic_summaries_go_inactive_and_partitions(harness):
    """A tree-like area: failures cut routers off from some borders only, and take a summary's prefixes away."""
    v, borders, out = synth(harness, 11, n_fail=80, l1_degree=2, cost_choices=[5],
                            summaries=[("10.2.0.0/16", None), ("10.1.0.5/32", None)])
    active = np.stack([b.words for b in borders])
    assert (active[:, 0] >> np.uint64(32) == 1).any() and (active[:, 1:] >> np.uint64(32) == 0).any()
    def keys(b, j, present):
        on = (b.cells[j]["flags"] & isis.CELL_PRESENT != 0) == present
        return {(int(k), bytes(p["bytes"]), int(n)) for k, p, n, o in zip(b.t.kind, b.t.prefix, b.t.len, on) if o}
    # a job where one border loses a key that another border still propagates
    assert any(keys(a, j, False) & keys(a, 0, True) & keys(b, j, True)
               for j in range(1, len(borders[0].cells)) for a in borders for b in borders if a is not b)
    for bt, cells, _ in out:
        assert kinds(cells).any()


def test_synthetic_equal_cost_borders(harness):
    """Every cost equal: R reaches several borders at one distance, so their keys merge next hops (ECMP), and a failure
    that raises one border's total hands the prefix to the others: NEXTHOPS in the delta."""
    v, borders, out = synth(harness, 31, n_fail=40, cost_choices=[10], backbone=range(3, 30), l1_degree=2, summaries=[])
    assert any((kinds(cells) & DELTA_NEXTHOPS).any() for _bt, cells, _ in out)
    assert any(((cells["nh_mask"] & (cells["nh_mask"] - np.uint64(1))) != 0).any() for _bt, cells, _ in out)


def test_synthetic_sr(harness):
    """SR on: tied borders give HL_CELL_MIXED_SID cells, which the decode refuses; every other cell decodes to the
    chain."""
    v, borders, out = synth(harness, 31, n_fail=12, cost_choices=[10], backbone=range(3, 30), l1_degree=2,
                            summaries=[], sr=True, mixed_ok=True)
    assert sum(n for _bt, _c, n in out) > 0


# ---- refusals ----------------------------------------------------------------------------------------------------
def refused(r, borders, derived):
    with pytest.raises(capi.HspfError) as e:
        isis.BackboneTable(r, borders, derived)
    return e.value.code


def test_refusals(harness):
    v, borders = view_borders(13, n_l1=30, n_l2=30, summaries=[("10.1.0.0/16", None)])
    r, der = isis.l1l2_backbone(v, 5), v["derived_all"]
    ts = [b.t for b in borders]
    isis.BackboneTable(r, ts, der)
    assert refused(dict(r, level_no=1), ts, der) == capi.HSPF_E_INVAL
    assert refused(dict(r, level_type=1), ts, der) == capi.HSPF_E_INVAL
    assert refused(v["l2"], ts, der) == capi.HSPF_E_INVAL                   # R is border 0
    assert refused(r, [ts[0], ts[1], ts[0]], der) == capi.HSPF_E_INVAL      # border 0 twice
    assert refused(r, [], der) == capi.HSPF_E_INVAL
    # a border without a valid zeroth fragment in R's image
    lv = copy.copy(r["level"])
    lv.lsps = lv.lsps.copy()
    z = int(np.nonzero((lv.lsps["lan_id"] == borders[1].lid) & (lv.lsps["fragment"] == 0))[0][0])
    lv.lsps["rem_lifetime"][z] = 0
    assert refused(dict(r, level=lv), ts, der) == capi.HSPF_E_INVAL
    # a derived byte on another router's entry
    lsps = r["level"].lsps
    other = int(np.nonzero(((lsps["lan_id"] >> 8) == isis.sysid(v["t1"].n_routers + 7)) & (lsps["n_ipreach"] > 0))[0][0])
    bad = der.copy()
    bad[int(lsps["ipreach_off"][other])] = 1
    assert refused(r, ts, bad) == capi.HSPF_E_INVAL
    # a derived byte on a border's configured entry (10.200.b/32 is none of its keys)
    own = int(np.nonzero((lsps["lan_id"] == borders[2].lid) & (lsps["fragment"] == 0))[0][0])
    bad = der.copy()
    bad[int(lsps["ipreach_off"][own])] = 1
    assert refused(r, ts, bad) == capi.HSPF_E_INVAL
    # a summary key equal to a configured entry of the border: propagation would overwrite it
    lv = copy.copy(r["level"])
    keys0 = [(int(k), bytes(p["bytes"]), int(n)) for k, p, n in zip(borders[0].t.kind, borders[0].t.prefix, borders[0].t.len)]
    summ = (isis.IP_V4_EXT, bytes(v["cfg"][0]["prefix"]["bytes"]), int(v["cfg"][0]["len"]))
    assert summ in keys0
    e = np.zeros(1, isis.IPREACH_DT)
    e["prefix"], e["len"], e["kind"], e["metric"] = v["cfg"][0]["prefix"], summ[2], summ[0], 3
    x = isis._with_ipreach(lv, {borders[0].lid: [tuple(e[0].tolist())]})
    der2 = np.zeros(len(x.ipreaches), np.uint8)
    # the same entries marked: the new entry sits at the end of border 0's zeroth fragment, after its derived ones
    i0 = int(np.nonzero((x.lsps["lan_id"] == borders[0].lid) & (x.lsps["fragment"] == 0))[0][0])
    end = int(x.lsps["ipreach_off"][i0]) + int(x.lsps["n_ipreach"][i0])
    for i in range(len(x.lsps)):
        a, n = int(x.lsps["ipreach_off"][i]), int(x.lsps["n_ipreach"][i])
        b, m = int(r["level"].lsps["ipreach_off"][i]), int(r["level"].lsps["n_ipreach"][i])
        der2[a:a + m] = der[b:b + m]
    assert der2[end - 1] == 0
    assert refused(dict(r, level=x), ts, der2) == capi.HSPF_E_UNSUPPORTED


def with_entry(r, derived, lid, entry):
    """R's image with `entry` appended to LAN id lid's zeroth fragment, and the derived mask moved along."""
    lv = r["level"]
    mask = []
    for i in range(len(lv.lsps)):
        a, n = int(lv.lsps["ipreach_off"][i]), int(lv.lsps["n_ipreach"][i])
        mask += [int(x) for x in derived[a:a + n]]
        if int(lv.lsps["lan_id"][i]) == lid and int(lv.lsps["fragment"][i]) == 0:
            mask.append(0)
    return dict(r, level=isis._with_ipreach(lv, {lid: [tuple(entry.tolist())]})), np.array(mask, np.uint8)


RT_L2_INTRA = 0               # HL_ISIS_RT_L2_INTRA


def test_equal_metrics_keep_walk_order(harness):
    """A backbone router after border 0 in vertex order advertises one of border 0's keys as external, at the total
    the border's slot reaches in the base job.  compute_routes meets the border first, so the route stays internal:
    a slot placed anywhere but at its border's vertex hands the route to the external entry."""
    v, borders = view_borders(23, n_l1=40, n_l2=30, summaries=[], cost_choices=[5, 10])
    r = isis.l1l2_backbone(v, 9)
    b0 = borders[0]
    b0.run(harness[0], [None])
    f = topology_flat(r, isis.MT_STANDARD)
    d = r_planes(r)[0][0]
    x = next(i for i in range(3, 30) if i != 9 and f.vertex(isis.sysid(40 + i) << 8) > f.vertex(b0.lid))
    dx, db = int(d[f.vertex(isis.sysid(40 + x) << 8)]), int(d[f.vertex(b0.lid)])
    e = next(e for e in b0.entries[0] if int(e["kind"]) == isis.IP_V4_EXT and db + int(e["metric"]) >= dx)
    e = e.copy()
    e["metric"], e["external"], e["has_psid"] = db + int(e["metric"]) - dx, 1, 0
    rx, der = with_entry(r, v["derived_all"], isis.sysid(40 + x) << 8, e)
    jobs = [{}] + [{k: o for k in range(3)} for o in view_jobs(v, 6)[1:]]
    bt, cells, _ = check(harness, rx, der, borders, jobs)
    key = (int(e["prefix"]["is_v6"]), bytes(e["prefix"]["bytes"]), int(e["len"]))
    got = isis.backbone_from_cells(rx, bt, cells[0], [q[:2] if q is not None else None for q in r_planes(rx)],
                                   [b.entries[0] for b in borders])
    route = next(q for q in got.routes if rkey(q) == key)
    # the tie is there: the external entry's total is the route's metric, and the route is internal
    assert int(route["metric"]) == dx + int(e["metric"]) and int(route["route_type"]) == RT_L2_INTRA


def test_sr_key_changes_record_between_jobs(harness):
    """SR on, one propagated key advertised by two L1 routers with different Prefix-SIDs.  In the base job the two
    records tie at border 0 (the first in LSP order wins); a failure that cuts the first one off hands the key to the
    second at the same metric.  At a backbone router that routes the key through border 0 only, the cell keeps its
    metric and next hops but names the other record (the delta reports OTHER), and the decode must take the job's
    Prefix-SID: the base job's entry would give another label."""
    v, _ = view_borders(41, n_l1=40, n_l2=30, summaries=[], cost_choices=[5], l1_degree=2, sr=True)
    l1 = v["l1"]
    f = topology_flat(l1, isis.MT_STANDARD)
    root0 = f.vertex(isis.sysid(0) << 8)
    jobs = view_jobs(v, 200)[1:]

    def dist(ov):
        return pyoracle.csr_spf(f.csr, root0, overrides=ov[0])["dist"]
    base = dist([[], []])
    d_jobs = [dist(o) for o in jobs]
    vert = {r: f.vertex(isis.sysid(r) << 8) for r in range(3, 40)}
    # the pair: equal distance from border 0, and a failure that moves the first one and leaves the second
    pair, job = next(((a, b), j) for a in range(3, 40) for b in range(a + 1, 40)
                     if base[vert[a]] == base[vert[b]]
                     for j, d in enumerate(d_jobs) if d[vert[a]] != base[vert[a]] and d[vert[b]] == base[vert[b]])
    tie = lambda sid: [isis.ipreach_rec(ospfv3.ip_rec("10.3.0.0"), 1, 0, 24, isis.IP_V4_EXT, 0, (0, 0, sid))]
    ent = {isis.sysid(pair[0]) << 8: tie(700), isis.sysid(pair[1]) << 8: tie(800)}
    borders = []
    for b in range(3):
        vb = isis.l1l2_view(41, n_l1=40, n_l2=30, summaries=[], cost_choices=[5], l1_degree=2, sr=True, root=b)
        x1 = dict(vb["l1"], level=isis._with_ipreach(vb["l1"]["level"], ent))
        borders.append(Border(x1, vb["l2"], vb["cfg"], vb["l2_derived"]))
    key = (0, bytes(ospfv3.ip_rec("10.3.0.0")[0]), 24)
    all_jobs = [{}, {k: jobs[job] for k in range(3)}]
    # a backbone router that reaches border 0 strictly closer than the others: the key is border 0's alone
    for i in range(3, 30):
        r = isis.l1l2_backbone(v, i)
        fr, d = topology_flat(r, isis.MT_STANDARD), r_planes(r)[0][0]
        db = [int(d[fr.vertex(isis.sysid(b) << 8)]) for b in range(3)]
        if db[0] + 10 < min(db[1:]):
            break
    bt, cells, _ = check(harness, r, v["derived_all"], borders, all_jobs, mixed_ok=True)   # other keys may tie
    p = next(k for k, (q, n) in enumerate(zip(bt.prefix, bt.len)) if (0, bytes(q["bytes"]), int(n)) == key)
    assert not (cells[:, p]["flags"] & isis.CELL_MIXED_SID).any()
    b0 = borders[0]
    k0 = next(k for k in range(b0.t.n_keys) if int(b0.t.len[k]) == 24 and bytes(b0.t.prefix[k]["bytes"]) == key[1])
    assert b0.t.n_records > b0.t.n_keys - 1                 # the key has two records
    w0, w1 = b0.cells[0][k0], b0.cells[1][k0]
    assert int(w0["metric"]) == int(w1["metric"]) and int(w0["winner"]) + 1 == int(w1["winner"])
    c0, c1 = cells[0][p], cells[1][p]
    assert int(c0["metric"]) == int(c1["metric"]) and int(c0["nh_mask"]) == int(c1["nh_mask"])
    assert int(c1["winner"]) == int(c0["winner"]) + 1
    jw, rw, tw = reference(cells, cells[:1])
    assert any(int(x["job"]) == 1 and int(x["prefix"]) == p and int(x["kind"]) == DELTA_OTHER for x in rw)
    planes = [q[:2] if q is not None else None for q in r_planes(r)]
    lab = lambda rib: int(next(q for q in rib.routes if rkey(q) == key)["sr_label"])
    c = cells[1].copy()
    c["flags"] &= ~np.uint8(isis.CELL_MIXED_SID)            # the other keys' tied cells, decoded by check() apart
    got = isis.backbone_from_cells(r, bt, c, planes, [b.entries[1] for b in borders])
    stale = isis.backbone_from_cells(r, bt, c, planes, [b.entries[0] for b in borders])
    assert got.rc == capi.HSPF_OK and stale.rc == capi.HSPF_OK
    assert lab(got) != lab(stale)                            # the job's entry decides the label
