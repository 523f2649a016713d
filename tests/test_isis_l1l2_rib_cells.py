"""CPU: the routing table of an IS-IS L1/L2 router for every job of a batch (update_rib, holo-isis route.rs:182-249).

The device kernels' bodies (isis_summary_eval and isis_l1l2_cell_eval, holo_b200/csrc/isis_l1l2_rib_cells.h) are
compiled into a test harness and run on the CPU over the oracle's SPT planes.  The cells, decoded by the product's
hspf_isis_l1l2_rib_from_cells, must give byte for byte the host chain over the same planes:
hspf_isis_rib_merge(hspf_isis_rib_add_summaries(L2 routes, hspf_isis_summaries(L1 routes, cfg)), L1 routes) — and,
for what-if jobs, the chain over LSDBs that carry the change, with the router's own L2 LSP re-originated for the
job (configured entries + hspf_isis_l1_to_l2 over the job's L1 SPT + the job's active summaries)."""
import copy
import ctypes as C
import ipaddress
import subprocess
from pathlib import Path

import numpy as np
import pytest

import golden_util as gu
from holo_b200 import capi, isis, ospfv3
from oracle import pyoracle

ROOT = Path(__file__).resolve().parent.parent
TOPOS = ((isis.TOPO_STD, isis.MT_STANDARD), (isis.TOPO_MT6, isis.MT_IPV6))


@pytest.fixture(scope="module")
def harness(built):
    out = ROOT / "tests" / "_build" / "libisis_l1l2_rib_cells_harness.so"
    src = ROOT / "tests" / "native" / "isis_l1l2_rib_cells_harness.cc"
    hdrs = [ROOT / "holo_b200" / "csrc" / n for n in ("isis_l1l2_rib_cells.h", "isis_route_cells.h", "route_cells.h")]
    if not out.exists() or out.stat().st_mtime < max(p.stat().st_mtime for p in [src, *hdrs]):
        out.parent.mkdir(parents=True, exist_ok=True)
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                        "-o", str(out), str(src)], check=True)
    lib = C.CDLL(str(out))
    lib.harness_isis_l1l2_rib_cells.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 6
    return lib


def topology_flat(inst, mt):
    lv = copy.copy(inst["level"])
    lv.mt_id, lv.metric_mode = mt, isis.MODE_NORMAL
    return isis.Flat(lv)


def oracle_planes(inst, roots, nv, ov=None):
    """[std, mt6] of one level: the oracle's (dist, hops, nh) of the local system, None without a root."""
    out = [None, None]
    for t, mt in TOPOS:
        if roots[t] == isis.NO_ROOT:
            continue
        f = topology_flat(inst, mt)
        assert f.csr.n_vertices == nv[t] and f.vertex(inst["system_id"] << 8) == roots[t]
        c = pyoracle.csr_spf(f.csr, roots[t], overrides=(ov or {}).get(t, ()), nh_words=1)
        assert c["status"] == 0
        out[t] = (np.ascontiguousarray(c["dist"], np.uint32), np.ascontiguousarray(c["hops"], np.uint16),
                  np.ascontiguousarray(c["nh_mask"], np.uint64).reshape(-1))
    return out


def job_planes(l1, l2, t, ov1=None, ov2=None):
    return oracle_planes(l1, t.root[0], t.n_vertices[0], ov1) + oracle_planes(l2, t.root[1], t.n_vertices[1], ov2)


def cells_on_cpu(harness, t, jobs):
    """jobs: one list of four plane triples per job (each job gets its own rows)."""
    n = len(jobs)
    arrs = []
    for k in range(4):
        have = [j[k] for j in jobs if j[k] is not None]
        arrs.append(None if not have else tuple(np.ascontiguousarray(np.concatenate([h[i] for h in have])) for i in range(3)))
    ptr = lambda i: (C.c_void_p * 4)(*[a[i].ctypes.data if a is not None else None for a in arrs])
    rows = np.repeat(np.arange(n, dtype=np.uint32), 2)
    words = np.zeros((n, max(t.n_summaries, 1)), np.uint64)
    cells = np.zeros((n, t.n_prefixes), isis.CELL_DT)
    harness.harness_isis_l1l2_rib_cells(t.handle, n, ptr(0), ptr(1), ptr(2), rows.ctypes.data, words.ctypes.data,
                                        cells.ctypes.data)
    return cells, words[:, : t.n_summaries]


def decode(l1, l2, t, cells, words, planes, ovs=None):
    return isis.l1l2_rib_from_cells(l1, l2, t, cells, words, [p[:2] if p is not None else None for p in planes], ovs)


def level_routes(inst, ov=None):
    def spf(csr, root):
        c = pyoracle.csr_spf(csr, root, overrides=ov or (), nh_words=1)
        return c["dist"], c["hops"]
    return isis.routes_from_planes(inst, spf)


def chain(l1_rib, l2_rib, cfg):
    act = isis.summaries(l1_rib, cfg)
    return isis.rib_merge(isis.rib_add_summaries(l2_rib, act), l1_rib), act


def same_rib(a, b):
    assert a.rc == capi.HSPF_OK, a.rc
    assert a.routes.tobytes() == b.routes.tobytes()
    assert a.nexthops.tobytes() == b.nexthops.tobytes()


def without(inst, mask):
    """The instance with the IP reachability entries `mask` marks left out."""
    lv = copy.copy(inst["level"])
    lsps, keep = lv.lsps.copy(), []
    for i in range(len(lsps)):
        a, n = int(lsps["ipreach_off"][i]), int(lsps["n_ipreach"][i])
        mine = [k for k in range(a, a + n) if not mask[k]]
        lsps["ipreach_off"][i], lsps["n_ipreach"][i] = len(keep), len(mine)
        keep += mine
    lv.lsps, lv.ipreaches = lsps, lv.ipreaches[keep]
    return dict(inst, level=lv)


def check(harness, l1, l2, cfg, mask):
    """Base job: decoded harness cells == the host chain over the same planes (L2 without the derived entries), and
    the words == hspf_isis_summaries."""
    t = isis.L1L2RibTable(l1, l2, cfg, mask)
    planes = job_planes(l1, l2, t)
    cells, words = cells_on_cpu(harness, t, [planes])
    got = decode(l1, l2, t, cells[0], words[0], planes)
    l1r = level_routes(l1)
    want, act = chain(l1r, level_routes(without(l2, mask) if mask is not None else l2), cfg)
    same_rib(got, want)
    active = {(bytes(a["prefix"]["bytes"]), int(a["len"])): int(a["metric"]) for a in act}
    for s in range(t.n_summaries):
        k = (bytes(cfg[s]["prefix"]["bytes"]), int(cfg[s]["len"]))
        assert (int(words[0][s]) >> 32 == 1) == (k in active)
        if k in active:
            assert int(words[0][s]) & 0xFFFFFFFF == active[k]
    return t, cells[0], words[0], got


# ---- reference goldens -------------------------------------------------------------------------------------
SNAPS = [s for s in gu.load_isis() if s["level_type"] == "level-all" and len(s["levels"]) == 2]


def golden_pair(snap):
    lv = {l["level"]: l for l in snap["levels"]}
    l1, l2 = gu.isis_instance_image(snap, lv[1]), gu.isis_instance_image(snap, lv[2])
    return l1, l2


def own_derived(l1, l2):
    """The router's own L2 entries that its own L1 LSP does not carry (the propagated set of test_isis_l1l2)."""
    me = l1["system_id"]
    key = lambda r: (int(r["prefix"]["is_v6"]), bytes(r["prefix"]["bytes"]), int(r["len"]))
    def own(inst):
        lv = inst["level"]
        for i in range(len(lv.lsps)):
            if int(lv.lsps["lan_id"][i]) == me << 8:
                a = int(lv.lsps["ipreach_off"][i])
                yield from range(a, a + int(lv.lsps["n_ipreach"][i]))
    mine = {key(l1["level"].ipreaches[k]) for k in own(l1)}
    mask = np.zeros(len(l2["level"].ipreaches), np.uint8)
    for k in own(l2):
        mask[k] = key(l2["level"].ipreaches[k]) not in mine
    return mask


@pytest.mark.parametrize("snap", SNAPS, ids=[f"{s['topo']}-{s['rt']}" for s in SNAPS])
def test_goldens_decode_to_the_host_chain_and_the_reference_routes(harness, snap):
    l1, l2 = golden_pair(snap)
    mask = own_derived(l1, l2)
    none = isis.summary_cfg([])
    t, cells, words, got = check(harness, l1, l2, none, mask)
    assert mask.any()
    # shadowing: the table without the derived entries decodes to the routes of the table with them
    t0, cells0, words0, got0 = check(harness, l1, l2, none, None)
    same_rib(got, got0)
    # and against the routes the reference installed
    acts, _ = isis.rib_diff(None, got)
    inst_routes = {}
    for a in acts:
        r = got.routes[int(a["route"])]
        inst_routes[f"{ospfv3.ip_str(r['prefix'])}/{int(r['len'])}"] = int(r["metric"])
    want = {p: v["metric"] for p, v in snap["ibus_routes"].items()}
    assert inst_routes == want


CHAINS = [(s, n) for s in gu.load_isis() for n in s.get("summary_chains", {})]


@pytest.mark.parametrize("snap,name", CHAINS, ids=[n for _s, n in CHAINS])
def test_summary_step_chains(harness, snap, name):
    n_active = 0
    for st in snap["summary_chains"][name]:
        l1, l2 = golden_pair(st)
        cfg = isis.summary_cfg([(p, m) for p, m in st["summaries"]])
        t, cells, words, got = check(harness, l1, l2, cfg, own_derived(l1, l2))
        n_active += int((words >> 32 == 1).sum())
        rib_want = {r["prefix"]: r["metric"] for r in st["local_rib"]}
        for r in got.routes[(got.routes["flags"] & isis.ROUTE_SUMMARY) != 0]:
            assert rib_want.get(f"{ospfv3.ip_str(r['prefix'])}/{int(r['len'])}") == int(r["metric"])
    assert n_active > 0


# ---- synthetic two-level domains ----------------------------------------------------------------------------
CFGS = {
    "none": [],
    "area": [("10.0.0.0/8", None)],
    "nested": [("10.0.0.0/8", None), ("10.1.0.0/16", 7), ("10.2.0.0/16", None)],
    "equal-l1": [("10.2.3.0/24", 40)],
    "equal-l2": [("10.200.0.5/32", None), ("10.1.0.0/16", None)],
    "cfg-metric": [("10.1.0.0/16", 1000)],
    "ipv6": [("2001:db8::/32", None), ("10.1.0.0/16", None)],
    "default": [("0.0.0.0/0", None)],
}


def view_check(harness, v):
    t, cells, words, got = check(harness, v["l1"], v["l2"], v["cfg"], v["l2_derived"])
    assert got.rc == capi.HSPF_OK
    return t, cells, words, got


@pytest.mark.parametrize("cfg", list(CFGS))
@pytest.mark.parametrize("mtype", [isis.METRIC_WIDE, isis.METRIC_STANDARD, isis.METRIC_BOTH])
def test_synthetic_domains_summary_configurations(harness, cfg, mtype):
    for root in (0, 2):
        v = isis.l1l2_view(3, n_l1=80, n_l2=60, root=root, metric_type=mtype, summaries=CFGS[cfg])
        t, cells, words, got = view_check(harness, v)
        win = cells["winner"][cells["flags"] & isis.CELL_PRESENT != 0]
        assert (win < t.n_l1).any() and ((win >= t.n_l1) & (win < t.n_contributors)).any()
        if cfg in ("area", "nested", "cfg-metric", "default"):
            assert (words >> 32 == 1).any()


@pytest.mark.parametrize("mt6,sr,max_paths,attached", [
    (True, False, 4, True), (True, True, 2, True), (False, True, 1, True), (False, False, 16, False),
    (True, False, 16, False), (False, True, 2, False)])
def test_synthetic_domains_topologies(harness, mt6, sr, max_paths, attached):
    n_default = 0
    for seed, root in ((5, 0), (6, 1), (7, 2)):
        v = isis.l1l2_view(seed, n_l1=90, n_l2=70, root=root, mt6=mt6, sr=sr, max_paths=max_paths, attached=attached,
                           summaries=CFGS["nested"] + ([("2001:db8::/32", None)] if mt6 else []),
                           cost_choices=[5, 10])
        t, cells, words, got = view_check(harness, v)
        assert int(got.routes["n_nh"].max()) <= max_paths
        n_default += int(((got.routes["len"] == 0)).sum())
        if mt6:
            assert t.root[0][isis.TOPO_MT6] != isis.NO_ROOT
    assert (n_default > 0) == (not attached)


# ---- what-if jobs ------------------------------------------------------------------------------------------
def link_edges(f, a, b):
    row, col = f.csr.row_ptr, f.csr.col
    va, vb = f.vertex(a << 8), f.vertex(b << 8)
    return [e for e in range(row[va], row[va + 1]) if col[e] == vb] + [e for e in range(row[vb], row[vb + 1]) if col[e] == va]


def cut(inst, a, b):
    """The LSDB without the adjacency a-b (both directions; p2p links only)."""
    lv = copy.copy(inst["level"])
    reaches = lv.reaches.copy()
    for x, y in ((a, b), (b, a)):
        for i in np.nonzero(lv.lsps["lan_id"] == (x << 8))[0]:
            o, n = int(lv.lsps["reach_off"][i]), int(lv.lsps["n_reach"][i])
            for k in range(o, o + n):
                if int(reaches["neighbor"][k]) == y << 8:
                    reaches["neighbor"][k] = 0xFFFFFF0000
    lv.reaches = reaches
    return dict(inst, level=lv)


def reoriginate(l1x, l2, mask, cfg, metric_type):
    """The L2 instance whose own LSP carries what the router re-originates after the L1 change: its configured
    entries, hspf_isis_l1_to_l2 over the job's L1 SPT, and the job's active summaries."""
    l1_routes = pyoracle.isis_compute_routes(l1x)
    act = isis.summaries(l1_routes, cfg)
    lv = l1x["level"]
    sysid = l1x["system_id"]
    lv.mt_id = isis.MT_STANDARD
    std = pyoracle.isis_compute_spt(lv, sysid)
    v6 = None
    if l1x["mt_ipv6"]:
        lv.mt_id = isis.MT_IPV6
        v6 = pyoracle.isis_compute_spt(lv, sysid)
        lv.mt_id = isis.MT_STANDARD
    prop = isis.l1_to_l2(lv, sysid, std, v6, metric_type, metric_type, cfg, act)
    base = without(l2, mask)
    lv2 = base["level"]
    entries = {sysid << 8: [tuple(x.tolist()) for x in prop]}
    return dict(base, level=isis._with_ipreach(lv2, entries)), l1_routes


def whatif(harness, v, level, a, b, mtype=isis.METRIC_WIDE):
    """Job: link a-b (system ids) of `level` disabled through overrides.  Decoded cells == the chain over the LSDBs
    carrying the change, with the own L2 LSP re-originated."""
    l1, l2, cfg, mask = v["l1"], v["l2"], v["cfg"], v["l2_derived"]
    t = isis.L1L2RibTable(l1, l2, cfg, mask)
    inst = l1 if level == 1 else l2
    ov = [(e, capi.COST_DISABLED) for e in link_edges(topology_flat(inst, isis.MT_STANDARD), a, b)]
    assert len(ov) == 2
    ovd = {isis.TOPO_STD: ov}
    planes = job_planes(l1, l2, t, ovd if level == 1 else None, ovd if level == 2 else None)
    cells, words = cells_on_cpu(harness, t, [planes])
    ovs = [ov, (), (), ()] if level == 1 else [(), (), ov, ()]
    got = decode(l1, l2, t, cells[0], words[0], planes, ovs)
    l1x = cut(l1, a, b) if level == 1 else l1
    l2x = cut(l2, a, b) if level == 2 else l2
    l2r, l1_routes = reoriginate(l1x, l2x, mask, cfg, mtype)
    want, act = chain(l1_routes, pyoracle.isis_compute_routes(l2r), cfg)
    same_rib(got, want)
    return t, cells[0], words[0], got


def p2p_links(t, lo, hi, sys_of):
    seen, out = set(), []
    for k in range(t.n_p2p):
        x, y = int(t.p2p_a[k]), int(t.p2p_b[k])
        key = tuple(sorted((x, y)))
        if key in seen:
            continue
        seen.add(key)
        if lo <= x < hi or lo <= y < hi:
            out.append((sys_of(x), sys_of(y)))
    dup = {k for k in seen if sum(1 for j in range(t.n_p2p) if tuple(sorted((int(t.p2p_a[j]), int(t.p2p_b[j])))) == k) > 1}
    return [(x, y) for x, y in out if tuple(sorted((x - isis.SYSID_BASE, y - isis.SYSID_BASE))) not in dup]


def test_whatif_l1_failures(harness):
    """L1 link failures: summaries go inactive or change metric, prefixes move from L1 routes to L2 routes, the area
    partitions."""
    v = isis.l1l2_view(11, n_l1=40, n_l2=40, summaries=[("10.2.0.0/16", None), ("10.1.0.5/32", None)], cost_choices=[5],
                       l1_degree=2)
    base = check(harness, v["l1"], v["l2"], v["cfg"], v["l2_derived"])
    links = p2p_links(v["t1"], 0, 40, isis.sysid)
    f1 = topology_flat(v["l1"], isis.MT_STANDARD)
    root = f1.vertex(v["l1"]["system_id"] << 8)
    routers = sum(1 for x in f1.ids if int(x) & 0xFF == 0)
    n_moved = n_summary = n_changed = n_partitioned = 0
    for a, b in links:
        t, cells, words, got = whatif(harness, v, 1, a, b)
        n_changed += got.routes.tobytes() != base[3].routes.tobytes()
        n_summary += not np.array_equal(words, base[2])
        l2_won = (cells["winner"] >= t.n_l1) & (base[1]["winner"] < t.n_l1) & (cells["flags"] & isis.CELL_PRESENT != 0)
        n_moved += int(l2_won.sum())
        # the job's L1 SPT leaves part of the area's routers unreached
        d = pyoracle.csr_spf(f1.csr, root, overrides=[(e, capi.COST_DISABLED) for e in link_edges(f1, a, b)])["dist"]
        reached = sum(1 for x, dx in zip(f1.ids, d) if int(x) & 0xFF == 0 and dx != 0xFFFFFFFF)
        n_partitioned += reached < routers
    assert n_changed and n_moved and n_summary and n_partitioned


def test_whatif_l2_failures(harness):
    v = isis.l1l2_view(12, n_l1=40, n_l2=40, summaries=[("10.1.0.0/16", None)], cost_choices=[5, 10])
    sys2 = lambda i: isis.sysid(i) if i < 3 else isis.sysid(40 + i)
    n_changed = 0
    base = check(harness, v["l1"], v["l2"], v["cfg"], v["l2_derived"])[3]
    for a, b in p2p_links(v["t2"], 3, 40, sys2)[:16]:
        got = whatif(harness, v, 2, a, b)[3]
        n_changed += got.routes.tobytes() != base.routes.tobytes()
    assert n_changed


# ---- refusals ----------------------------------------------------------------------------------------------
def refused(l1, l2, cfg=None, mask=None):
    with pytest.raises(capi.HspfError) as e:
        isis.L1L2RibTable(l1, l2, cfg, mask)
    return e.value.code


def test_refusals():
    v = isis.l1l2_view(13, n_l1=30, n_l2=30)
    l1, l2, cfg, mask = v["l1"], v["l2"], v["cfg"], v["l2_derived"]
    assert refused(dict(l1, level_type=2), l2, cfg, mask) == capi.HSPF_E_INVAL
    assert refused(l1, dict(l2, level_type=1), cfg, mask) == capi.HSPF_E_INVAL
    assert refused(l1, dict(l2, system_id=l2["system_id"] + 1), cfg, mask) == capi.HSPF_E_INVAL
    assert refused(l1, dict(l2, max_paths=7), cfg, mask) == capi.HSPF_E_INVAL
    assert refused(l2, l1, cfg, None) == capi.HSPF_E_INVAL
    assert refused(dict(l1, level_no=2), l2, cfg, mask) == capi.HSPF_E_INVAL
    two = isis.summary_cfg([("10.0.0.0/8", None), ("10.1.0.0/16", None)])
    assert refused(l1, l2, two[::-1].copy(), mask) == capi.HSPF_E_INVAL
    assert refused(l1, l2, np.concatenate([two[:1], two[:1]]), mask) == capi.HSPF_E_INVAL
    bad = mask.copy()
    lsps2 = l2["level"].lsps
    other = int(np.nonzero(((lsps2["lan_id"] >> 8) != l2["system_id"]) & (lsps2["n_ipreach"] > 0))[0][0])
    lsp = l2["level"].lsps[other]
    bad[int(lsp["ipreach_off"])] = 1
    assert int(lsp["n_ipreach"]) > 0 and refused(l1, l2, cfg, bad) == capi.HSPF_E_INVAL
    # an entry no LSP lists
    lv = copy.copy(l2["level"])
    lv.ipreaches = np.concatenate([lv.ipreaches, lv.ipreaches[:1]])
    stray = np.concatenate([mask, np.ones(1, np.uint8)])
    assert refused(l1, dict(l2, level=lv), cfg, stray) == capi.HSPF_E_INVAL
    isis.L1L2RibTable(l1, dict(l2, level=lv), cfg, np.concatenate([mask, np.zeros(1, np.uint8)]))
    isis.L1L2RibTable(l1, l2, cfg, mask)


def test_propagation_outside_the_l1_routes_is_refused():
    """Entries propagation would carry into the own L2 LSP but compute_routes would not route: unsupported, unless a
    summary covers them."""
    v = isis.l1l2_view(14, n_l1=30, n_l2=30, summaries=[])
    l1, l2 = v["l1"], v["l2"]
    lv = copy.copy(l1["level"])
    lsps = lv.lsps.copy()
    # a fragment 1 whose system has no valid zeroth LSP: expire router 5's zeroth fragment, give it a fragment 1
    i = int(np.nonzero((lsps["lan_id"] == isis.sysid(5) << 8) & (lsps["fragment"] == 0))[0][0])
    lsps["rem_lifetime"][i] = 0
    one = lsps[i:i + 1].copy()
    one["fragment"], one["rem_lifetime"], one["n_reach"] = 1, 1200, 0
    lv.lsps = np.sort(np.concatenate([lsps, one]), order=["lan_id", "fragment"])
    bad = dict(l1, level=lv)
    assert refused(bad, l2, v["cfg"], v["l2_derived"]) == capi.HSPF_E_UNSUPPORTED
    covered = isis.summary_cfg([("10.0.0.0/8", None), ("2001:db8::/32", None)])
    isis.L1L2RibTable(bad, l2, covered, v["l2_derived"])
    # an extended IPv4 entry above the wide-metric limit
    big = copy.copy(l1["level"])
    big.ipreaches = big.ipreaches.copy()
    k = int(np.nonzero(big.ipreaches["kind"] == isis.IP_V4_EXT)[0][-1])
    big.ipreaches["metric"][k] = 0xFE000001
    assert refused(dict(l1, level=big), l2, v["cfg"], v["l2_derived"]) == capi.HSPF_E_UNSUPPORTED
    # MT-IPv6 entries under an instance with IPv6 disabled
    m = isis.l1l2_view(14, n_l1=30, n_l2=30, mt6=True, summaries=[])
    off = copy.copy(m["l1"]["level"])
    off.ipv6_enabled = False
    assert refused(dict(m["l1"], level=off), m["l2"], m["cfg"], m["l2_derived"]) == capi.HSPF_E_UNSUPPORTED


def test_decode_refusals(harness):
    v = isis.l1l2_view(15, n_l1=30, n_l2=30, summaries=[("10.1.0.0/16", None)])
    l1, l2 = v["l1"], v["l2"]
    t, cells, words, got = check(harness, l1, l2, v["cfg"], v["l2_derived"])
    planes = job_planes(l1, l2, t)
    s = int(np.nonzero(cells["winner"] >= t.n_contributors)[0][0])
    w = words.copy()
    w[:] = 0                                   # a summary cell whose word is inactive
    with pytest.raises(capi.HspfError):
        decode(l1, l2, t, cells, w, planes)
    c = cells.copy()
    p1 = int(np.nonzero(c["winner"] < t.n_l1)[0][0])
    c["winner"][p1] = t.n_l1 + 0 if t.off[1][p1] > t.n_l1 else t.n_contributors - 1   # outside the prefix's range
    with pytest.raises(capi.HspfError):
        decode(l1, l2, t, c, words, planes)
    c = cells.copy()
    c["flags"][s] |= isis.CELL_MIXED_SID
    assert decode(l1, l2, t, c, words, planes).rc == capi.HSPF_E_UNSUPPORTED
    with pytest.raises(capi.HspfError):        # not the instances of the table
        decode(l2, l1, t, cells, words, planes)
