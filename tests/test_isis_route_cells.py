"""CPU: the batched IS-IS route stage (holo-isis/src/spf.rs:838-941, compute_routes, for every job of a batch).

The device kernel's body (isis_route_cell_eval, holo_b200/csrc/isis_route_cells.h) is compiled into a test
harness and run on the CPU over the oracle's SPT planes; the cells, decoded by the product's host function
hspf_isis_routes_from_cells, must give byte for byte the table hspf_isis_routes_from_planes gives for the
same planes (routes, next hops, SR labels), or — for what-if overrides — the oracle's table on an LSDB that
carries the change.  tests/test_isis_route_cells_gpu.py makes the same comparisons with cells computed on
the device."""
import copy
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import golden_util as gu
from holo_b200 import capi, isis, ospfv3, synth
from isis_synth import synth_instance
from oracle import pyoracle

ROOT = Path(__file__).resolve().parent.parent
TOPOS = ((isis.TOPO_STD, isis.MT_STANDARD), (isis.TOPO_MT6, isis.MT_IPV6))


@pytest.fixture(scope="module")
def harness(built):
    out = ROOT / "tests" / "_build" / "libisis_route_cells_harness.so"
    src = ROOT / "tests" / "native" / "isis_route_cells_harness.cc"
    hdrs = [ROOT / "holo_b200" / "csrc" / n for n in ("isis_route_cells.h", "route_cells.h")]
    if not out.exists() or out.stat().st_mtime < max(p.stat().st_mtime for p in [src, *hdrs]):
        out.parent.mkdir(parents=True, exist_ok=True)
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                        "-o", str(out), str(src)], check=True)
    lib = C.CDLL(str(out))
    lib.harness_isis_route_cells.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 7
    return lib


def topology_flat(inst, mt):
    lv = copy.copy(inst["level"])
    lv.mt_id, lv.metric_mode = mt, isis.MODE_NORMAL
    return isis.Flat(lv)


def oracle_planes(inst, rt, ov=None):
    """Per topology with a root: the oracle's planes (nh_words 1) of the local system, with that
    topology's overrides."""
    out = {}
    for t, mt in TOPOS:
        if rt.root[t] == isis.NO_ROOT:
            continue
        f = topology_flat(inst, mt)
        assert f.csr.n_vertices == rt.n_vertices[t] and f.vertex(inst["system_id"] << 8) == rt.root[t]
        c = pyoracle.csr_spf(f.csr, rt.root[t], overrides=(ov or {}).get(t, ()), nh_words=1)
        assert c["status"] == 0
        out[t] = (np.ascontiguousarray(c["dist"], np.uint32), np.ascontiguousarray(c["hops"], np.uint16),
                  np.ascontiguousarray(c["nh_mask"], np.uint64).reshape(-1))
    return out


def cells_on_cpu(harness, rt, planes):
    cells = np.zeros(rt.n_prefixes, isis.CELL_DT)
    ptrs = []
    for t in (isis.TOPO_STD, isis.TOPO_MT6):
        ptrs += [a.ctypes.data for a in planes[t]] if t in planes else [None] * 3
    harness.harness_isis_route_cells(rt.handle, 1, *ptrs, cells.ctypes.data)
    return cells


def decode(inst, rt, cells, planes, ov=None):
    dh = lambda t: planes[t][:2] if t in planes else None
    ov = ov or {}
    return isis.routes_from_cells(inst, rt, cells, dh(isis.TOPO_STD), dh(isis.TOPO_MT6),
                                  ov.get(isis.TOPO_STD, ()), ov.get(isis.TOPO_MT6, ()))


def from_planes(inst):
    return isis.routes_from_planes(inst, lambda csr, root: (lambda c: (c["dist"], c["hops"]))(
        pyoracle.csr_spf(csr, root, nh_words=1)))


def same_rib(a, b):
    assert a.rc == capi.HSPF_OK, a.rc
    assert len(a.routes) == len(b.routes) and len(a.nexthops) == len(b.nexthops)
    assert a.routes.tobytes() == b.routes.tobytes()
    assert a.nexthops.tobytes() == b.nexthops.tobytes()


def check(harness, inst):
    """cells over the oracle's planes, decoded == hspf_isis_routes_from_planes over the same planes."""
    rt = isis.RouteTable(inst)
    planes = oracle_planes(inst, rt)
    cells = cells_on_cpu(harness, rt, planes)
    got = decode(inst, rt, cells, planes)
    if got.rc == capi.HSPF_OK:
        same_rib(got, from_planes(inst))
    return rt, cells, got


SNAPS = gu.load_isis()
LEVELS = [(s, i) for s in SNAPS for i in range(len(s["levels"]))]


@pytest.mark.parametrize("snap,li", LEVELS, ids=[f"{s['topo']}-{s['rt']}-{s['levels'][i]['level']}" for s, i in LEVELS])
def test_cells_decode_exactly_on_reference_goldens(harness, snap, li):
    inst = gu.isis_instance_image(snap, snap["levels"][li])
    rt, cells, got = check(harness, inst)
    assert got.rc == capi.HSPF_OK
    assert int((cells["flags"] & isis.CELL_PRESENT != 0).sum()) == len(got.routes)


AFTER = [(s, n) for s in SNAPS for n in s.get("after", {})]


@pytest.mark.parametrize("snap,name", AFTER, ids=[f"{n}-{s['topo']}-{s['rt']}" for s, n in AFTER])
def test_cells_decode_exactly_on_step_after_states(harness, snap, name):
    """Overload and ATT bits, expired LSPs, removed adjacencies, af / interface changes."""
    after = snap["after"][name]
    for level in after["levels"]:
        inst = gu.isis_instance_image(after, level)
        inst["att_ignore"] = int(bool(after.get("att_ignore", False)))
        assert check(harness, inst)[2].rc == capi.HSPF_OK


@pytest.mark.parametrize("seed,kw,mtype,frag,sr", [
    (3, dict(cost_lo=1, cost_hi=30, lan_fraction=0.15), isis.METRIC_WIDE, 3, False),
    (4, dict(cost_choices=[10], lan_fraction=0.2), isis.METRIC_WIDE, 0, True),         # ECMP: merged next hops
    (5, dict(cost_lo=1, cost_hi=20), isis.METRIC_BOTH, 2, True),
    (6, dict(cost_choices=[5, 10]), isis.METRIC_WIDE, 2, True),
    (7, dict(cost_lo=1, cost_hi=9, lan_fraction=0.3), isis.METRIC_BOTH, 1, False),
])
@pytest.mark.parametrize("max_paths", [1, 2, 4])
def test_cells_decode_exactly_on_synthetic_instances(harness, seed, kw, mtype, frag, sr, max_paths):
    t = synth.random_topology(150, 600, synth.SEED_BASE + seed, **kw)
    n_multi = n_labels = 0
    for root in range(0, 150, 13):
        inst = synth_instance(t, root, mtype, frag, sr=sr)
        inst["max_paths"] = max_paths
        rt, cells, got = check(harness, inst)
        assert got.rc == capi.HSPF_OK
        n_multi += int((got.routes["n_nh"] > 1).sum())
        n_labels += int(got.nexthops["has_label"].sum())
        assert int(got.routes["n_nh"].max()) <= max_paths
    if max_paths > 1 and "cost_choices" in kw:
        assert n_multi > 0
    assert (n_labels > 0) == sr


def with_ipreach(inst, lan_id, recs):
    """The instance with `recs` appended to the IP reachability of lan_id's zeroth fragment."""
    lv = copy.copy(inst["level"])
    lsps, old = lv.lsps.copy(), lv.ipreaches
    new = []
    for i in range(len(lsps)):
        a, n = int(lsps["ipreach_off"][i]), int(lsps["n_ipreach"][i])
        ent = list(old[a:a + n])
        if int(lsps["lan_id"][i]) == lan_id and int(lsps["fragment"][i]) == 0:
            ent += [np.array(r, isis.IPREACH_DT) for r in recs]
        lsps["ipreach_off"][i], lsps["n_ipreach"][i] = len(new), len(ent)
        new += ent
    lv.lsps = lsps
    lv.ipreaches = np.array(new, isis.IPREACH_DT) if new else np.zeros(0, isis.IPREACH_DT)
    return dict(inst, level=lv)


def v4(s):
    return ospfv3.ip_rec(s)


def mt6_instance(t, root, frag=0, sr=False):
    """Standard and MT-IPv6 topologies: TLV 222 adjacencies whose metrics differ from the standard ones away from
    the root; per router an MT-IPv6 /128 (TLV 237) and a TLV 236 /128 the instance must ignore; adjacencies with
    IPv6 addresses."""
    inst = synth_instance(t, root, isis.METRIC_WIDE, frag, sr=sr)
    mt = isis.synth_level(t, isis.METRIC_WIDE, mt_id=isis.MT_IPV6, max_reach_per_fragment=frag)
    lv = copy.copy(inst["level"])
    lsps = lv.lsps.copy()
    assert np.array_equal(lsps["lan_id"], mt.lsps["lan_id"]) and np.array_equal(lsps["fragment"], mt.lsps["fragment"])
    lsps["reach_off"], lsps["n_reach"] = mt.lsps["reach_off"], mt.lsps["n_reach"]
    lsps["flags"] |= np.where(lsps["fragment"] == 0, isis.LSPF_NLPID_IPV6, 0).astype(np.uint8)
    reaches = mt.reaches.copy()
    me = isis.sysid(root) << 8
    for i in range(len(lsps)):
        a, n = int(lsps["reach_off"][i]), int(lsps["n_reach"][i])
        for k in range(a, a + n):
            if reaches["kind"][k] == isis.REACH_MT and int(lsps["lan_id"][i]) != me and int(reaches["neighbor"][k]) != me:
                reaches["metric"][k] = (int(reaches["metric"][k]) * 7) % 23 + 1
    lv.lsps, lv.reaches, lv.ipv6_enabled = lsps, reaches, True
    inst = dict(inst, level=lv, mt_ipv6=1)
    adjs = inst["adjs"].copy()
    adjs["topo_ipv6"], adjs["has_ipv6"] = 1, 1
    for k in range(len(adjs)):
        adjs["ipv6"][k] = ospfv3.ip_rec(f"fe80::{k + 1:x}")
    inst["adjs"] = adjs
    for r in range(t.n_routers):
        psid = (isis.PSID_P, 0, 600 + r) if sr and r % 2 else None
        inst = with_ipreach(inst, isis.sysid(r) << 8, [
            isis.ipreach_rec(ospfv3.ip_rec(f"2001:db8::{r + 1:x}"), 2, isis.MT_IPV6, 128, isis.IP_MT_V6, 0, psid),
            isis.ipreach_rec(ospfv3.ip_rec(f"2001:db9::{r + 1:x}"), 2, 0, 128, isis.IP_V6)])
    return inst


@pytest.mark.parametrize("sr", [False, True])
def test_mt_ipv6_prefixes_read_the_mt_planes(harness, sr):
    t = synth.random_topology(120, 500, synth.SEED_BASE + 31, cost_lo=1, cost_hi=20, lan_fraction=0.1)
    n_v6 = 0
    for root in (0, 17, 64):
        inst = mt6_instance(t, root, frag=2, sr=sr)
        rt, cells, got = check(harness, inst)
        assert got.rc == capi.HSPF_OK
        assert rt.root[isis.TOPO_MT6] != isis.NO_ROOT
        v6 = rt.prefix["is_v6"][np.searchsorted(rt.off, np.arange(rt.n_contributors), side="right") - 1] == 1
        assert np.array_equal(rt.contribs["topology"] == isis.TOPO_MT6, v6)
        # TLV 236 entries are ignored with MT-IPv6 enabled
        assert not any(ospfv3.ip_str(p).startswith("2001:db9:") for p in rt.prefix)
        n_v6 += int((got.routes["prefix"]["is_v6"] == 1).sum())
        # the distances differ between the topologies, and the metrics say which planes were read
        assert n_v6 and len(got.routes) > len(got.routes[got.routes["prefix"]["is_v6"] == 1])


def adjacency_edges(f, a, b):
    row, col = f.csr.row_ptr, f.csr.col
    va, vb = f.vertex(isis.sysid(a) << 8), f.vertex(isis.sysid(b) << 8)
    ab = [e for e in range(row[va], row[va + 1]) if col[e] == vb]
    ba = [e for e in range(row[vb], row[vb + 1]) if col[e] == va]
    return ab, ba


def set_reach_metric(inst, owner, nbr, metric):
    """The LSDB with owner's IS reachability to nbr set to `metric` (None: the entry names a system that owns no
    LSP, so the adjacency is gone)."""
    lv = copy.copy(inst["level"])
    lsps, reaches = lv.lsps, lv.reaches.copy()
    n_hit = 0
    for i in np.nonzero(lsps["lan_id"] == (isis.sysid(owner) << 8))[0]:
        a, n = int(lsps["reach_off"][i]), int(lsps["n_reach"][i])
        for k in range(a, a + n):
            if int(reaches["neighbor"][k]) == isis.sysid(nbr) << 8:
                n_hit += 1
                if metric is None:
                    reaches["neighbor"][k] = 0xFFFFFF0000
                else:
                    reaches["metric"][k] = metric
    assert n_hit == 1
    lv.reaches = reaches
    return dict(inst, level=lv)


def whatif(harness, inst, ov, want_inst):
    rt = isis.RouteTable(inst)
    planes = oracle_planes(inst, rt, {isis.TOPO_STD: ov})
    cells = cells_on_cpu(harness, rt, planes)
    got = decode(inst, rt, cells, planes, {isis.TOPO_STD: ov})
    same_rib(got, pyoracle.isis_compute_routes(want_inst))
    return got


def single_p2p(t):
    pairs = {}
    for k in range(t.n_p2p):
        key = tuple(sorted((int(t.p2p_a[k]), int(t.p2p_b[k]))))
        pairs[key] = pairs.get(key, 0) + 1
    return [(k, int(t.p2p_a[k]), int(t.p2p_b[k])) for k in range(t.n_p2p)
            if pairs[tuple(sorted((int(t.p2p_a[k]), int(t.p2p_b[k]))))] == 1]


@pytest.mark.parametrize("sr", [False, True])
def test_whatif_adjacency_away_from_the_root_disabled(harness, sr):
    t = synth.random_topology(150, 600, synth.SEED_BASE + 33, cost_choices=[5, 10], lan_fraction=0.1)
    root = 3
    inst = synth_instance(t, root, sr=sr)
    f = topology_flat(inst, isis.MT_STANDARD)
    base = from_planes(inst)
    n_changed = 0
    for k, a, b in single_p2p(t)[:40:4]:
        if root in (a, b):
            continue
        ab, ba = adjacency_edges(f, a, b)
        ov = [(ab[0], capi.COST_DISABLED), (ba[0], capi.COST_DISABLED)]
        got = whatif(harness, inst, ov, set_reach_metric(set_reach_metric(inst, a, b, None), b, a, None))
        n_changed += got.routes.tobytes() != base.routes.tobytes()
    assert n_changed > 0


def test_whatif_raised_cost_on_a_root_link(harness):
    """The root's interface metric goes up: its own LSP and the interface configuration carry the new metric.
    The decode gets the new interface metric and the edge override; the oracle the changed LSDB."""
    t = synth.random_topology(150, 600, synth.SEED_BASE + 35, cost_lo=1, cost_hi=12)
    n_changed = 0
    for root in (0, 9, 40):
        inst = synth_instance(t, root, sr=True)
        f = topology_flat(inst, isis.MT_STANDARD)
        base = from_planes(inst)
        for k, a, b in single_p2p(t):
            if root not in (a, b):
                continue
            nbr = b if a == root else a
            ab, _ = adjacency_edges(f, root, nbr)
            new_cost = int(f.csr.cost[ab[0]]) + 9
            ifaces = inst["ifaces"].copy()
            i = next(i for i in range(len(ifaces)) if not ifaces["is_broadcast"][i]
                     and int(inst["adjs"]["system_id"][ifaces["adj_off"][i]]) == isis.sysid(nbr))
            ifaces["metric"][i] = new_cost
            local = dict(inst, ifaces=ifaces)
            got = whatif(harness, local, [(ab[0], new_cost)], set_reach_metric(local, root, nbr, new_cost))
            n_changed += got.routes.tobytes() != base.routes.tobytes() or got.nexthops.tobytes() != base.nexthops.tobytes()
    assert n_changed > 0


def equal_distance_pair(inst):
    f = topology_flat(inst, isis.MT_STANDARD)
    root = f.vertex(inst["system_id"] << 8)
    d = pyoracle.csr_spf(f.csr, root, nh_words=1)["dist"]
    by_d = {}
    for v in range(f.csr.n_vertices):
        lid = int(f.ids[v])
        if lid & 0xFF == 0 and v != root and d[v] != 0xFFFFFFFF:
            by_d.setdefault(int(d[v]), []).append((lid >> 8) - isis.SYSID_BASE)
    return next(rs for _, rs in sorted(by_d.items()) if len(rs) >= 2)[:2]


def test_equal_metric_prefix_sids_from_two_routers_are_flagged(harness):
    """Two routers at equal distance advertise one prefix with Prefix-SIDs under SR: the labels depend on the
    order of the updates, the cell is flagged and the decode refuses.  The same prefix twice from one router
    (TLV 128 and TLV 135 under METRIC_BOTH) is an ordinary merge: no flag, exact routes."""
    t = synth.random_topology(60, 240, synth.SEED_BASE + 37, cost_choices=[10])
    inst = synth_instance(t, 0, isis.METRIC_BOTH, sr=True)
    a, b = equal_distance_pair(inst)
    pfx = v4("198.51.100.0")
    two = inst
    for r, sid in ((a, 70), (b, 71)):
        two = with_ipreach(two, isis.sysid(r) << 8, [isis.ipreach_rec(pfx, 5, 0, 24, isis.IP_V4_EXT, 0, (isis.PSID_P, 0, sid))])
    rt, cells, got = check(harness, two)
    p = next(i for i in range(rt.n_prefixes) if ospfv3.ip_str(rt.prefix[i]) == "198.51.100.0" and rt.len[i] == 24)
    assert cells["flags"][p] & isis.CELL_MIXED_SID and cells["flags"][p] & isis.CELL_PRESENT
    assert got.rc == capi.HSPF_E_UNSUPPORTED
    # without SR nothing depends on the order: exact
    assert check(harness, dict(two, sr_enabled=0))[2].rc == capi.HSPF_OK
    one = with_ipreach(inst, isis.sysid(a) << 8, [isis.ipreach_rec(pfx, 5, 0, 24, isis.IP_V4_INTERNAL),
                                                  isis.ipreach_rec(pfx, 5, 0, 24, isis.IP_V4_EXT, 0, (isis.PSID_P, 0, 70))])
    rt, cells, got = check(harness, one)
    p = next(i for i in range(rt.n_prefixes) if ospfv3.ip_str(rt.prefix[i]) == "198.51.100.0" and rt.len[i] == 24)
    assert rt.off[p + 1] - rt.off[p] == 2
    assert not cells["flags"][p] & isis.CELL_MIXED_SID and got.rc == capi.HSPF_OK
    # two entries with Prefix-SIDs from one router: the labels are that router's, exact
    one = with_ipreach(inst, isis.sysid(a) << 8, [isis.ipreach_rec(pfx, 5, 0, 24, isis.IP_V4_EXT, 0, (isis.PSID_P, 0, 70)),
                                                  isis.ipreach_rec(pfx, 5, 0, 24, isis.IP_V4_EXT, 0, (isis.PSID_P, 0, 71))])
    assert check(harness, one)[2].rc == capi.HSPF_OK


FUZZ_STATS = {}


def collide(inst, t, rng):
    """A small pool of prefixes advertised by many routers with few distinct metrics (ties are common), as
    TLV 135 entries with equal, different or no Prefix-SIDs, and under METRIC_BOTH also as TLV 128 entries."""
    pool = [(f"198.51.{100 + i}.0", 24) for i in range(4)]
    both = inst["level"].metric_type == isis.METRIC_BOTH
    for r in rng.choice(t.n_routers, min(t.n_routers, 14), replace=False):
        recs = []
        for _ in range(int(rng.integers(1, 3))):
            p, ln = pool[int(rng.integers(0, len(pool)))]
            m = int(rng.choice([0, 5, 5, 10]))
            if both and rng.random() < 0.3:
                recs.append(isis.ipreach_rec(v4(p), m, 0, ln, isis.IP_V4_INTERNAL))
            else:
                psid = None if rng.random() < 0.4 else (int(rng.choice([isis.PSID_P, 0, isis.PSID_P | isis.PSID_E])), 0,
                                                        int(rng.choice([900, 900, 901])))
                recs.append(isis.ipreach_rec(v4(p), m, 0, ln, isis.IP_V4_EXT, 0, psid))
        inst = with_ipreach(inst, isis.sysid(int(r)) << 8, recs)
    return inst


@pytest.mark.parametrize("seed", range(12))
def test_colliding_prefixes_fuzz(harness, seed):
    """Every way contributions can meet on one prefix (one or several vertices, equal and unequal metrics,
    equal, different or no Prefix-SIDs, TLV 128 beside TLV 135): the decoded cells equal the planes' table, or
    the decode refuses the job with the flag set — never a wrong route."""
    rng = np.random.default_rng(700 + seed)
    V = int(rng.integers(30, 90))
    t = synth.random_topology(V, int(V * rng.uniform(2.5, 5)), synth.SEED_BASE + 90 + seed,
                              cost_choices=[int(x) for x in rng.choice([5, 10, 10, 20], 2)],
                              lan_fraction=float(rng.uniform(0.1, 0.35)))
    sr = bool(rng.random() < 0.75)
    mtype = int(rng.choice([isis.METRIC_WIDE, isis.METRIC_BOTH]))
    frag = int(rng.choice([0, 2]))
    mp = int(rng.choice([1, 2, 4]))
    mut_seed = int(rng.integers(0, 1 << 30))
    n_ok = n_refused = 0
    for root in rng.choice(V, 8, replace=False):
        inst = synth_instance(t, int(root), mtype, frag, sr=sr)
        inst["max_paths"] = mp
        inst = collide(inst, t, np.random.default_rng(mut_seed))
        rt, cells, got = check(harness, inst)
        assert int((np.diff(rt.off.astype(np.int64)) > 2).sum()) > 0
        if got.rc == capi.HSPF_E_UNSUPPORTED:
            assert sr and (cells["flags"] & isis.CELL_MIXED_SID).any()
            n_refused += 1
            continue
        assert got.rc == capi.HSPF_OK
        n_ok += 1
    FUZZ_STATS[seed] = (n_ok, n_refused)


def test_colliding_prefixes_fuzz_covers_both_outcomes():
    if len(FUZZ_STATS) < 12:
        pytest.skip("runs after the whole fuzz")
    ok = sum(a for a, _ in FUZZ_STATS.values())
    refused = sum(b for _, b in FUZZ_STATS.values())
    assert refused > 0 and ok > refused


def test_table_shape_and_order():
    t = synth.random_topology(120, 500, synth.SEED_BASE + 39, lan_fraction=0.1)
    for inst in (synth_instance(t, 3, isis.METRIC_BOTH, 2, sr=True), mt6_instance(t, 3, sr=True)):
        inst = with_ipreach(inst, isis.sysid(5) << 8, [isis.ipreach_rec(v4("10.0.0.3"), 1, 0, 32, isis.IP_V4_EXT)])
        rt = isis.RouteTable(inst)
        key = [(int(p["is_v6"]), bytes(p["bytes"]), int(n)) for p, n in zip(rt.prefix, rt.len)]
        assert key == sorted(key) and len(set(key)) == len(key)                  # NetKey order, unique
        assert rt.off[0] == 0 and rt.off[-1] == rt.n_contributors and np.all(np.diff(rt.off.astype(np.int64)) >= 1)
        owner = np.searchsorted(rt.off, np.arange(rt.n_contributors), side="right") - 1
        v6 = rt.prefix["is_v6"][owner] == 1
        want = np.where(v6 & bool(inst["mt_ipv6"]), isis.TOPO_MT6, isis.TOPO_STD)
        assert np.array_equal(rt.contribs["topology"], want)                    # one topology per prefix
        n_tlv236 = t.n_routers if inst["mt_ipv6"] else 0                       # ignored with MT-IPv6 enabled
        assert rt.n_contributors == int(inst["level"].lsps["n_ipreach"].sum()) - n_tlv236
        p = next(i for i in range(rt.n_prefixes) if ospfv3.ip_str(rt.prefix[i]) == "10.0.0.3")
        assert rt.off[p + 1] - rt.off[p] == 2 and rt.contribs["metric"][rt.off[p] + 1] == 1
        sr_rel = rt.contribs["sr"] == 1
        assert np.array_equal(sr_rel, rt.contribs["has_psid"] == 1) and sr_rel.any()
