"""CPU: what an IS-IS L1/L2 router propagates into its L2 LSP, for every job of a batch (lsp_propagate_l1_to_l2,
holo-isis lsdb.rs:1149-1357).

The device kernels' bodies (isis_summary_eval and isis_l1_to_l2_cell_eval, holo_b200/csrc/isis_l1_to_l2_cells.h) are
compiled into a test harness and run on the CPU over the oracle's L1 SPT planes.  The cells, decoded by the
product's hspf_isis_l1_to_l2_from_cells, must give byte for byte what hspf_isis_l1_to_l2 and the oracle's
restatement return over the job's L1 SPTs (rebuilt from the same planes under the same overrides) and the job's
active summaries (hspf_isis_summaries over the job's L1 routes)."""
import copy
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from holo_b200 import capi, isis, ospfv3
from holo_b200.route_table import DELTA_LOST, DELTA_METRIC, DELTA_NEXTHOPS, DELTA_OTHER
from oracle import pyoracle
from test_isis_l1l2_rib_cells import SNAPS, TOPOS, golden_pair, oracle_planes, p2p_links, topology_flat
from test_route_delta import reference

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def harness(built):
    out = ROOT / "tests" / "_build" / "libisis_l1_to_l2_cells_harness.so"
    src = ROOT / "tests" / "native" / "isis_l1_to_l2_cells_harness.cc"
    hdrs = [ROOT / "holo_b200" / "csrc" / n
            for n in ("isis_l1_to_l2_cells.h", "isis_l1l2_rib_cells.h", "isis_route_cells.h", "route_cells.h")]
    if not out.exists() or out.stat().st_mtime < max(p.stat().st_mtime for p in [src, *hdrs]):
        out.parent.mkdir(parents=True, exist_ok=True)
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                        "-o", str(out), str(src)], check=True)
    lib = C.CDLL(str(out))
    lib.harness_isis_l1_to_l2_cells.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 6
    return lib


def tables(l1, l2, cfg, up_down=None):
    rib = isis.L1L2RibTable(l1, l2, cfg)
    return rib, isis.L1ToL2Table(l1, l2, rib, up_down)


def cells_on_cpu(harness, t, jobs):
    """jobs: per job its [std, mt6] L1 plane triples (None without a root); row j is job j."""
    n = len(jobs)
    arrs = []
    for k in range(2):
        have = [j[k] for j in jobs if j[k] is not None]
        arrs.append(None if not have else tuple(np.ascontiguousarray(np.concatenate([h[i] for h in have])) for i in range(3)))
    ptr = lambda i: (C.c_void_p * 2)(*[a[i].ctypes.data if a is not None else None for a in arrs])
    rows = np.arange(n, dtype=np.uint32)
    words = np.zeros((n, max(t.n_summaries, 1)), np.uint64)
    cells = np.zeros((n, max(t.n_keys, 1)), isis.CELL_DT)
    harness.harness_isis_l1_to_l2_cells(t.handle, n, ptr(0), ptr(1), ptr(2), rows.ctypes.data, words.ctypes.data,
                                        cells.ctypes.data)
    return cells[:, : t.n_keys].copy(), words[:, : t.n_summaries].copy()


def host(l1, l2, t, planes, ovs, cfg, up_down, oracle=False):
    """hspf_isis_l1_to_l2 (or the oracle's) over the job's L1 SPTs, rebuilt from `planes` under `ovs`, and the job's
    active summaries."""
    spts = []
    for tt, mt in TOPOS:
        if tt == isis.TOPO_MT6 and not l1["mt_ipv6"]:
            spts.append(None)
            continue
        f = topology_flat(l1, mt)
        if planes[tt] is None:                   # no root in the topology: nothing is on its SPT
            spts.append(isis._spt_of(f, np.full(f.csr.n_vertices, 0xFFFFFFFF, np.uint32)))
        else:
            spts.append(f.spt_from_planes(t.rib.root[0][tt], planes[tt][0], planes[tt][1], ovs[tt]))
    it = iter([p for p in planes if p is not None])
    act = isis.summaries(isis.routes_from_planes(l1, lambda csr, root: next(it)[:2]), cfg)
    kw = dict(lib=pyoracle.lib(), name="oracle_isis_l1_to_l2") if oracle else {}
    return isis.l1_to_l2(l1["level"], l1["system_id"], spts[0], spts[1], l1["level"].metric_type,
                         l2["level"].metric_type, cfg, act, up_down=up_down, **kw)


def failure(l1, a, b):
    """[std, mt6] overrides that disable every edge between LAN ids a and b."""
    out = []
    for tt, mt in TOPOS:
        if tt == isis.TOPO_MT6 and not l1["mt_ipv6"]:
            out.append([])
            continue
        f = topology_flat(l1, mt)
        va, vb = f.vertex(a), f.vertex(b)
        if isis.NO_ROOT in (va, vb):
            out.append([])
            continue
        row, col = f.csr.row_ptr, f.csr.col
        out.append([(e, capi.COST_DISABLED) for x, y in ((va, vb), (vb, va)) for e in range(int(row[x]), int(row[x + 1]))
                    if int(col[e]) == y])
    return out


def adjacencies(l1):
    """Each adjacency of the L1 LSDB once, as the LAN ids of its ends in the standard topology."""
    f = topology_flat(l1, isis.MT_STANDARD)
    row, col = f.csr.row_ptr, f.csr.col
    out = set()
    for u in range(f.csr.n_vertices):
        for e in range(int(row[u]), int(row[u + 1])):
            a, b = int(f.ids[u]), int(f.ids[int(col[e])])
            out.add((min(a, b), max(a, b)))
    return sorted(out)


def check(harness, l1, l2, cfg, up_down=None, jobs=None):
    """Jobs: one per override pair ([std, mt6]; None: the base job alone).  Each job's decoded harness cells ==
    hspf_isis_l1_to_l2 == oracle_isis_l1_to_l2, byte for byte."""
    jobs = jobs or [[[], []]]
    rib, t = tables(l1, l2, cfg, up_down)
    planes = [oracle_planes(l1, rib.root[0], rib.n_vertices[0], {0: o[0], 1: o[1]}) for o in jobs]
    cells, words = cells_on_cpu(harness, t, planes)
    for j, o in enumerate(jobs):
        got = isis.l1_to_l2_from_cells(l1, t, cells[j], words[j])
        want = host(l1, l2, t, planes[j], o, cfg, up_down)
        ref = host(l1, l2, t, planes[j], o, cfg, up_down, oracle=True)
        assert got.tobytes() == want.tobytes(), j
        assert want.tobytes() == ref.tobytes(), j
    return t, cells, words, planes


def kinds(cells):
    """The route-delta kinds of every job against job 0, per (job, key)."""
    jw, rw, tw = reference(cells, cells[:1])
    return jw, rw


# ---- reference goldens -------------------------------------------------------------------------------------
NONE = isis.summary_cfg([])


@pytest.mark.parametrize("snap", SNAPS, ids=[f"{s['topo']}-{s['rt']}" for s in SNAPS])
def test_goldens_base_job_and_every_adjacency_failure(harness, snap):
    l1, l2 = golden_pair(snap)
    jobs = [[[], []]] + [failure(l1, a, b) for a, b in adjacencies(l1)]
    t, cells, words, _ = check(harness, l1, l2, NONE, jobs=jobs)
    assert t.n_keys > 0 and (cells[0]["flags"] & isis.CELL_PRESENT).any()
    assert not (cells["nh_mask"]).any()


PAIRS = ((isis.METRIC_WIDE, isis.METRIC_WIDE), (isis.METRIC_BOTH, isis.METRIC_STANDARD),
         (isis.METRIC_BOTH, isis.METRIC_BOTH), (isis.METRIC_STANDARD, isis.METRIC_STANDARD))


@pytest.mark.parametrize("seed", range(12))
def test_perturbed_goldens(harness, seed):
    """Random up/down bits, metrics, Prefix-SID flags, summary configurations and metric-type pairs."""
    rng = np.random.default_rng(seed)
    snap = SNAPS[seed % len(SNAPS)]
    l1, l2 = golden_pair(snap)
    lv = copy.copy(l1["level"])
    lv.ipreaches = lv.ipreaches.copy()
    n = len(lv.ipreaches)
    ud = (rng.random(n) < 0.15).astype(np.uint8)
    lv.ipreaches["metric"] = rng.integers(1, 70, n)
    if seed % 3 == 0:
        lv.ipreaches["has_psid"] = 1
        lv.ipreaches["psid_flags"] = rng.integers(0, 256, n)
    cfg = isis.summary_cfg([("10.0.0.0/8", None), ("10.0.0.0/16", 7), ("2001:db8::/32", 30), ("1.0.0.0/8", None)][: 1 + seed % 4])
    for l1t, l2t in PAIRS:
        a, b = copy.copy(lv), copy.copy(l2["level"])
        a.metric_type, b.metric_type = l1t, l2t
        x1, x2 = dict(l1, level=a), dict(l2, level=b)
        adj = adjacencies(x1)
        jobs = [[[], []]] + [failure(x1, p, q) for p, q in adj[:: max(1, len(adj) // 4)]]
        check(harness, x1, x2, cfg, ud, jobs)


# ---- synthetic two-level domains ----------------------------------------------------------------------------
def view_jobs(v, n_fail=12):
    l1 = v["l1"]
    links = p2p_links(v["t1"], 0, v["t1"].n_routers, isis.sysid)
    return [[[], []]] + [failure(l1, a << 8, b << 8) for a, b in links[:n_fail]]


@pytest.mark.parametrize("mtype", [isis.METRIC_WIDE, isis.METRIC_STANDARD, isis.METRIC_BOTH])
@pytest.mark.parametrize("mt6,v4,v6", [(False, True, False), (True, True, True), (True, False, True), (True, True, False)])
def test_synthetic_domains(harness, mtype, mt6, v4, v6):
    summ = [("10.2.0.0/16", None), ("10.1.0.3/32", 9)] + ([("2001:db8:1::4/128", None), ("2001:db8::/32", None)] if mt6 else [])
    if mt6 and not v6:               # MT-IPv6 entries with IPv6 off: a summary covers them (else the rib table refuses)
        summ = [s for s in summ if ":" not in s[0]] + [("2001:db8::/32", None)]
    v = isis.l1l2_view(31, n_l1=60, n_l2=40, mt6=mt6, metric_type=mtype, summaries=summ, cost_choices=[5, 10], l1_degree=2)
    l1 = v["l1"]
    lv = copy.copy(l1["level"])
    lv.ipv4_enabled, lv.ipv6_enabled = v4, (v6 if mt6 else lv.ipv6_enabled)
    l1 = dict(l1, level=lv)
    t, cells, words, _ = check(harness, l1, v["l2"], v["cfg"], jobs=view_jobs(dict(v, l1=l1)))
    present = cells["flags"] & isis.CELL_PRESENT != 0
    assert present.any()
    if not v4:
        assert not np.isin(t.kind, [isis.IP_V4_INTERNAL, isis.IP_V4_EXT, isis.IP_V4_EXTERNAL]).any()
    if mt6 and v6:
        assert (t.kind == isis.IP_V6).any()


# ---- the cases the stage must get right ---------------------------------------------------------------------
def test_failures_lose_keys_drop_summaries_and_swap_winners(harness):
    """A tree-like area with equal costs: failures cut originators off (LOST), take a summary's only covered
    prefix away (the summary key LOST), change totals (METRIC) and, where two originators tie, hand the key to the
    other one (OTHER); no NEXTHOPS ever."""
    v = isis.l1l2_view(11, n_l1=40, n_l2=40, summaries=[("10.2.0.0/16", None), ("10.1.0.5/32", None)], cost_choices=[5],
                       l1_degree=2)
    l1 = v["l1"]
    # two routers at the same distance from the root advertise 10.3.0.0/24 at one metric: a tie
    rib = isis.L1L2RibTable(l1, v["l2"], v["cfg"])
    d = oracle_planes(l1, rib.root[0], rib.n_vertices[0])[0][0]
    f = topology_flat(l1, isis.MT_STANDARD)
    at = {}
    for r in range(1, 40):
        at.setdefault(int(d[f.vertex(isis.sysid(r) << 8)]), []).append(r)
    pair = next(rs[:2] for _d, rs in sorted(at.items()) if len(rs) > 1)
    tie = [isis.ipreach_rec(ospfv3.ip_rec("10.3.0.0"), 5, 0, 24, isis.IP_V4_EXT)]
    l1 = dict(l1, level=isis._with_ipreach(l1["level"], {isis.sysid(r) << 8: tie for r in pair}))
    t, cells, words, planes = check(harness, l1, v["l2"], v["cfg"], jobs=view_jobs(dict(v, l1=l1), n_fail=60))
    jw, rw = kinds(cells)
    k = rw["kind"]
    assert (k & DELTA_LOST).any() and (k & DELTA_METRIC).any() and (k & DELTA_OTHER).any()
    assert not (k & DELTA_NEXTHOPS).any()
    summary_keys = np.nonzero(cells[0]["winner"] >= t.n_records)[0]
    lost_summary = [r for r in rw if int(r["prefix"]) in summary_keys and int(r["kind"]) & DELTA_LOST]
    assert lost_summary and not (words[[int(r["job"]) for r in lost_summary]] >> np.uint64(32) == 1).all()
    # the tied key: the first originator in LSP order holds it; a failure that cuts it off hands it to the other
    # at the same metric (OTHER)
    key = int(np.nonzero((t.len == 24) & (t.prefix["bytes"][:, 1] == 3))[0][0])
    w0 = int(cells[0]["winner"][key])
    swaps = [r for r in rw if int(r["prefix"]) == key and int(r["kind"]) == DELTA_OTHER]
    assert swaps and all(int(cells[int(r["job"])]["winner"][key]) == w0 + 1 for r in swaps)


def test_narrow_totals_cap_at_63(harness):
    v = isis.l1l2_view(41, n_l1=50, n_l2=30, metric_type=isis.METRIC_STANDARD, summaries=[], cost_choices=[20])
    t, cells, words, planes = check(harness, v["l1"], v["l2"], v["cfg"], jobs=view_jobs(v, n_fail=6))
    narrow = t.kind == isis.IP_V4_INTERNAL
    m = cells[:, narrow]["metric"][cells[:, narrow]["flags"] & isis.CELL_PRESENT != 0]
    assert (m == 63).any() and (m < 63).any() and m.max() == 63


def test_wide_totals_near_the_top(harness):
    """MT-IPv6 entries at 2^32 - 16: totals below the top stay exact, the others stop at 2^32 - 1."""
    v = isis.l1l2_view(42, n_l1=50, n_l2=30, mt6=True, summaries=[], cost_choices=[5, 10])
    l1 = v["l1"]
    lv = copy.copy(l1["level"])
    lv.ipreaches = lv.ipreaches.copy()
    mt = lv.ipreaches["kind"] == isis.IP_MT_V6
    lv.ipreaches["metric"] = np.where(mt, 0xFFFFFFF0, lv.ipreaches["metric"])
    l1 = dict(l1, level=lv)
    t, cells, words, planes = check(harness, l1, v["l2"], v["cfg"], jobs=view_jobs(dict(v, l1=l1), n_fail=6))
    v6 = t.kind == isis.IP_V6
    m = cells[:, v6]["metric"][cells[:, v6]["flags"] & isis.CELL_PRESENT != 0]
    assert (m == 0xFFFFFFFF).any() and ((m >= 0xFFFFFFF0) & (m < 0xFFFFFFFF)).any()


# ---- refusals ----------------------------------------------------------------------------------------------
def refused(l1, l2, rib, ud=None):
    with pytest.raises(capi.HspfError) as e:
        isis.L1ToL2Table(l1, l2, rib, ud)
    return e.value.code


def test_refusals(harness):
    v = isis.l1l2_view(13, n_l1=30, n_l2=30, summaries=[("10.1.0.0/16", None)])
    l1, l2 = v["l1"], v["l2"]
    rib = isis.L1L2RibTable(l1, l2, v["cfg"])
    assert refused(dict(l1, level_type=2), l2, rib) == capi.HSPF_E_INVAL
    assert refused(l1, dict(l2, level_type=1), rib) == capi.HSPF_E_INVAL
    assert refused(l2, l1, rib) == capi.HSPF_E_INVAL
    assert refused(l1, dict(l2, system_id=l2["system_id"] + 1), rib) == capi.HSPF_E_INVAL
    other = isis.l1l2_view(14, n_l1=31, n_l2=30)                     # another area: vertex counts differ
    assert refused(other["l1"], l2, rib) == capi.HSPF_E_INVAL
    moved = isis.l1l2_view(13, n_l1=30, n_l2=30, root=1)             # the same area, another root
    assert refused(moved["l1"], moved["l2"], rib) == capi.HSPF_E_INVAL
    t = isis.L1ToL2Table(l1, l2, rib)
    # the decode refuses cells that are not the table's, and another instance
    planes = oracle_planes(l1, rib.root[0], rib.n_vertices[0])
    cells, words = cells_on_cpu(harness, t, [planes])
    s = int(np.nonzero(cells[0]["winner"] >= t.n_records)[0][0])
    with pytest.raises(capi.HspfError):
        isis.l1_to_l2_from_cells(l1, t, cells[0], np.zeros_like(words[0]))       # a summary cell, its word inactive
    c = cells[0].copy()
    p = int(np.nonzero((c["winner"] < t.n_records) & (c["flags"] & isis.CELL_PRESENT != 0))[0][0])
    c["winner"][p] = t.n_records - 1 if c["winner"][p] == 0 else 0                 # a record of another key
    with pytest.raises(capi.HspfError):
        isis.l1_to_l2_from_cells(l1, t, c, words[0])
    with pytest.raises(capi.HspfError):
        isis.l1_to_l2_from_cells(l2, t, cells[0], words[0])
    assert s >= 0
