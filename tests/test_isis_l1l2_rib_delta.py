"""CPU: the route-delta stage over the routing-table cells of IS-IS L1/L2 routers (hspf_isis_l1l2_rib_delta[16]).

The cells of a what-if batch come from the walk harness (test_isis_l1l2_rib_cells); the delta harness (the body of the
route-delta passes compiled for the host) must equal the numpy reference with every base mapping, status word and
capacity it distinguishes.  At route level, the records of each job name exactly the prefixes its decoded table
loses, gains or reaches at another metric, and every prefix hspf_isis_rib_diff installs or uninstalls."""
import numpy as np
import pytest

from holo_b200 import capi, isis
from holo_b200.route_table import DELTA_GAINED, DELTA_LOST, DELTA_METRIC, DELTA_OTHER
from test_isis_l1l2_rib_cells import (cells_on_cpu, decode, harness, job_planes, link_edges, p2p_links,  # noqa: F401
                                      topology_flat)
from test_route_delta import check_stage, harnesses  # noqa: F401


def batch(harness, v, n_l1, n_l2):
    """Job 0 unperturbed, then n_l1 jobs each disabling one L1 adjacency and n_l2 jobs one L2 adjacency."""
    l1, l2 = v["l1"], v["l2"]
    t = isis.L1L2RibTable(l1, l2, v["cfg"], v["l2_derived"])
    jobs = [((), ())]
    f1, f2 = topology_flat(l1, isis.MT_STANDARD), topology_flat(l2, isis.MT_STANDARD)
    sys2 = lambda i: isis.sysid(i) if i < 3 else isis.sysid(v["t1"].n_routers + i)
    for a, b in p2p_links(v["t1"], 0, v["t1"].n_routers, isis.sysid)[:n_l1]:
        jobs.append(([(e, capi.COST_DISABLED) for e in link_edges(f1, a, b)], ()))
    for a, b in p2p_links(v["t2"], 3, v["t2"].n_routers, sys2)[:n_l2]:
        jobs.append(((), [(e, capi.COST_DISABLED) for e in link_edges(f2, a, b)]))
    planes = [job_planes(l1, l2, t, {isis.TOPO_STD: o1}, {isis.TOPO_STD: o2}) for o1, o2 in jobs]
    cells, words = cells_on_cpu(harness, t, planes)
    return t, jobs, planes, cells, words


def keys(t, rib):
    index = {(bytes(p["bytes"]), int(p["is_v6"]), int(n)): i for i, (p, n) in enumerate(zip(t.prefix, t.len))}
    return {index[(bytes(r["prefix"]["bytes"]), int(r["prefix"]["is_v6"]), int(r["len"]))]: r for r in rib.routes}, index


def touched(index, base_rib, rib):
    """Prefix indices of every install / uninstall hspf_isis_rib_diff lists going from base_rib to rib."""
    _, installed = isis.rib_diff(None, base_rib)
    acts, _ = isis.rib_diff(isis.IsisRib(installed, base_rib.nexthops), rib)
    out = set()
    for a in acts:
        # HL_RIB_UNINSTALL_OLD (3) names a route of the base table
        r = (base_rib.routes if a["kind"] == 3 else rib.routes)[int(a["route"])]
        out.add(index[(bytes(r["prefix"]["bytes"]), int(r["prefix"]["is_v6"]), int(r["len"]))])
    return out


@pytest.mark.parametrize("seed,mtype", [(31, isis.METRIC_WIDE), (32, isis.METRIC_BOTH)])
def test_stage_against_the_numpy_reference(harness, harnesses, seed, mtype):
    v = isis.l1l2_view(seed, n_l1=40, n_l2=40, metric_type=mtype, l1_degree=2, cost_choices=[5, 10],
                       summaries=[("10.2.0.0/16", None), ("10.1.0.5/32", None)])
    t, jobs, planes, cells, words = batch(harness, v, 12, 8)
    job_out, records, total = check_stage(harnesses, cells, n_base=2)
    assert total > 0 and job_out["n_metric"].sum() > 0 and job_out["n_other"].sum() > 0


def test_records_match_decoded_tables_and_rib_diff(harness, harnesses):
    """L1 failures move prefixes from their L1 route to another border router's L2 route (a new winner: OTHER) and
    deactivate a summary; L2 failures change L2 metrics.  Records and decoded tables agree."""
    v = isis.l1l2_view(33, n_l1=40, n_l2=40, l1_degree=2, cost_choices=[5],
                       summaries=[("10.2.0.0/16", None), ("10.1.0.5/32", None)])
    t, jobs, planes, cells, words = batch(harness, v, 40, 12)
    job_out, records, total = check_stage(harnesses, cells)
    base_rib = decode(v["l1"], v["l2"], t, cells[0], words[0], planes[0], [(), (), (), ()])
    assert base_rib.rc == capi.HSPF_OK
    base, index = keys(t, base_rib)
    n_moved = n_summary_lost = 0
    for j in range(1, len(jobs)):
        o1, o2 = jobs[j]
        rib = decode(v["l1"], v["l2"], t, cells[j], words[j], planes[j], [o1, (), o2, ()])
        assert rib.rc == capi.HSPF_OK
        rows, _ = keys(t, rib)
        r = records[records["job"] == j]
        assert set(r["prefix"][r["kind"] == DELTA_LOST].tolist()) == set(base) - set(rows)
        assert set(r["prefix"][r["kind"] == DELTA_GAINED].tolist()) == set(rows) - set(base)
        assert (set(r["prefix"][(r["kind"] & DELTA_METRIC) != 0].tolist())
                == {p for p in set(base) & set(rows) if base[p]["metric"] != rows[p]["metric"]})
        assert touched(index, base_rib, rib) <= set(r["prefix"].tolist()), j
        moved = (cells[0]["winner"] < t.n_l1) & (cells[j]["winner"] >= t.n_l1) & (cells[j]["flags"] & isis.CELL_PRESENT != 0)
        other = set(r["prefix"][(r["kind"] & DELTA_OTHER) != 0].tolist())
        assert set(np.nonzero(moved)[0].tolist()) <= other
        n_moved += int(moved.sum())
        # a summary the job deactivates: its prefix changes (another border router's L2 route, or none)
        off = np.nonzero((words[0] >> np.uint64(32) == 1) & (words[j] >> np.uint64(32) == 0))[0]
        summary_prefix = {int(np.nonzero(t.sum_of == s)[0][0]) for s in off}
        assert summary_prefix <= set(r["prefix"].tolist())
        n_summary_lost += len(summary_prefix)
    assert n_moved > 0 and n_summary_lost > 0
