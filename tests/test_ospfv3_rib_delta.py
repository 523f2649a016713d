"""CPU: the route-delta stage over OSPFv3 routing-table cells (hspf_ospfv2_rib_delta[16] over the tables of
hspf_ospfv3_ribtable_create).

The stage's CPU restatement (tests/native/rib_delta_harness.cc) over the cells the routing-table harness computes for
OSPFv3 what-if jobs must equal the numpy reference of tests/test_ospf_rib_delta.py, with base_of, caps and status
words.  The route-level tie decodes the base and each job (hspf_ospfv3_rib_from_cells) and checks that the records
name the prefixes whose presence or metric changed, and every prefix hspf_ospfv3_rib_diff would touch."""
import numpy as np
import pytest

from holo_b200 import capi, ospf_rib, ospfv3, synth
from holo_b200.route_table import DELTA_GAINED, DELTA_LOST, DELTA_METRIC
from test_ospf_rib_cells import harness, harness_cells, planes_of  # noqa: F401  (harness: the fixture)
from test_ospf_rib_delta import delta_harness, harness_stage, perturbed, reference  # noqa: F401
from test_ospfv2_route_cells import gather_for
from test_ospfv3_rib_cells import flags_of, view
from test_route_delta import same_stage


def link_pairs(flat):
    """(e, reverse e) of every router-to-router edge of the flat's CSR, each link once."""
    csr = flat.csr
    src = np.repeat(np.arange(csr.n_vertices), np.diff(csr.row_ptr))
    out, seen = [], set()
    for e in range(csr.n_edges):
        u, v = int(src[e]), int(csr.col[e])
        if e in seen or not (flat.is_router[u] and flat.is_router[v]):
            continue
        back = [f for f in range(csr.row_ptr[v], csr.row_ptr[v + 1]) if csr.col[f] == u and f not in seen]
        if back:
            seen.update((e, back[0]))
            out.append((e, back[0]))
    return out


def whatif_overrides(flat, n_jobs, seed):
    """Job 0 plain; job j > 0 disables one router-to-router link in both directions, or raises one edge's cost."""
    rng = np.random.default_rng(seed)
    pairs = link_pairs(flat)
    ov = [[]]
    for j in range(1, n_jobs):
        if j % 3:
            a, b = pairs[int(rng.integers(len(pairs)))]
            ov.append([(a, capi.COST_DISABLED), (b, capi.COST_DISABLED)])
        else:
            ov.append([(int(rng.integers(flat.csr.n_edges)), int(rng.integers(1, 60)))])
    return ov


def whatif_batch(harness, flat, rt, roots, overrides):  # noqa: F811
    V = flat.csr.n_vertices
    planes = [planes_of(flat.csr, r if r < V else 0, overrides=o) for r, o in zip(roots, overrides)]
    stack = tuple(np.stack([p[i].reshape(-1) for p in planes]) for i in range(3))
    cells, st = harness_cells(harness, rt, roots, stack)
    return cells, st, planes


def internal_root(area, flat):
    fl = flags_of(area)
    return next(flat.router_vertex(r) for r in sorted(fl) if not fl[r] & 0x01 and flat.router_vertex(r) != 0xFFFFFFFF)


SEEDS = [(1, dict(cost_choices=[10]), 16, 0), (2, dict(cost_choices=[10, 20], lan_fraction=0.15), 16, 0),
         (3, dict(cost_choices=[10, 20], lan_fraction=0.15), 2, 3), (5, dict(cost_choices=[5, 10], lan_fraction=0.2), 16, 0)]


@pytest.mark.parametrize("seed,kw,mp,frag", SEEDS, ids=[f"seed{s[0]}" for s in SEEDS])
def test_stage_over_whatif_cells(harness, delta_harness, seed, kw, mp, frag):  # noqa: F811
    """Jobs of one internal root with link cuts and cost changes, one ABR root and one root out of range; the stage
    against job 0 and against a perturbed row, with base_of (one row out of range), status words and every cap."""
    t = synth.random_topology(60, 240, synth.SEED_BASE + 500 + seed, **kw)
    area, sums, ext = view(t, 0, 1900 + seed, mp, frag)
    flat = ospfv3.Flat(area)
    rt = ospf_rib.RibTable(flat, area.area_id, sums, ext)
    rv = internal_root(area, flat)
    abr = flat.router_vertex(next(r for r, f in flags_of(area).items() if f & 0x01))
    n = 14
    roots = [rv] * n
    roots[5], roots[9] = abr, flat.csr.n_vertices
    cells, st, _ = whatif_batch(harness, flat, rt, roots, whatif_overrides(flat, n, seed))
    assert st[5] == ospf_rib.JS_NOT_INTERNAL and st[9] == capi.JS_INVALID
    st[7] |= capi.JS_SATURATED
    d = delta_harness
    base = np.stack([cells[0], perturbed(cells[0])])
    full = reference(cells, base[:1], status=st)
    same_stage(harness_stage(d, cells, base[:1], status=st), full)
    job_out, _, total = full
    assert total > 0 and job_out["n_metric"].sum() > 0 and job_out["n_nexthops"].sum() > 0
    assert (job_out["status"][[5, 7, 9]] != 0).all() and not job_out["n_changed"][[5, 7, 9]].any()
    for cap in sorted({0, 1, max(total // 2, 1), total}):
        same_stage(harness_stage(d, cells, base[:1], status=st, cap=cap), reference(cells, base[:1], status=st, cap=cap))
    base_of = np.arange(n) % 3                                         # row 2 is out of range
    got = harness_stage(d, cells, base, base_of, st)
    same_stage(got, reference(cells, base, base_of, st))
    assert (got[0]["status"][base_of == 2] == capi.JS_INVALID).all()
    vs_perturbed = reference(cells, base[1:], status=st)[0]
    assert all(vs_perturbed[k].sum() > 0 for k in ("n_lost", "n_gained", "n_other"))


# ---- route-level tie ----------------------------------------------------------------------------------------------
def prefix_index(rt):
    return {(bytes(int(b) for b in p["bytes"]), int(l)): i for i, (p, l) in enumerate(zip(rt.prefix, rt.plen))}


def route_rows(index, rib):
    """{prefix index: metric} of a decoded table."""
    return {index[(bytes(int(b) for b in r["prefix"]["bytes"]), int(r["len"]))]: int(r["metric"]) for r in rib.routes}


def touched_prefixes(index, base_rib, rib):
    """Prefix indices of every install / uninstall hspf_ospfv3_rib_diff lists going from base_rib to rib."""
    _, installed = ospf_rib.rib_diff(None, base_rib, v3=True)
    acts, _ = ospf_rib.rib_diff(ospf_rib.Rib(installed, base_rib.nexthops), rib, v3=True)
    out = set()
    for a in acts:
        r = (base_rib.routes if a["kind"] == ospf_rib.RIB_UNINSTALL_OLD else rib.routes)[int(a["route"])]
        out.add(index[(bytes(int(b) for b in r["prefix"]["bytes"]), int(r["len"]))])
    return out


@pytest.mark.parametrize("seed", [2, 5])
def test_records_match_decoded_tables(harness, delta_harness, seed):  # noqa: F811
    t = synth.random_topology(60, 240, synth.SEED_BASE + 540 + seed, cost_choices=[10, 20], lan_fraction=0.15)
    fl = flags_of(view(t, 0, 1980 + seed)[0])
    root = next(r for r in sorted(fl) if not fl[r] & 0x01) - ospfv3.RID_BASE      # the first internal router
    area, sums, ext = view(t, root, 1980 + seed)
    flat = ospfv3.Flat(area)
    rv = flat.router_vertex(area.router_id)
    rt = ospf_rib.RibTable(flat, area.area_id, sums, ext)
    n = 24
    cells, st, planes = whatif_batch(harness, flat, rt, [rv] * n, whatif_overrides(flat, n, seed))
    assert not st.any()
    job_out, records, total = harness_stage(delta_harness, cells, cells[:1])
    same_stage((job_out, records, total), reference(cells, cells[:1]))
    assert total > 0
    index = prefix_index(rt)

    def decode(j):
        d, h, m = planes[j]
        gv, gn = gather_for(flat, rv, (d, h, m.reshape(-1)))
        return ospf_rib.rib_from_cells_v3(area, rt, cells[j], gv, gn), gn

    base_rib, base_gn = decode(0)
    assert base_rib.rc == capi.HSPF_OK
    base_rows = route_rows(index, base_rib)
    checked = diffed = 0
    for j in range(1, n):
        rib, gn = decode(j)
        if rib.rc != capi.HSPF_OK:
            continue
        rows = route_rows(index, rib)
        r = records[records["job"] == j]
        assert set(r["prefix"][r["kind"] == DELTA_LOST].tolist()) == set(base_rows) - set(rows)
        assert set(r["prefix"][r["kind"] == DELTA_GAINED].tolist()) == set(rows) - set(base_rows)
        assert (set(r["prefix"][(r["kind"] & DELTA_METRIC) != 0].tolist())
                == {p for p in set(base_rows) & set(rows) if base_rows[p] != rows[p]})
        checked += 1
        if (gn == base_gn).all():                  # the transit networks next to the root keep their atom sets
            assert touched_prefixes(index, base_rib, rib) <= set(r["prefix"].tolist()), j
            diffed += 1
    assert checked >= n // 2 and diffed >= n // 3
