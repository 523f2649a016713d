"""CPU: the route-delta stage over OSPFv2 routing-table cells (hl_ospf_rib_cell; hspf_ospfv2_rib_delta[16]).

The classification the device stage compiles (holo_b200/csrc/route_delta.h with OspfRibCellLayout) runs in a CPU
harness (tests/native/rib_delta_harness.cc, over the stage of route_delta_harness.cc): hand-built cell pairs give exactly their kind, and the whole stage equals a numpy reference over
the cells the routing-table harness computes for what-if jobs.  The route-level tie decodes the base and each job
(hspf_ospfv2_rib_from_cells) and checks that the records name the prefixes whose presence or metric changed, and every
prefix update_global_rib would touch.  tests/test_ospf_rib_delta_gpu.py compares the device stage with the same
reference."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from holo_b200 import capi, ospf_rib, ospfv2, synth
from holo_b200.route_table import (DELTA_DT, DELTA_GAINED, DELTA_JOB_DT, DELTA_LOST, DELTA_METRIC, DELTA_NEXTHOPS,
                                   DELTA_OTHER)
from test_ospf_rib_cells import flags_of, harness, harness_cells, planes_of, view  # noqa: F401
from test_ospfv2_route_cells import gather_for
from test_route_delta import same_stage

ROOT = Path(__file__).resolve().parent.parent
PRESENT, CONNECTED = ospfv2.CELL_PRESENT, ospfv2.CELL_CONNECTED
METRIC_MAX = 0x03FFFFFF                # HL_RIB_CELL_METRIC_MAX


@pytest.fixture(scope="module")
def delta_harness(built, tmp_path_factory):
    """tests/native/rib_delta_harness.cc: the route-delta stage over routing-table cells, compiled on the CPU."""
    so = tmp_path_factory.mktemp("harness") / "librib_delta_harness.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                    "-o", str(so), str(ROOT / "tests" / "native" / "rib_delta_harness.cc")], check=True)
    d = C.CDLL(str(so))
    d.harness_rib_delta_kind.argtypes = [C.c_void_p, C.c_void_p]
    d.harness_rib_delta_kind.restype = C.c_uint32
    d.harness_rib_route_delta.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
    return d


# ---- numpy reference of the stage over RIB_CELL_DT ---------------------------------------------------------------
def classify(J, B):
    """HL_DELTA_* of routing-table cells J against B (same shape), from the cell fields."""
    jp, bp = (ospf_rib.cell_flags(J) & PRESENT) != 0, (ospf_rib.cell_flags(B) & PRESENT) != 0
    both = jp & bp
    k = np.zeros(J.shape, np.uint8)
    k[bp & ~jp] = DELTA_LOST
    k[jp & ~bp] = DELTA_GAINED
    k[both & (ospf_rib.cell_metric(J) != ospf_rib.cell_metric(B))] |= DELTA_METRIC
    k[both & (J["nh_mask"] != B["nh_mask"])] |= DELTA_NEXTHOPS
    other = ((J["winner"] != B["winner"]) | (J["aux"] != B["aux"]) | (ospf_rib.cell_path(J) != ospf_rib.cell_path(B))
             | (ospf_rib.cell_flags(J) != ospf_rib.cell_flags(B)))
    k[both & other] |= DELTA_OTHER
    return k


def reference(cells, base, base_of=None, status=None, cap=None):
    """(job summaries, the first min(total, cap) records, total) of the stage over cells [n_jobs, P]."""
    n, P = cells.shape
    job_out = np.zeros(n, DELTA_JOB_DT)
    recs = []
    for j in range(n):
        b = 0 if base_of is None else int(base_of[j])
        st = capi.JS_INVALID if b >= len(base) else (0 if status is None else int(status[j]))
        job_out[j]["status"] = st
        if st:
            continue
        k = classify(cells[j], base[b])
        nz = np.nonzero(k)[0]
        job_out[j]["n_changed"] = len(nz)
        for name, bit in (("n_lost", DELTA_LOST), ("n_gained", DELTA_GAINED), ("n_metric", DELTA_METRIC),
                          ("n_nexthops", DELTA_NEXTHOPS), ("n_other", DELTA_OTHER)):
            job_out[j][name] = int(((k & bit) != 0).sum())
        r = np.zeros(len(nz), DELTA_DT)
        r["job"], r["prefix"], r["kind"] = j, nz, k[nz]
        r["metric"] = np.where(k[nz] == DELTA_LOST, ospf_rib.cell_metric(base[b][nz]), ospf_rib.cell_metric(cells[j][nz]))
        recs.append(r)
    records = np.concatenate(recs) if recs else np.zeros(0, DELTA_DT)
    total = len(records)
    return job_out, records[: total if cap is None else min(total, cap)], total


def harness_stage(d, cells, base, base_of=None, status=None, cap=None):
    """The rib-delta harness's stage over routing-table cells, the same triple as reference()."""
    n, P = cells.shape
    cells, base = np.ascontiguousarray(cells, ospf_rib.RIB_CELL_DT), np.ascontiguousarray(base, ospf_rib.RIB_CELL_DT)
    bo = None if base_of is None else np.ascontiguousarray(base_of, np.uint32)
    st = None if status is None else np.ascontiguousarray(status, np.uint32)
    cap = n * P if cap is None else cap
    job_out = np.zeros(n, DELTA_JOB_DT)
    records = np.zeros(max(cap, 1), DELTA_DT)
    total = C.c_uint64()
    d.harness_rib_route_delta(cells.ctypes.data, n, P, base.ctypes.data, len(base),
                              None if bo is None else bo.ctypes.data, None if st is None else st.ctypes.data,
                              job_out.ctypes.data, records.ctypes.data, cap, C.byref(total))
    return job_out, records[: min(total.value, cap)], total.value


def perturbed(row):
    """A base row that differs from `row` in every way a routing-table cell can: metric, atoms, presence (both ways),
    winner, path type and aux."""
    r = row.copy()
    m = ospf_rib.cell_metric(r)
    r["mpf"][::3] = (r["mpf"][::3] & ~np.uint32(METRIC_MAX)) | ((m[::3] + 1) & METRIC_MAX)
    r["nh_mask"][1::5] ^= 1
    r["mpf"][2::7] ^= np.uint32(PRESENT << 28)
    absent = np.nonzero((ospf_rib.cell_flags(row) & PRESENT) == 0)[0]
    r["mpf"][absent[:1]] |= np.uint32(PRESENT << 28)          # LOST wherever the job lacks that prefix too
    r["winner"][3::11] += 1
    r["mpf"][5::17] ^= np.uint32(1 << 26)
    r["aux"][4::13] ^= 2
    return r


# ---- one cell pair at a time ------------------------------------------------------------------------------------
def cell(nh=0b0110, aux=0b0010, winner=3, metric=10, path=ospf_rib.PATH_INTRA, flags=PRESENT):
    c = np.zeros(1, ospf_rib.RIB_CELL_DT)
    c["nh_mask"], c["aux"], c["winner"] = nh, aux, winner
    c["mpf"] = metric | (path << 26) | (flags << 28)
    return c


EMPTY = dict(nh=0, aux=0, winner=ospf_rib.NO_RECORD, metric=0, path=0, flags=0)
CASES = [
    ("same", {}, {}, 0),
    ("lost", {}, EMPTY, DELTA_LOST),
    ("gained", EMPTY, {}, DELTA_GAINED),
    ("metric", {}, dict(metric=11), DELTA_METRIC),
    ("metric at max", {}, dict(metric=METRIC_MAX), DELTA_METRIC),
    ("metric from max", dict(metric=METRIC_MAX), dict(metric=METRIC_MAX - 1), DELTA_METRIC),
    ("nexthops", {}, dict(nh=0b0100), DELTA_NEXTHOPS),
    ("intra to inter", {}, dict(winner=40, aux=0, path=ospf_rib.PATH_INTER), DELTA_OTHER),
    ("intra to inter, metric", {}, dict(winner=40, aux=0, path=ospf_rib.PATH_INTER, metric=30), DELTA_OTHER | DELTA_METRIC),
    ("inter to type-1", dict(winner=40, aux=0, path=ospf_rib.PATH_INTER), dict(winner=90, aux=0, path=ospf_rib.PATH_TYPE1),
     DELTA_OTHER),
    ("inter to type-2", dict(winner=40, aux=0, path=ospf_rib.PATH_INTER),
     dict(winner=91, aux=7, path=ospf_rib.PATH_TYPE2, metric=20), DELTA_OTHER | DELTA_METRIC),
    ("type-2 metric", dict(winner=91, aux=7, path=ospf_rib.PATH_TYPE2), dict(winner=92, aux=8, path=ospf_rib.PATH_TYPE2),
     DELTA_OTHER),
    ("aux only", {}, dict(aux=0b0100), DELTA_OTHER),
    ("connected", {}, dict(flags=PRESENT | CONNECTED), DELTA_OTHER),
    ("everything", {}, dict(nh=1, metric=12, winner=0, aux=0), DELTA_METRIC | DELTA_NEXTHOPS | DELTA_OTHER),
    ("both empty", EMPTY, EMPTY, 0),
    ("both absent, words differ", EMPTY, dict(EMPTY, nh=5, aux=3, winner=2, metric=7, path=3), 0),
]


@pytest.mark.parametrize("name,b,j,want", CASES, ids=[c[0] for c in CASES])
def test_kind_of_one_cell(delta_harness, name, b, j, want):
    B, J = cell(**b), cell(**j)
    assert delta_harness.harness_rib_delta_kind(J.ctypes.data, B.ctypes.data) == want
    assert classify(J, B)[0] == want
    # as a one-job batch: the record carries the job's metric, the base's when the prefix was lost
    job_out, records, total = harness_stage(delta_harness, J[None], B[None])
    same_stage((job_out, records, total), reference(J[None], B[None]))
    assert total == int(want != 0)
    if want:
        assert records[0]["metric"] == ospf_rib.cell_metric(B if want == DELTA_LOST else J)[0]


def test_lost_record_carries_the_base_metric(delta_harness):
    B = np.concatenate([cell(metric=METRIC_MAX), cell(metric=77, winner=5)])
    J = np.concatenate([cell(**EMPTY), cell(**EMPTY)])
    _, records, _ = harness_stage(delta_harness, J[None], B[None])
    assert records["kind"].tolist() == [DELTA_LOST] * 2 and records["metric"].tolist() == [METRIC_MAX, 77]


# ---- what-if batches ----------------------------------------------------------------------------------------------
def link_pairs(flat):
    """(e, reverse e) of every router-to-router link of the flat's CSR, each link once."""
    csr = flat.csr
    src = np.repeat(np.arange(csr.n_vertices), np.diff(csr.row_ptr))
    out, seen = [], set()
    for e in range(csr.n_edges):
        if flat.link_index[e] == 0xFFFFFFFF or e in seen:
            continue
        u, v = int(src[e]), int(csr.col[e])
        back = [f for f in range(csr.row_ptr[v], csr.row_ptr[v + 1]) if csr.col[f] == u and flat.link_index[f] != 0xFFFFFFFF]
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


def internal_root(area, flat, start=0):
    fl = flags_of(area)
    return next(flat.router_vertex(r) for r in sorted(fl)[start:] if not fl[r] & 0x01)


def whatif_batch(harness, flat, rt, roots, overrides):  # noqa: F811
    """Harness cells and status words of jobs rooted at `roots` with `overrides`, and each job's wide planes."""
    V = flat.csr.n_vertices
    planes = [planes_of(flat.csr, r if r < V else 0, overrides=o) for r, o in zip(roots, overrides)]
    stack = tuple(np.stack([p[i].reshape(-1) for p in planes]) for i in range(3))
    cells, st = harness_cells(harness, rt, roots, stack)
    return cells, st, planes


SEEDS = [(1, dict(cost_choices=[10]), 16), (2, dict(cost_choices=[10, 20], lan_fraction=0.15), 16),
         (3, dict(cost_choices=[10, 20], lan_fraction=0.15), 2), (5, dict(cost_choices=[5, 10], lan_fraction=0.2), 16)]


@pytest.mark.parametrize("seed,kw,mp", SEEDS, ids=[f"seed{s[0]}" for s in SEEDS])
def test_stage_over_whatif_cells(harness, delta_harness, seed, kw, mp):  # noqa: F811
    """Jobs of one internal root with link cuts and cost changes, one ABR root and one root out of range; the stage
    against job 0 and against a perturbed row, with base_of (one row out of range), status words and every cap."""
    t = synth.random_topology(60, 240, synth.SEED_BASE + 300 + seed, **kw)
    area, sums, ext = view(t, 0, 900 + seed, mp)
    flat = ospfv2.Flat(area)
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
    assert total > 0 and all(job_out[k].sum() > 0 for k in ("n_metric", "n_nexthops", "n_other"))
    assert (job_out["status"][[5, 7, 9]] != 0).all() and not job_out["n_changed"][[5, 7, 9]].any()
    for cap in sorted({0, 1, max(total // 2, 1), total}):
        same_stage(harness_stage(d, cells, base[:1], status=st, cap=cap), reference(cells, base[:1], status=st, cap=cap))
    base_of = np.arange(n) % 3                                         # row 2 is out of range
    got = harness_stage(d, cells, base, base_of, st)
    same_stage(got, reference(cells, base, base_of, st))
    assert (got[0]["status"][base_of == 2] == capi.JS_INVALID).all()
    vs_perturbed = reference(cells, base[1:], status=st)[0]
    assert vs_perturbed["n_lost"].sum() > 0 and vs_perturbed["n_gained"].sum() > 0


# ---- route-level tie ----------------------------------------------------------------------------------------------
def route_rows(rt, rib):
    """{prefix index: metric} of a decoded table."""
    index = {k: i for i, k in enumerate(zip(rt.prefix.tolist(), rt.plen.tolist()))}
    return {index[(int(r["prefix"]), bin(int(r["mask"])).count("1"))]: int(r["metric"]) for r in rib.routes}


def check_tie(records, j, base_rows, job_rows):
    """records of job j == the prefixes present in one table only (LOST / GAINED) and those whose metric differs
    (METRIC).  Returns the prefixes reported for j."""
    r = records[records["job"] == j]
    assert set(r["prefix"][r["kind"] == DELTA_LOST].tolist()) == set(base_rows) - set(job_rows)
    assert set(r["prefix"][r["kind"] == DELTA_GAINED].tolist()) == set(job_rows) - set(base_rows)
    assert (set(r["prefix"][(r["kind"] & DELTA_METRIC) != 0].tolist())
            == {p for p in set(base_rows) & set(job_rows) if base_rows[p] != job_rows[p]})
    return set(r["prefix"].tolist())


def touched_prefixes(rt, base_rib, rib):
    """Prefix indices of every install / uninstall update_global_rib lists going from base_rib to rib."""
    _, installed = ospf_rib.rib_diff(None, base_rib)
    acts, _ = ospf_rib.rib_diff(ospf_rib.Rib(installed, base_rib.nexthops), rib)
    index = {k: i for i, k in enumerate(zip(rt.prefix.tolist(), rt.plen.tolist()))}
    out = set()
    for a in acts:
        src = base_rib.routes if a["kind"] == ospf_rib.RIB_UNINSTALL_OLD else rib.routes
        r = src[int(a["route"])]
        out.add(index[(int(r["prefix"]), bin(int(r["mask"])).count("1"))])
    return out


def tie(area, flat, rt, rv, cells, planes, records, job_ids):
    """The route-level tie over decoded tables of jobs `job_ids` against job 0.  Returns (jobs checked, jobs whose
    update_global_rib actions were checked)."""
    def decode(j):
        d, h, m = planes[j]
        gv, gn = gather_for(flat, rv, (d, h, m.reshape(-1)))
        return ospf_rib.rib_from_cells(area, rt, cells[j], gv, gn), gn

    base_rib, base_gn = decode(0)
    assert base_rib.rc == capi.HSPF_OK
    base_rows = route_rows(rt, base_rib)
    checked = diffed = 0
    for j in job_ids:
        rib, gn = decode(j)
        if rib.rc != capi.HSPF_OK:
            continue
        reported = check_tie(records, j, base_rows, route_rows(rt, rib))
        checked += 1
        if (gn == base_gn).all():                  # the transit networks next to the root keep their atom sets
            assert touched_prefixes(rt, base_rib, rib) <= reported, j
            diffed += 1
    return checked, diffed


@pytest.mark.parametrize("seed", [2, 5])
def test_records_match_decoded_tables(harness, delta_harness, seed):  # noqa: F811
    kw = dict(cost_choices=[10, 20], lan_fraction=0.15)
    t = synth.random_topology(60, 240, synth.SEED_BASE + 340 + seed, **kw)
    fl = flags_of(view(t, 0, 980 + seed)[0])
    root = next(r for r in sorted(fl) if not fl[r] & 0x01) - ospfv2.RID_BASE      # the first internal router
    area, sums, ext = view(t, root, 980 + seed)
    flat = ospfv2.Flat(area)
    rv = flat.router_vertex(area.router_id)
    rt = ospf_rib.RibTable(flat, area.area_id, sums, ext)
    n = 24
    cells, st, planes = whatif_batch(harness, flat, rt, [rv] * n, whatif_overrides(flat, n, seed))
    assert not st.any()
    job_out, records, total = harness_stage(delta_harness, cells, cells[:1])
    same_stage((job_out, records, total), reference(cells, cells[:1]))
    assert total > 0
    checked, diffed = tie(area, flat, rt, rv, cells, planes, records, range(1, n))
    assert checked >= n // 2 and diffed >= n // 3
