"""CPU: the route-delta stage's classification (holo_b200/csrc/route_delta.h: route_delta_kind), compiled into a test
harness with a CPU restatement of the stage (summaries, record order, capacity), checked cell by cell against a
table of cases for both cell layouts and, over the cells the existing CPU harnesses compute on synthetic and golden
instances, against a numpy reference of the whole stage.  tests/test_route_delta_gpu.py compares the device stage
with the same numpy reference."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import golden_util as gu
from holo_b200 import capi, isis, ospfv2, synth
from holo_b200.route_table import (DELTA_DT, DELTA_GAINED, DELTA_JOB_DT, DELTA_LOST, DELTA_METRIC, DELTA_NEXTHOPS,
                                   DELTA_OTHER)
from isis_synth import synth_instance
from oracle import pyoracle

ROOT = Path(__file__).resolve().parent.parent
NAMES = ("route_cells_harness", "isis_route_cells_harness", "route_delta_harness")


@pytest.fixture(scope="module")
def harnesses(built, tmp_path_factory):
    """The two cell harnesses and the delta harness (tests/native), compiled in a temporary directory."""
    out = tmp_path_factory.mktemp("harness")
    libs = {}
    for name in NAMES:
        so = out / f"lib{name}.so"
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                        "-o", str(so), str(ROOT / "tests" / "native" / f"{name}.cc")], check=True)
        libs[name] = C.CDLL(str(so))
    libs["route_cells_harness"].harness_route_cells.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 4
    libs["isis_route_cells_harness"].harness_isis_route_cells.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 7
    d = libs["route_delta_harness"]
    d.harness_delta_kind.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
    d.harness_delta_kind.restype = C.c_uint32
    d.harness_route_delta.argtypes = [C.c_int, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
    return {"ospf": libs["route_cells_harness"], "isis": libs["isis_route_cells_harness"], "delta": d}


# ---- numpy reference of the stage -------------------------------------------------------------------------------
def classify(J, B, is_isis):
    """HL_DELTA_* of job cells J against base cells B (same shape), from the cell fields."""
    jp, bp = (J["flags"] & 1) != 0, (B["flags"] & 1) != 0
    both = jp & bp
    k = np.zeros(J.shape, np.uint8)
    k[bp & ~jp] = DELTA_LOST
    k[jp & ~bp] = DELTA_GAINED
    k[both & (J["metric"] != B["metric"])] |= DELTA_METRIC
    k[both & (J["nh_mask"] != B["nh_mask"])] |= DELTA_NEXTHOPS
    other = (J["winner"] != B["winner"]) | (J["flags"] != B["flags"])
    if not is_isis:
        other |= J["lasthop_mask"] != B["lasthop_mask"]
    k[both & other] |= DELTA_OTHER
    return k


def reference(cells, base, base_of=None, status=None, cap=None):
    """(job summaries, the first min(total, cap) records, total) of the stage over cells [n_jobs, P]."""
    is_isis = cells.dtype == isis.CELL_DT
    n, P = cells.shape
    job_out = np.zeros(n, DELTA_JOB_DT)
    recs = []
    for j in range(n):
        b = 0 if base_of is None else int(base_of[j])
        st = capi.JS_INVALID if b >= len(base) else (0 if status is None else int(status[j]))
        job_out[j]["status"] = st
        if st:
            continue
        k = classify(cells[j], base[b], is_isis)
        nz = np.nonzero(k)[0]
        job_out[j]["n_changed"] = len(nz)
        for name, bit in (("n_lost", DELTA_LOST), ("n_gained", DELTA_GAINED), ("n_metric", DELTA_METRIC),
                          ("n_nexthops", DELTA_NEXTHOPS), ("n_other", DELTA_OTHER)):
            job_out[j][name] = int(((k & bit) != 0).sum())
        r = np.zeros(len(nz), DELTA_DT)
        r["job"], r["prefix"], r["kind"] = j, nz, k[nz]
        r["metric"] = np.where(k[nz] == DELTA_LOST, base[b]["metric"][nz], cells[j]["metric"][nz])
        recs.append(r)
    records = np.concatenate(recs) if recs else np.zeros(0, DELTA_DT)
    total = len(records)
    return job_out, records[: total if cap is None else min(total, cap)], total


def harness_stage(d, cells, base, base_of=None, status=None, cap=None):
    """The CPU harness's stage, the same triple as reference()."""
    n, P = cells.shape
    cells, base = np.ascontiguousarray(cells), np.ascontiguousarray(base)
    bo = None if base_of is None else np.ascontiguousarray(base_of, np.uint32)
    st = None if status is None else np.ascontiguousarray(status, np.uint32)
    cap = n * P if cap is None else cap
    job_out = np.zeros(n, DELTA_JOB_DT)
    records = np.zeros(max(cap, 1), DELTA_DT)
    total = C.c_uint64()
    d.harness_route_delta(int(cells.dtype == isis.CELL_DT), cells.ctypes.data, n, P, base.ctypes.data, len(base),
                          None if bo is None else bo.ctypes.data, None if st is None else st.ctypes.data,
                          job_out.ctypes.data, records.ctypes.data, cap, C.byref(total))
    return job_out, records[: min(total.value, cap)], total.value


def same_stage(a, b):
    assert a[2] == b[2]
    assert a[0].tobytes() == b[0].tobytes()
    assert a[1].tobytes() == b[1].tobytes()


# ---- one cell pair at a time ------------------------------------------------------------------------------------
def base_cell(dt):
    c = np.zeros(1, dt)
    c["nh_mask"], c["winner"], c["metric"], c["flags"] = 0b0110, 3, 10, ospfv2.CELL_PRESENT
    if dt == ospfv2.CELL_DT:
        c["lasthop_mask"] = 0b0010
    return c


OSPF_ONLY = {"lasthop"}
ISIS_WIDE = {"metric32"}
CASES = [
    ("same", {}, 0),
    ("metric", {"metric": 11}, DELTA_METRIC),
    ("metric32", {"metric": 10 + (1 << 20)}, DELTA_METRIC),
    ("nexthops", {"nh_mask": 0b0100}, DELTA_NEXTHOPS),
    ("metric+nexthops", {"metric": 9, "nh_mask": 0b1000}, DELTA_METRIC | DELTA_NEXTHOPS),
    ("winner", {"winner": 4}, DELTA_OTHER),
    ("flags", {"flags": ospfv2.CELL_PRESENT | ospfv2.CELL_CONNECTED}, DELTA_OTHER),
    ("lasthop", {"lasthop_mask": 0b0100}, DELTA_OTHER),
    ("all three", {"metric": 12, "nh_mask": 1, "winner": 0}, DELTA_METRIC | DELTA_NEXTHOPS | DELTA_OTHER),
    ("lost", {"flags": 0, "nh_mask": 0xF0, "winner": 9, "metric": 99}, DELTA_LOST),
    ("gained", None, DELTA_GAINED),
    ("both absent, words differ", "absent", 0),
]


@pytest.mark.parametrize("layout", ["ospf", "isis"])
@pytest.mark.parametrize("name,change,want", CASES, ids=[c[0] for c in CASES])
def test_kind_of_one_cell(harnesses, layout, name, change, want):
    dt = ospfv2.CELL_DT if layout == "ospf" else isis.CELL_DT
    if (name in OSPF_ONLY and layout == "isis") or (name in ISIS_WIDE and layout == "ospf"):
        pytest.skip("field of the other layout")
    B, J = base_cell(dt), base_cell(dt)
    if change is None:                                # GAINED: the base is absent, every other word differs
        B["flags"], B["nh_mask"], B["winner"], B["metric"] = 0, 0xF0, 0xFFFFFFFF, 0
        if layout == "ospf":
            B["lasthop_mask"] = 0xF0
    elif change == "absent":
        B["flags"], J["flags"] = 0, 0
        J["nh_mask"], J["winner"], J["metric"] = 5, 2, 7
    else:
        for k, v in change.items():
            J[k] = v
    got = harnesses["delta"].harness_delta_kind(int(layout == "isis"), J.ctypes.data, B.ctypes.data)
    assert got == want
    assert classify(J, B, layout == "isis")[0] == want


# ---- the whole stage over cells of the existing CPU harnesses ---------------------------------------------------
def ospf_batch(harnesses, t, root, n_jobs, seed):
    """Cells [n_jobs, P] of OSPFv2 what-if jobs of one root: job 0 plain, job j > 0 disables one edge or raises one
    cost (the oracle's planes)."""
    from test_ospfv2_route_cells import cells_on_cpu
    area = ospfv2.synth_area(t, root=root, sr=True)
    flat = ospfv2.Flat(area)
    rt = ospfv2.RouteTable(flat)
    rv = flat.router_vertex(area.router_id)
    rng = np.random.default_rng(seed)
    E = flat.csr.n_edges
    rows = []
    for j in range(n_jobs):
        ov = [] if j == 0 else [(int(rng.integers(E)), capi.COST_DISABLED if j % 2 else int(rng.integers(1, 60)))]
        c = pyoracle.csr_spf(flat.csr, rv, overrides=ov, nh_words=1)
        assert c["status"] == 0
        planes = (np.ascontiguousarray(c["dist"], np.uint32), np.ascontiguousarray(c["hops"], np.uint16),
                  np.ascontiguousarray(c["nh_mask"], np.uint64).reshape(-1))
        rows.append(cells_on_cpu(harnesses["ospf"], rt, planes))
    return np.stack(rows)


def isis_batch(harnesses, inst, n_jobs, seed):
    from test_isis_route_cells import cells_on_cpu, oracle_planes, topology_flat
    rt = isis.RouteTable(inst)
    E = topology_flat(inst, isis.MT_STANDARD).csr.n_edges
    rng = np.random.default_rng(seed)
    rows = []
    for j in range(n_jobs):
        ov = {} if j == 0 or E == 0 else {isis.TOPO_STD: [(int(rng.integers(E)),
                                                             capi.COST_DISABLED if j % 2 else int(rng.integers(1, 60)))]}
        rows.append(cells_on_cpu(harnesses["isis"], rt, oracle_planes(inst, rt, ov)))
    return rt, np.stack(rows)


def check_stage(harnesses, cells, n_base=1):
    """Reference and harness agree with every base mapping, status and capacity the stage distinguishes."""
    d = harnesses["delta"]
    n = len(cells)
    base = cells[:n_base]
    full = reference(cells, base)
    same_stage(harness_stage(d, cells, base), full)
    total = full[2]
    for cap in sorted({0, 1, max(total // 2, 1), total}):
        same_stage(harness_stage(d, cells, base, cap=cap), reference(cells, base, cap=cap))
    base_of = np.arange(n) % (n_base + 1)                 # row n_base is out of range
    status = np.zeros(n, np.uint32)
    status[1::3] = capi.JS_SATURATED
    same_stage(harness_stage(d, cells, base, base_of, status), reference(cells, base, base_of, status))
    return full


@pytest.mark.parametrize("seed,kw", [(21, dict(cost_choices=[5, 10], lan_fraction=0.1)), (22, dict(cost_lo=1, cost_hi=30))])
def test_stage_over_ospfv2_cells(harnesses, seed, kw):
    t = synth.random_topology(120, 500, synth.SEED_BASE + seed, **kw)
    cells = ospf_batch(harnesses, t, 3, 12, seed)
    job_out, records, total = check_stage(harnesses, cells, n_base=2)
    assert total > 0 and job_out["n_other"].sum() > 0
    assert job_out["n_metric"].sum() > 0 and job_out["n_nexthops"].sum() > 0


@pytest.mark.parametrize("seed,mtype,frag,sr", [(23, isis.METRIC_WIDE, 0, True), (24, isis.METRIC_WIDE, 2, False)])
def test_stage_over_isis_cells(harnesses, seed, mtype, frag, sr):
    t = synth.random_topology(120, 500, synth.SEED_BASE + seed, cost_lo=1, cost_hi=20, lan_fraction=0.1)
    _, cells = isis_batch(harnesses, synth_instance(t, 5, mtype, frag, sr=sr), 12, seed)
    job_out, _, total = check_stage(harnesses, cells, n_base=2)
    assert total > 0 and job_out["n_metric"].sum() > 0


def test_stage_over_isis_goldens(harnesses):
    """Every golden level as a two-job batch: the plain SPT and one with an edge raised; the base is job 0."""
    n = 0
    for snap in gu.load_isis():
        for level in snap["levels"]:
            inst = gu.isis_instance_image(snap, level)
            rt = isis.RouteTable(inst)
            if rt.n_prefixes == 0 or rt.root[isis.TOPO_STD] == isis.NO_ROOT:
                continue
            _, cells = isis_batch(harnesses, inst, 3, 7)
            check_stage(harnesses, cells)
            n += 1
    assert n >= 30


def test_lost_and_gained_prefixes_from_a_disabled_root_link(harnesses):
    """Removing every link of a leaf router loses its prefixes: LOST records with the base's metric."""
    t = synth.random_topology(80, 320, synth.SEED_BASE + 25, cost_choices=[10])
    cells = ospf_batch(harnesses, t, 0, 1, 1)
    from test_ospfv2_route_cells import cells_on_cpu
    area = ospfv2.synth_area(t, root=0, sr=True)
    flat = ospfv2.Flat(area)
    rt = ospfv2.RouteTable(flat)
    rv = flat.router_vertex(area.router_id)
    csr = flat.csr
    other = next(v for v in range(csr.n_vertices) if flat.is_router[v] and v != rv)
    ov = [(e, capi.COST_DISABLED) for u in range(csr.n_vertices) for e in range(csr.row_ptr[u], csr.row_ptr[u + 1])
          if csr.col[e] == other]
    c = pyoracle.csr_spf(csr, rv, overrides=ov, nh_words=1)
    planes = (np.ascontiguousarray(c["dist"], np.uint32), np.ascontiguousarray(c["hops"], np.uint16),
              np.ascontiguousarray(c["nh_mask"], np.uint64).reshape(-1))
    cut = cells_on_cpu(harnesses["ospf"], rt, planes)
    batch = np.stack([cells[0], cut])
    job_out, records, _ = check_stage(harnesses, batch)
    lost = records[records["kind"] == DELTA_LOST]
    assert len(lost) > 0 and job_out[1]["n_lost"] == len(lost)
    assert (lost["metric"] == cells[0][lost["prefix"]]["metric"]).all()
    # and the other way round: with the cut job as the base, the same prefixes are gained
    _, back, _ = reference(np.stack([cut, cells[0]]), cut[None])
    assert (back[back["kind"] == DELTA_GAINED]["prefix"] == lost["prefix"]).all()
