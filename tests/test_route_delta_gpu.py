"""GPU: the route-delta stage (hspf_ospfv2_routes_delta[16], hspf_isis_routes_delta[16]; holo_b200/csrc/route_stage.cuh).
The SPT planes are written on the device; every case compares the device summaries, records and total byte for byte
with the numpy reference of tests/test_route_delta.py, applied to the cells the existing route kernel writes over the
same device planes.  The route-level tests decode base and job tables on the host and check that the records name
exactly the prefixes whose presence or metric changed, and every prefix update_global_rib would touch."""
import ctypes as C

import numpy as np
import pytest

from holo_b200 import capi, isis, ospfv2, synth
from holo_b200.route_table import DELTA_DT, DELTA_GAINED, DELTA_JOB_DT, DELTA_LOST, DELTA_METRIC
from test_isis_route_cells import decode, topology_flat
from test_isis_route_cells_gpu import DeviceTopology, c3_small, device_cells, job_planes  # noqa: F401
from test_ospfv2_route_cells import gather_for
from test_route_delta import reference
from test_route_stage_gpu import Case, harnesses  # noqa: F401

pytestmark = pytest.mark.gpu

SENTINEL = 0xAB
GUARD = 64
u32p = C.POINTER(C.c_uint32)


def to_device(arr, offset=0):
    """A device byte buffer holding `arr` at `offset` (the start 16-byte aligned), and the pointer to it."""
    import torch
    raw = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
    buf = torch.full((offset + len(raw) + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
    buf[offset:offset + len(raw)] = torch.from_numpy(raw.copy()).cuda()
    return buf, buf.data_ptr() + offset


def delta(ctx, rt, n, rs_std, rs_mt6, base, base_of=None, cap=None, base_offset=0):
    """The device stage over the batch's planes against `base` [n_base, P] cells (host), uploaded `base_offset` bytes
    into a buffer.  Returns (job summaries, records written, total); the bytes after the record buffer are checked."""
    import torch
    P = rt.n_prefixes
    cap = n * P if cap is None else cap
    base_buf, base_ptr = to_device(base, base_offset)
    bo = to_device(np.asarray(base_of, np.uint32))[0] if base_of is not None else None
    job_out = torch.full((n * DELTA_JOB_DT.itemsize,), SENTINEL, dtype=torch.uint8, device="cuda")
    records = torch.full((cap * DELTA_DT.itemsize + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
    total = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    args = (base_ptr, len(base), bo.data_ptr() if bo is not None else 0, job_out.data_ptr(),
            records.data_ptr() if cap else 0, cap, total.data_ptr())
    if isinstance(rt, isis.RouteTable):
        isis.routes_delta_device(ctx, rt, n, rs_std, rs_mt6, *args)
    else:
        ospfv2.routes_delta_device(ctx, rt, n, rs_std, *args)
    ctx.sync()
    t = int(total.item())
    rec = records.cpu().numpy()
    w = min(t, cap) * DELTA_DT.itemsize
    assert (rec[w:] == SENTINEL).all()
    return (np.frombuffer(job_out.cpu().numpy().tobytes(), DELTA_JOB_DT),
            np.frombuffer(rec[:w].tobytes(), DELTA_DT), t)


def same(got, want):
    assert got[2] == want[2]
    assert got[0].tobytes() == want[0].tobytes()
    assert got[1].tobytes() == want[1].tobytes()


def case_delta(case, base, **kw):
    if case.kind == "isis":
        return delta(case.ctx, case.rt, case.n, case.tops[isis.TOPO_STD].rs, case.tops[isis.TOPO_MT6].rs, base, **kw)
    return delta(case.ctx, case.rt, case.n, case.tops[0].rs, None, base, **kw)


def perturbed(row):
    """A base row that differs from `row` in every way a cell can: metric, atom set, presence (both ways), winner,
    and for OSPF the last-hop atoms."""
    r = row.copy()
    r["metric"][::3] += 1
    r["nh_mask"][1::5] ^= 1
    r["flags"][2::7] ^= ospfv2.CELL_PRESENT
    r["winner"][3::11] += 1
    if "lasthop_mask" in r.dtype.names:
        r["lasthop_mask"][4::13] ^= 2
    return r


@pytest.fixture(scope="module", params=["ospfv2-wide", "ospfv2-narrow", "ospfv3", "isis"])
def dcase(request, ctx, harnesses):  # noqa: F811
    """A Case with its cells from the existing kernel and two base rows: row 0 a perturbed copy of job 0's cells (so
    every kind of change occurs, whatever the jobs do), row 1 job 0's own cells."""
    c = Case(ctx, request.param, harnesses)
    c.cells = c.launch()[0]
    c.base = np.stack([perturbed(c.cells[0]), c.cells[0]])
    return c


def test_partial_last_tile_against_job_zero(dcase):
    assert (dcase.n * dcase.rt.n_prefixes) % 32
    base = dcase.base[:1]
    want = reference(dcase.cells, base)
    assert want[0]["n_lost"].sum() + want[0]["n_gained"].sum() > 0
    assert all(want[0][k].sum() > 0 for k in ("n_metric", "n_nexthops", "n_other"))
    same(case_delta(dcase, base), want)
    same(case_delta(dcase, base, base_of=np.zeros(dcase.n)), want)        # base_of all 0 == NULL


@pytest.mark.parametrize("offset", [8, 24])
def test_misaligned_base_cells(dcase, offset):
    base = dcase.base
    bo = np.arange(dcase.n) % 2
    same(case_delta(dcase, base, base_of=bo, base_offset=offset), reference(dcase.cells, base, bo))


def test_out_of_range_base_row(dcase):
    base = dcase.base
    bo = np.arange(dcase.n) % 3                                            # row 2 does not exist
    got = case_delta(dcase, base, base_of=bo)
    same(got, reference(dcase.cells, base, bo))
    assert (got[0]["status"][bo == 2] == capi.JS_INVALID).all()


def test_capacity(dcase):
    base = dcase.base[:1]
    total = reference(dcase.cells, base)[2]
    for cap in sorted({0, 1, total // 2, total}):
        got = case_delta(dcase, base, cap=cap)
        same(got, reference(dcase.cells, base, cap=cap))
        assert len(got[1]) == min(cap, total)


def test_two_launches_give_identical_bytes(dcase):
    base = dcase.base[:1]
    a, b = case_delta(dcase, base), case_delta(dcase, base)
    same(a, b)


def test_refused_jobs(dcase):
    """A status word set in either topology (by turns for IS-IS): the summary carries it, no records."""
    refuse = (1, 3)
    poked = [(dcase.tops[i % len(dcase.tops)], j) for i, j in enumerate(refuse)]
    import torch
    torch.cuda.synchronize()
    for d, j in poked:
        d.status[j] = 2
    try:
        got = case_delta(dcase, dcase.base[:1])
    finally:
        for d, j in poked:
            d.status[j] = 0
    status = np.zeros(dcase.n, np.uint32)
    status[list(refuse)] = 2
    same(got, reference(dcase.cells, dcase.base[:1], status=status))
    assert not np.isin(got[1]["job"], refuse).any()


def test_argument_checks(dcase):
    import torch
    job_out = torch.zeros(dcase.n * 32, dtype=torch.uint8, device="cuda")
    total = torch.zeros(1, dtype=torch.int64, device="cuda")
    base, ptr = to_device(dcase.cells[:1])
    rs = dcase.tops[0].rs
    for args in ((ptr, 0, 0, job_out.data_ptr(), 0, 0, total.data_ptr()),       # n_base 0
                 (ptr, 1, 0, 0, 0, 0, total.data_ptr()),                          # no job_out
                 (ptr + 4, 1, 0, job_out.data_ptr(), 0, 0, total.data_ptr())):    # base not 8-byte aligned
        with pytest.raises(capi.HspfError) as e:
            if dcase.kind == "isis":
                isis.routes_delta_device(dcase.ctx, dcase.rt, dcase.n, rs, dcase.tops[isis.TOPO_MT6].rs, *args)
            else:
                ospfv2.routes_delta_device(dcase.ctx, dcase.rt, dcase.n, rs, *args)
        assert e.value.code == capi.HSPF_E_INVAL


def test_several_roots_in_one_batch(ctx, harnesses):  # noqa: F811
    """OSPFv2: jobs of three roots interleaved, each compared with its own root's plain SPT through base_of."""
    import torch
    t = synth.random_topology(150, 600, synth.SEED_BASE + 63, cost_choices=[5, 10], lan_fraction=0.1)
    area = ospfv2.synth_area(t, root=2, sr=True)
    flat = ospfv2.Flat(area)
    rt = ospfv2.RouteTable(flat)
    rt.upload(ctx)
    csr = flat.csr
    roots = [v for v in range(csr.n_vertices) if flat.is_router[v] and 2 <= capi.atom_count(csr, v) <= 64][:3]
    P, E = rt.n_prefixes, csr.n_edges
    n = next(k for k in range(20, 60) if (k * P) % 32)
    ov = [[((31 * j) % E, capi.COST_DISABLED if j % 2 else 40)] for j in range(n)]

    def topo(rs_roots, overrides):
        d = DeviceTopology(ctx, csr, rs_roots[0], len(rs_roots), overrides)
        d.keep[0] = torch.tensor(np.asarray(rs_roots, np.int32), device="cuda")
        d.js.roots = C.cast(d.keep[0].data_ptr(), u32p)
        d.run()
        ctx.sync()
        assert not d.status.any().item()
        return d

    def cells_of(d, k):
        buf = torch.zeros(k * P * 24, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        ospfv2.routes_batch_device(ctx, rt, k, d.rs, buf.data_ptr())
        ctx.sync()
        return np.frombuffer(buf.cpu().numpy().tobytes(), ospfv2.CELL_DT).reshape(k, P)

    base_of = np.arange(n) % 3
    jobs = topo([roots[b] for b in base_of], ov)
    base = cells_of(topo(roots, None), 3)
    cells = cells_of(jobs, n)
    got = delta(ctx, rt, n, jobs.rs, None, base, base_of=base_of)
    same(got, reference(cells, base, base_of))
    assert got[2] > 0
    assert reference(cells, base)[2] != got[2]            # every job against row 0 is another answer


# ---- the c3_small IS-IS batch and the route-level tie ------------------------------------------------------------
@pytest.fixture(scope="module")
def isis_whatif(ctx, c3_small):  # noqa: F811
    """2 000 systems, 256 jobs each removing one adjacency (job 0 removes none); the base row is the plain SPT."""
    t, inst, adj = c3_small
    n = 256
    ov = [[]] + [[(ab, capi.COST_DISABLED), (ba, capi.COST_DISABLED)] for (_a, _b, ab, ba) in
                 (adj[(7 * j) % len(adj)] for j in range(1, n))]
    rt = isis.RouteTable(inst)
    rt.upload(ctx)
    cells, tops = device_cells(ctx, inst, rt, n, ov)
    return inst, rt, cells, tops, ov


def test_c3_small_isis_batch(ctx, isis_whatif):
    inst, rt, cells, tops, _ = isis_whatif
    got = delta(ctx, rt, len(cells), tops[isis.TOPO_STD].rs, None, cells[:1])
    same(got, reference(cells, cells[:1]))
    assert got[2] > 0 and (got[0]["n_changed"] > 0).sum() > 50
    summary = delta(ctx, rt, len(cells), tops[isis.TOPO_STD].rs, None, cells[:1], cap=0)
    assert summary[0].tobytes() == got[0].tobytes() and summary[2] == got[2]


def prefix_index(rt, routes, key):
    index = {k: i for i, k in enumerate(key(rt))}
    return np.array([index[k] for k in key(routes)], np.int64)


def isis_keys(x):
    if isinstance(x, isis.RouteTable):
        return [(bytes(p["bytes"]), int(p["is_v6"]), int(n)) for p, n in zip(x.prefix, x.len)]
    return [(bytes(r["prefix"]["bytes"]), int(r["prefix"]["is_v6"]), int(r["len"])) for r in x]


def check_tie(records, j, base_rows, job_rows):
    """records of job j == the prefixes present in one table and not the other (LOST / GAINED) and those whose
    metric differs (METRIC).  *_rows: {prefix index: metric}."""
    r = records[records["job"] == j]
    lost = set(r["prefix"][r["kind"] == DELTA_LOST].tolist())
    gained = set(r["prefix"][r["kind"] == DELTA_GAINED].tolist())
    metric = set(r["prefix"][(r["kind"] & DELTA_METRIC) != 0].tolist())
    assert lost == set(base_rows) - set(job_rows)
    assert gained == set(job_rows) - set(base_rows)
    assert metric == {p for p in set(base_rows) & set(job_rows) if base_rows[p] != job_rows[p]}
    return set(r["prefix"].tolist())


def test_isis_records_match_decoded_tables(ctx, isis_whatif):
    inst, rt, cells, tops, ov = isis_whatif
    _, records, _ = delta(ctx, rt, len(cells), tops[isis.TOPO_STD].rs, None, cells[:1])
    base_planes = job_planes(tops, 0)
    base_rib = decode(inst, rt, cells[0], base_planes)
    assert base_rib.rc == capi.HSPF_OK
    _, base_installed = isis.rib_diff(None, base_rib)
    base_rib_i = isis.IsisRib(base_installed, base_rib.nexthops, base_rib.rc)
    base_rows = dict(zip(prefix_index(rt, base_rib.routes, isis_keys).tolist(), base_rib.routes["metric"].tolist()))
    f = topology_flat(inst, isis.MT_STANDARD)
    root = rt.root[isis.TOPO_STD]
    nbrs = np.unique(f.csr.col[f.csr.row_ptr[root]:f.csr.row_ptr[root + 1]])
    checked = diffed = 0
    for j in range(1, len(cells), 5):
        planes = job_planes(tops, j)
        rib = decode(inst, rt, cells[j], planes, {isis.TOPO_STD: ov[j]})
        if rib.rc != capi.HSPF_OK:
            continue
        rows = dict(zip(prefix_index(rt, rib.routes, isis_keys).tolist(), rib.routes["metric"].tolist()))
        reported = check_tie(records, j, base_rows, rows)
        checked += 1
        d, h, _ = planes[isis.TOPO_STD]
        bd, bh, _ = base_planes[isis.TOPO_STD]
        if (d[nbrs] == bd[nbrs]).all() and (h[nbrs] == bh[nbrs]).all():
            acts, _ = isis.rib_diff(base_rib_i, rib)
            touched = set()
            for a in acts:
                src = base_rib.routes if a["kind"] == 3 else rib.routes
                touched.add(int(prefix_index(rt, src[int(a["route"]):int(a["route"]) + 1], isis_keys)[0]))
            assert touched <= reported, j
            diffed += 1
    assert checked >= 45 and diffed >= 30


def test_ospfv2_records_match_decoded_tables(ctx, harnesses):  # noqa: F811
    """OSPFv2 what-if batch of the local root: the records against the decoded tables of each job."""
    import torch
    t = synth.random_topology(200, 800, synth.SEED_BASE + 65, cost_choices=[5, 10], lan_fraction=0.1)
    area = ospfv2.synth_area(t, root=0, sr=True)
    flat = ospfv2.Flat(area)
    rt = ospfv2.RouteTable(flat)
    rt.upload(ctx)
    csr = flat.csr
    rv = flat.router_vertex(area.router_id)
    P, E, n = rt.n_prefixes, csr.n_edges, 64
    ov = [[]] + [[((53 * j) % E, capi.COST_DISABLED if j % 2 else 45)] for j in range(1, n)]
    d = DeviceTopology(ctx, csr, rv, n, ov)
    d.run()
    ctx.sync()
    buf = torch.zeros(n * P * 24, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ospfv2.routes_batch_device(ctx, rt, n, d.rs, buf.data_ptr())
    ctx.sync()
    cells = np.frombuffer(buf.cpu().numpy().tobytes(), ospfv2.CELL_DT).reshape(n, P)
    got = delta(ctx, rt, n, d.rs, None, cells[:1])
    same(got, reference(cells, cells[:1]))
    key = lambda x: (list(zip(x.prefix.tolist(), x.plen.tolist())) if isinstance(x, ospfv2.RouteTable) else
                     [(int(r["prefix"]), bin(int(r["mask"])).count("1")) for r in x])

    def table(j):
        planes = d.planes(j)
        gv, gn = gather_for(flat, rv, planes)
        res = ospfv2.routes_from_cells(area, rt, cells[j], gv, gn)
        if res.rc != capi.HSPF_OK:
            return None
        return dict(zip(prefix_index(rt, res.routes, key).tolist(), res.routes["metric"].tolist()))

    base_rows = table(0)
    assert base_rows is not None
    checked = 0
    for j in range(1, n):
        rows = table(j)
        if rows is None:
            continue
        check_tie(got[1], j, base_rows, rows)
        checked += 1
    assert checked > n // 2
