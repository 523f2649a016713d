"""GPU: the route-delta stage over OSPFv2 routing-table cells (hspf_ospfv2_rib_delta[16]).  The SPT planes are written
on the device; every case compares the device summaries, records and total byte for byte with the numpy reference of
tests/test_ospf_rib_delta.py, applied to the cells hspf_ospfv2_rib_cells stores over the same device planes.  The
route-level test decodes base and job tables on the host and ties the records to them."""
import numpy as np
import pytest

from holo_b200 import capi, ospf_rib, ospfv2, synth
from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
from test_ospf_rib_cells import view
from test_ospf_rib_cells_gpu import KW, Batch, dev_u32, small  # noqa: F401
from test_ospf_rib_delta import perturbed, reference, tie, whatif_overrides
from test_route_delta_gpu import GUARD, SENTINEL, same, to_device

pytestmark = pytest.mark.gpu


def rib_delta(b, base, base_of=None, cap=None, base_offset=0, roots=None, refuse=()):
    """The device stage over batch b's planes against `base` [n_base, P] cells (host), uploaded `base_offset` bytes into
    a buffer; roots: the call's root array (default: the batch's); refuse: jobs whose status word is set for this call.
    Returns (job summaries, records written, total); the bytes after the record buffer are checked."""
    import torch
    n, P = b.n, b.rt.n_prefixes
    cap = n * P if cap is None else cap
    _base_buf, base_ptr = to_device(base, base_offset)
    bo = to_device(np.asarray(base_of, np.uint32))[0] if base_of is not None else None
    d_roots = b.d_roots if roots is None else dev_u32(roots)
    job_out = torch.full((n * DELTA_JOB_DT.itemsize,), SENTINEL, dtype=torch.uint8, device="cuda")
    records = torch.full((cap * DELTA_DT.itemsize + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
    total = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    for j in refuse:
        b.top.status[j] = 2
    torch.cuda.synchronize()
    try:
        ospf_rib.rib_delta_device(b.ctx, b.rt, n, b.top.rs, d_roots.data_ptr(), base_ptr, len(base),
                                  bo.data_ptr() if bo is not None else 0, job_out.data_ptr(),
                                  records.data_ptr() if cap else 0, cap, total.data_ptr())
        b.ctx.sync()
    finally:
        for j in refuse:
            b.top.status[j] = 0
    t = int(total.item())
    rec = records.cpu().numpy()
    w = min(t, cap) * DELTA_DT.itemsize
    assert (rec[w:] == SENTINEL).all()
    return (np.frombuffer(job_out.cpu().numpy().tobytes(), DELTA_JOB_DT),
            np.frombuffer(rec[:w].tobytes(), DELTA_DT), t)


@pytest.fixture(scope="module")
def cells(small):  # noqa: F811
    """The small batch's device cells and cell-kernel status words, and two base rows: row 0 a perturbed copy of job 0's
    cells (every kind of change occurs), row 1 job 0's own cells."""
    c, st, _ = small.launch()
    return c, st, np.stack([perturbed(c[0]), c[0]])


def test_partial_last_tile_against_a_perturbed_row(small, cells):  # noqa: F811
    c, st, base = cells
    assert (small.n * small.rt.n_prefixes) % 32
    want = reference(c, base[:1], status=st)
    assert all(want[0][k].sum() > 0 for k in ("n_lost", "n_gained", "n_metric", "n_nexthops", "n_other"))
    same(rib_delta(small, base[:1]), want)
    same(rib_delta(small, base[:1], base_of=np.zeros(small.n)), want)          # base_of all 0 == NULL


@pytest.mark.parametrize("offset", [8, 24])
def test_misaligned_base_cells(small, cells, offset):  # noqa: F811
    c, st, base = cells
    bo = np.arange(small.n) % 2
    same(rib_delta(small, base, base_of=bo, base_offset=offset), reference(c, base, bo, st))


def test_out_of_range_base_row(small, cells):  # noqa: F811
    c, st, base = cells
    bo = np.arange(small.n) % 3                                                # row 2 does not exist
    got = rib_delta(small, base, base_of=bo)
    same(got, reference(c, base, bo, st))
    assert (got[0]["status"][bo == 2] == capi.JS_INVALID).all()


def test_capacity(small, cells):  # noqa: F811
    c, st, base = cells
    total = reference(c, base[:1], status=st)[2]
    for cap in sorted({0, 1, total // 2, total}):
        got = rib_delta(small, base[:1], cap=cap)
        same(got, reference(c, base[:1], status=st, cap=cap))
        assert len(got[1]) == min(cap, total)


def test_two_launches_give_identical_bytes(small, cells):  # noqa: F811
    base = cells[2][:1]
    same(rib_delta(small, base), rib_delta(small, base))


def test_refused_jobs(small, cells):  # noqa: F811
    """A status word, roots out of range and the batch's ABR roots: the summary carries what the cell kernel's
    job_status_out holds, and the job has no records."""
    base = cells[2][:1]
    roots = list(small.roots)
    roots[4], roots[5] = small.top.V, small.top.V + 1000
    c, st, _ = small.launch(roots=roots, refuse=(1, 2))
    got = rib_delta(small, base, roots=roots, refuse=(1, 2))
    assert got[0]["status"].tolist() == st.tolist()
    refused = np.nonzero(st)[0]
    assert {1, 2, 4, 5, 6, 7} <= set(refused.tolist()) and (st[[6, 7]] == ospf_rib.JS_NOT_INTERNAL).all()
    assert not np.isin(got[1]["job"], refused).any() and not got[0]["n_changed"][refused].any()
    same(got, reference(c, base, status=st))


def test_argument_checks(small, cells):  # noqa: F811
    import torch
    job_out = torch.zeros(small.n * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device="cuda")
    total = torch.zeros(1, dtype=torch.int64, device="cuda")
    _buf, ptr = to_device(cells[2][:1])
    roots = small.d_roots.data_ptr()
    for args in ((roots, ptr, 0, 0, job_out.data_ptr(), 0, 0, total.data_ptr()),        # n_base 0
                 (roots, ptr, 1, 0, 0, 0, 0, total.data_ptr()),                           # no job_out
                 (roots, ptr + 4, 1, 0, job_out.data_ptr(), 0, 0, total.data_ptr()),      # base not 8-byte aligned
                 (0, ptr, 1, 0, job_out.data_ptr(), 0, 0, total.data_ptr())):             # no roots
        with pytest.raises(capi.HspfError) as e:
            ospf_rib.rib_delta_device(small.ctx, small.rt, small.n, small.top.rs, *args)
        assert e.value.code == capi.HSPF_E_INVAL
    # no jobs: no roots needed, the total is zeroed
    ospf_rib.rib_delta_device(small.ctx, small.rt, 0, small.top.rs, 0, ptr, 1, 0, job_out.data_ptr(), 0, 0,
                              total.data_ptr())
    small.ctx.sync()
    assert int(total.item()) == 0


def small_overrides(small):  # noqa: F811
    """The overrides test_ospf_rib_cells_gpu's `small` fixture gives its jobs."""
    E = small.flat.csr.n_edges
    return [[]] * 3 + [[((97 * j) % E, capi.COST_DISABLED)] for j in range(3, small.n)]


@pytest.mark.parametrize("small", ["wide"], indirect=True)
def test_wide_and_narrow_planes_agree(ctx, small, cells):  # noqa: F811
    assert not small.narrow
    other = Batch(ctx, small.t, small.seed, small.roots, small_overrides(small), narrow=True)
    base = cells[2]
    bo = np.arange(small.n) % 2
    same(rib_delta(other, base, base_of=bo), rib_delta(small, base, base_of=bo))


def test_several_roots_in_one_batch(ctx, small):  # noqa: F811
    """Jobs of three internal roots interleaved, each compared with its own root's plain job through base_of."""
    roots = [r for r, s in zip(small.roots[:6], small.launch()[1][:6]) if not s][:3]
    assert len(roots) == 3 and len(set(roots)) == 3
    n = small.n
    base_of = np.arange(n) % 3
    E = small.flat.csr.n_edges
    jobs = Batch(ctx, small.t, small.seed, [roots[b] for b in base_of],
                 [[((31 * j) % E, capi.COST_DISABLED if j % 2 else 40)] for j in range(n)], narrow=small.narrow)
    plain = Batch(ctx, small.t, small.seed, roots, None, narrow=small.narrow)
    base = plain.launch()[0]
    c, st, _ = jobs.launch()
    got = rib_delta(jobs, base, base_of=base_of)
    same(got, reference(c, base, base_of, st))
    assert got[2] > 0 and not st.any()
    assert reference(c, base, status=st)[2] != got[2]          # every job against row 0 is another answer


# ------------------------------------------------------------------------------ 2 000-router area
def test_records_match_decoded_tables_on_2000_routers(ctx):
    """A what-if batch of one internal root, each job disabling one link (or raising one cost): the device records
    name the prefixes whose presence or metric changed in the decoded tables, and every prefix update_global_rib
    touches while the root's transit networks keep their atoms."""
    t = synth.random_topology(2000, 8000, synth.SEED_BASE + 362, cost_choices=[10, 20], lan_fraction=0.05)
    area, _, _ = view(t, 0, 972, **KW)
    flat = ospfv2.Flat(area)
    rv = flat.router_vertex(area.router_id)
    n = 64
    b = Batch(ctx, t, 972, [rv] * n, whatif_overrides(flat, n, 7), **KW)
    c, st, _ = b.launch()
    assert not st.any()
    got = rib_delta(b, c[:1])
    same(got, reference(c, c[:1]))
    assert got[2] > 0 and (got[0]["n_changed"] > 0).sum() > n // 4
    summary = rib_delta(b, c[:1], cap=0)
    assert summary[0].tobytes() == got[0].tobytes() and summary[2] == got[2]
    planes = [b.planes(j) for j in range(n)]
    checked, diffed = tie(area, flat, b.rt, rv, c, planes, got[1], range(1, n))
    assert checked >= n // 2 and diffed >= n // 3
