"""GPU: the route-delta stage (holo_b200/csrc/route_stage.cuh: launch_route_delta) past 2^32 cells per call and up to
its limit of 2^36 cells (include/holo_spf_lsdb.h, "Route-delta stage on the device"), over both cell layouts and both
grids of the shared launcher: hspf_ospfv2_abr_rib_delta[16] (routing-table cells, 4 blocks per SM) and
hspf_isis_l1l2_rib_delta[16] (IS-IS cells, 8 blocks per SM, behind the summary pass).  One job more than the limit is
refused before anything is enqueued, by those two and by hspf_isis_l1_to_l2_delta[16].

A job's cells depend only on its plane rows, so a batch of billions of cells is built from a few row combinations,
each given to many jobs by a seeded permutation: warp tiles straddle jobs of different combinations, and the last one
of them is refused (a row out of range).  The expected output is the numpy reference of the stage
(tests/test_ospf_rib_delta.py for routing-table cells, tests/test_route_delta.py for IS-IS cells) over the cells the
existing cell kernel writes for the combinations, computed once per (combination, base row) and expanded to every
job: the summaries by indexing, the total as a sum, the first `cap` records by expanding only the jobs they fall in.
test_expansion_equals_reference checks that expansion against the reference run on a small explicit batch, on the
CPU.  Each case keeps below ~4 GB of device memory (the record workspace is 9 bytes per warp tile: ~2.4 GB at 2^33
cells) and runs on a context of its own, closed at the end of the module."""
import time

import numpy as np
import pytest

import test_ospf_rib_delta as rib_delta
import test_route_delta as route_delta
from holo_b200 import capi, isis, ospf_rib
from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT, DELTA_LOST, DELTA_METRIC

MAX_CELLS = 1 << 36               # the most cells of one route-delta call (route_stage.cuh: kDeltaMaxCells)
SENTINEL = 0xAB
GUARD = 64
SEED = 0x5CA1E


# ---- the expected output of a batch made of a few combinations --------------------------------------------------
def reference(cells, base, base_of=None, status=None, cap=None):
    """The numpy reference of the stage for the cells' layout."""
    fn = rib_delta.reference if cells.dtype == ospf_rib.RIB_CELL_DT else route_delta.reference
    return fn(cells, base, base_of, status, cap)


class Expected:
    """The stage's output over a batch whose job j has the cells and status word of combination combo_of[j]
    (cells [C, P], status [C]) and base row base_of[j] of base [n_base, P]: the reference runs once per (combination,
    base row) pair that occurs, every row >= n_base being one pair."""

    def __init__(self, cells, status, base, combo_of, base_of):
        nb = len(base)
        key = combo_of.astype(np.int64) * (nb + 1) + np.minimum(base_of, nb)
        pairs, self.pair_of = np.unique(key, return_inverse=True)
        self.summ = np.zeros(len(pairs), DELTA_JOB_DT)
        self.recs, counts = [], np.zeros(len(pairs), np.int64)
        for i, k in enumerate(pairs):
            c, b = divmod(int(k), nb + 1)
            s, r, t = reference(cells[c:c + 1], base, base_of=[b], status=[int(status[c])])
            self.summ[i], counts[i] = s[0], t
            self.recs.append(r)
        self.per_job = counts[self.pair_of]
        self.total = int(self.per_job.sum())

    def summaries(self):
        return self.summ[self.pair_of]

    def records(self, cap):
        """The first min(total, cap) records, in (job, prefix) order: only the jobs they fall in are expanded."""
        jobs = np.nonzero(self.per_job)[0]
        k = int(np.searchsorted(np.cumsum(self.per_job[jobs]), cap)) + 1
        parts = []
        for j in jobs[:k]:
            r = self.recs[self.pair_of[j]].copy()
            r["job"] = j
            parts.append(r)
        return (np.concatenate(parts) if parts else np.zeros(0, DELTA_DT))[:cap]


def spread(n, n_combos, seed):
    """combo_of [n]: each combination to n / n_combos jobs, in a seeded order."""
    return (np.random.default_rng(seed).permutation(n) % n_combos).astype(np.uint32)


def raised(cells):
    """Base rows from cells: every prefix present, at a metric one above the cell's, so that every cell of a job
    that is compared is LOST (the job lacks the prefix) or METRIC."""
    r = cells.copy()
    if r.dtype == ospf_rib.RIB_CELL_DT:
        m = (ospf_rib.cell_metric(r) + 1) & rib_delta.METRIC_MAX
        r["mpf"] = (r["mpf"] & ~np.uint32(rib_delta.METRIC_MAX)) | m | np.uint32(rib_delta.PRESENT << 28)
    else:
        r["metric"] += np.uint32(1)
        r["flags"] |= isis.CELL_PRESENT
    return r


def perturbed(cells):
    """Base rows from cells that differ from them in every way a cell can (tests/test_*_delta*.py: perturbed)."""
    if cells.dtype == ospf_rib.RIB_CELL_DT:
        return np.stack([rib_delta.perturbed(c) for c in cells])
    from test_route_delta_gpu import perturbed as isis_perturbed
    return np.stack([isis_perturbed(c) for c in cells])


def random_cells(dt, shape, rng):
    """Cells whose fields take few values, so that every kind of change and no change all occur."""
    c = np.zeros(shape, dt)
    c["nh_mask"] = rng.integers(0, 3, shape)
    c["winner"] = rng.integers(0, 3, shape)
    flags = rng.choice([0, 1, 1, 3], shape)
    if dt == ospf_rib.RIB_CELL_DT:
        c["aux"] = rng.integers(0, 2, shape)
        c["mpf"] = rng.integers(0, 4, shape) | (rng.integers(0, 2, shape) << 26) | (flags << 28)
    else:
        c["metric"] = rng.choice([0, 1, 2, 0xFFFFFFFF], shape)
        c["flags"] = flags
    return c


@pytest.mark.parametrize("dt", [ospf_rib.RIB_CELL_DT, isis.CELL_DT], ids=["rib-cells", "isis-cells"])
def test_expansion_equals_reference(dt):
    """CPU: Expected over combinations equals the reference over the explicit batch, for every cap."""
    rng = np.random.default_rng(SEED)
    C, P, n = 4, 37, 90
    cells = random_cells(dt, (C, P), rng)
    status = np.array([0, 0, capi.JS_SATURATED, 0], np.uint32)
    base = np.concatenate([random_cells(dt, (2, P), rng), raised(cells[:1])])
    combo_of = spread(n, C, SEED)
    base_of = rng.integers(0, len(base) + 2, n).astype(np.uint32)           # some rows out of range
    exp = Expected(cells, status, base, combo_of, base_of)
    full = reference(cells[combo_of], base, base_of, status[combo_of])
    assert exp.total == full[2] and exp.total > 0
    assert exp.summaries().tobytes() == full[0].tobytes()
    assert set(full[0]["status"]) == {0, capi.JS_SATURATED, capi.JS_INVALID}
    for cap in sorted({0, 1, 2, 50, full[2] // 2, full[2] - 1, full[2], full[2] + 7}):
        assert exp.records(cap).tobytes() == full[1][:cap].tobytes(), cap
    raised_only = Expected(cells, status, raised(cells), combo_of, combo_of)
    compared = status[combo_of] == 0
    assert raised_only.total == P * compared.sum()
    s = raised_only.summaries()
    assert (s["n_changed"][compared] == P).all() and (s["n_lost"] + s["n_metric"] == s["n_changed"]).all()


# ---- the device stages -------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sctx(built):
    """A context of this module's own: its grow-only route-delta workspace is freed when the module ends."""
    c = capi.Context(0)
    yield c
    c.close()


@pytest.fixture(autouse=True)
def release_cache():
    yield
    try:
        import torch
        if torch.cuda.is_available():
            torch.cuda.empty_cache()
    except ImportError:
        pass


class Stage:
    """One delta entry point over a domain's tables and device planes.  combos [C, width]: plane rows, the last
    combination refused (a row out of range); cells [C, P], status [C] and (IS-IS) summary words [C, S] from the
    cell kernel; call(n, rows, words, base, n_base, base_of, job_out, records, cap, n_records) the delta over device
    pointers."""

    def __init__(self, ctx, kind, narrow):
        self.kind, self.narrow = kind, narrow
        if kind == "abr":
            from test_ospf_abr_rib_gpu import AbrBatch
            b = AbrBatch(ctx, 11, n_rows=4, narrow=narrow, V=600, E=2400)
            self.P, self.S = b.rt.n_prefixes, 0
            self.combos = np.array([[0, 0, 0], [1, 0, 0], [0, 2, 0], [0, 0, 3], [3, 1, 2], [b.n_rows[0], 0, 0]],
                                   np.uint32)
            self.cells, self.status, _ = b.launch(rows=self.combos)
            self.words = np.zeros((len(self.combos), 0), np.uint64)
            planes = [t.rs for t in b.top]
            self.call = lambda n, rows, words, *rest: ospf_rib.abr_rib_delta_device(ctx, b.rt, n, planes, b.n_rows, rows,
                                                                                     *rest)
        elif kind == "l1l2":
            from test_isis_l1l2_rib_gpu import L1L2Batch
            b = L1L2Batch(ctx, 12, n_rows=(4, 3), narrow=narrow, n_l1=4000, n_l2=300, summaries=[("10.1.0.0/28", None)])
            self.P, self.S = b.t.n_prefixes, b.t.n_summaries
            self.combos = np.array([[0, 0], [1, 0], [0, 1], [2, 2], [3, 1], [b.n_rows[0], 0]], np.uint32)
            self.cells, self.words, self.status = b.launch(rows=self.combos)
            l1, l2 = (b.rs(0), b.rs(1)), (b.rs(2), b.rs(3))
            self.call = lambda n, *rest: isis.l1l2_rib_delta_device(ctx, b.t, n, l1, l2, b.n_rows, *rest)
        else:
            from test_isis_l1_to_l2_gpu import Batch
            b = Batch(ctx, 13, n_rows=4, narrow=narrow, n_l1=4000, n_l2=300, summaries=[("10.1.0.0/28", None)])
            self.P, self.S = b.t.n_keys, b.t.n_summaries
            self.combos = np.array([[0]], np.uint32)
            self.call = lambda n, *rest: isis.l1_to_l2_delta_device(ctx, b.t, n, b.rs(), b.n_rows, *rest)
        self.batch = b
        assert self.P >= 3000 and self.P % 32, self.P
        assert kind == "l1_to_l2" or (self.status[-1] == capi.JS_INVALID and not self.status[:-1].any())


@pytest.fixture(scope="module")
def stages(sctx):
    made = {}

    def get(kind, narrow):
        if (kind, narrow) not in made:
            made[(kind, narrow)] = Stage(sctx, kind, narrow)
        return made[(kind, narrow)]
    return get


def run(ctx, st, combo_of, base, base_of, cap):
    """The device stage over len(combo_of) jobs, job j on the rows of combination combo_of[j] against row base_of[j]
    of base.  Returns (summaries, records written, total, summary words or None, seconds from the call to the end of
    a device synchronise); the record buffer past the records written still holds its sentinel bytes."""
    import torch
    n = len(combo_of)
    rows = torch.from_numpy(np.ascontiguousarray(st.combos[combo_of]).view(np.int32).reshape(-1)).cuda()
    d_base = torch.from_numpy(np.ascontiguousarray(base).view(np.uint8).reshape(-1).copy()).cuda()
    d_of = torch.from_numpy(np.ascontiguousarray(base_of, np.uint32).view(np.int32)).cuda()
    words = torch.full((max(n * st.S, 1),), -1, dtype=torch.int64, device="cuda")
    job_out = torch.full((n * DELTA_JOB_DT.itemsize,), SENTINEL, dtype=torch.uint8, device="cuda")
    records = torch.full((cap * DELTA_DT.itemsize + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
    total = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    st.call(n, rows.data_ptr(), words.data_ptr() if st.S else 0, d_base.data_ptr(), len(base), d_of.data_ptr(),
            job_out.data_ptr(), records.data_ptr() if cap else 0, cap, total.data_ptr())
    ctx.sync()
    secs = time.perf_counter() - t0
    del rows, d_base, d_of
    t = int(total.item())
    w = min(t, cap) * DELTA_DT.itemsize
    assert bool((records[w:] == SENTINEL).all())
    recs = np.frombuffer(records[:w].cpu().numpy().tobytes(), DELTA_DT)
    del records
    summ = job_out.cpu().numpy().view(DELTA_JOB_DT)
    del job_out
    wh = words.cpu().numpy().view(np.uint64)[: n * st.S].reshape(n, st.S) if st.S else None
    return summ, recs, t, wh, secs


def same_summaries(got, want):
    g, w = got.view(np.uint32).reshape(-1, 8), want.view(np.uint32).reshape(-1, 8)
    assert g.shape == w.shape
    bad = np.nonzero((g != w).any(axis=1))[0]
    assert not len(bad), f"{len(bad)} jobs differ, first {bad[0]}: got {got[bad[0]]}, want {want[bad[0]]}"


def check_words(st, combo_of, words):
    """IS-IS: the summary pass wrote each job its combination's words."""
    if st.S:
        bad = np.nonzero((words != st.words[combo_of]).any(axis=1))[0]
        assert not len(bad), f"{len(bad)} jobs' summary words differ, first {bad[0]}"


def jobs_above(cells, P):
    """The fewest jobs of P cells past `cells` cells whose last warp tile is partial."""
    n = cells // P + 1
    while (n * P) % 32 == 0:
        n += 1
    return n


STAGES = [("abr", False), ("abr", True), ("l1l2", False), ("l1l2", True)]
STAGE_IDS = ["abr_rib_delta", "abr_rib_delta16", "l1l2_rib_delta", "l1l2_rib_delta16"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,narrow", STAGES, ids=STAGE_IDS)
def test_every_cell_changed_past_2_32(sctx, stages, kind, narrow, record_property):
    """Just over 2^33 cells, each job against its combination's cells raised: every compared cell is a change, the
    total passes 2^32 (64-bit atomics, scan offsets past 2^32), and with cap 2^20 pass B stores the first tiles'
    records and skips the others."""
    st = stages(kind, narrow)
    n = jobs_above(1 << 33, st.P)
    combo_of = spread(n, len(st.combos), SEED + 1)
    base = raised(st.cells)
    cap = 1 << 20
    exp = Expected(st.cells, st.status, base, combo_of, combo_of)
    assert exp.total == st.P * int((st.status[combo_of] == 0).sum()) and exp.total > 1 << 32
    summ, recs, total, words, secs = run(sctx, st, combo_of, base, combo_of, cap)
    record_property("jobs", n)
    record_property("cells", n * st.P)
    record_property("delta_s", round(secs, 3))
    assert total == exp.total
    same_summaries(summ, exp.summaries())
    want = exp.records(cap)
    assert len(recs) == cap and recs.tobytes() == want.tobytes()
    assert np.isin(want["kind"], [DELTA_LOST, DELTA_METRIC]).all() and (want["kind"] == DELTA_METRIC).any()
    check_words(st, combo_of, words)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,narrow", STAGES, ids=STAGE_IDS)
def test_records_from_the_far_end(sctx, stages, kind, narrow, record_property):
    """The same size, each job against its own combination's cells (no change), except a dozen jobs whose cells lie
    past index 2^32: they get perturbed base rows, one of them a refused row and one a base row past n_base.  Every
    record is compared."""
    st = stages(kind, narrow)
    C, P = len(st.combos), st.P
    n = jobs_above(1 << 33, P)
    combo_of = spread(n, C, SEED + 2)
    first = -(-(1 << 32) // P)                                    # the first job whose cells start at 2^32 or later
    far = np.unique(np.linspace(first, n - 1, 12).astype(np.int64))
    assert len(far) == 12
    combo_of[far] = np.arange(len(far)) % (C - 1)                 # comparable combinations ...
    combo_of[far[7]] = C - 1                                      # ... but one refused
    base = np.concatenate([st.cells, perturbed(st.cells[combo_of[far]])])
    base_of = combo_of.copy()
    base_of[far] = C + np.arange(len(far))
    base_of[far[3]] = len(base)                                   # no such base row: HSPF_JS_INVALID
    exp = Expected(st.cells, st.status, base, combo_of, base_of)
    assert np.array_equal(np.nonzero(exp.per_job)[0], np.delete(far, [3, 7]))
    cap = exp.total + 5
    summ, recs, total, words, secs = run(sctx, st, combo_of, base, base_of, cap)
    record_property("jobs", n)
    record_property("delta_s", round(secs, 3))
    assert total == exp.total and len(recs) == total
    assert recs.tobytes() == exp.records(cap).tobytes()
    assert (recs["job"].astype(np.int64) * P + recs["prefix"] >= 1 << 32).all()
    same_summaries(summ, exp.summaries())
    assert summ[far[3]]["status"] == capi.JS_INVALID and summ[far[7]]["status"] == capi.JS_INVALID
    check_words(st, combo_of, words)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,narrow", [("abr", False), ("l1l2", True)], ids=["abr_rib_delta", "l1l2_rib_delta16"])
def test_the_largest_accepted_batch(sctx, stages, kind, narrow, record_property):
    """n_jobs = floor(2^36 / P), summaries only: each job against its combination's cells raised or perturbed (a
    seeded choice per job).  Every job's summary and the total are compared."""
    st = stages(kind, narrow)
    C, P = len(st.combos), st.P
    n = MAX_CELLS // P
    combo_of = spread(n, C, SEED + 3)
    base = np.concatenate([raised(st.cells), perturbed(st.cells)])
    base_of = combo_of + C * np.random.default_rng(SEED + 4).integers(0, 2, n).astype(np.uint32)
    exp = Expected(st.cells, st.status, base, combo_of, base_of)
    assert exp.total > 1 << 34
    summ, recs, total, words, secs = run(sctx, st, combo_of, base, base_of, 0)
    record_property("jobs", n)
    record_property("cells", n * P)
    record_property("delta_s", round(secs, 3))
    assert total == exp.total and len(recs) == 0
    same_summaries(summ, exp.summaries())
    check_words(st, combo_of, words)


@pytest.mark.gpu
@pytest.mark.parametrize("narrow", [False, True], ids=["wide", "16"])
@pytest.mark.parametrize("kind", ["abr", "l1l2", "l1_to_l2"])
def test_one_job_more_is_refused(sctx, stages, kind, narrow):
    """n_jobs = floor(2^36 / P) + 1: HSPF_E_INVAL, no launch (for IS-IS not even the summary pass), and job_out,
    n_records and the summary words keep their sentinel bytes.  Every buffer is sized for the whole batch and every
    row is valid, so a stage that accepted the call would run it to the end."""
    import torch
    st = stages(kind, narrow)
    n = MAX_CELLS // st.P + 1
    assert (n - 1) * st.P <= MAX_CELLS < n * st.P
    rows = torch.zeros(n * st.combos.shape[1], dtype=torch.int32, device="cuda")
    words = torch.full((max(n * st.S, 1) * 8,), SENTINEL, dtype=torch.uint8, device="cuda")
    base = torch.zeros(st.P * 24, dtype=torch.uint8, device="cuda")
    job_out = torch.full((n * DELTA_JOB_DT.itemsize,), SENTINEL, dtype=torch.uint8, device="cuda")
    total = torch.full((8,), SENTINEL, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    before = sctx.launch_count
    rc = capi.HSPF_OK
    try:
        st.call(n, rows.data_ptr(), words.data_ptr() if st.S else 0, base.data_ptr(), 1, 0, job_out.data_ptr(), 0, 0,
                total.data_ptr())
    except capi.HspfError as e:
        rc = e.code
    sctx.sync()
    assert (rc, sctx.launch_count - before) == (capi.HSPF_E_INVAL, 0)
    assert bool((job_out == SENTINEL).all()) and bool((total == SENTINEL).all()) and bool((words == SENTINEL).all())
