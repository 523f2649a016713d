"""GPU: what IS-IS L1/L2 routers propagate into their L2 LSP (hspf_isis_l1_to_l2_cells[16], _delta[16]).  One SPT
batch per L1 topology runs on the device; a job picks one L1 row.  The device cells and summary words must equal,
byte for byte, the CPU harness (the same walk compiled for the host) over those planes; sampled jobs decode to
hspf_isis_l1_to_l2 over their planes; the delta equals the reference comparison of the stored cells."""
import numpy as np
import pytest

from holo_b200 import capi, isis
from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT, DELTA_NEXTHOPS
from test_isis_l1_to_l2_cells import cells_on_cpu, harness, host  # noqa: F401
from test_isis_l1l2_rib_cells import TOPOS, topology_flat
from test_isis_route_cells_gpu import DeviceTopology
from test_route_delta import reference

pytestmark = pytest.mark.gpu

SENTINEL = 0xAB
GUARD = 64
SUMM = [("10.2.0.0/16", None), ("10.1.0.5/32", None), ("10.1.0.9/32", 3)]


def dev_u32(a):
    import torch
    return torch.tensor(np.asarray(a, np.uint32).view(np.int32).reshape(-1), device="cuda")


class Batch:
    """A domain's tables on the device and one L1 batch per topology (row 0 unperturbed, the others disabling one
    adjacency each)."""

    def __init__(self, ctx, seed, n_rows=8, narrow=False, **kw):
        self.ctx, self.narrow = ctx, narrow
        self.v = v = isis.l1l2_view(seed, **kw)
        self.rib = isis.L1L2RibTable(v["l1"], v["l2"], v["cfg"])
        self.rib.upload(ctx)
        self.t = isis.L1ToL2Table(v["l1"], v["l2"], self.rib)
        self.t.upload(ctx)
        rng = np.random.default_rng(seed)
        self.n_rows = n_rows
        self.top, self.ov = [], []
        for tt, mt in TOPOS:
            if self.rib.root[0][tt] == isis.NO_ROOT:
                self.top.append(None)
                self.ov.append(None)
                continue
            f = topology_flat(v["l1"], mt)
            ov = [[]] + [[(int(e), capi.COST_DISABLED)] for e in rng.integers(0, f.csr.n_edges, n_rows - 1)]
            d = DeviceTopology(ctx, f.csr, self.rib.root[0][tt], n_rows, ov, narrow)
            d.run()
            self.top.append(d)
            self.ov.append(ov)
        ctx.sync()
        self.rows = np.arange(n_rows, dtype=np.uint32)

    def rs(self):
        return tuple(t.rs if t is not None else None for t in self.top)

    def host_planes(self, k):
        t = self.top[k]
        if t is None:
            return None
        d = t.dist.cpu().numpy().view(np.uint16 if self.narrow else np.uint32).reshape(t.n, t.V)
        h = t.hops.cpu().numpy().view(np.uint16).reshape(t.n, t.V)
        m = t.nh.cpu().numpy().view(np.uint16 if self.narrow else np.uint64).reshape(t.n, t.V)
        if self.narrow:        # the harness reads wide planes: widen, unreached stays unreached
            d = d.astype(np.uint32)
            d[d == 0xFFFF] = 0xFFFFFFFF
            m = m.astype(np.uint64)
        return d, h, m

    def job(self, r):
        out = []
        for k in range(2):
            p = self.host_planes(k)
            out.append(None if p is None else tuple(x[r] for x in p))
        return out

    def launch(self, rows=None, offset=0):
        import torch
        rows = self.rows if rows is None else np.asarray(rows, np.uint32)
        n, K, S = len(rows), self.t.n_keys, self.t.n_summaries
        nbytes = n * K * isis.CELL_DT.itemsize
        buf = torch.full((offset + nbytes + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
        words = torch.full((max(n * S, 1),), -1, dtype=torch.int64, device="cuda")
        st = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
        d_rows = dev_u32(rows)
        torch.cuda.synchronize()
        isis.l1_to_l2_cells_device(self.ctx, self.t, n, self.rs(), self.n_rows, d_rows.data_ptr(), words.data_ptr(),
                                   st.data_ptr(), buf.data_ptr() + offset)
        self.ctx.sync()
        host = buf.cpu().numpy()
        assert (host[:offset] == SENTINEL).all() and (host[offset + nbytes:] == SENTINEL).all()
        cells = host[offset: offset + nbytes].copy().view(isis.CELL_DT).reshape(n, K)
        return cells, words.cpu().numpy().view(np.uint64)[: n * S].reshape(n, S), st.cpu().numpy().view(np.uint32)[:n]

    def harness(self, harness, rows=None):
        rows = self.rows if rows is None else rows
        return cells_on_cpu(harness, self.t, [self.job(r) for r in rows])


@pytest.mark.parametrize("narrow", [False, True])
@pytest.mark.parametrize("mt6", [False, True])
def test_device_cells_and_words_equal_harness(ctx, harness, narrow, mt6):
    b = Batch(ctx, 51, narrow=narrow, n_l1=60, n_l2=40, mt6=mt6, l1_degree=2, cost_choices=[5, 10],
              summaries=SUMM + ([("2001:db8:1::4/128", None)] if mt6 else []))
    cells, words, st = b.launch(offset=8)
    want, wwords = b.harness(harness)
    assert not st.any()
    assert cells.tobytes() == want.tobytes() and words.tobytes() == wwords.tobytes()
    assert (words >> np.uint64(32) == 1).any() and (cells["winner"] >= b.t.n_records).any()
    again = b.launch(offset=8)
    assert again[0].tobytes() == cells.tobytes() and again[1].tobytes() == words.tobytes()   # repeat launches
    m = next(m for m in range(len(b.rows), 0, -1) if (m * b.t.n_keys) % 32)                 # a partial warp tile
    part = b.launch(rows=b.rows[:m])
    assert part[0].tobytes() == want[:m].tobytes() and part[1].tobytes() == wwords[:m].tobytes()


def test_refused_jobs_and_rows_out_of_range(ctx, harness):
    import torch
    b = Batch(ctx, 52, n_l1=50, n_l2=30, summaries=SUMM)
    b.top[0].status[2] = 1                           # L1 row 2 refused by its planes
    torch.cuda.synchronize()
    rows = np.asarray([0, 2, 1, b.n_rows, 3], np.uint32)
    cells, words, st = b.launch(rows=rows)
    assert list(st) == [0, 1, 0, capi.JS_INVALID, 0]
    want, wwords = b.harness(harness, rows=rows[[0, 2, 4]])
    assert cells[[0, 2, 4]].tobytes() == want.tobytes() and words[[0, 2, 4]].tobytes() == wwords.tobytes()
    for j in (1, 3):
        assert not cells[j]["flags"].any() and (cells[j]["winner"] == 0xFFFFFFFF).all() and not words[j].any()
    b.top[0].status[2] = 0


@pytest.mark.parametrize("narrow", [False, True])
def test_sampled_jobs_decode_to_the_host_function(ctx, harness, narrow):
    b = Batch(ctx, 53, narrow=narrow, n_l1=50, n_l2=30, mt6=True, l1_degree=2, summaries=SUMM)
    cells, words, st = b.launch()
    v = b.v
    for j in (0, 1, len(b.rows) // 2, len(b.rows) - 1):
        planes = b.job(j)
        ovs = [b.ov[k][j] if b.ov[k] is not None else [] for k in range(2)]
        got = isis.l1_to_l2_from_cells(v["l1"], b.t, cells[j], words[j])
        want = host(v["l1"], v["l2"], b.t, planes, ovs, v["cfg"], None)
        assert got.tobytes() == want.tobytes(), j


def test_delta_equals_comparison_of_stored_cells(ctx, harness):
    import torch
    b = Batch(ctx, 54, n_rows=24, n_l1=60, n_l2=30, l1_degree=2, cost_choices=[5], summaries=SUMM)
    cells, words, st = b.launch()
    n, K, S = len(b.rows), b.t.n_keys, b.t.n_summaries
    base = cells[:2].copy()
    base_of = (np.arange(n) % 2).astype(np.uint32)
    base_of[-1] = 2                                  # out of range: HSPF_JS_INVALID, not compared
    d_base = torch.from_numpy(base.view(np.uint8).reshape(-1).copy()).cuda()
    d_of = dev_u32(base_of)
    d_rows = dev_u32(b.rows)
    for narrow in (False, True):
        nb = b if not narrow else Batch(ctx, 54, n_rows=24, narrow=True, n_l1=60, n_l2=30, l1_degree=2, cost_choices=[5],
                                        summaries=SUMM)
        for cap in (0, 7, n * K):
            job_out = torch.zeros(n * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device="cuda")
            recs = torch.zeros(max(cap, 1) * DELTA_DT.itemsize, dtype=torch.uint8, device="cuda")
            total = torch.zeros(1, dtype=torch.int64, device="cuda")
            w = torch.zeros(max(n * S, 1), dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            isis.l1_to_l2_delta_device(ctx, nb.t, n, nb.rs(), nb.n_rows, d_rows.data_ptr(), w.data_ptr(),
                                       d_base.data_ptr(), 2, d_of.data_ptr(), job_out.data_ptr(),
                                       recs.data_ptr() if cap else 0, cap, total.data_ptr())
            ctx.sync()
            jw, rw, tw = reference(cells, base, base_of, cap=cap)
            got_job = job_out.cpu().numpy().view(DELTA_JOB_DT)
            assert got_job.tobytes() == jw.tobytes()
            assert got_job[-1]["status"] == capi.JS_INVALID
            assert int(total.item()) == tw and tw > 0
            if cap:
                got = recs.cpu().numpy().view(DELTA_DT)[: min(cap, tw)]
                assert got.tobytes() == rw.tobytes()
                assert not (got["kind"] & DELTA_NEXTHOPS).any()
            assert w.cpu().numpy().view(np.uint64)[: n * S].reshape(n, S).tobytes() == words.tobytes()


@pytest.mark.parametrize("narrow", [False, True])
def test_argument_refusals_launch_nothing(ctx, narrow):
    import torch
    b = Batch(ctx, 55, narrow=narrow, n_l1=40, n_l2=30, summaries=SUMM)
    n, K, S = len(b.rows), b.t.n_keys, b.t.n_summaries
    cells = torch.zeros(n * K * 3, dtype=torch.int64, device="cuda")
    words = torch.zeros(n * S, dtype=torch.int64, device="cuda")
    rows = dev_u32(b.rows)
    base = torch.zeros(K * 3, dtype=torch.int64, device="cuda")
    jo = torch.zeros(n * 8, dtype=torch.int32, device="cuda")
    tot = torch.zeros(1, dtype=torch.int64, device="cuda")

    def cells_call(**kw):
        a = dict(n=n, l1=b.rs(), rows=rows.data_ptr(), words=words.data_ptr(), cells=cells.data_ptr())
        a.update(kw)
        isis.l1_to_l2_cells_device(ctx, b.t, a["n"], a["l1"], b.n_rows, a["rows"], a["words"], 0, a["cells"])

    def delta_call(**kw):
        a = dict(n=n, rows=rows.data_ptr(), words=words.data_ptr(), base=base.data_ptr(), n_base=1, jo=jo.data_ptr(),
                 tot=tot.data_ptr())
        a.update(kw)
        isis.l1_to_l2_delta_device(ctx, b.t, a["n"], b.rs(), b.n_rows, a["rows"], a["words"], a["base"], a["n_base"], 0,
                                   a["jo"], 0, 0, a["tot"])

    for call, kw in ((cells_call, dict(rows=0)), (cells_call, dict(words=0)), (cells_call, dict(cells=0)),
                     (cells_call, dict(words=words.data_ptr() + 4)), (cells_call, dict(l1=(None, None))),
                     (delta_call, dict(rows=0)), (delta_call, dict(words=0)), (delta_call, dict(base=0)),
                     (delta_call, dict(n_base=0)), (delta_call, dict(jo=0)), (delta_call, dict(tot=0)),
                     (delta_call, dict(base=base.data_ptr() + 4))):
        before = ctx.launch_count
        with pytest.raises(capi.HspfError) as e:
            call(**kw)
        assert e.value.code == capi.HSPF_E_INVAL and ctx.launch_count == before, kw
    # a rib table that was not uploaded
    rib = isis.L1L2RibTable(b.v["l1"], b.v["l2"], b.v["cfg"])
    t = isis.L1ToL2Table(b.v["l1"], b.v["l2"], rib)
    t.upload(ctx)
    before = ctx.launch_count
    with pytest.raises(capi.HspfError):
        isis.l1_to_l2_cells_device(ctx, t, n, b.rs(), b.n_rows, rows.data_ptr(), words.data_ptr(), 0, cells.data_ptr())
    assert ctx.launch_count == before
    cells_call(n=0)                                    # nothing to do
    delta_call(n=0)
    assert ctx.launch_count == before
    cells_call()
    assert ctx.launch_count == before + 2              # the summary pass and the cells
