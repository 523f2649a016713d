"""GPU: the routing table of IS-IS L1/L2 routers (hspf_isis_l1l2_rib_cells[16], _delta[16]).  One SPT batch per level
and topology runs on the device; a job picks one L1 row and one L2 row.  The device cells and summary words must
equal, byte for byte, the CPU harness (the same walk compiled for the host) over those planes; sampled jobs decode to
the host chain; the delta equals the reference comparison of the stored cells."""
import numpy as np
import pytest

from holo_b200 import capi, isis
from holo_b200.route_table import DELTA_DT, DELTA_JOB_DT
from test_isis_l1l2_rib_cells import (chain, cells_on_cpu, decode, harness, level_routes, same_rib,  # noqa: F401
                                      topology_flat, without)
from test_isis_route_cells_gpu import DeviceTopology
from test_route_delta import reference

pytestmark = pytest.mark.gpu

SENTINEL = 0xAB
GUARD = 64
TOPOS = ((isis.TOPO_STD, isis.MT_STANDARD), (isis.TOPO_MT6, isis.MT_IPV6))


def dev_u32(a):
    import torch
    return torch.tensor(np.asarray(a, np.uint32).view(np.int32).reshape(-1), device="cuda")


class L1L2Batch:
    """A domain's table on the device and one batch of rows per level (row 0 unperturbed, the others disabling one
    adjacency each), n_rows[0] L1 rows and n_rows[1] L2 rows."""

    def __init__(self, ctx, seed, n_rows=(5, 3), narrow=False, **kw):
        self.ctx, self.narrow = ctx, narrow
        self.v = v = isis.l1l2_view(seed, **kw)
        self.t = isis.L1L2RibTable(v["l1"], v["l2"], v["cfg"], v["l2_derived"])
        self.t.upload(ctx)
        rng = np.random.default_rng(seed)
        self.n_rows = list(n_rows)
        self.top, self.ov = [], []
        for l, inst in ((0, v["l1"]), (1, v["l2"])):
            for t, mt in TOPOS:
                if self.t.root[l][t] == isis.NO_ROOT:
                    self.top.append(None)
                    self.ov.append(None)
                    continue
                f = topology_flat(inst, mt)
                ov = [[]] + [[(int(e), capi.COST_DISABLED)] for e in rng.integers(0, f.csr.n_edges, n_rows[l] - 1)]
                d = DeviceTopology(ctx, f.csr, self.t.root[l][t], n_rows[l], ov, narrow)
                d.run()
                self.top.append(d)
                self.ov.append(ov)
        ctx.sync()
        jobs = [[a, b] for a in range(n_rows[0]) for b in range(n_rows[1])]
        self.rows = np.asarray(jobs, np.uint32)

    def rs(self, k):
        return self.top[k].rs if self.top[k] is not None else None

    def host_planes(self, k):
        t = self.top[k]
        if t is None:
            return None
        d = t.dist.cpu().numpy().view(np.uint16 if self.narrow else np.uint32).reshape(t.n, t.V)
        h = t.hops.cpu().numpy().view(np.uint16).reshape(t.n, t.V)
        m = t.nh.cpu().numpy().view(np.uint16 if self.narrow else np.uint64).reshape(t.n, t.V)
        if self.narrow:        # the harness reads wide planes: widen, unreached stays unreached
            d = np.where(d == 0xFFFF, 0xFFFFFFFF, d).astype(np.uint32)
            m = m.astype(np.uint64)
        return d, h, m

    def job(self, rows):
        """The four plane triples of the job with (L1 row, L2 row)."""
        out = []
        for k in range(4):
            p = self.host_planes(k)
            out.append(None if p is None else tuple(x[rows[k // 2]] for x in p))
        return out

    def launch(self, rows=None, offset=0):
        import torch
        rows = self.rows if rows is None else np.asarray(rows, np.uint32)
        n, P, S = rows.shape[0], self.t.n_prefixes, self.t.n_summaries
        nbytes = n * P * isis.CELL_DT.itemsize
        buf = torch.full((offset + nbytes + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
        words = torch.full((max(n * S, 1),), -1, dtype=torch.int64, device="cuda")
        st = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
        d_rows = dev_u32(rows)
        torch.cuda.synchronize()
        isis.l1l2_rib_cells_device(self.ctx, self.t, n, (self.rs(0), self.rs(1)), (self.rs(2), self.rs(3)), self.n_rows,
                                   d_rows.data_ptr(), words.data_ptr(), st.data_ptr(), buf.data_ptr() + offset)
        self.ctx.sync()
        host = buf.cpu().numpy()
        assert (host[:offset] == SENTINEL).all() and (host[offset + nbytes:] == SENTINEL).all()
        cells = host[offset: offset + nbytes].copy().view(isis.CELL_DT).reshape(n, P)
        return cells, words.cpu().numpy().view(np.uint64)[: n * S].reshape(n, S), st.cpu().numpy().view(np.uint32)[:n]

    def harness(self, harness, rows=None):
        rows = self.rows if rows is None else rows
        return cells_on_cpu(harness, self.t, [self.job(r) for r in rows])


@pytest.mark.parametrize("narrow", [False, True])
@pytest.mark.parametrize("mt6", [False, True])
def test_device_cells_and_words_equal_harness(ctx, harness, narrow, mt6):
    b = L1L2Batch(ctx, 21, narrow=narrow, n_l1=60, n_l2=50, mt6=mt6,
                  summaries=[("10.0.0.0/8", None), ("10.1.0.0/16", 9), ("10.2.0.0/16", None)]
                  + ([("2001:db8::/32", None)] if mt6 else []))
    cells, words, st = b.launch(offset=8)
    want, wwords = b.harness(harness)
    assert not st.any()
    assert cells.tobytes() == want.tobytes() and words.tobytes() == wwords.tobytes()
    assert (words >> np.uint64(32) == 1).any()
    again = b.launch(offset=8)
    assert again[0].tobytes() == cells.tobytes() and again[1].tobytes() == words.tobytes()   # repeat launches
    # L1 and L2 batches of different sizes, a batch ending in a partial warp tile
    m = next(m for m in range(len(b.rows), 0, -1) if (m * b.t.n_prefixes) % 32)
    part = b.launch(rows=b.rows[:m])
    assert part[0].tobytes() == want[:m].tobytes() and part[1].tobytes() == wwords[:m].tobytes()


def test_refused_jobs_and_rows_out_of_range(ctx, harness):
    import torch
    b = L1L2Batch(ctx, 22, n_l1=50, n_l2=40)
    b.top[0].status[2] = 1                           # L1 row 2 refused
    b.top[2].status[1] = 4                           # L2 row 1 refused
    torch.cuda.synchronize()
    rows = np.asarray([[0, 0], [2, 0], [0, 1], [1, 2], [5, 0], [0, 3]], np.uint32)
    cells, words, st = b.launch(rows=rows)
    assert list(st) == [0, 1, 4, 0, capi.JS_INVALID, capi.JS_INVALID]
    want, wwords = b.harness(harness, rows=rows[[0, 3]])
    assert cells[[0, 3]].tobytes() == want.tobytes() and words[[0, 3]].tobytes() == wwords.tobytes()
    for j in (1, 2, 4, 5):
        assert not (cells[j]["flags"]).any() and (cells[j]["winner"] == 0xFFFFFFFF).all() and not words[j].any()
    b.top[0].status[2] = 0
    b.top[2].status[1] = 0


def test_sampled_jobs_decode_to_the_host_chain(ctx, harness):
    b = L1L2Batch(ctx, 23, n_l1=50, n_l2=40, summaries=[("10.1.0.0/16", None), ("10.2.0.0/16", 20)])
    cells, words, st = b.launch()
    v = b.v
    for j in (0, 1, len(b.rows) // 2, len(b.rows) - 1):
        r = b.rows[j]
        planes = b.job(r)
        ovs = [b.ov[k][r[k // 2]] if b.ov[k] is not None else () for k in range(4)]
        got = decode(v["l1"], v["l2"], b.t, cells[j], words[j], planes, ovs)
        want, _ = chain(level_routes(v["l1"], ovs[0]), level_routes(without(v["l2"], v["l2_derived"]), ovs[2]), v["cfg"])
        same_rib(got, want)


def test_delta_equals_comparison_of_stored_cells(ctx, harness):
    import torch
    b = L1L2Batch(ctx, 24, n_l1=60, n_l2=50, summaries=[("10.1.0.0/16", None)])
    cells, words, st = b.launch()
    n, P, S = len(b.rows), b.t.n_prefixes, b.t.n_summaries
    base = cells[:2].copy()
    base_of = (np.arange(n) % 2).astype(np.uint32)
    d_base = torch.from_numpy(base.view(np.uint8).reshape(-1).copy()).cuda()
    d_of = dev_u32(base_of)
    for narrow in (False, True):
        nb = b if not narrow else L1L2Batch(ctx, 24, narrow=True, n_l1=60, n_l2=50, summaries=[("10.1.0.0/16", None)])
        for cap in (0, 7, n * P):
            job_out = torch.zeros(n * DELTA_JOB_DT.itemsize, dtype=torch.uint8, device="cuda")
            recs = torch.zeros(max(cap, 1) * DELTA_DT.itemsize, dtype=torch.uint8, device="cuda")
            total = torch.zeros(1, dtype=torch.int64, device="cuda")
            w = torch.zeros(n * S, dtype=torch.int64, device="cuda")
            d_rows = dev_u32(b.rows)
            torch.cuda.synchronize()
            isis.l1l2_rib_delta_device(ctx, nb.t, n, (nb.rs(0), nb.rs(1)), (nb.rs(2), nb.rs(3)), nb.n_rows,
                                       d_rows.data_ptr(), w.data_ptr(), d_base.data_ptr(), 2, d_of.data_ptr(),
                                       job_out.data_ptr(), recs.data_ptr() if cap else 0, cap, total.data_ptr())
            ctx.sync()
            jw, rw, tw = reference(cells, base, base_of, cap=cap)
            got_job = job_out.cpu().numpy().view(DELTA_JOB_DT)
            assert got_job.tobytes() == jw.tobytes()
            assert int(total.item()) == tw
            if cap:
                assert recs.cpu().numpy().view(DELTA_DT)[: min(cap, tw)].tobytes() == rw.tobytes()
            assert w.cpu().numpy().view(np.uint64).reshape(n, S).tobytes() == words.tobytes()


@pytest.mark.parametrize("narrow", [False, True])
def test_argument_refusals_launch_nothing(ctx, narrow):
    import torch
    b = L1L2Batch(ctx, 25, narrow=narrow, n_l1=40, n_l2=30, summaries=[("10.1.0.0/16", None)])
    n, P, S = len(b.rows), b.t.n_prefixes, b.t.n_summaries
    cells = torch.zeros(n * P * 3, dtype=torch.int64, device="cuda")
    words = torch.zeros(n * S, dtype=torch.int64, device="cuda")
    rows = dev_u32(b.rows)
    base = torch.zeros(P * 3, dtype=torch.int64, device="cuda")
    jo = torch.zeros(n * 8, dtype=torch.int32, device="cuda")
    tot = torch.zeros(1, dtype=torch.int64, device="cuda")
    l1, l2 = (b.rs(0), b.rs(1)), (b.rs(2), b.rs(3))

    def cells_call(**kw):
        a = dict(n=n, l1=l1, l2=l2, rows=rows.data_ptr(), words=words.data_ptr(), cells=cells.data_ptr())
        a.update(kw)
        isis.l1l2_rib_cells_device(ctx, b.t, a["n"], a["l1"], a["l2"], b.n_rows, a["rows"], a["words"], 0, a["cells"])

    def delta_call(**kw):
        a = dict(n=n, rows=rows.data_ptr(), words=words.data_ptr(), base=base.data_ptr(), n_base=1, jo=jo.data_ptr(),
                 tot=tot.data_ptr())
        a.update(kw)
        isis.l1l2_rib_delta_device(ctx, b.t, a["n"], l1, l2, b.n_rows, a["rows"], a["words"], a["base"], a["n_base"], 0,
                                   a["jo"], 0, 0, a["tot"])

    for call, kw in ((cells_call, dict(rows=0)), (cells_call, dict(words=0)), (cells_call, dict(cells=0)),
                     (cells_call, dict(words=words.data_ptr() + 4)), (cells_call, dict(l1=(None, None))),
                     (cells_call, dict(l1=(None, None), l2=(None, None))),
                     (delta_call, dict(rows=0)), (delta_call, dict(words=0)), (delta_call, dict(base=0)),
                     (delta_call, dict(n_base=0)), (delta_call, dict(jo=0)), (delta_call, dict(tot=0)),
                     (delta_call, dict(base=base.data_ptr() + 4))):
        before = ctx.launch_count
        with pytest.raises(capi.HspfError) as e:
            call(**kw)
        assert e.value.code == capi.HSPF_E_INVAL and ctx.launch_count == before, kw
    before = ctx.launch_count
    cells_call(n=0)                                    # nothing to do
    delta_call(n=0)
    assert ctx.launch_count == before
    cells_call()
    assert ctx.launch_count == before + 2              # the summary pass and the cells
