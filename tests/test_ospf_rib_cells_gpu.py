"""GPU: the batched routing-table stage for roots attached to one area (hspf_ospfv2_rib_cells[16]).  The SPT planes are
written on the device and never leave it before the kernel reads them; the device cells must equal, byte for byte, the
CPU harness (the same walk compiled for the host) over those planes, and sampled jobs decode to what the host
stages (area_from_planes + update_rib_full) give over the same planes."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from holo_b200 import capi, ospf_rib, ospfv2, synth
from test_isis_route_cells_gpu import DeviceTopology
from test_ospf_rib_cells import host_rib, same_rib, view
from test_ospfv2_route_cells import gather_for

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
SENTINEL = 0xAB
GUARD = 64


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    out = tmp_path_factory.mktemp("harness") / "libospf_rib_cells_harness.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                    "-o", str(out), str(ROOT / "tests" / "native" / "ospf_rib_cells_harness.cc")], check=True)
    lib = C.CDLL(str(out))
    lib.harness_rib_cells.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 7
    return lib


def dev_u32(a):
    import torch
    return torch.tensor(np.asarray(a, np.uint32).view(np.int32), device="cuda")


class Batch:
    """A table on the device and a batch of jobs computed on the device: job j is rooted at roots[j] (set in the
    SPT batch's root array) with overrides[j]."""

    def __init__(self, ctx, t, seed, roots, overrides=None, narrow=False, **kw):
        import torch
        self.ctx, self.t, self.seed, self.kw, self.narrow = ctx, t, seed, kw, narrow
        self.area, self.sums, self.ext = view(t, 0, seed, **kw)
        self.flat = ospfv2.Flat(self.area)
        self.rt = ospf_rib.RibTable(self.flat, self.area.area_id, self.sums, self.ext)
        self.rt.upload(ctx)
        self.n, self.roots = len(roots), [int(r) for r in roots]
        self.top = DeviceTopology(ctx, self.flat.csr, self.roots[0], self.n, overrides, narrow)
        self.top.keep[0].copy_(dev_u32(self.roots))
        self.top.run()
        ctx.sync()
        self.d_roots = dev_u32(self.roots)
        torch.cuda.synchronize()

    def launch(self, offset=0, roots=None, refuse=(), gather=()):
        """The kernel over the batch's planes, cells `offset` bytes into a 16-byte aligned buffer with a guard after
        them.  roots: the kernel's root array (default: the batch's); refuse: jobs whose status word is set for this
        launch.  Returns (cells, status_out, gathered nh)."""
        import torch
        P, n = self.rt.n_prefixes, self.n
        nbytes = n * P * ospf_rib.RIB_CELL_DT.itemsize
        buf = torch.full((offset + nbytes + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
        assert buf.data_ptr() % 16 == 0
        for j in refuse:
            self.top.status[j] = 2
        d_roots = self.d_roots if roots is None else dev_u32(roots)
        st = torch.zeros(n, dtype=torch.int32, device="cuda")
        gj, gv = dev_u32([j for j, _ in gather] or [0]), dev_u32([v for _, v in gather] or [0])
        gnh = torch.zeros(max(len(gather), 1), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        ospf_rib.rib_cells_device(self.ctx, self.rt, n, self.top.rs, d_roots.data_ptr(), buf.data_ptr() + offset,
                                  st.data_ptr(), len(gather), gj.data_ptr(), gv.data_ptr(), gnh.data_ptr())
        self.ctx.sync()
        for j in refuse:
            self.top.status[j] = 0
        host = buf.cpu().numpy()
        assert (host[:offset] == SENTINEL).all() and (host[offset + nbytes:] == SENTINEL).all()
        cells = np.frombuffer(host[offset:offset + nbytes].tobytes(), ospf_rib.RIB_CELL_DT).reshape(n, P)
        return cells, st.cpu().numpy().view(np.uint32), gnh.cpu().numpy().view(np.uint64)[: len(gather)]

    def planes(self, j):
        return self.top.planes(j)

    def expected(self, harness, roots=None, status=None):
        roots = self.roots if roots is None else roots
        V = self.top.V
        pl = [self.planes(j) for j in range(self.n)]
        stack = [np.ascontiguousarray(np.stack([p[i] for p in pl])) for i in range(3)]
        st0 = self.top.status.cpu().numpy().view(np.uint32).copy() if status is None else np.asarray(status, np.uint32)
        cells = np.zeros((self.n, self.rt.n_prefixes), ospf_rib.RIB_CELL_DT)
        out = np.zeros(self.n, np.uint32)
        r = np.ascontiguousarray(roots, np.uint32)
        harness.harness_rib_cells(self.rt.handle, self.n, r.ctypes.data, st0.ctypes.data, stack[0].ctypes.data,
                                  stack[1].ctypes.data, stack[2].ctypes.data, cells.ctypes.data, out.ctypes.data)
        assert V == self.rt.flat.csr.n_vertices
        return cells, out

    def decode_and_check(self, j, root_index):
        """Job j (rooted at router `root_index` of the topology): the device cells decoded equal the host stages over
        the job's planes."""
        area, sums, ext = view(self.t, root_index, self.seed, **self.kw)
        flat = ospfv2.Flat(area)
        rv = flat.router_vertex(area.router_id)
        assert rv == self.roots[j]
        d, h, m = self.planes(j)
        cells, st, _ = self.launch()
        assert st[j] == 0
        gv, gn = gather_for(flat, rv, (d, h, m))
        got = ospf_rib.rib_from_cells(area, self.rt, cells[j], gv, gn)
        m4 = np.zeros((len(m), 4), np.uint64)
        m4[:, 0] = m
        want = host_rib(area, sums, ext, lambda csr, root, nhw: (d, h, m4[:, :nhw]))
        same_rib(got, want)
        return got


def router_vertices(flat):
    return [v for v in range(flat.csr.n_vertices) if flat.is_router[v]]


@pytest.fixture(scope="module", params=["wide", "narrow"])
def small(request, ctx):
    narrow = request.param == "narrow"
    t = synth.random_topology(150, 600, synth.SEED_BASE + 361, cost_choices=[5, 10], lan_fraction=0.1)
    area, _, _ = view(t, 0, 971)
    flat = ospfv2.Flat(area)
    fits = [v for v in router_vertices(flat) if capi.atom_count(flat.csr, v) <= 16]
    is_abr = lambda v: int(area.router_lsas["flags"][int(np.nonzero(area.router_lsas["adv_rtr"] == flat.ids[v])[0][0])]) & 1
    rv = [v for v in fits if not is_abr(v)][:40]
    rv = rv[:6] + [v for v in fits if is_abr(v)][:2] + rv[6:]           # jobs 6 and 7: ABR roots
    # the job count makes jobs * prefixes not a multiple of 32: a partial last warp tile
    P = ospf_rib.RibTable(flat, 1, *view(t, 0, 971)[1:]).n_prefixes
    n = next(k for k in range(20, 60) if (k * P) % 32)
    E = flat.csr.n_edges
    ov = [[]] * 3 + [[((97 * j) % E, capi.COST_DISABLED)] for j in range(3, n)]
    return Batch(ctx, t, 971, [rv[j % len(rv)] for j in range(n)], ov, narrow)


def test_partial_last_tile_and_status(small, harness):
    assert (small.n * small.rt.n_prefixes) % 32
    cells, st, _ = small.launch()
    want, want_st = small.expected(harness)
    assert st.tolist() == want_st.tolist()
    assert cells.tobytes() == want.tobytes()
    paths = set(ospf_rib.cell_path(cells[(ospf_rib.cell_flags(cells) & 1) != 0]).tolist())
    assert paths == {0, 1, 2, 3}
    assert (st == ospf_rib.JS_NOT_INTERNAL).any() and (st == 0).any()


@pytest.mark.parametrize("offset", [8, 24])
def test_misaligned_cell_buffer(small, offset):
    assert small.launch(offset)[0].tobytes() == small.launch()[0].tobytes()


def test_two_launches_give_identical_bytes(small):
    a, b = small.launch(), small.launch()
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


def test_refused_jobs(small, harness):
    V = small.top.V
    roots = list(small.roots)
    roots[4] = V                                                  # out of range
    roots[5] = V + 1000
    cells, st, _ = small.launch(roots=roots, refuse=(1, 2))
    status = small.top.status.cpu().numpy().view(np.uint32).copy()
    status[[1, 2]] = 2
    want, want_st = small.expected(harness, roots=roots, status=status)
    assert st.tolist() == want_st.tolist()
    assert st[1] & 2 and st[2] & 2 and st[4] == capi.JS_INVALID and st[5] == capi.JS_INVALID
    assert cells.tobytes() == want.tobytes()
    for j in (1, 2, 4, 5):
        assert (cells["winner"][j] == ospf_rib.NO_RECORD).all() and not cells["mpf"][j].any()


def test_gather(small):
    V = small.top.V
    pairs = [(j, v) for j in range(small.n) for v in (0, V // 2, V - 1)] + [(small.n, 0), (0, V)]
    _, _, got = small.launch(8, gather=pairs)
    want = [int(small.planes(j)[2][v]) if j < small.n and v < V else 0 for j, v in pairs]
    assert got.tolist() == want


def test_small_batch_decodes(small):
    """The jobs rooted at the batch's first routers, without overrides, decode to the host stages."""
    ids = small.flat.ids
    for j in range(3):
        root_index = int(ids[small.roots[j]]) - ospfv2.RID_BASE
        if small.launch()[1][j]:
            continue
        small.decode_and_check(j, root_index)


# ------------------------------------------------------------------------------ 2 000-router area
KW = dict(n_abr=6, n_asbr=6, n_inter=1500, n_ext=1000, n_overlap=300, n_fresh=600, n_ext_only=200)


def test_multi_root_batch_on_2000_routers(ctx, harness):
    t = synth.random_topology(2000, 8000, synth.SEED_BASE + 362, cost_choices=[10, 20], lan_fraction=0.05)
    area, _, _ = view(t, 0, 972, **KW)
    flat = ospfv2.Flat(area)
    roots = [flat.router_vertex(ospfv2.RID_BASE + i) for i in range(0, 2000, 31)]
    b = Batch(ctx, t, 972, roots, None, **KW)
    assert not b.top.status.any().item()
    cells, st, _ = b.launch()
    want, want_st = b.expected(harness)
    assert st.tolist() == want_st.tolist() and cells.tobytes() == want.tobytes()
    n_ok, paths = 0, set()
    for j in (0, 7, 21, len(roots) - 1):
        if st[j]:
            continue
        got = b.decode_and_check(j, int(flat.ids[roots[j]]) - ospfv2.RID_BASE)
        paths |= set(got.routes["path_type"].tolist())
        n_ok += 1
    assert n_ok >= 3 and paths == {0, 1, 2, 3}


def test_override_batch_on_2000_routers(ctx, harness):
    t = synth.random_topology(2000, 8000, synth.SEED_BASE + 362, cost_choices=[10, 20], lan_fraction=0.05)
    area, _, _ = view(t, 0, 972, **KW)
    flat = ospfv2.Flat(area)
    rv = flat.router_vertex(area.router_id)
    csr = flat.csr
    out = [e for e in range(csr.row_ptr[rv], csr.row_ptr[rv + 1])]
    ov = [[]] + [[(out[j % len(out)], capi.COST_DISABLED)] if j % 2 else [((53 * j) % csr.n_edges, 1)] for j in range(1, 48)]
    b = Batch(ctx, t, 972, [rv] * 48, ov, **KW)
    cells, st, _ = b.launch()
    want, want_st = b.expected(harness)
    assert st.tolist() == want_st.tolist() and cells.tobytes() == want.tobytes()
    assert len({cells[j].tobytes() for j in range(48)}) > 1
    for j in (0, 1, 2, 17):
        if not st[j]:
            b.decode_and_check(j, 0)
