"""GPU: the warp-tiled cell store and the launch every route kernel shares (holo_b200/csrc/route_stage.cuh), for each
table type and plane width: OSPFv2 with wide and 16-bit planes, OSPFv3 through hspf_ospfv2_routes_batch, and IS-IS
over both topologies.  The SPT planes are written on the device and never leave it before the route kernel reads
them; every case compares the device cells with the CPU harness (the same walk compiled for the host) over those
planes."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from holo_b200 import capi, isis, ospfv2, ospfv3, synth
from test_isis_route_cells import mt6_instance, topology_flat
from test_isis_route_cells_gpu import DeviceTopology, harness_cells
from test_ospfv2_route_cells import cells_on_cpu

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
SENTINEL = 0xAB
GUARD = 64                 # bytes after the cells that the kernel must leave alone


@pytest.fixture(scope="module")
def harnesses(built, tmp_path_factory):
    """Both CPU harnesses (tests/native), compiled for this module in a temporary directory."""
    out = tmp_path_factory.mktemp("harness")
    libs = {}
    for name in ("route_cells_harness", "isis_route_cells_harness"):
        so = out / f"lib{name}.so"
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                        "-o", str(so), str(ROOT / "tests" / "native" / f"{name}.cc")], check=True)
        libs[name] = C.CDLL(str(so))
    ospf, isis_ = libs["route_cells_harness"], libs["isis_route_cells_harness"]
    ospf.harness_route_cells.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 4
    ospf.harness_route_cells16.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 4
    isis_.harness_isis_route_cells.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 7
    return {"ospf": ospf, "isis": isis_}


class Case:
    """One table type and plane width: the table on the device and a batch of jobs whose planes were computed on
    the device.  Job 0 is the plain SPT, job j > 0 disables one edge; the batch size makes jobs * prefixes not a
    multiple of 32, so the last warp tile is partial."""

    def __init__(self, ctx, kind, harnesses):
        self.ctx, self.kind, self.narrow = ctx, kind, kind == "ospfv2-narrow"
        t = synth.random_topology(150, 600, synth.SEED_BASE + 61, cost_choices=[5, 10], lan_fraction=0.1)
        if kind == "isis":
            inst = mt6_instance(t, 2)
            self.rt = isis.RouteTable(inst)
            assert isis.NO_ROOT not in self.rt.root
            flats = {isis.TOPO_STD: topology_flat(inst, isis.MT_STANDARD), isis.TOPO_MT6: topology_flat(inst, isis.MT_IPV6)}
            roots = dict(enumerate(self.rt.root))
            self.cell_dt, self.harness = isis.CELL_DT, harnesses["isis"]
        else:
            mod = ospfv3 if kind == "ospfv3" else ospfv2
            area = ospfv3.synth_area(t, root=2) if kind == "ospfv3" else ospfv2.synth_area(t, root=2, sr=True)
            flat = mod.Flat(area)
            self.rt = mod.RouteTable(flat)
            csr = flat.csr
            # a root with at most 16 first-hop atoms has 16-bit planes too
            root = next(v for v in range(csr.n_vertices) if flat.is_router[v] and 2 <= capi.atom_count(csr, v) <= 16)
            flats, roots = {0: flat}, {0: root}
            self.cell_dt, self.harness = ospfv2.CELL_DT, harnesses["ospf"]
        self.rt.upload(ctx)
        P = self.rt.n_prefixes
        self.n = next(k for k in range(6, 40) if (k * P) % 32)
        E = flats[0].csr.n_edges
        ov = [[]] + [[((97 * j) % E, capi.COST_DISABLED)] for j in range(1, self.n)]
        self.tops = {tt: DeviceTopology(ctx, f.csr, roots[tt], self.n, ov if tt == 0 else None, self.narrow)
                     for tt, f in flats.items()}
        for d in self.tops.values():
            d.run()
        ctx.sync()
        assert not any(d.status.any().item() for d in self.tops.values())

    def expected(self, j):
        if self.kind == "isis":
            return harness_cells(self.harness, self.rt, self.tops, j)
        return cells_on_cpu(self.harness, self.rt, self.tops[0].planes(j), self.narrow)

    def launch(self, offset=0, refuse=(), gather=()):
        """The route kernel over the batch's planes, cells written `offset` bytes into a buffer whose start is
        16-byte aligned.  refuse: jobs whose status word is set for this launch (IS-IS: in the standard and the
        MT-IPv6 topology by turns).  gather: (job, vertex) pairs of the OSPF gather.  Returns the cells and the
        gathered values."""
        import torch
        P, n = self.rt.n_prefixes, self.n
        nbytes = n * P * self.cell_dt.itemsize
        buf = torch.full((offset + nbytes + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
        assert buf.data_ptr() % 16 == 0
        poked = [(self.tops[i % len(self.tops)], j) for i, j in enumerate(refuse)]
        for d, j in poked:
            d.status[j] = 2
        dev = lambda a: torch.tensor(np.asarray(a, np.uint32).view(np.int32), device="cuda")
        gj, gv = dev([j for j, _ in gather]), dev([v for _, v in gather])
        gnh = torch.zeros(len(gather), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        ptr = buf.data_ptr() + offset
        if self.kind == "isis":
            isis.routes_batch_device(self.ctx, self.rt, n, self.tops[isis.TOPO_STD].rs, self.tops[isis.TOPO_MT6].rs, ptr)
        else:
            ospfv2.routes_batch_device(self.ctx, self.rt, n, self.tops[0].rs, ptr, len(gather), gj.data_ptr(),
                                       gv.data_ptr(), gnh.data_ptr())
        self.ctx.sync()
        for d, j in poked:
            d.status[j] = 0
        host = buf.cpu().numpy()
        assert (host[:offset] == SENTINEL).all() and (host[offset + nbytes:] == SENTINEL).all()
        cells = np.frombuffer(host[offset:offset + nbytes].tobytes(), self.cell_dt).reshape(n, P)
        return cells, gnh.cpu().numpy().view(np.uint64)


@pytest.fixture(scope="module", params=["ospfv2-wide", "ospfv2-narrow", "ospfv3", "isis"])
def case(request, ctx, harnesses):
    return Case(ctx, request.param, harnesses)


@pytest.fixture(scope="module", params=["ospfv2-wide", "ospfv2-narrow"])
def ospfv2_case(request, ctx, harnesses):
    return Case(ctx, request.param, harnesses)


def test_partial_last_tile(case):
    assert (case.n * case.rt.n_prefixes) % 32
    cells, _ = case.launch()
    for j in range(case.n):
        assert cells[j].tobytes() == case.expected(j).tobytes(), j
    assert (cells["flags"] & ospfv2.CELL_PRESENT).any()


@pytest.mark.parametrize("offset", [8, 24])
def test_misaligned_cell_buffer(case, offset):
    assert case.launch(offset)[0].tobytes() == case.launch()[0].tobytes()


def test_refused_jobs_get_empty_cells(case):
    refuse = (1, 2)
    cells, _ = case.launch(refuse=refuse)
    empty = np.zeros(case.rt.n_prefixes, case.cell_dt)
    empty["winner"] = 0xFFFFFFFF
    for j in range(case.n):
        assert cells[j].tobytes() == (empty if j in refuse else case.expected(j)).tobytes(), j


def test_gather_with_a_misaligned_cell_buffer(ospfv2_case):
    c = ospfv2_case
    V = c.tops[0].V
    pairs = [(j, v) for j in range(c.n) for v in (0, 1, V // 2, V - 1)] + [(c.n, 0), (0, V)]     # last two: out of range
    cells, got = c.launch(8, gather=pairs)
    assert cells.tobytes() == c.launch()[0].tobytes()
    want = [int(c.tops[0].planes(j)[2][v]) if j < c.n and v < V else 0 for j, v in pairs]
    assert got.tolist() == want
