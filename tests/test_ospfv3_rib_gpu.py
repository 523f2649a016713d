"""GPU: the batched route stages over OSPFv3 areas.  The SPT planes are written on the device and never leave it before
the route kernels read them:
  * intra-area cells (hspf_ospfv2_routes_batch[16] over the tables of hspf_ospfv3_rtable_create) equal the CPU harness
    byte for byte and decode to the oracle's run_area routes;
  * routing-table cells (hspf_ospfv2_rib_cells[16] over the tables of hspf_ospfv3_ribtable_create) equal the CPU
    harness byte for byte, with a partial last tile, refused jobs and gather, and decode (hspf_ospfv3_rib_from_cells)
    to the host stages over the same planes, the golden snapshots' local-rib included;
  * the route-delta stage (hspf_ospfv2_rib_delta[16]) equals the numpy reference of tests/test_ospf_rib_delta.py
    applied to those device cells."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import golden_util as gu
from holo_b200 import capi, ospf_rib, ospfv2, ospfv3, synth
from oracle import pyoracle
from test_isis_route_cells_gpu import DeviceTopology
from test_ospf_rib_cells import same_rib
from test_ospf_rib_cells_gpu import Batch, dev_u32, harness  # noqa: F401  (harness: the fixture)
from test_ospf_rib_delta import perturbed, reference
from test_ospf_rib_delta_gpu import rib_delta
from test_ospfv2_route_cells import gather_for
from test_ospfv3_rib_cells import flags_of, host_rib, rib_dict, view
from test_ospfv3_rib_delta import whatif_overrides
from test_ospfv3_route_cells import same_routes
from test_route_delta_gpu import same

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def route_harness(built, tmp_path_factory):
    """tests/native/route_cells_harness.cc: the intra-area walk on the CPU."""
    out = tmp_path_factory.mktemp("harness") / "libroute_cells_harness.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I", str(ROOT / "include"), "-o", str(out),
                    str(ROOT / "tests" / "native" / "route_cells_harness.cc")], check=True)
    lib = C.CDLL(str(out))
    lib.harness_route_cells.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 4
    lib.harness_route_cells16.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 4
    return lib


class Batch3(Batch):
    """Batch over the OSPFv3 view of topology t (test_ospfv3_rib_cells.view): the routing table on the device and jobs
    rooted at roots[j] with overrides[j], computed on the device."""

    def __init__(self, ctx, t, seed, roots, overrides=None, narrow=False, frag=0, **kw):
        import torch
        self.ctx, self.t, self.seed, self.kw, self.narrow, self.frag = ctx, t, seed, kw, narrow, frag
        self.area, self.sums, self.ext = view(t, 0, seed, frag=frag, **kw)
        self.flat = ospfv3.Flat(self.area)
        self.rt = ospf_rib.RibTable(self.flat, self.area.area_id, self.sums, self.ext)
        self.rt.upload(ctx)
        self.n, self.roots = len(roots), [int(r) for r in roots]
        self.top = DeviceTopology(ctx, self.flat.csr, self.roots[0], self.n, overrides, narrow)
        self.top.keep[0].copy_(dev_u32(self.roots))
        self.top.run()
        ctx.sync()
        self.d_roots = dev_u32(self.roots)
        torch.cuda.synchronize()

    def decode_and_check(self, j, root_index):
        area, sums, ext = view(self.t, root_index, self.seed, frag=self.frag, **self.kw)
        flat = ospfv3.Flat(area)
        rv = flat.router_vertex(area.router_id)
        assert rv == self.roots[j]
        d, h, m = self.planes(j)
        cells, st, _ = self.launch()
        assert st[j] == 0
        gv, gn = gather_for(flat, rv, (d, h, m))
        got = ospf_rib.rib_from_cells_v3(area, self.rt, cells[j], gv, gn)
        m4 = np.zeros((len(m), 4), np.uint64)
        m4[:, 0] = m
        same_rib(got, host_rib(area, sums, ext, lambda csr, root, nhw: (d, h, m4[:, :nhw])))
        return got


def internal_and_abr_roots(area, flat, limit=16):
    fl = flags_of(area)
    fits = [flat.router_vertex(r) for r in sorted(fl) if flat.router_vertex(r) != 0xFFFFFFFF]
    fits = [v for v in fits if capi.atom_count(flat.csr, v) <= limit]
    is_abr = lambda v: fl[int(flat.router_ids[v])] & 1
    return [v for v in fits if not is_abr(v)], [v for v in fits if is_abr(v)]


@pytest.fixture(scope="module", params=["wide", "narrow"])
def small(request, ctx):
    narrow = request.param == "narrow"
    t = synth.random_topology(150, 600, synth.SEED_BASE + 561, cost_choices=[5, 10], lan_fraction=0.1)
    area, sums, ext = view(t, 0, 1971, frag=3)
    flat = ospfv3.Flat(area)
    ok, abr = internal_and_abr_roots(area, flat)
    rv = ok[:6] + abr[:2] + ok[6:40]                                    # jobs 6 and 7: ABR roots
    P = ospf_rib.RibTable(flat, 1, sums, ext).n_prefixes
    n = next(k for k in range(20, 60) if (k * P) % 32)                   # a partial last warp tile
    E = flat.csr.n_edges
    ov = [[]] * 3 + [[((97 * j) % E, capi.COST_DISABLED)] for j in range(3, n)]
    return Batch3(ctx, t, 1971, [rv[j % len(rv)] for j in range(n)], ov, narrow, frag=3)


def test_partial_last_tile_and_status(small, harness):  # noqa: F811
    assert (small.n * small.rt.n_prefixes) % 32 and small.rt.v3
    cells, st, _ = small.launch()
    want, want_st = small.expected(harness)
    assert st.tolist() == want_st.tolist()
    assert cells.tobytes() == want.tobytes()
    paths = set(ospf_rib.cell_path(cells[(ospf_rib.cell_flags(cells) & 1) != 0]).tolist())
    assert paths == {0, 1, 2, 3}
    assert (st == ospf_rib.JS_NOT_INTERNAL).any() and (st == 0).any()
    a, b = small.launch(), small.launch()
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


def test_refused_jobs_and_gather(small, harness):  # noqa: F811
    V = small.top.V
    roots = list(small.roots)
    roots[4], roots[5] = V, V + 1000                              # out of range
    cells, st, _ = small.launch(roots=roots, refuse=(1, 2))
    status = small.top.status.cpu().numpy().view(np.uint32).copy()
    status[[1, 2]] = 2
    want, want_st = small.expected(harness, roots=roots, status=status)
    assert st.tolist() == want_st.tolist() and cells.tobytes() == want.tobytes()
    assert st[4] == capi.JS_INVALID and st[5] == capi.JS_INVALID
    for j in (1, 2, 4, 5):
        assert (cells["winner"][j] == ospf_rib.NO_RECORD).all() and not cells["mpf"][j].any()
    pairs = [(j, v) for j in range(small.n) for v in (0, V // 2, V - 1)] + [(small.n, 0), (0, V)]
    _, _, got = small.launch(8, gather=pairs)
    assert got.tolist() == [int(small.planes(j)[2][v]) if j < small.n and v < V else 0 for j, v in pairs]


def test_small_batch_decodes(small):
    for j in range(3):
        small.decode_and_check(j, int(small.flat.router_ids[small.roots[j]]) - ospfv3.RID_BASE)


# ------------------------------------------------------------------------------ intra-area stage over v3 tables
@pytest.mark.parametrize("narrow", [False, True], ids=["wide", "narrow"])
def test_intra_area_routes_batch_over_v3_tables(ctx, route_harness, narrow):
    """hspf_ospfv2_routes_batch[16] over an OSPFv3 rtable: the device cells equal the CPU harness over the same device
    planes, and each job decodes (hspf_ospfv3_routes_from_cells) to the oracle's run_area routes for its root."""
    import torch
    t = synth.random_topology(120, 500, synth.SEED_BASE + 562, cost_choices=[10, 20], lan_fraction=0.1)
    area = ospfv3.synth_area(t, root=0, max_links_per_fragment=2)
    flat = ospfv3.Flat(area)
    rt = ospfv3.RouteTable(flat)
    rt.upload(ctx)
    roots = [v for v in range(flat.csr.n_vertices) if flat.is_router[v] and capi.atom_count(flat.csr, v) <= 16][:37]
    n, P = len(roots), rt.n_prefixes
    top = DeviceTopology(ctx, flat.csr, roots[0], n, None, narrow)
    top.keep[0].copy_(dev_u32(roots))
    top.run()
    ctx.sync()
    buf = torch.zeros(n * P * ospfv2.CELL_DT.itemsize, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ospfv2.routes_batch_device(ctx, rt, n, top.rs, buf.data_ptr())
    ctx.sync()
    cells = np.frombuffer(buf.cpu().numpy().tobytes(), ospfv2.CELL_DT).reshape(n, P)
    for j, rv in enumerate(roots):
        d, h, m = top.planes(j)
        want = np.zeros(P, ospfv2.CELL_DT)
        if narrow:
            d16 = np.where(d == 0xFFFFFFFF, 0xFFFF, d).astype(np.uint16)
            route_harness.harness_route_cells16(rt.handle, 1, d16.ctypes.data, np.ascontiguousarray(h).ctypes.data,
                                                m.astype(np.uint16).ctypes.data, want.ctypes.data)
        else:
            route_harness.harness_route_cells(rt.handle, 1, np.ascontiguousarray(d, np.uint32).ctypes.data,
                                              np.ascontiguousarray(h).ctypes.data, np.ascontiguousarray(m, np.uint64).ctypes.data,
                                              want.ctypes.data)
        assert cells[j].tobytes() == want.tobytes(), j
        if j % 6:
            continue
        a = ospfv3.synth_area(t, root=int(flat.router_ids[rv]) - ospfv3.RID_BASE, max_links_per_fragment=2)
        gv, gn = gather_for(flat, rv, (d, h, np.asarray(m, np.uint64)))
        same_routes(ospfv3.routes_from_cells(a, rt, cells[j], gv, gn), pyoracle.ospfv3_run_area(a))


# ------------------------------------------------------------------------------ goldens through the device
SNAPS = [s for s in gu.load_ospfv3() if len(s["areas"]) == 1]


def test_golden_snapshots_through_the_device(ctx, harness):  # noqa: F811
    """Every single-area OSPFv3 snapshot as a one-job batch on the device: cells equal the harness, and the decoded
    table equals the host stages and the reference's local-rib."""
    for snap in SNAPS:
        keys = gu.global_sort_keys(snap)
        area_j = snap["areas"][0]
        img = gu.ospfv3_area_image(snap, area_j, keys)
        sums = gu.ospfv3_inter_area_lsas(area_j)
        b = object.__new__(Batch3)
        b.ctx, b.narrow = ctx, False
        b.flat = ospfv3.Flat(img)
        b.rt = ospf_rib.RibTable(b.flat, img.area_id, sums)
        b.rt.upload(ctx)
        rv = b.flat.router_vertex(img.router_id)
        b.n, b.roots = 1, [rv]
        b.top = DeviceTopology(ctx, b.flat.csr, rv, 1)
        b.top.run()
        ctx.sync()
        b.d_roots = dev_u32([rv])
        cells, st, _ = b.launch()
        want, want_st = b.expected(harness)
        assert st.tolist() == want_st.tolist() == [0] and cells.tobytes() == want.tobytes(), snap["topo"]
        d, h, m = b.planes(0)
        gv, gn = gather_for(b.flat, rv, (d, h, m))
        got = ospf_rib.rib_from_cells_v3(img, b.rt, cells[0], gv, gn)
        m4 = np.zeros((len(m), 4), np.uint64)
        m4[:, 0] = m
        same_rib(got, host_rib(img, sums, None, lambda csr, root, nhw: (d, h, m4[:, :nhw])))
        mine, ref = rib_dict(got, {v: k for k, v in keys.items()}), gu.golden_rib(snap)
        assert {k: v[:2] for k, v in mine.items()} == {k: v[:2] for k, v in ref.items()}, (snap["topo"], snap["rt"])


# ------------------------------------------------------------------------------ route-delta stage
@pytest.fixture(scope="module")
def cells(small):
    c, st, _ = small.launch()
    return c, st, np.stack([perturbed(c[0]), c[0]])


def test_delta_against_a_perturbed_row(small, cells):
    c, st, base = cells
    want = reference(c, base[:1], status=st)
    # every prefix stays reachable in these jobs: no LOST record here (the OSPFv2 tests meet that kind)
    assert all(want[0][k].sum() > 0 for k in ("n_gained", "n_metric", "n_nexthops", "n_other"))
    same(rib_delta(small, base[:1]), want)
    bo = np.arange(small.n) % 3                                                # row 2 does not exist
    got = rib_delta(small, base, base_of=bo, base_offset=8)
    same(got, reference(c, base, bo, st))
    assert (got[0]["status"][bo == 2] == capi.JS_INVALID).all()


def test_delta_capacity_and_refusals(small, cells):
    c, st, base = cells
    total = reference(c, base[:1], status=st)[2]
    for cap in sorted({0, 1, total // 2, total}):
        got = rib_delta(small, base[:1], cap=cap)                              # checks the bytes after the records
        same(got, reference(c, base[:1], status=st, cap=cap))
    roots = list(small.roots)
    roots[4] = small.top.V
    c2, st2, _ = small.launch(roots=roots, refuse=(1,))
    got = rib_delta(small, base[1:], roots=roots, refuse=(1,))
    assert got[0]["status"].tolist() == st2.tolist() and {1, 4, 6, 7} <= set(np.nonzero(st2)[0].tolist())
    same(got, reference(c2, base[1:], status=st2))


def test_whatif_batch_on_600_routers(ctx, harness):  # noqa: F811
    """One internal root, each job disabling one link or raising one cost, wide and narrow planes: cells equal the
    harness, the delta equals the reference over the cells, sampled jobs decode to the host stages."""
    kw = dict(n_abr=5, n_asbr=5, n_inter=400, n_ext=300, n_overlap=80, n_fresh=150, n_ext_only=60)
    t = synth.random_topology(600, 2400, synth.SEED_BASE + 563, cost_choices=[10, 20], lan_fraction=0.05)
    area, _, _ = view(t, 0, 1972, **kw)
    flat = ospfv3.Flat(area)
    ok, _ = internal_and_abr_roots(area, flat)
    rv = ok[0]
    n = 48
    ov = whatif_overrides(flat, n, 11)
    wide = Batch3(ctx, t, 1972, [rv] * n, ov, **kw)
    narrow = Batch3(ctx, t, 1972, [rv] * n, ov, narrow=True, **kw)
    c, st, _ = wide.launch()
    want, want_st = wide.expected(harness)
    assert not st.any() and c.tobytes() == want.tobytes()
    assert narrow.launch()[0].tobytes() == c.tobytes()
    got = rib_delta(wide, c[:1])
    same(got, reference(c, c[:1]))
    same(rib_delta(narrow, c[:1]), got)
    assert got[2] > 0 and (got[0]["n_changed"] > 0).sum() > n // 4
    for j in (0, 1, 2, 17):
        wide.decode_and_check(j, int(flat.router_ids[rv]) - ospfv3.RID_BASE)
