"""OSPFv2 side of the engine from Python: LSDB images (include/holo_lsdb.h) as numpy
structured arrays, the `run_area` call (holo-ospf/src/spf.rs:587-729 +
route.rs:343-446 replaced by hspf_ospfv2_run_area), the flattener for batch use,
and a synthetic LSDB builder for the BASELINE.json shapes.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import capi, route_table
from .synth import Topology

LINK_P2P, LINK_TRANSIT, LINK_STUB, LINK_VLINK = 1, 2, 3, 4
IF_P2P, IF_BROADCAST, IF_NBMA, IF_P2MP, IF_VLINK, IF_LOOPBACK = range(6)
MAX_AGE = 3600
PSID_NP, PSID_M, PSID_E, PSID_V, PSID_L = 0x40, 0x20, 0x10, 0x08, 0x04

LINK_DT = np.dtype([("link_id", "<u4"), ("link_data", "<u4"), ("metric", "<u2"), ("link_type", "u1"), ("_pad", "u1")],
                   align=True)
ROUTER_LSA_DT = np.dtype([("adv_rtr", "<u4"), ("lsa_id", "<u4"), ("age", "<u2"), ("flags", "u1"), ("options", "u1"),
                          ("link_off", "<u4"), ("n_links", "<u4")], align=True)
NETWORK_LSA_DT = np.dtype([("adv_rtr", "<u4"), ("lsa_id", "<u4"), ("mask", "<u4"), ("age", "<u2"), ("_pad", "<u2"),
                           ("att_off", "<u4"), ("n_att", "<u4")], align=True)
IFACE_DT = np.dtype([("ifindex", "<u4"), ("sort_key", "<u4"), ("if_type", "u1"), ("_pad", "u1", (3,)),
                     ("addr_off", "<u4"), ("n_addrs", "<u4"), ("nbr_off", "<u4"), ("n_nbrs", "<u4")], align=True)
IPV4_NET_DT = np.dtype([("addr", "<u4"), ("mask", "<u4")], align=True)
NBR_DT = np.dtype([("router_id", "<u4"), ("src", "<u4")], align=True)
SRGB_DT = np.dtype([("first", "<u4"), ("range", "<u4"), ("first_is_index", "u1"), ("_pad", "u1", (3,))], align=True)
RI_LSA_DT = np.dtype([("adv_rtr", "<u4"), ("lsa_id", "<u4"), ("age", "<u2"), ("has_sr_algo", "u1"),
                      ("sr_algo_has_spf", "u1"), ("srgb_off", "<u4"), ("n_srgb", "<u4")], align=True)
EXT_PREFIX_DT = np.dtype([("adv_rtr", "<u4"), ("prefix", "<u4"), ("mask", "<u4"), ("age", "<u2"), ("route_type", "u1"),
                          ("has_sid", "u1"), ("sid_flags", "u1"), ("sid_is_label", "u1"), ("_pad", "u1", (2,)),
                          ("sid_value", "<u4")], align=True)
NEXTHOP_DT = np.dtype([("iface", "<u4"), ("addr", "<u4"), ("nbr_router_id", "<u4"), ("sr_label", "<u4"),
                       ("has_addr", "u1"), ("has_nbr", "u1"), ("has_label", "u1"), ("_pad", "u1")], align=True)
SPT_VERTEX_DT = np.dtype([("id", "<u4"), ("distance", "<u4"), ("hops", "<u2"), ("is_router", "u1"), ("_pad", "u1"),
                          ("nh_off", "<u4"), ("n_nh", "<u4")], align=True)
ROUTE_RTR_DT = np.dtype([("router_id", "<u4"), ("metric", "<u4"), ("flags", "u1"), ("options", "u1"),
                         ("_pad", "u1", (2,)), ("nh_off", "<u4"), ("n_nh", "<u4")], align=True)
ROUTE_NET_DT = np.dtype([("prefix", "<u4"), ("mask", "<u4"), ("metric", "<u4"), ("flags", "u1"), ("origin_type", "u1"),
                         ("has_prefix_sid", "u1"), ("has_sr_label", "u1"), ("origin_adv_rtr", "<u4"),
                         ("origin_lsa_id", "<u4"), ("prefix_sid_value", "<u4"), ("prefix_sid_flags", "u1"),
                         ("prefix_sid_is_label", "u1"), ("_pad", "u1", (2,)), ("sr_label", "<u4"), ("nh_off", "<u4"),
                         ("n_nh", "<u4")], align=True)


class AreaStruct(C.Structure):
    _fields_ = [
        ("router_id", C.c_uint32), ("area_id", C.c_uint32), ("max_paths", C.c_uint16), ("sr_enabled", C.c_uint8),
        ("_pad", C.c_uint8),
        ("n_router_lsas", C.c_uint32), ("router_lsas", C.c_void_p),
        ("n_links", C.c_uint32), ("links", C.c_void_p),
        ("n_network_lsas", C.c_uint32), ("network_lsas", C.c_void_p),
        ("n_attached", C.c_uint32), ("attached", C.c_void_p),
        ("n_ifaces", C.c_uint32), ("ifaces", C.c_void_p),
        ("n_iface_addrs", C.c_uint32), ("iface_addrs", C.c_void_p),
        ("n_nbrs", C.c_uint32), ("nbrs", C.c_void_p),
        ("n_ri_lsas", C.c_uint32), ("ri_lsas", C.c_void_p),
        ("n_srgbs", C.c_uint32), ("srgbs", C.c_void_p),
        ("n_ext_prefixes", C.c_uint32), ("ext_prefixes", C.c_void_p),
    ]


class ResultStruct(C.Structure):
    _fields_ = [
        ("vertices_cap", C.c_uint32), ("n_vertices", C.c_uint32), ("vertices", C.c_void_p),
        ("routers_cap", C.c_uint32), ("n_routers", C.c_uint32), ("routers", C.c_void_p),
        ("routes_cap", C.c_uint32), ("n_routes", C.c_uint32), ("routes", C.c_void_p),
        ("nexthops_cap", C.c_uint32), ("n_nexthops", C.c_uint32), ("nexthops", C.c_void_p),
        ("transit_capability", C.c_uint8), ("root_found", C.c_uint8), ("_pad", C.c_uint8 * 2),
    ]


# order of hspf_abi_sizes()
ABI_SIZES = [
    C.sizeof(capi.CsrStruct), C.sizeof(capi.JobsStruct), C.sizeof(capi.ResultStruct),
    LINK_DT.itemsize, ROUTER_LSA_DT.itemsize, NETWORK_LSA_DT.itemsize, IFACE_DT.itemsize, IPV4_NET_DT.itemsize,
    NBR_DT.itemsize, SRGB_DT.itemsize, RI_LSA_DT.itemsize, EXT_PREFIX_DT.itemsize, C.sizeof(AreaStruct),
    NEXTHOP_DT.itemsize, SPT_VERTEX_DT.itemsize, ROUTE_RTR_DT.itemsize, ROUTE_NET_DT.itemsize, C.sizeof(ResultStruct),
]


def abi_sizes_expected():
    from . import isis, ospf_rib, ospfv3
    return (ABI_SIZES + isis.ABI_SIZES + ospfv3.ABI_SIZES + ospf_rib.ABI_SIZES +
            [isis.RNL_DT.itemsize, CELL_DT.itemsize, TRIGGER_DT.itemsize, C.sizeof(SpfComputationStruct),
             ospf_rib.RIB_RTR_DT.itemsize, C.sizeof(ospf_rib.RtrTablesStruct),
             isis.LSP_TRIGGER_DT.itemsize, ospfv3.IP_PREFIX_DT.itemsize, ospfv3.TRIGGER6_DT.itemsize,
             C.sizeof(ospfv3.SpfComputation6Struct), isis.CELL_DT.itemsize,
             route_table.DELTA_DT.itemsize, route_table.DELTA_JOB_DT.itemsize])


def abi_sizes_from_library():
    lib = capi.load_library()
    out = (C.c_uint32 * 128)()
    n = lib.hspf_abi_sizes(out, 128)
    return [int(out[i]) for i in range(n)]


def _arr(x, dt):
    a = np.zeros(len(x), dtype=dt) if not isinstance(x, np.ndarray) else x
    return np.ascontiguousarray(a, dtype=dt)


@dataclass
class Ospfv2Area:
    """hl_ospfv2_area as numpy structured arrays."""
    router_id: int
    area_id: int = 0
    max_paths: int = 16
    sr_enabled: bool = False
    router_lsas: np.ndarray = field(default_factory=lambda: np.zeros(0, ROUTER_LSA_DT))
    links: np.ndarray = field(default_factory=lambda: np.zeros(0, LINK_DT))
    network_lsas: np.ndarray = field(default_factory=lambda: np.zeros(0, NETWORK_LSA_DT))
    attached: np.ndarray = field(default_factory=lambda: np.zeros(0, np.uint32))
    ifaces: np.ndarray = field(default_factory=lambda: np.zeros(0, IFACE_DT))
    iface_addrs: np.ndarray = field(default_factory=lambda: np.zeros(0, IPV4_NET_DT))
    nbrs: np.ndarray = field(default_factory=lambda: np.zeros(0, NBR_DT))
    ri_lsas: np.ndarray = field(default_factory=lambda: np.zeros(0, RI_LSA_DT))
    srgbs: np.ndarray = field(default_factory=lambda: np.zeros(0, SRGB_DT))
    ext_prefixes: np.ndarray = field(default_factory=lambda: np.zeros(0, EXT_PREFIX_DT))
    ifnames: list = field(default_factory=list)     # diagnostic only

    def as_struct(self) -> AreaStruct:
        s = AreaStruct()
        s.router_id, s.area_id = self.router_id, self.area_id
        s.max_paths, s.sr_enabled = self.max_paths, int(self.sr_enabled)
        for name, dt in (("router_lsas", ROUTER_LSA_DT), ("links", LINK_DT), ("network_lsas", NETWORK_LSA_DT),
                         ("attached", np.dtype("<u4")), ("ifaces", IFACE_DT), ("iface_addrs", IPV4_NET_DT),
                         ("nbrs", NBR_DT), ("ri_lsas", RI_LSA_DT), ("srgbs", SRGB_DT),
                         ("ext_prefixes", EXT_PREFIX_DT)):
            a = np.ascontiguousarray(getattr(self, name), dtype=dt)
            setattr(self, name, a)
            setattr(s, "n_" + name, len(a))
            setattr(s, name, a.ctypes.data if len(a) else None)
        return s


@dataclass
class Ospfv2Result:
    vertices: np.ndarray
    routers: np.ndarray
    routes: np.ndarray
    nexthops: np.ndarray
    transit_capability: bool
    root_found: bool
    rc: int = 0

    def nh(self, rec):
        """Next hops of a vertex / router / route record as tuples."""
        return [tuple(int(x[k]) for k in ("iface", "has_addr", "addr", "has_nbr", "nbr_router_id", "has_label", "sr_label"))
                for x in self.nexthops[int(rec["nh_off"]): int(rec["nh_off"]) + int(rec["n_nh"])]]


def _call_run_area(fn, area: Ospfv2Area, prefix_args=(), tail_args=()):
    s = area.as_struct()
    nv = len(area.router_lsas) + len(area.network_lsas) + 1
    n_routes = len(area.links) + len(area.network_lsas) + 1
    caps = [nv, nv, n_routes, 64 * (2 * nv + n_routes) + 64]
    for _ in range(2):
        verts = np.zeros(caps[0], SPT_VERTEX_DT)
        rtrs = np.zeros(caps[1], ROUTE_RTR_DT)
        routes = np.zeros(caps[2], ROUTE_NET_DT)
        nhs = np.zeros(caps[3], NEXTHOP_DT)
        r = ResultStruct()
        r.vertices_cap, r.vertices = caps[0], verts.ctypes.data
        r.routers_cap, r.routers = caps[1], rtrs.ctypes.data
        r.routes_cap, r.routes = caps[2], routes.ctypes.data
        r.nexthops_cap, r.nexthops = caps[3], nhs.ctypes.data
        rc = fn(*prefix_args, C.byref(s), *tail_args, C.byref(r))
        if rc == capi.HSPF_E_NOMEM and r.n_nexthops > caps[3]:
            caps = [max(caps[0], r.n_vertices), max(caps[1], r.n_routers), max(caps[2], r.n_routes), r.n_nexthops]
            continue
        break
    return Ospfv2Result(verts[: r.n_vertices].copy(), rtrs[: r.n_routers].copy(), routes[: r.n_routes].copy(),
                        nhs[: r.n_nexthops].copy(), bool(r.transit_capability), bool(r.root_found), rc)


def run_area(ctx: capi.Context, area: Ospfv2Area) -> Ospfv2Result:
    """run_area + update_rib_intra_area of the local router on the GPU engine."""
    lib = ctx.lib
    lib.hspf_ospfv2_run_area.argtypes = [C.c_void_p, C.POINTER(AreaStruct), C.POINTER(ResultStruct)]
    res = _call_run_area(lib.hspf_ospfv2_run_area, area, (ctx.handle,))
    if res.rc not in (capi.HSPF_OK,):
        raise capi.HspfError(res.rc, ctx.last_error())
    return res


def area_from_planes(area: Ospfv2Area, spf) -> Ospfv2Result:
    """hspf_ospfv2_area_from_planes: the post-SPT half of run_area over planes supplied by
    `spf(csr, root_vertex, nh_words) -> (dist u32[V], hops u16[V], nh_mask u64[V, nh_words])` on the
    flattened CSR of the area (host only; the planes may come from hspf_run_batch or, in tests, from
    the oracle)."""
    lib = capi.load_library()
    lib.hspf_ospfv2_area_from_planes.argtypes = [C.POINTER(AreaStruct), C.POINTER(C.c_uint32), C.POINTER(C.c_uint16),
                                                 C.POINTER(C.c_uint64), C.c_uint32, C.POINTER(ResultStruct)]
    f = Flat(area)
    root = f.router_vertex(area.router_id)
    nhw = 4
    if root == 0xFFFFFFFF:
        V = f.csr.n_vertices
        d, h, m = np.zeros(V, np.uint32), np.zeros(V, np.uint16), np.zeros((V, nhw), np.uint64)
    else:
        d, h, m = spf(f.csr, root, nhw)
    d = np.ascontiguousarray(d, np.uint32)
    h = np.ascontiguousarray(h, np.uint16)
    m = np.ascontiguousarray(m, np.uint64)
    tail = (d.ctypes.data_as(C.POINTER(C.c_uint32)), h.ctypes.data_as(C.POINTER(C.c_uint16)),
            m.ctypes.data_as(C.POINTER(C.c_uint64)), nhw)
    res = _call_run_area(lib.hspf_ospfv2_area_from_planes, area, (), tail)
    if res.rc != capi.HSPF_OK:
        raise capi.HspfError(res.rc, "hspf_ospfv2_area_from_planes failed")
    return res


class Flat:
    """hspf_ospfv2_flatten result: CSR + vertex table (host only)."""

    def __init__(self, area: Ospfv2Area):
        lib = capi.load_library()
        lib.hspf_ospfv2_flatten.argtypes = [C.POINTER(AreaStruct), C.POINTER(C.c_void_p)]
        lib.hspf_ospfv2_flat_free.argtypes = [C.c_void_p]
        lib.hspf_ospfv2_flat_free.restype = None
        lib.hspf_ospfv2_flat_csr.argtypes = [C.c_void_p, C.POINTER(capi.CsrStruct)]
        lib.hspf_ospfv2_flat_vertices.argtypes = [C.c_void_p, C.POINTER(C.POINTER(C.c_uint32)),
                                                  C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_uint32)]
        lib.hspf_ospfv2_flat_edge_tags.argtypes = [C.c_void_p, C.POINTER(C.POINTER(C.c_uint32)),
                                                   C.POINTER(C.POINTER(C.c_uint32))]
        lib.hspf_ospfv2_flat_router_vertex.argtypes = [C.c_void_p, C.c_uint32]
        lib.hspf_ospfv2_flat_router_vertex.restype = C.c_uint32
        lib.hspf_ospfv2_flat_network_vertex.argtypes = [C.c_void_p, C.c_uint32]
        lib.hspf_ospfv2_flat_network_vertex.restype = C.c_uint32
        self.lib = lib
        self.area = area
        self._s = area.as_struct()
        h = C.c_void_p()
        rc = lib.hspf_ospfv2_flatten(C.byref(self._s), C.byref(h))
        if rc != capi.HSPF_OK:
            raise capi.HspfError(rc, "hspf_ospfv2_flatten failed")
        self.handle = h
        self._load()

    def _load(self):
        lib, h = self.lib, self.handle
        cs = capi.CsrStruct()
        lib.hspf_ospfv2_flat_csr(h, C.byref(cs))
        V, E = cs.n_vertices, cs.n_edges
        as_np = lambda p, n, dt: np.ctypeslib.as_array(p, shape=(n,)).astype(dt).copy() if n else np.zeros(0, dt)
        self.csr = capi.Csr(as_np(cs.row_ptr, V + 1, np.uint32), as_np(cs.col, E, np.uint32),
                            as_np(cs.cost, E, np.uint32), as_np(cs.vflags, V, np.uint8),
                            reject_above=cs.reject_above, saturate_at=cs.saturate_at, flags=cs.flags, delta=cs.delta)
        ids, isr, n = C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint8)(), C.c_uint32()
        lib.hspf_ospfv2_flat_vertices(h, C.byref(ids), C.byref(isr), C.byref(n))
        self.ids = as_np(ids, n.value, np.uint32)
        self.is_router = as_np(isr, n.value, np.uint8)
        li, lp = C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint32)()
        lib.hspf_ospfv2_flat_edge_tags(h, C.byref(li), C.byref(lp))
        self.link_index = as_np(li, E, np.uint32)
        self.link_pos = as_np(lp, E, np.uint32)

    def router_vertex(self, router_id: int) -> int:
        return int(self.lib.hspf_ospfv2_flat_router_vertex(self.handle, router_id))

    def network_vertex(self, dr_addr: int) -> int:
        return int(self.lib.hspf_ospfv2_flat_network_vertex(self.handle, dr_addr))

    def __del__(self):
        try:
            if self.handle:
                self.lib.hspf_ospfv2_flat_free(self.handle)
                self.handle = None
        except Exception:
            pass


# ------------------------------------------------------------------- trigger-keyed recomputation
TRIGGER_DT = np.dtype([("adv_rtr", "<u4"), ("lsa_id", "<u4"), ("mask", "<u4"), ("lsa_type", "u1"), ("opaque_type", "u1"),
                       ("_pad", "u1", (2,))])
SPF_FULL, SPF_PARTIAL = 1, 2
FLAT_UNCHANGED, FLAT_COSTS, FLAT_REBUILT = 0, 1, 2


class SpfComputationStruct(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("n_inter_network", C.c_uint32), ("n_inter_router", C.c_uint32),
                ("n_external", C.c_uint32), ("cap", C.c_uint32), ("inter_network", C.c_void_p),
                ("inter_router", C.c_void_p), ("external", C.c_void_p)]


def spf_computation_type(triggers, fn=None):
    """hspf_ospfv2_spf_computation_type -> (kind, inter_network [(addr, mask)], inter_router [id], external)."""
    tr = np.ascontiguousarray(triggers, TRIGGER_DT)
    if fn is None:
        fn = capi.load_library().hspf_ospfv2_spf_computation_type
    fn.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(SpfComputationStruct)]
    cap = max(len(tr), 1)
    net, rtr, ext = np.zeros(cap, IPV4_NET_DT), np.zeros(cap, np.uint32), np.zeros(cap, IPV4_NET_DT)
    s = SpfComputationStruct(0, 0, 0, 0, cap, net.ctypes.data, rtr.ctypes.data, ext.ctypes.data)
    rc = fn(tr.ctypes.data, len(tr), C.byref(s))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, "spf_computation_type failed")
    pairs = lambda a, k: [(int(x["addr"]), int(x["mask"])) for x in a[:k]]
    return s.kind, pairs(net, s.n_inter_network), [int(x) for x in rtr[: s.n_inter_router]], pairs(ext, s.n_external)


def flat_update(flat: "Flat", new_area: Ospfv2Area, triggers):
    """hspf_ospfv2_flat_update: returns (kind, edges, costs); the Flat object's numpy views are refreshed."""
    lib = flat.lib
    lib.hspf_ospfv2_flat_update.argtypes = [C.c_void_p, C.POINTER(AreaStruct), C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32),
                                            C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    tr = np.ascontiguousarray(triggers, TRIGGER_DT)
    cap = max(int(flat.csr.n_edges), 1)
    edges, costs = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
    kind, n = C.c_uint32(), C.c_uint32()
    s = new_area.as_struct()
    rc = lib.hspf_ospfv2_flat_update(flat.handle, C.byref(s), tr.ctypes.data, len(tr), C.byref(kind), edges.ctypes.data,
                                     costs.ctypes.data, cap, C.byref(n))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, "hspf_ospfv2_flat_update failed")
    flat.area, flat._s = new_area, s            # the native flat now refers to the new image
    flat._load()
    return kind.value, edges[: n.value].copy(), costs[: n.value].copy()


# ------------------------------------------------------------------- batched route stage
CELL_DT = np.dtype([("nh_mask", "<u8"), ("lasthop_mask", "<u8"), ("winner", "<u4"), ("metric", "<u2"),
                    ("flags", "u1"), ("_pad", "u1")])
CONTRIB_DT = np.dtype([("vertex", "<u4"), ("origin_id", "<u4"), ("metric", "<u2"), ("sid_class", "<u2"),
                       ("is_network", "u1"), ("_pad", "u1", (3,))])
CELL_PRESENT, CELL_CONNECTED, CELL_MIXED_SID = 1, 2, 4


class RouteTable(route_table.RouteTable):
    """hspf_ospfv2_rtable: the area's prefixes in route-table order and their advertisers (host);
    `upload(ctx)` copies it to the device for hspf_ospfv2_routes_batch."""

    api, contrib_dt = "hspf_ospfv2", CONTRIB_DT

    def __init__(self, flat: Flat):
        self.flat = flat                      # the table is built from the flat's area image
        super().__init__(capi.load_library().hspf_ospfv2_rtable_create, flat.handle)
        pp, pl = C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint32)()
        self._call("arrays", C.byref(pp), C.byref(pl), None, None)
        self.prefix = route_table.copy_records(pp, self.n_prefixes, np.uint32)
        self.plen = route_table.copy_records(pl, self.n_prefixes, np.uint32)


@dataclass
class BatchRoutes:
    cells: np.ndarray          # [n_roots, P] CELL_DT
    status: np.ndarray         # [n_roots] job status words
    gather_off: np.ndarray     # [n_roots + 1]
    gather_v: np.ndarray
    gather_nh: np.ndarray
    device_ms: tuple           # (SPT batch, route kernel)
    rc: int = 0

    def gather(self, j):
        a, b = int(self.gather_off[j]), int(self.gather_off[j + 1])
        return self.gather_v[a:b], self.gather_nh[a:b]


def run_area_batch(ctx: capi.Context, area: Ospfv2Area, root_router_ids, n_prefixes=None) -> BatchRoutes:
    """hspf_ospfv2_run_area_batch: SPT + intra-area route cells of every listed root router, on the device."""
    lib = ctx.lib
    roots = np.ascontiguousarray(root_router_ids, np.uint32)
    n = len(roots)
    s = area.as_struct()
    if n_prefixes is None:
        n_prefixes = len(area.links) + len(area.network_lsas)       # upper bound
    u32p, u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
    for _ in range(2):
        cells = np.zeros((n, max(n_prefixes, 1)), CELL_DT)
        status = np.zeros(n, np.uint32)
        goff = np.zeros(n + 1, np.uint32)
        gcap = 128 * max(n, 1)
        gv, gnh = np.zeros(gcap, np.uint32), np.zeros(gcap, np.uint64)
        P = C.c_uint32()
        ms = (C.c_double * 2)()
        rc = lib.hspf_ospfv2_run_area_batch(ctx.handle, C.byref(s), roots.ctypes.data_as(u32p), n, cells.ctypes.data,
                                            cells.size, C.byref(P), status.ctypes.data_as(u32p), goff.ctypes.data_as(u32p),
                                            gv.ctypes.data_as(u32p), gnh.ctypes.data_as(u64p), gcap, ms)
        if rc == capi.HSPF_E_NOMEM and P.value != cells.shape[1]:
            n_prefixes = P.value
            continue
        break
    if rc not in (capi.HSPF_OK, capi.HSPF_E_JOB_STATUS):
        raise capi.HspfError(rc, ctx.last_error())
    if P.value != cells.shape[1]:             # the call wrote rows of P cells into the flat buffer
        cells = cells.reshape(-1)[: n * P.value].reshape(n, P.value)
    G = int(goff[n])
    return BatchRoutes(cells, status, goff, gv[:G].copy(), gnh[:G].copy(), (ms[0], ms[1]), rc)


def routes_batch_device(ctx: capi.Context, rt: RouteTable, n_jobs: int, rs, cells_ptr: int, n_gather: int = 0,
                        gather_job_ptr: int = 0, gather_v_ptr: int = 0, gather_nh_ptr: int = 0):
    """hspf_ospfv2_routes_batch / _batch16 over DEVICE planes (rs: capi.ResultStruct or capi.Result16Struct
    holding device pointers); cells_ptr: device buffer of n_jobs * rt.n_prefixes cells.  Enqueued on the ctx
    stream; the table must have been uploaded."""
    lib = ctx.lib
    narrow = isinstance(rs, capi.Result16Struct)
    fn = lib.hspf_ospfv2_routes_batch16 if narrow else lib.hspf_ospfv2_routes_batch
    rc = fn(ctx.handle, rt.handle, n_jobs, C.byref(rs), cells_ptr, n_gather, gather_job_ptr or None,
            gather_v_ptr or None, gather_nh_ptr or None)
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, ctx.last_error())


def routes_delta_device(ctx: capi.Context, rt: RouteTable, n_jobs: int, rs, base_ptr: int, n_base: int, base_of_ptr: int,
                        job_out_ptr: int, records_ptr: int, cap: int, n_records_ptr: int):
    """hspf_ospfv2_routes_delta / _delta16 over DEVICE planes (rs as for routes_batch_device): each job's cells compared
    with its base row of base_ptr ([n_base, rt.n_prefixes] cells; base_of_ptr: [n_jobs] u32 rows, 0 for row 0 of
    every job), without storing them.  job_out_ptr: [n_jobs] route_table.DELTA_JOB_DT; records_ptr: [cap]
    route_table.DELTA_DT in (job, prefix) order (0 or cap 0: summaries only); n_records_ptr: u64 total.  All device
    pointers; enqueued on the ctx stream."""
    lib = ctx.lib
    narrow = isinstance(rs, capi.Result16Struct)
    fn = lib.hspf_ospfv2_routes_delta16 if narrow else lib.hspf_ospfv2_routes_delta
    rc = fn(ctx.handle, rt.handle, n_jobs, C.byref(rs), base_ptr or None, n_base, base_of_ptr or None, job_out_ptr or None,
            records_ptr or None, cap, n_records_ptr or None)
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, ctx.last_error())


def routes_from_cells(area: Ospfv2Area, rt: RouteTable, cells: np.ndarray, gather_v, gather_nh) -> Ospfv2Result:
    """hspf_ospfv2_routes_from_cells (host): one job's cells -> routes and next hops as run_area returns them
    for area.router_id.  rc HSPF_E_UNSUPPORTED is returned in the result (caller: area_from_planes)."""
    lib = capi.load_library()
    cells = np.ascontiguousarray(cells, CELL_DT)
    assert cells.shape == (rt.n_prefixes,)
    gv = np.ascontiguousarray(gather_v, np.uint32)
    gn = np.ascontiguousarray(gather_nh, np.uint64)
    res = _call_run_area(lib.hspf_ospfv2_routes_from_cells, area, (),
                         (rt.handle, cells.ctypes.data, gv.ctypes.data_as(C.POINTER(C.c_uint32)),
                          gn.ctypes.data_as(C.POINTER(C.c_uint64)), len(gv)))
    if res.rc not in (capi.HSPF_OK, capi.HSPF_E_UNSUPPORTED):
        raise capi.HspfError(res.rc, "hspf_ospfv2_routes_from_cells failed")
    return res


# ------------------------------------------------------------------------------ synthetic
RID_BASE = 0x0A000001        # 10.0.0.1 + i
P2P_BASE = 0xAC100000        # 172.16.0.0/12, one /30 per adjacency
LAN_BASE = 0xC0A80000        # 192.168.0.0/16..., one /24 per LAN


def synth_area(t: Topology, root: int = 0, sr: bool = False, max_paths: int = 16,
               reverse_sort_keys: bool = True) -> Ospfv2Area:
    """OSPFv2 single-area LSDB for topology `t` as seen by router `root`
    (SURVEY.md §8d): per router one Router-LSA with, per adjacency, a p2p link + a
    /30 stub link, per LAN a transit link, and a /32 loopback stub (metric 0); one
    Network-LSA per LAN originated by its first member (the DR).  With sr=True every
    router advertises SR-Algo SPF, SRGB 16000+8000 and a Prefix-SID (index i, NP
    flag) for its loopback."""
    R = t.n_routers
    rid = lambda i: RID_BASE + int(i)
    per = [[] for _ in range(R)]      # per router: list of (link_id, link_data, metric, type)
    root_ifaces = []                  # (if_type, [(nbr_rid, nbr_src)], own_addr, mask)
    for k in range(t.n_p2p):
        a, b = int(t.p2p_a[k]), int(t.p2p_b[k])
        net = P2P_BASE + 4 * k
        per[a].append((rid(b), net + 1, int(t.p2p_cost_ab[k]), LINK_P2P))
        per[a].append((net, 0xFFFFFFFC, int(t.p2p_cost_ab[k]), LINK_STUB))
        per[b].append((rid(a), net + 2, int(t.p2p_cost_ba[k]), LINK_P2P))
        per[b].append((net, 0xFFFFFFFC, int(t.p2p_cost_ba[k]), LINK_STUB))
        if a == root:
            root_ifaces.append((IF_P2P, [(rid(b), net + 2)], net + 1, 0xFFFFFFFC))
        if b == root:
            root_ifaces.append((IF_P2P, [(rid(a), net + 1)], net + 2, 0xFFFFFFFC))
    net_lsas, attached = [], []
    for li, (members, costs) in enumerate(t.lans):
        net = LAN_BASE + 256 * li
        dr = members[0]
        dr_addr = net + 1
        for pos, (m, c) in enumerate(zip(members, costs)):
            per[m].append((dr_addr, net + 1 + pos, int(c), LINK_TRANSIT))
            if m == root:
                nb = [(rid(o), net + 1 + p2) for p2, o in enumerate(members) if o != m]
                root_ifaces.append((IF_BROADCAST, nb, net + 1 + pos, 0xFFFFFF00))
        net_lsas.append((rid(dr), dr_addr, 0xFFFFFF00, len(attached), len(members)))
        attached += sorted(rid(m) for m in members)
    for i in range(R):
        per[i].append((rid(i), 0xFFFFFFFF, 0, LINK_STUB))
    n_links = sum(len(p) for p in per)
    links = np.zeros(n_links, LINK_DT)
    rl = np.zeros(R, ROUTER_LSA_DT)
    off = 0
    for i in range(R):
        rl[i] = (rid(i), rid(i), 1, 0, 0x02, off, len(per[i]), )
        for (lid, ld, m, ty) in per[i]:
            links[off] = (lid, ld, m, ty, 0)
            off += 1
    nl = np.zeros(len(net_lsas), NETWORK_LSA_DT)
    for i, (adv, lsid, mask, ao, na) in enumerate(net_lsas):
        nl[i] = (adv, lsid, mask, 1, 0, ao, na)
    order = np.lexsort((nl["lsa_id"], nl["adv_rtr"])) if len(nl) else np.zeros(0, np.int64)
    nl = nl[order]
    # local interfaces of the root, in link order == name order; the root's link_pos
    # counts non-stub links in Router-LSA order, which is the order generated above
    ifaces = np.zeros(len(root_ifaces), IFACE_DT)
    nbrs, addrs = [], []
    for i, (ty, nb, own, mask) in enumerate(root_ifaces):
        sk = (len(root_ifaces) - i) if reverse_sort_keys else i + 1
        ifaces[i] = (100 + i, sk, ty, (0, 0, 0), len(addrs), 1, len(nbrs), len(nb))
        addrs.append((own, mask))
        nbrs += nb
    area = Ospfv2Area(router_id=rid(root), max_paths=max_paths, sr_enabled=sr)
    area.router_lsas, area.links, area.network_lsas = rl, links, nl
    area.attached = np.asarray(attached, dtype=np.uint32)
    area.ifaces = ifaces
    area.iface_addrs = np.asarray(addrs, dtype=IPV4_NET_DT) if addrs else np.zeros(0, IPV4_NET_DT)
    area.nbrs = np.asarray(nbrs, dtype=NBR_DT) if nbrs else np.zeros(0, NBR_DT)
    area.ifnames = [f"eth{i:05d}" for i in range(len(root_ifaces))]
    if sr:
        ri = np.zeros(R, RI_LSA_DT)
        sg = np.zeros(R, SRGB_DT)
        ep = np.zeros(R, EXT_PREFIX_DT)
        for i in range(R):
            ri[i] = (rid(i), 0x04000000, 1, 1, 1, i, 1)
            sg[i] = (16000, 8000, 0, (0, 0, 0))
            ep[i] = (rid(i), rid(i), 0xFFFFFFFF, 1, 1, 1, PSID_NP, 0, (0, 0), i % 8000)
        area.ri_lsas, area.srgbs, area.ext_prefixes = ri, sg, ep
    return area
