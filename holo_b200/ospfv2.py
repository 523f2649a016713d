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
             route_table.DELTA_DT.itemsize, route_table.DELTA_JOB_DT.itemsize, ospf_rib.RIB_CELL_DT.itemsize])


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
    route_table.call_stage(ctx, "hspf_ospfv2_routes_batch", rs, rt.handle, n_jobs, C.byref(rs), cells_ptr, n_gather,
                           gather_job_ptr or None, gather_v_ptr or None, gather_nh_ptr or None)


def routes_delta_device(ctx: capi.Context, rt: RouteTable, n_jobs: int, rs, base_ptr: int, n_base: int, base_of_ptr: int,
                        job_out_ptr: int, records_ptr: int, cap: int, n_records_ptr: int):
    """hspf_ospfv2_routes_delta / _delta16 over DEVICE planes (rs as for routes_batch_device): each job's cells compared
    with its base row of base_ptr ([n_base, rt.n_prefixes] cells; base_of_ptr: [n_jobs] u32 rows, 0 for row 0 of
    every job), without storing them.  job_out_ptr: [n_jobs] route_table.DELTA_JOB_DT; records_ptr: [cap]
    route_table.DELTA_DT in (job, prefix) order (0 or cap 0: summaries only); n_records_ptr: u64 total.  All device
    pointers; enqueued on the ctx stream."""
    route_table.call_stage(ctx, "hspf_ospfv2_routes_delta", rs, rt.handle, n_jobs, C.byref(rs), base_ptr or None, n_base,
                           base_of_ptr or None, job_out_ptr or None, records_ptr or None, cap, n_records_ptr or None)


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


def inter_area_view(area: Ospfv2Area, seed: int, n_abr: int = 4, n_asbr: int = 3, n_inter: int = 60, n_ext: int = 50,
                    unreachable_abr: bool = True, n_overlap: int = 8, n_fresh: int = 10, n_ext_only: int = 8):
    """A single-area LSDB as one area of a multi-area domain: returns (area, summaries, externals) for
    ospf_rib (hl_ospfv2_summary_lsa[] in LsaKey order, hl_ospfv2_external_lsa[] in LSDB order).  Seeded and
    independent of area.router_id, so every root of one topology sees the same LSDB.
      * n_abr routers get the B flag, n_asbr others the E flag; with unreachable_abr a router with B|E and no
        adjacency is added (its LSAs exist, no job reaches it);
      * type-3 LSAs from the ABRs (and from a router without the B flag and an unknown router, which no job may
        use) for intra-area prefixes, new prefixes, prefixes with host bits and the default route; type-4 LSAs
        for in-area ASBRs (the last one usable replaces the ASBR's intra-area entry) and ASBRs outside the area;
        type-5 LSAs of type 1 and 2 from those ASBRs, from routers without the E flag, from unknown routers and
        from ordinary routers (self-originated for the job rooted there);
      * metrics from small sets, so that ties are common; some LSAs at maxage or at LSInfinity.
    Prefixes: n_overlap of the area's own, n_fresh new /24s (< 2048) and three with host bits or the default route,
    for both LSA types; n_ext_only /24s named by type-5 LSAs only, the first four by type-2 LSAs only."""
    from . import ospf_rib
    rng = np.random.default_rng(seed)
    a = Ospfv2Area(**{k: getattr(area, k) for k in area.__dataclass_fields__})
    rl, links = area.router_lsas.copy(), area.links.copy()
    rids = [int(x) for x in rl["adv_rtr"]]
    pick = [int(x) for x in rng.permutation(rids)]
    abrs, asbrs, plain = pick[:n_abr], pick[n_abr:n_abr + n_asbr], pick[n_abr + n_asbr:]
    for i, r in enumerate(rids):
        rl["flags"][i] |= (0x01 if r in abrs else 0) | (0x02 if r in asbrs else 0)
    lost = []
    if unreachable_abr:
        lost = [max(rids) + 0x100]
        rl = np.concatenate([rl, np.array([(lost[0], lost[0], 1, 0x03, 0x02, len(links), 1)], ROUTER_LSA_DT)])
        links = np.concatenate([links, np.array([(lost[0], 0xFFFFFFFF, 0, LINK_STUB, 0)], LINK_DT)])
    a.router_lsas, a.links = rl, links
    stubs = sorted({(int(l["link_id"]) & int(l["link_data"]), int(l["link_data"])) for l in links if l["link_type"] == LINK_STUB})
    nets = [(int(n["lsa_id"]) & int(n["mask"]), int(n["mask"])) for n in area.network_lsas]
    intra = [stubs[int(i)] for i in rng.choice(len(stubs), min(len(stubs), n_overlap), replace=False)] + nets[:2]
    fresh = [(0x0AC80000 + (i << 8), 0xFFFFFF00) for i in range(n_fresh)]
    pool = intra + fresh + [(0x0AC80005, 0xFFFFFF00), (0x0AC80105, 0xFFFFFF00), (0, 0)]
    metric = lambda: int(rng.choice([1, 10, 10, 20, 30])) if rng.random() > 0.05 else ospf_rib.LSA_INFINITY
    maxage = lambda: int(rng.random() < 0.06)
    sums = []
    advs3 = abrs + lost + plain[:1] + [0x7F000001]                # the last two: never an ABR of the area
    for _ in range(n_inter):
        p, m = pool[int(rng.integers(0, len(pool)))]
        sums.append((int(rng.choice(advs3)), p, m, metric(), 3, maxage(), (0, 0)))
    outside = [0x0B000001 + i for i in range(3)]                  # ASBRs in other areas
    for asbr in asbrs[:2] + outside:
        for abr in rng.choice(abrs + lost, int(rng.integers(1, 4)), replace=False):
            sums.append((int(abr), asbr, 0, metric(), 4, maxage(), (0, 0)))
    sums.sort(key=lambda x: (x[4], x[0], x[1]))
    summaries = np.asarray(sums, ospf_rib.SUMMARY_LSA_DT)
    ext = []
    advs5 = asbrs + outside + lost + plain[:3] + abrs[:1] + [0x7F000002]
    pool5 = pool + [(0x0C000000 + (i << 8), 0xFFFFFF00) for i in range(n_ext_only)]     # prefixes only externals name
    for _ in range(n_ext):
        p, m = pool5[int(rng.integers(0, len(pool5)))]
        e_bit = 1 if 0x0C000000 <= p < 0x0C000400 else int(rng.integers(0, 2))   # four prefixes of type-2 LSAs only
        ext.append((int(rng.choice(advs5)), p, m, int(rng.choice([1, 5, 5, 20])) if rng.random() > 0.05 else ospf_rib.LSA_INFINITY,
                    0, int(rng.integers(0, 4)), e_bit, maxage(), (0, 0)))
    ext.sort(key=lambda x: (x[0], x[1]))
    externals = np.asarray(ext, ospf_rib.EXTERNAL_LSA_DT)
    return a, summaries, externals


ABR_ROUTER_ID = 0x0AFF0001   # 10.255.0.1: the router abr_view roots every area at
ABR_TIE_ASBR = 0x0B0000F1    # an ASBR outside the domain that every non-backbone area of abr_view names


def _dist_from(flat: Flat, root: int):
    """Unperturbed SPT distances of `flat` from `root` (the generator's own Dijkstra, to place equal-cost routes)."""
    import heapq
    c = flat.csr
    dist = np.full(c.n_vertices, np.iinfo(np.int64).max, np.int64)
    dist[root] = 0
    heap = [(0, root)]
    while heap:
        d, v = heapq.heappop(heap)
        if d > dist[v]:
            continue
        for e in range(int(c.row_ptr[v]), int(c.row_ptr[v + 1])):
            w, nd = int(c.col[e]), d + int(c.cost[e])
            if nd < dist[w]:
                dist[w] = nd
                heapq.heappush(heap, (nd, w))
    return dist


def _with_stubs(area: Ospfv2Area, adds: dict) -> Ospfv2Area:
    """area with stub links appended to Router-LSAs: adds {router_id: [(prefix, mask, metric)]}.  Appended after each
    LSA's own links, so the root's non-stub link positions do not move."""
    rl, links = area.router_lsas.copy(), []
    for i in range(len(rl)):
        o, n = int(rl["link_off"][i]), int(rl["n_links"][i])
        extra = [(p, m, metric, LINK_STUB, 0) for (p, m, metric) in adds.get(int(rl["adv_rtr"][i]), [])]
        rl["link_off"][i] = len(links)
        rl["n_links"][i] = n + len(extra)
        links += [tuple(x) for x in area.links[o: o + n].tolist()] + extra
    a = Ospfv2Area(**{k: getattr(area, k) for k in area.__dataclass_fields__})
    a.router_lsas, a.links = rl, np.asarray(links, LINK_DT) if links else np.zeros(0, LINK_DT)
    return a


def abr_view(topos: list, seed: int, area_ids=None, roots=None, max_paths: int = 16, n_shared: int = 6,
             v_flag_area: int | None = 1, **inter_kw):
    """A multi-area domain as one ABR sees it: returns (areas [Ospfv2Area], summaries [SUMMARY_LSA_DT[] per area],
    externals EXTERNAL_LSA_DT[]), the areas in instance order.  Area k is synth_area(topos[k], root=roots[k]) with its
    router ids, addresses, interface sort keys and ifindexes moved into ranges of its own; the root becomes router
    ABR_ROUTER_ID in every area, with the B flag.  Seeded.
      * area 0 (area_ids[0], 0 by default) carries inter_area_view's type-3/4/5 load (type-4 LSAs naming the root
        dropped); every other area gets type-3 LSAs from two ABRs of its own, for some of area 0's prefixes and new
        ones (read only while one area is active, and by the transit-area step), and a type-4 LSA;
      * shared prefixes: area 0's first LAN is also a LAN of area 1 (transit-network overwrite across areas); n_shared
        stubs of area 0's neighbours of the root are also stubs of a neighbour of the root in the other areas, half at
        the same metric (atoms merge across areas), half not;
      * an ASBR in each non-backbone area (its farthest router) with externals of its own, also named by a backbone
        type-4 LSA at metric 1; an ASBR named by a type-4 LSA of every non-backbone area at one forwarding metric;
      * with v_flag_area, a router of that area (not the root) gets the V flag."""
    from . import ospf_rib
    rng = np.random.default_rng(seed)
    A = len(topos)
    area_ids = list(area_ids) if area_ids is not None else list(range(A))
    roots = list(roots) if roots is not None else [0] * A
    areas = []
    for k, (t, r) in enumerate(zip(topos, roots)):
        a = synth_area(t, root=r, max_paths=max_paths)
        root_rid = RID_BASE + r

        def rmap(x, k=k, root_rid=root_rid):
            x = np.asarray(x, np.uint64)
            out = x.copy()
            is_rid = (x >> 24) == 10
            out = np.where(is_rid, x + (k << 20), out)
            out = np.where(x == root_rid, ABR_ROUTER_ID, out)
            out = np.where((x >> 20) == (P2P_BASE >> 20), x + (k << 18), out)
            lan = (x >> 16) == (LAN_BASE >> 16)
            lan_to = x + (k << 16)
            if k == 1:                       # area 1's LAN 0 is area 0's LAN 0, hosts moved up by 100
                lan_to = np.where(lan & (((x - LAN_BASE) >> 8) == 0), x + 100, lan_to)
            out = np.where(lan, lan_to, out)
            return out.astype(np.uint32)

        a.router_id = ABR_ROUTER_ID
        a.area_id = area_ids[k]
        rl = a.router_lsas.copy()
        rl["adv_rtr"], rl["lsa_id"] = rmap(rl["adv_rtr"]), rmap(rl["lsa_id"])
        links = a.links.copy()
        links["link_id"] = rmap(links["link_id"])
        non_stub = links["link_type"] != LINK_STUB
        links["link_data"] = np.where(non_stub, rmap(links["link_data"]), links["link_data"])
        nl = a.network_lsas.copy()
        nl["adv_rtr"], nl["lsa_id"] = rmap(nl["adv_rtr"]), rmap(nl["lsa_id"])
        a.attached = rmap(a.attached)
        nb = a.nbrs.copy()
        for f in nb.dtype.names:
            if nb.dtype[f] == np.uint32:
                nb[f] = rmap(nb[f])
        ia = a.iface_addrs.copy()
        ia["addr"] = rmap(ia["addr"])
        ifs = a.ifaces.copy()
        ifs["sort_key"] += 1000 * k
        ifs["ifindex"] += 1000 * k
        order = np.lexsort((rl["lsa_id"], rl["adv_rtr"]))
        rl = rl[order]
        rl["flags"][rl["adv_rtr"] == ABR_ROUTER_ID] |= 0x01
        a.router_lsas, a.links, a.nbrs, a.iface_addrs, a.ifaces = rl, links, nb, ia, ifs
        a.network_lsas = nl[np.lexsort((nl["lsa_id"], nl["adv_rtr"]))] if len(nl) else nl
        areas.append(a)
    # type-3/4/5 load of area 0 (the backbone unless area_ids say otherwise)
    a0, sums0, ext = inter_area_view(areas[0], seed, **inter_kw)
    a0.router_lsas["flags"][a0.router_lsas["adv_rtr"] == ABR_ROUTER_ID] |= 0x01
    sums0 = sums0[~((sums0["lsa_type"] == 4) & (sums0["lsa_id"] == ABR_ROUTER_ID))]
    areas[0] = a0
    flat0 = Flat(a0)
    d0 = _dist_from(flat0, flat0.router_vertex(ABR_ROUTER_ID))
    stubs0 = [(int(l["link_id"]), int(l["link_data"]), int(l["metric"]), int(r["adv_rtr"]))
              for r in a0.router_lsas for l in a0.links[int(r["link_off"]): int(r["link_off"]) + int(r["n_links"])]
              if l["link_type"] == LINK_STUB and int(r["adv_rtr"]) != ABR_ROUTER_ID]
    summaries, ext_rows = [sums0], [tuple(x) for x in ext.tolist()]
    bb_abrs = [int(r) for r, f in zip(a0.router_lsas["adv_rtr"], a0.router_lsas["flags"])
               if f & 0x01 and int(r) != ABR_ROUTER_ID and flat0.router_vertex(int(r)) != 0xFFFFFFFF
               and d0[flat0.router_vertex(int(r))] < 1 << 40]
    extra4 = []
    inter_prefixes = sorted({(int(s["lsa_id"]), int(s["mask"])) for s in sums0 if s["lsa_type"] == 3})
    for k in range(1, A):
        a = areas[k]
        flat = Flat(a)
        rv = flat.router_vertex(ABR_ROUTER_ID)
        dk = _dist_from(flat, rv)
        others = [int(x) for x in a.router_lsas["adv_rtr"] if int(x) != ABR_ROUTER_ID]
        reach = {int(flat.ids[v]): int(dk[v]) for v in range(len(flat.ids)) if flat.is_router[v] and dk[v] < 1 << 40}
        pick = [int(x) for x in rng.permutation([r for r in others if r in reach])]
        abrs, vrtr = pick[:2], pick[3]
        asbr = max((r for r in pick[2:] if r != vrtr), key=lambda r: (reach[r], r))     # the farthest router
        # shared stubs: the same prefix at a router of this area, half of them at the metric that ties area 0's route
        adds = {}
        shared = [stubs0[int(i)] for i in rng.choice(len(stubs0), min(n_shared, len(stubs0)), replace=False)]
        for j, (p, m, metric, adv) in enumerate(shared):
            want = int(d0[flat0.router_vertex(adv)]) + metric
            cand = [(rid, d) for rid, d in reach.items() if rid != ABR_ROUTER_ID and d <= want - 1]
            if not cand or want > 0xFFFF:
                continue
            rid, d = cand[int(rng.integers(0, len(cand)))]
            m2 = want - d if j % 2 == 0 else want - d + int(rng.choice([-1, 5]))
            adds.setdefault(rid, []).append((p, m, max(int(m2), 1)))
        a = _with_stubs(a, adds)
        rl = a.router_lsas
        for rid in abrs:
            rl["flags"][rl["adv_rtr"] == rid] |= 0x01
        rl["flags"][rl["adv_rtr"] == asbr] |= 0x02
        if v_flag_area is not None and k == v_flag_area:
            rl["flags"][rl["adv_rtr"] == vrtr] |= 0x04
        areas[k] = a
        pool = [(p, m) for (p, m, _, _) in shared] + inter_prefixes[:6] + [(0x0AD00000 + (k << 12) + (i << 8), 0xFFFFFF00)
                                                                          for i in range(4)]
        sums = []
        for (p, m) in pool:
            for abr in abrs[: int(rng.integers(1, 3))]:
                sums.append((abr, p, m, int(rng.choice([1, 5, 10, 20])), 3, 0, (0, 0)))
        sums.append((abrs[0], 0x0B000001, 0, 10, 4, 0, (0, 0)))
        # an ASBR outside the area named by every non-backbone area at one forwarding metric: with one active area
        # the entries tie across areas and the higher area id wins
        sums.append((abrs[0], ABR_TIE_ASBR, 0, max(1, 1000 - reach[abrs[0]]), 4, 0, (0, 0)))
        # this area's ASBR, also named by a backbone type-4 LSA through the nearest backbone ABR at metric 1: an
        # intra-area entry through a non-backbone area beats the (usually shorter) backbone entry
        if bb_abrs:
            near = min(bb_abrs, key=lambda r: (int(d0[flat0.router_vertex(r)]), r))
            extra4.append((near, asbr, 0, 1, 4, 0, (0, 0)))
        sums.sort(key=lambda x: (x[4], x[0], x[1]))
        summaries.append(np.asarray(sums, ospf_rib.SUMMARY_LSA_DT))
        for i in range(3):
            ext_rows.append((asbr, 0x0E000000 + (k << 16) + (i << 8), 0xFFFFFF00, int(rng.choice([1, 5, 20])), 0, k,
                             int(i % 2), 0, (0, 0)))
        if inter_prefixes:                                           # an ASBR of area 0's view seen from this area too
            ext_rows.append((0x0B000001, 0x0E000000 + (k << 16) + 0xF00, 0xFFFFFF00, 7, 0, 0, 1, 0, (0, 0)))
    if A > 1:
        for i in range(2):
            ext_rows.append((ABR_TIE_ASBR, 0x0E0F0000 + (i << 8), 0xFFFFFF00, 3, 0, 9, i, 0, (0, 0)))
    if extra4:
        s0 = sorted([tuple(x) for x in summaries[0].tolist()] + extra4, key=lambda x: (x[4], x[0], x[1]))
        summaries[0] = np.asarray(s0, ospf_rib.SUMMARY_LSA_DT)
    ext_rows.sort(key=lambda x: (x[0], x[1]))
    return areas, summaries, np.asarray(ext_rows, ospf_rib.EXTERNAL_LSA_DT)


def _area_remap(a: Ospfv2Area, k: int, idmap: dict) -> Ospfv2Area:
    """A copy of synth_area's image as area k of a multi-area domain: router ids moved up by k << 20, then renamed by
    idmap (the routers of this area that are also routers of area 0 keep their area-0 ids), p2p and LAN addresses,
    interface sort keys and ifindexes moved into ranges of area k."""
    a = Ospfv2Area(**{f: getattr(a, f) for f in a.__dataclass_fields__})

    def rmap(x):
        x = np.asarray(x, np.uint64)
        out = np.where((x >> 24) == 10, x + (k << 20), x)
        for old, new in idmap.items():
            out = np.where(out == old + (k << 20), new, out)
        out = np.where((x >> 20) == (P2P_BASE >> 20), x + (k << 18), out)
        out = np.where((x >> 16) == (LAN_BASE >> 16), x + (k << 16), out)
        return out.astype(np.uint32)

    a.router_id = int(rmap([a.router_id])[0])
    a.area_id = k
    rl = a.router_lsas.copy()
    rl["adv_rtr"], rl["lsa_id"] = rmap(rl["adv_rtr"]), rmap(rl["lsa_id"])
    links = a.links.copy()
    links["link_id"] = rmap(links["link_id"])
    non_stub = links["link_type"] != LINK_STUB
    links["link_data"] = np.where(non_stub, rmap(links["link_data"]), links["link_data"])
    nl = a.network_lsas.copy()
    nl["adv_rtr"], nl["lsa_id"] = rmap(nl["adv_rtr"]), rmap(nl["lsa_id"])
    a.attached = rmap(a.attached)
    nb = a.nbrs.copy()
    for f in nb.dtype.names:
        if nb.dtype[f] == np.uint32:
            nb[f] = rmap(nb[f])
    ia = a.iface_addrs.copy()
    ia["addr"] = rmap(ia["addr"])
    ifs = a.ifaces.copy()
    ifs["sort_key"] += 1000 * k
    ifs["ifindex"] += 1000 * k
    order = np.lexsort((rl["lsa_id"], rl["adv_rtr"]))
    a.router_lsas, a.links, a.nbrs, a.iface_addrs, a.ifaces = rl[order], links, nb, ia, ifs
    a.network_lsas = nl[np.lexsort((nl["lsa_id"], nl["adv_rtr"]))] if len(nl) else nl
    return a


def _set_flags(a: Ospfv2Area, flags: dict) -> Ospfv2Area:
    rl = a.router_lsas.copy()
    for rid, f in flags.items():
        rl["flags"][rl["adv_rtr"] == rid] |= f
    a.router_lsas = rl
    return a


def backbone_view(t0: Topology, t1: Topology, seed: int, r: int = 0, borders=((1, 0), (2, 1), (3, 2)),
                  max_paths: int = 16, n_ext_keys: int = 3, area1_asbrs: int = 0, area1_ext: int = 4):
    """A backbone router R of area 0 and the area border routers ("borders") of one other area 1, each as its own
    image.  Seeded.  Area 0 is synth_area(t0) (router i is RID_BASE + i), area 1 synth_area(t1) moved into ranges of
    its own, except that border (i0, i1) is router i0 of t0 and router i1 of t1, with one router id and the B flag in
    both areas.  Returns a dict:
      r_area        R's area-0 image (router r of t0);
      summaries0    area 0's type-3 LSAs (LsaKey order): each border's for the area-1 stub prefixes it reaches, at
                    its distance plus the stub metric (what a job replaces);
      externals     an ASBR of area 0 (the E flag) with type-5 LSAs for n_ext_keys area-1 loopbacks (prefixes that
                    are also keys) and for one prefix of its own;
      borders       per border (areas [area 0 image, area 1 image], area ids, summaries per area) in that area order,
                    except that the first border lists area 1 first;
      shared        a /24 that is a stub of a neighbour of the first border in area 0 and in area 1, at metrics that
                    tie at that border (its route there is intra-area in both areas and carries area-0 atoms).
    area1_asbrs = k > 0 (drawn from a generator of its own, so that every other part is as without it): k routers of
    area 1 get the E flag ("area1_asbrs" in the dict) and area1_ext type-5 LSAs each, both E-bit values, on /24s that
    the next ASBR shares in half, plus the area-0 ASBR's own /24 at its type-2 metric; summaries0 then also holds each
    border's type-4 LSAs for those it reaches in area 1, at that distance.  A border left out of a backbone table keeps
    its type-3 / type-4 LSAs as another ABR's static ones."""
    from . import ospf_rib
    rng = np.random.default_rng(seed)
    rid0 = lambda i: RID_BASE + int(i)
    idmap = {rid0(i1): rid0(i0) for i0, i1 in borders}
    bids = [rid0(i0) for i0, _ in borders]
    cand = [i for i in range(t0.n_routers) if i != r and rid0(i) not in bids]
    asbr = rid0(cand[int(rng.integers(0, len(cand)))])
    f0 = {b: 0x01 for b in bids}
    f0[asbr] = 0x02
    img0 = lambda i: _set_flags(synth_area(t0, root=i, max_paths=max_paths), f0)
    img1 = lambda i: _set_flags(_area_remap(synth_area(t1, root=i, max_paths=max_paths), 1, idmap), {b: 0x01 for b in bids})
    r_area = img0(r)
    b0 = [img0(i0) for i0, _ in borders]
    b1 = [img1(i1) for _, i1 in borders]
    asbrs1 = []
    if area1_asbrs:
        rng1 = np.random.default_rng([seed, 0xA5B])
        cand1 = sorted({int(x["adv_rtr"]) for x in b1[0].router_lsas} - set(bids))
        asbrs1 = sorted(cand1[int(i)] for i in rng1.choice(len(cand1), min(area1_asbrs, len(cand1)), replace=False))
        b1 = [_set_flags(a, {x: 0x02 for x in asbrs1}) for a in b1]
    # the shared prefix: a nearest neighbour of the first border in each area, at metrics that tie there
    def nearest(a):
        fl = Flat(a)
        d = _dist_from(fl, fl.router_vertex(a.router_id))
        vs = [v for v in range(len(fl.ids)) if fl.is_router[v] and 0 < d[v] < 1 << 40]
        v = min(vs, key=lambda v: (int(d[v]), int(fl.ids[v])))
        return int(fl.ids[v]), int(d[v])
    (n0, d0), (n1, d1) = nearest(b0[0]), nearest(b1[0])
    shared = (0x0AEE0000, 0xFFFFFF00)
    m0, m1 = 10 + max(0, d1 - d0), 10 + max(0, d0 - d1)
    add0, add1 = {n0: [(shared[0], shared[1], m0)]}, {n1: [(shared[0], shared[1], m1)]}
    r_area = _with_stubs(r_area, add0)
    b0 = [_with_stubs(a, add0) for a in b0]
    b1 = [_with_stubs(a, add1) for a in b1]
    # the borders' type-3 LSAs into area 0: area-1 stubs that are not area-0 prefixes
    stubs0 = {(int(l["link_id"]), int(l["link_data"])) for l in r_area.links if l["link_type"] == LINK_STUB}
    sums0 = []
    for bid, a in zip(bids, b1):
        fl = Flat(a)
        d = _dist_from(fl, fl.router_vertex(bid))
        seen = set()
        for x in a.router_lsas:
            v = fl.router_vertex(int(x["adv_rtr"]))
            if v == 0xFFFFFFFF or d[v] >= 1 << 40:
                continue
            for l in a.links[int(x["link_off"]): int(x["link_off"]) + int(x["n_links"])]:
                key = (int(l["link_id"]), int(l["link_data"]))
                if l["link_type"] != LINK_STUB or key in stubs0 or key in seen:
                    continue
                seen.add(key)
                sums0.append((bid, key[0], key[1], int(d[v]) + int(l["metric"]), 3, 0, (0, 0)))
    for bid, a in zip(bids, b1) if asbrs1 else ():
        fl = Flat(a)
        d = _dist_from(fl, fl.router_vertex(bid))
        sums0 += [(bid, x, 0, int(d[fl.router_vertex(x)]), 4, 0, (0, 0)) for x in asbrs1
                  if d[fl.router_vertex(x)] < 1 << 40]
    sums0.sort(key=lambda x: (x[4], x[0], x[1]))
    summaries0 = np.asarray(sums0, ospf_rib.SUMMARY_LSA_DT)
    loops = sorted({int(x["adv_rtr"]) for x in b1[0].router_lsas} - set(bids))
    keys = [loops[int(i)] for i in rng.choice(len(loops), min(n_ext_keys, len(loops)), replace=False)]
    ext = [(asbr, k, 0xFFFFFFFF, int(rng.choice([5, 30])), 0, 7, int(j % 2), 0, (0, 0)) for j, k in enumerate(keys)]
    ext.append((asbr, 0x0E0A0000, 0xFFFFFF00, 12, 0, 8, 1, 0, (0, 0)))
    for m, x in enumerate(asbrs1):
        ext.append((x, 0x0E0A0000, 0xFFFFFF00, 12, 0, 9, 1, 0, (0, 0)))
        for q in range(area1_ext):
            pfx = 0x0F000000 | ((m * area1_ext // 2 + q) << 8)
            ext.append((x, pfx, 0xFFFFFF00, int(rng1.integers(1, 40)), 0, 10 + m, (q + m) % 2, 0, (0, 0)))
    ext.sort(key=lambda x: (x[0], x[1]))
    externals = np.asarray(ext, ospf_rib.EXTERNAL_LSA_DT)
    empty = np.zeros(0, ospf_rib.SUMMARY_LSA_DT)
    out_borders = []
    for j, (a0, a1) in enumerate(zip(b0, b1)):
        pair = [(a0, 0, summaries0[summaries0["adv_rtr"] != a0.router_id]), (a1, 1, empty)]
        if j == 0:
            pair = pair[::-1]
        out_borders.append(([p[0] for p in pair], [p[1] for p in pair], [p[2] for p in pair]))
    return {"r_area": r_area, "summaries0": summaries0, "externals": externals, "borders": out_borders,
            "shared": shared, "asbr": asbr, "area1_asbrs": asbrs1}


def abr_backbone_view(t0: Topology, t1: Topology, t2: Topology, seed: int, r: int = 0, r2: int = 0,
                      borders=((1, 0), (2, 1), (3, 2)), max_paths: int = 16, n_ext_keys: int = 3, area1_asbrs: int = 0,
                      area1_ext: int = 4):
    """An area border router R of area 0 and area 2, and the borders of area 1, each as its own image: backbone_view's
    domain (areas 0 and 1, the three borders, the area-0 ASBR, with area1_asbrs / area1_ext its area-1 ASBRs and
    their type-5 and the borders' type-4 LSAs), with R (router r of t0) also router r2 of area 2, synth_area(t2) moved
    into ranges of its own, and the B flag in both of R's areas.  Seeded; area 2 draws from a generator of its own.
    Returns a dict:
      r_areas       R's images [area 0, area 2] (area ids `area_ids` [0, 2]), `summaries` per area: backbone_view's
                    summaries0 and none for area 2 (R is its only ABR);
      externals     backbone_view's, plus an area-2 ASBR's ("area2_asbr", the E flag) type-5 LSAs: 0x0E0A0000/24, which
                    the area-0 ASBR and every area-1 ASBR also advertise, and a /24 of its own;
      area2_shared  (prefix, mask) of an area-1 stub that is also a stub of an area-2 router (intra-area at R);
      borders, shared, asbr, area1_asbrs  as backbone_view's (R has the B flag in the borders' area-0 images)."""
    from . import ospf_rib
    v = backbone_view(t0, t1, seed, r=r, borders=borders, max_paths=max_paths, n_ext_keys=n_ext_keys,
                      area1_asbrs=area1_asbrs, area1_ext=area1_ext)
    rng = np.random.default_rng([seed, 0xAB2])
    R = RID_BASE + int(r)
    a2 = _set_flags(_area_remap(synth_area(t2, root=r2, max_paths=max_paths), 2, {RID_BASE + int(r2): R}), {R: 0x01})
    fl = Flat(a2)
    d = _dist_from(fl, fl.router_vertex(R))
    reach = sorted(int(fl.ids[x]) for x in range(len(fl.ids)) if fl.is_router[x] and 0 < d[x] < 1 << 40)
    t3 = v["summaries0"][v["summaries0"]["lsa_type"] == 3]
    pick = t3[int(rng.integers(0, len(t3)))]
    shared2 = (int(pick["lsa_id"]), int(pick["mask"]))
    a2 = _with_stubs(a2, {reach[int(rng.integers(0, len(reach)))]: [(shared2[0], shared2[1], 1)]})
    asbr2 = reach[int(rng.integers(0, len(reach)))]
    a2 = _set_flags(a2, {asbr2: 0x02})
    ext = [tuple(x) for x in v["externals"].tolist()]
    ext += [(asbr2, 0x0E0A0000, 0xFFFFFF00, 12, 0, 12, 1, 0, (0, 0)),
            (asbr2, 0x0E0C0000, 0xFFFFFF00, int(rng.integers(1, 40)), 0, 12, 0, 0, (0, 0))]
    ext.sort(key=lambda x: (x[0], x[1]))
    r_area0 = _set_flags(v["r_area"], {R: 0x01})
    out_borders = [([_set_flags(a, {R: 0x01}) if a.area_id == 0 else a for a in areas], ids, sums)
                   for areas, ids, sums in v["borders"]]
    return {"r_areas": [r_area0, a2], "area_ids": [0, 2],
            "summaries": [v["summaries0"], np.zeros(0, ospf_rib.SUMMARY_LSA_DT)],
            "externals": np.asarray(ext, ospf_rib.EXTERNAL_LSA_DT), "area2_shared": shared2, "area2_asbr": asbr2,
            "borders": out_borders, "shared": v["shared"], "asbr": v["asbr"], "area1_asbrs": v["area1_asbrs"]}


def _rerooted(img: Ospfv2Area, fresh: Ospfv2Area) -> Ospfv2Area:
    """img's LSDB as seen by fresh's root: the root's own fields (router id, interfaces, neighbours) from fresh."""
    a = Ospfv2Area(**{k: getattr(img, k) for k in img.__dataclass_fields__})
    for k in ("router_id", "ifaces", "iface_addrs", "nbrs", "ifnames"):
        setattr(a, k, getattr(fresh, k))
    return a


def third_area_view(t0: Topology, t1: Topology, t2: Topology, seed: int, spf, n_c: int = 2, max_paths: int = 16,
                    n_ext_keys: int = 3, area1_asbrs: int = 0, area1_ext: int = 4):
    """An internal router R of area 2, the area border routers C of area 2 and area 0 (n_c of them, 2 or 3), and the
    borders B of area 1, each as its own image: backbone_view's areas 0 and 1 (its three borders, the area-0 ASBR,
    area1_asbrs area-1 ASBRs with their type-5 and type-4 LSAs), with synth_area(t2) moved into ranges of area 2 whose
    routers 0 .. n_c - 1 are the C's (routers 0, then the first routers of t0 past the borders that are not the
    area-0 ASBR; the B flag in areas 0 and 2) and whose router n_c is R.  Area 2 also holds an ASBR ("area2_asbr") with
    0x0E0A0000/24 and a /24 of its own, and a stub of an area-1 prefix ("area2_shared").  Seeded; area 2 draws from a
    generator of its own.  `spf(csr, root_vertex, nh_words)` gives unperturbed planes, as area_from_planes takes them.
    Returns a dict:
      r_area        R's area-2 image;
      summaries2    area 2's type-3/4 LSAs (LsaKey order): each C's hspf_ospfv2_net_summaries into area 2 over its
                    update_rib_full at the unperturbed job;
      externals     backbone_view's plus the area-2 ASBR's;
      c_areas       per C (areas [area 0, area 2], area ids [0, 2], summaries per area: area 0's, none for area 2);
      borders       per B as backbone_view's (the C's have the B flag in its area-0 image);
      asbr, area1_asbrs, area2_asbr, area2_shared, shared."""
    from . import ospf_rib
    if n_c not in (2, 3):
        raise ValueError("n_c is 2 or 3")
    v = backbone_view(t0, t1, seed, r=0, max_paths=max_paths, n_ext_keys=n_ext_keys, area1_asbrs=area1_asbrs,
                      area1_ext=area1_ext)
    rng = np.random.default_rng([seed, 0xC3A])
    c0 = [0] + [i for i in range(4, t0.n_routers) if RID_BASE + i != v["asbr"]][:n_c - 1]
    cids = [RID_BASE + i for i in c0]
    cflag = {c: 0x01 for c in cids}
    idmap = {RID_BASE + k: c for k, c in enumerate(cids)}
    img2 = lambda i: _set_flags(_area_remap(synth_area(t2, root=i, max_paths=max_paths), 2, idmap), dict(cflag))
    ra = img2(n_c)
    fl = Flat(ra)
    d = _dist_from(fl, fl.router_vertex(ra.router_id))
    reach = sorted(int(fl.ids[x]) for x in range(len(fl.ids))
                   if fl.is_router[x] and 0 < d[x] < 1 << 40 and int(fl.ids[x]) not in cids)
    t3 = v["summaries0"][v["summaries0"]["lsa_type"] == 3]
    pick = t3[int(rng.integers(0, len(t3)))]
    shared2 = (int(pick["lsa_id"]), int(pick["mask"]))
    adds = {reach[int(rng.integers(0, len(reach)))]: [(shared2[0], shared2[1], 1)]}
    asbr2 = reach[int(rng.integers(0, len(reach)))]
    area2 = lambda i: _set_flags(_with_stubs(img2(i), adds), {asbr2: 0x02})
    ext = [tuple(x) for x in v["externals"].tolist()]
    ext += [(asbr2, 0x0E0A0000, 0xFFFFFF00, 12, 0, 12, 1, 0, (0, 0)),
            (asbr2, 0x0E0C0000, 0xFFFFFF00, int(rng.integers(1, 40)), 0, 12, 0, 0, (0, 0))]
    ext.sort(key=lambda x: (x[0], x[1]))
    externals = np.asarray(ext, ospf_rib.EXTERNAL_LSA_DT)
    a0 = _set_flags(v["r_area"], dict(cflag))
    empty = np.zeros(0, ospf_rib.SUMMARY_LSA_DT)
    c_areas = [([_rerooted(a0, synth_area(t0, root=i, max_paths=max_paths)) if k else a0, area2(k)], [0, 2],
                [v["summaries0"], empty]) for k, i in enumerate(c0)]
    sums = []
    for areas, ids, csums in c_areas:
        rid = areas[0].router_id
        rib_areas = [ospf_rib.RibArea(a.area_id, area_from_planes(a, spf), a.ifaces, s, True)
                     for a, s in zip(areas, csums)]
        rib = ospf_rib.update_rib_full(rid, max_paths, rib_areas, externals)
        sums += [tuple(x) for x in ospf_rib.net_summaries(rid, rib, ospf_rib.router_tables(rid, rib_areas), rib_areas,
                                                          [ospf_rib.area_config()] * 2, 1).tolist()]
    sums.sort(key=lambda x: (x[4], x[0], x[1]))
    borders = [([_set_flags(a, dict(cflag)) if a.area_id == 0 else a for a in areas], ids, bs)
               for areas, ids, bs in v["borders"]]
    return {"r_area": area2(n_c), "summaries2": np.asarray(sums, ospf_rib.SUMMARY_LSA_DT), "externals": externals,
            "c_areas": c_areas, "borders": borders, "asbr": v["asbr"], "area1_asbrs": v["area1_asbrs"],
            "area2_asbr": asbr2, "area2_shared": shared2, "shared": v["shared"]}


def nonbackbone_view(t0: Topology, t1: Topology, seed: int, spf, r: int | None = None,
                     borders=((1, 0), (2, 1), (3, 2)), max_paths: int = 16, n_ext_keys: int = 3, n_ext: int = 0):
    """An internal router R of area 1 and the area border routers ("borders") between area 0 and area 1, each as its
    own image: backbone_view's domain seen from area 1.  Seeded.  Areas, borders, the area-0 ASBR (the E flag) with
    its type-5 LSAs and the shared /24 are backbone_view(t0, t1, seed, ...)'s; R is router r of t1 (default: the first
    that is not a border).  `spf(csr, root_vertex, nh_words)` gives unperturbed planes, as area_from_planes takes them.
    Returns a dict:
      r_area        R's area-1 image;
      summaries1    area 1's type-3/4 LSAs (LsaKey order): each border's hspf_ospfv2_net_summaries into area 1 over
                    its update_rib_full at the unperturbed job (type-4: the area-0 ASBR);
      externals     backbone_view's, plus n_ext /24s of the area-0 ASBR, both E-bit values (drawn from a generator of
                    its own, so that every other part is as without them);
      borders       per border (areas, area ids, summaries per area) as backbone_view's (the first border lists area 1
                    first; a border's area-1 summaries are empty: with two active areas it reads only area 0's);
      shared        the /24 that ties at the first border between area 0 and area 1;
      asbr          the area-0 ASBR's router id."""
    from . import ospf_rib
    v = backbone_view(t0, t1, seed, borders=borders, max_paths=max_paths, n_ext_keys=n_ext_keys)
    bids = [RID_BASE + int(i0) for i0, _ in borders]
    idmap = {RID_BASE + int(i1): RID_BASE + int(i0) for i0, i1 in borders}
    if r is None:
        r = next(i for i in range(t1.n_routers) if i not in {int(i1) for _, i1 in borders})
    ra = _set_flags(_area_remap(synth_area(t1, root=r, max_paths=max_paths), 1, idmap), {b: 0x01 for b in bids})
    # the shared /24's stub in area 1, as the first border's area-1 image has it
    a1 = next(a for a in v["borders"][0][0] if a.area_id == 1)
    add1 = {}
    for x in a1.router_lsas:
        for l in a1.links[int(x["link_off"]): int(x["link_off"]) + int(x["n_links"])]:
            if l["link_type"] == LINK_STUB and (int(l["link_id"]), int(l["link_data"])) == v["shared"]:
                add1.setdefault(int(x["adv_rtr"]), []).append((v["shared"][0], v["shared"][1], int(l["metric"])))
    ra = _with_stubs(ra, add1)
    ext = v["externals"]
    if n_ext:
        rng = np.random.default_rng([seed, 0x0E1])
        more = [(v["asbr"], 0x0F800000 | (q << 8), 0xFFFFFF00, int(rng.integers(1, 40)), 0, 11, q % 2, 0, (0, 0))
                for q in range(n_ext)]
        ext = np.asarray(sorted([tuple(x) for x in ext.tolist()] + more, key=lambda x: (x[0], x[1])),
                         ospf_rib.EXTERNAL_LSA_DT)
    sums = []
    for areas, ids, bsums in v["borders"]:
        rid = areas[0].router_id
        rib_areas = [ospf_rib.RibArea(a.area_id, area_from_planes(a, spf), a.ifaces, s, True)
                     for a, s in zip(areas, bsums)]
        rib = ospf_rib.update_rib_full(rid, max_paths, rib_areas, ext)
        sums += [tuple(x) for x in ospf_rib.net_summaries(rid, rib, ospf_rib.router_tables(rid, rib_areas), rib_areas,
                                                          [ospf_rib.area_config()] * len(areas), ids.index(1)).tolist()]
    sums.sort(key=lambda x: (x[4], x[0], x[1]))
    return {"r_area": ra, "summaries1": np.asarray(sums, ospf_rib.SUMMARY_LSA_DT), "externals": ext,
            "borders": v["borders"], "shared": v["shared"], "asbr": v["asbr"]}
