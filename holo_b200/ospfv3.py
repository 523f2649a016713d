"""OSPFv3 side of the engine from Python: LSDB images (include/holo_lsdb.h), the
run_area call (holo-ospf/src/spf.rs:587-729 with the OSPFv3 hooks of
holo-ospf/src/ospfv3/spf.rs replaced by hspf_ospfv3_run_area) and a synthetic builder."""
from __future__ import annotations

import ctypes as C
import ipaddress
from dataclasses import dataclass, field

import numpy as np

from . import capi, route_table
from .ospfv2 import CONTRIB_DT, ROUTE_RTR_DT, IF_P2P, IF_BROADCAST, LINK_P2P, LINK_TRANSIT, MAX_AGE
from .synth import Topology

OPT_R, OPT_V6 = 0x01, 0x02
PFX_NU = 0x01
REF_ROUTER, REF_NETWORK = 1, 2

IP_DT = np.dtype([("bytes", "u1", (16,)), ("is_v6", "u1"), ("_pad", "u1", (3,))], align=True)
LINK_DT = np.dtype([("iface_id", "<u4"), ("nbr_iface_id", "<u4"), ("nbr_router_id", "<u4"), ("metric", "<u2"),
                    ("link_type", "u1"), ("_pad", "u1")], align=True)
ROUTER_LSA_DT = np.dtype([("adv_rtr", "<u4"), ("lsa_id", "<u4"), ("age", "<u2"), ("flags", "u1"), ("options", "u1"),
                          ("link_off", "<u4"), ("n_links", "<u4")], align=True)
NETWORK_LSA_DT = np.dtype([("adv_rtr", "<u4"), ("lsa_id", "<u4"), ("age", "<u2"), ("_pad", "<u2"), ("att_off", "<u4"),
                           ("n_att", "<u4")], align=True)
PREFIX_DT = np.dtype([("addr", IP_DT), ("len", "u1"), ("options", "u1"), ("metric", "<u2")], align=True)
IAP_LSA_DT = np.dtype([("adv_rtr", "<u4"), ("lsa_id", "<u4"), ("age", "<u2"), ("ref_type", "u1"), ("_pad", "u1"),
                       ("ref_lsa_id", "<u4"), ("ref_adv_rtr", "<u4"), ("prefix_off", "<u4"), ("n_prefixes", "<u4")],
                      align=True)
LINK_LSA_DT = np.dtype([("iface", "<u4"), ("adv_rtr", "<u4"), ("lsa_id", "<u4"), ("age", "<u2"), ("_pad", "<u2"),
                        ("linklocal", IP_DT)], align=True)
IFACE_DT = np.dtype([("ifindex", "<u4"), ("sort_key", "<u4"), ("if_type", "u1"), ("_pad", "u1", (3,))], align=True)
NEXTHOP6_DT = np.dtype([("iface", "<u4"), ("nbr_router_id", "<u4"), ("addr", IP_DT), ("has_addr", "u1"),
                        ("has_nbr", "u1"), ("_pad", "u1", (2,))], align=True)
SPT_VERTEX6_DT = np.dtype([("router_id", "<u4"), ("iface_id", "<u4"), ("distance", "<u4"), ("hops", "<u2"),
                           ("is_router", "u1"), ("_pad", "u1"), ("nh_off", "<u4"), ("n_nh", "<u4")], align=True)
ROUTE_NET6_DT = np.dtype([("prefix", IP_DT), ("len", "u1"), ("flags", "u1"), ("origin_type", "u1"),
                          ("prefix_options", "u1"), ("metric", "<u4"), ("origin_adv_rtr", "<u4"),
                          ("origin_lsa_id", "<u4"), ("nh_off", "<u4"), ("n_nh", "<u4")], align=True)


class AreaStruct(C.Structure):
    _fields_ = [
        ("router_id", C.c_uint32), ("area_id", C.c_uint32), ("max_paths", C.c_uint16), ("af_ipv6", C.c_uint8),
        ("_pad", C.c_uint8),
        ("n_router_lsas", C.c_uint32), ("router_lsas", C.c_void_p),
        ("n_links", C.c_uint32), ("links", C.c_void_p),
        ("n_network_lsas", C.c_uint32), ("network_lsas", C.c_void_p),
        ("n_attached", C.c_uint32), ("attached", C.c_void_p),
        ("n_iap_lsas", C.c_uint32), ("iap_lsas", C.c_void_p),
        ("n_prefixes", C.c_uint32), ("prefixes", C.c_void_p),
        ("n_ifaces", C.c_uint32), ("ifaces", C.c_void_p),
        ("n_link_lsas", C.c_uint32), ("link_lsas", C.c_void_p),
    ]


class ResultStruct(C.Structure):
    _fields_ = [
        ("vertices_cap", C.c_uint32), ("n_vertices", C.c_uint32), ("vertices", C.c_void_p),
        ("routers_cap", C.c_uint32), ("n_routers", C.c_uint32), ("routers", C.c_void_p),
        ("routes_cap", C.c_uint32), ("n_routes", C.c_uint32), ("routes", C.c_void_p),
        ("nexthops_cap", C.c_uint32), ("n_nexthops", C.c_uint32), ("nexthops", C.c_void_p),
        ("transit_capability", C.c_uint8), ("root_found", C.c_uint8), ("_pad", C.c_uint8 * 2),
    ]


ABI_SIZES = [LINK_DT.itemsize, ROUTER_LSA_DT.itemsize, NETWORK_LSA_DT.itemsize, IP_DT.itemsize, PREFIX_DT.itemsize,
             IAP_LSA_DT.itemsize, LINK_LSA_DT.itemsize, IFACE_DT.itemsize, C.sizeof(AreaStruct), NEXTHOP6_DT.itemsize,
             SPT_VERTEX6_DT.itemsize, ROUTE_NET6_DT.itemsize, C.sizeof(ResultStruct)]

_FIELDS = (("router_lsas", ROUTER_LSA_DT), ("links", LINK_DT), ("network_lsas", NETWORK_LSA_DT),
           ("attached", np.dtype("<u4")), ("iap_lsas", IAP_LSA_DT), ("prefixes", PREFIX_DT), ("ifaces", IFACE_DT),
           ("link_lsas", LINK_LSA_DT))


def ip_rec(addr) -> tuple:
    a = ipaddress.ip_address(addr)
    b = a.packed if a.version == 6 else a.packed + bytes(12)
    return (tuple(b), 1 if a.version == 6 else 0, (0, 0, 0))


def ip_str(rec) -> str:
    b = bytes(int(x) for x in rec["bytes"])
    return str(ipaddress.IPv6Address(b)) if int(rec["is_v6"]) else str(ipaddress.IPv4Address(b[:4]))


@dataclass
class Ospfv3Area:
    router_id: int
    area_id: int = 0
    max_paths: int = 16
    af_ipv6: bool = True
    router_lsas: np.ndarray = field(default_factory=lambda: np.zeros(0, ROUTER_LSA_DT))
    links: np.ndarray = field(default_factory=lambda: np.zeros(0, LINK_DT))
    network_lsas: np.ndarray = field(default_factory=lambda: np.zeros(0, NETWORK_LSA_DT))
    attached: np.ndarray = field(default_factory=lambda: np.zeros(0, np.uint32))
    iap_lsas: np.ndarray = field(default_factory=lambda: np.zeros(0, IAP_LSA_DT))
    prefixes: np.ndarray = field(default_factory=lambda: np.zeros(0, PREFIX_DT))
    ifaces: np.ndarray = field(default_factory=lambda: np.zeros(0, IFACE_DT))
    link_lsas: np.ndarray = field(default_factory=lambda: np.zeros(0, LINK_LSA_DT))
    ifnames: list = field(default_factory=list)

    def as_struct(self) -> AreaStruct:
        s = AreaStruct()
        s.router_id, s.area_id, s.max_paths, s.af_ipv6 = self.router_id, self.area_id, self.max_paths, int(self.af_ipv6)
        for name, dt in _FIELDS:
            a = np.ascontiguousarray(getattr(self, name), dtype=dt)
            setattr(self, name, a)
            setattr(s, "n_" + name, len(a))
            setattr(s, name, a.ctypes.data if len(a) else None)
        return s


@dataclass
class Ospfv3Result:
    vertices: np.ndarray
    routers: np.ndarray
    routes: np.ndarray
    nexthops: np.ndarray
    transit_capability: bool
    root_found: bool
    rc: int = 0

    def nh(self, rec):
        return [(int(x["iface"]), ip_str(x["addr"]) if x["has_addr"] else None, int(x["nbr_router_id"]) if x["has_nbr"] else None)
                for x in self.nexthops[int(rec["nh_off"]): int(rec["nh_off"]) + int(rec["n_nh"])]]


def _call_run_area(fn, area: Ospfv3Area, prefix_args=(), tail_args=()):
    s = area.as_struct()
    nv = len(area.router_lsas) + len(area.network_lsas) + 1
    n_routes = len(area.prefixes) + 1
    caps = [nv, nv, n_routes, 64 * (2 * nv + n_routes) + 64]
    for _ in range(2):
        verts = np.zeros(caps[0], SPT_VERTEX6_DT)
        rtrs = np.zeros(caps[1], ROUTE_RTR_DT)
        routes = np.zeros(caps[2], ROUTE_NET6_DT)
        nhs = np.zeros(caps[3], NEXTHOP6_DT)
        r = ResultStruct()
        r.vertices_cap, r.vertices = caps[0], verts.ctypes.data
        r.routers_cap, r.routers = caps[1], rtrs.ctypes.data
        r.routes_cap, r.routes = caps[2], routes.ctypes.data
        r.nexthops_cap, r.nexthops = caps[3], nhs.ctypes.data
        rc = fn(*prefix_args, C.byref(s), *tail_args, C.byref(r))
        if rc == capi.HSPF_E_NOMEM:
            caps = [max(caps[0], r.n_vertices), max(caps[1], r.n_routers), max(caps[2], r.n_routes),
                    max(caps[3], r.n_nexthops)]
            continue
        break
    return Ospfv3Result(verts[: r.n_vertices].copy(), rtrs[: r.n_routers].copy(), routes[: r.n_routes].copy(),
                        nhs[: r.n_nexthops].copy(), bool(r.transit_capability), bool(r.root_found), rc)


def run_area(ctx: capi.Context, area: Ospfv3Area) -> Ospfv3Result:
    lib = ctx.lib
    lib.hspf_ospfv3_run_area.argtypes = [C.c_void_p, C.POINTER(AreaStruct), C.POINTER(ResultStruct)]
    res = _call_run_area(lib.hspf_ospfv3_run_area, area, (ctx.handle,))
    if res.rc != capi.HSPF_OK:
        raise capi.HspfError(res.rc, ctx.last_error())
    return res


def area_from_planes(area: Ospfv3Area, spf) -> Ospfv3Result:
    """hspf_ospfv3_area_from_planes over planes from `spf(csr, root_vertex, nh_words)` (host only;
    see holo_b200.ospfv2.area_from_planes)."""
    lib = capi.load_library()
    lib.hspf_ospfv3_area_from_planes.argtypes = [C.POINTER(AreaStruct), C.POINTER(C.c_uint32), C.POINTER(C.c_uint16),
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
    res = _call_run_area(lib.hspf_ospfv3_area_from_planes, area, (), tail)
    if res.rc != capi.HSPF_OK:
        raise capi.HspfError(res.rc, "hspf_ospfv3_area_from_planes failed")
    return res


class RouteTable(route_table.RouteTable):
    """hspf_ospfv3_rtable_create: the route table of an OSPFv3 area for the batched route stage (the object
    ospfv2.RouteTable wraps; upload and hspf_ospfv2_routes_batch[16] work on it unchanged)."""

    api, contrib_dt = "hspf_ospfv2", CONTRIB_DT

    def __init__(self, flat: "Flat"):
        self.flat = flat
        super().__init__(capi.load_library().hspf_ospfv3_rtable_create, flat.handle)
        pp, pl = C.c_void_p(), C.POINTER(C.c_uint32)()
        self.lib.hspf_ospfv3_rtable_prefixes6(self.handle, C.byref(pp), C.byref(pl))
        self.prefix = route_table.copy_records(pp, self.n_prefixes, IP_DT)
        self.plen = route_table.copy_records(pl, self.n_prefixes, np.uint32)


def routes_from_cells(area: Ospfv3Area, rt: RouteTable, cells: np.ndarray, gather_v, gather_nh) -> Ospfv3Result:
    """hspf_ospfv3_routes_from_cells (host): one job's cells -> the routes / next hops of hspf_ospfv3_run_area."""
    from . import ospfv2
    lib = capi.load_library()
    cells = np.ascontiguousarray(cells, ospfv2.CELL_DT)
    assert cells.shape == (rt.n_prefixes,)
    gv = np.ascontiguousarray(gather_v, np.uint32)
    gn = np.ascontiguousarray(gather_nh, np.uint64)
    res = _call_run_area(lib.hspf_ospfv3_routes_from_cells, area, (),
                         (rt.handle, cells.ctypes.data, gv.ctypes.data_as(C.POINTER(C.c_uint32)),
                          gn.ctypes.data_as(C.POINTER(C.c_uint64)), len(gv)))
    if res.rc not in (capi.HSPF_OK, capi.HSPF_E_UNSUPPORTED):
        raise capi.HspfError(res.rc, "hspf_ospfv3_routes_from_cells failed")
    return res


IP_PREFIX_DT = np.dtype([("addr", IP_DT), ("len", "u1"), ("_pad", "u1", (3,))], align=True)
TRIGGER6_DT = np.dtype([("adv_rtr", "<u4"), ("lsa_id", "<u4"), ("router_id", "<u4"), ("prefix_off", "<u4"), ("n_prefixes", "<u4"),
                        ("function_code", "<u2"), ("_pad", "u1", (2,))], align=True)


class SpfComputation6Struct(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("n_intra", C.c_uint32), ("n_inter_network", C.c_uint32), ("n_inter_router", C.c_uint32),
                ("n_external", C.c_uint32), ("cap", C.c_uint32), ("intra", C.c_void_p), ("inter_network", C.c_void_p),
                ("inter_router", C.c_void_p), ("external", C.c_void_p)]


def spf_computation_type(triggers, fn=None):
    """hspf_ospfv3_spf_computation_type.  triggers: [(function_code, adv_rtr, lsa_id, router_id, [(addr, len), ...])]
    -> (kind, intra, inter_network, inter_router, external) with prefixes as (addr string, len)."""
    if fn is None:
        fn = capi.load_library().hspf_ospfv3_spf_computation_type
    fn.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(SpfComputation6Struct)]
    tr = np.zeros(len(triggers), TRIGGER6_DT)
    pf = []
    for i, (code, adv, lsa_id, router_id, prefixes) in enumerate(triggers):
        tr[i] = (adv, lsa_id, router_id, len(pf), len(prefixes), code, (0, 0))
        pf += [(ip_rec(a), ln, (0, 0, 0)) for a, ln in prefixes]
    pfa = np.asarray(pf, IP_PREFIX_DT) if pf else np.zeros(0, IP_PREFIX_DT)
    cap = max(len(pfa), len(tr), 1)
    a, b, c, d = np.zeros(cap, IP_PREFIX_DT), np.zeros(cap, IP_PREFIX_DT), np.zeros(cap, np.uint32), np.zeros(cap, IP_PREFIX_DT)
    s = SpfComputation6Struct(0, 0, 0, 0, 0, cap, a.ctypes.data, b.ctypes.data, c.ctypes.data, d.ctypes.data)
    rc = fn(tr.ctypes.data if len(tr) else None, len(tr), pfa.ctypes.data if len(pfa) else None, len(pfa), C.byref(s))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, "ospfv3 spf_computation_type failed")
    out = lambda arr, k: [(ip_str(x["addr"]), int(x["len"])) for x in arr[:k]]
    return s.kind, out(a, s.n_intra), out(b, s.n_inter_network), [int(x) for x in c[: s.n_inter_router]], out(d, s.n_external)


class Flat:
    def __init__(self, area: Ospfv3Area):
        lib = capi.load_library()
        lib.hspf_ospfv3_flatten.argtypes = [C.POINTER(AreaStruct), C.POINTER(C.c_void_p)]
        lib.hspf_ospfv3_flat_free.argtypes = [C.c_void_p]
        lib.hspf_ospfv3_flat_free.restype = None
        lib.hspf_ospfv3_flat_csr.argtypes = [C.c_void_p, C.POINTER(capi.CsrStruct)]
        lib.hspf_ospfv3_flat_vertices.argtypes = [C.c_void_p, C.POINTER(C.POINTER(C.c_uint32)),
                                                  C.POINTER(C.POINTER(C.c_uint32)), C.POINTER(C.POINTER(C.c_uint8)),
                                                  C.POINTER(C.c_uint32)]
        lib.hspf_ospfv3_flat_router_vertex.argtypes = [C.c_void_p, C.c_uint32]
        lib.hspf_ospfv3_flat_router_vertex.restype = C.c_uint32
        self.lib, self.area = lib, area
        self._s = area.as_struct()
        h = C.c_void_p()
        rc = lib.hspf_ospfv3_flatten(C.byref(self._s), C.byref(h))
        if rc != capi.HSPF_OK:
            raise capi.HspfError(rc, "hspf_ospfv3_flatten failed")
        self.handle = h
        self._load()

    def _load(self):
        lib, h = self.lib, self.handle
        cs = capi.CsrStruct()
        lib.hspf_ospfv3_flat_csr(h, C.byref(cs))
        V, E = cs.n_vertices, cs.n_edges
        as_np = lambda p, n, dt: np.ctypeslib.as_array(p, shape=(n,)).astype(dt).copy() if n else np.zeros(0, dt)
        self.csr = capi.Csr(as_np(cs.row_ptr, V + 1, np.uint32), as_np(cs.col, E, np.uint32),
                            as_np(cs.cost, E, np.uint32), as_np(cs.vflags, V, np.uint8),
                            reject_above=cs.reject_above, saturate_at=cs.saturate_at, flags=cs.flags, delta=cs.delta)
        rid, ifid, isr, n = C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint8)(), C.c_uint32()
        lib.hspf_ospfv3_flat_vertices(h, C.byref(rid), C.byref(ifid), C.byref(isr), C.byref(n))
        self.router_ids = as_np(rid, n.value, np.uint32)
        self.iface_ids = as_np(ifid, n.value, np.uint32)
        self.is_router = as_np(isr, n.value, np.uint8)

    def router_vertex(self, router_id: int) -> int:
        return int(self.lib.hspf_ospfv3_flat_router_vertex(self.handle, router_id))

    def update(self, new_area: "Ospfv3Area"):
        """hspf_ospfv3_flat_update -> (kind, edges, costs) with kind 0 unchanged / 1 costs / 2 rebuilt."""
        self.lib.hspf_ospfv3_flat_update.argtypes = [C.c_void_p, C.POINTER(AreaStruct), C.POINTER(C.c_uint32), C.c_void_p,
                                                     C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
        cap = max(int(self.csr.n_edges), 1)
        edges, costs = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
        kind, n = C.c_uint32(), C.c_uint32()
        s = new_area.as_struct()
        rc = self.lib.hspf_ospfv3_flat_update(self.handle, C.byref(s), C.byref(kind), edges.ctypes.data, costs.ctypes.data, cap,
                                              C.byref(n))
        if rc != capi.HSPF_OK:
            raise capi.HspfError(rc, "hspf_ospfv3_flat_update failed")
        self.area, self._s = new_area, s
        self._load()
        return kind.value, edges[: n.value].copy(), costs[: n.value].copy()

    def __del__(self):
        try:
            if self.handle:
                self.lib.hspf_ospfv3_flat_free(self.handle)
                self.handle = None
        except Exception:
            pass


# ------------------------------------------------------------------------------ synthetic
RID_BASE = 0x0A000001


def synth_area(t: Topology, root: int = 0, max_links_per_fragment: int = 0, max_paths: int = 16,
               rids=None, area_id: int = 0) -> Ospfv3Area:
    """OSPFv3 area LSDB for topology `t` seen by router `root`.  Interface ids are
    per-router link ordinals (1-based); Router-LSAs are split into fragments of
    `max_links_per_fragment` links when > 0 (RFC 5340 4.8.1 aggregate); one
    Intra-Area-Prefix-LSA per router (a /128 loopback, metric 0, plus one /64 per
    p2p link) and one per LAN (referencing the Network-LSA)."""
    R = t.n_routers
    rid = (lambda i: RID_BASE + int(i)) if rids is None else (lambda i: int(rids[int(i)]))
    per = [[] for _ in range(R)]          # (iface_id, nbr_iface_id, nbr_rid, metric, type)
    nif = [0] * R
    p2p_if = []
    for k in range(t.n_p2p):
        a, b = int(t.p2p_a[k]), int(t.p2p_b[k])
        nif[a] += 1; ia = nif[a]
        nif[b] += 1; ib = nif[b]
        p2p_if.append((ia, ib))
        per[a].append((ia, ib, rid(b), int(t.p2p_cost_ab[k]), LINK_P2P))
        per[b].append((ib, ia, rid(a), int(t.p2p_cost_ba[k]), LINK_P2P))
    lan_if = []
    net_lsas, attached = [], []
    for members, costs in t.lans:
        ids = []
        for m in members:
            nif[m] += 1
            ids.append(nif[m])
        dr, dr_if = members[0], ids[0]
        for m, c, i in zip(members, costs, ids):
            per[m].append((i, dr_if, rid(dr), int(c), LINK_TRANSIT))
        lan_if.append(ids)
        net_lsas.append((rid(dr), dr_if, len(attached), len(members)))
        attached += sorted(rid(m) for m in members)
    rl, links = [], []
    for i in range(R):
        chunks = [per[i]]
        if max_links_per_fragment > 0:
            chunks = [per[i][j:j + max_links_per_fragment] for j in range(0, len(per[i]), max_links_per_fragment)] or [[]]
        for frag, ch in enumerate(chunks):
            rl.append((rid(i), frag, 1, 0, OPT_R | OPT_V6, len(links), len(ch)))
            links += [(a, b, c, d, e, 0) for (a, b, c, d, e) in ch]
    area = Ospfv3Area(router_id=rid(root), max_paths=max_paths, area_id=area_id)
    rl.sort(key=lambda x: (x[0], x[1]))          # LsaKey order (adv_rtr, lsa_id)
    area.router_lsas = np.asarray(rl, dtype=ROUTER_LSA_DT)
    area.links = np.asarray(links, dtype=LINK_DT) if links else np.zeros(0, LINK_DT)
    nl = np.zeros(len(net_lsas), NETWORK_LSA_DT)
    for i, (adv, lsid, ao, na) in enumerate(net_lsas):
        nl[i] = (adv, lsid, 1, 0, ao, na)
    area.network_lsas = nl[np.lexsort((nl["lsa_id"], nl["adv_rtr"]))] if len(nl) else nl
    area.attached = np.asarray(attached, dtype=np.uint32)
    # prefixes
    iaps, prefixes = [], []
    for i in range(R):
        off = len(prefixes)
        prefixes.append((ip_rec(ipaddress.IPv6Address((0x20010DB8 << 96) | (0x1000 << 80) | (i + 1))), 128, 0, 0))
        iaps.append((rid(i), 0, 1, REF_ROUTER, 0, 0, rid(i), off, len(prefixes) - off))
    for k in range(t.n_p2p):
        a = int(t.p2p_a[k])
        off = len(prefixes)
        prefixes.append((ip_rec(ipaddress.IPv6Address((0x20010DB8 << 96) | (0x2000 << 80) | (k << 64))), 64, 0,
                         int(t.p2p_cost_ab[k])))
        iaps.append((rid(a), 1 + k, 1, REF_ROUTER, 0, 0, rid(a), off, 1))
    for li, (members, costs) in enumerate(t.lans):
        off = len(prefixes)
        prefixes.append((ip_rec(ipaddress.IPv6Address((0x20010DB8 << 96) | (0x3000 << 80) | (li << 64))), 64, 0, 0))
        iaps.append((rid(members[0]), 0x10000 + li, 1, REF_NETWORK, 0, lan_if[li][0], rid(members[0]), off, 1))
    ia = np.zeros(len(iaps), IAP_LSA_DT)
    for i, x in enumerate(iaps):
        ia[i] = x
    area.iap_lsas = ia[np.lexsort((ia["lsa_id"], ia["adv_rtr"]))]
    pa = np.zeros(len(prefixes), PREFIX_DT)
    for i, x in enumerate(prefixes):
        pa[i] = x
    area.prefixes = pa
    # local interfaces of the root + the neighbours' Link-LSAs
    ifaces, llsas, names = [], [], []
    ll = lambda r, i: ip_rec(ipaddress.IPv6Address((0xFE80 << 112) | (rid(r) << 32) | i))
    for k in range(t.n_p2p):
        a, b = int(t.p2p_a[k]), int(t.p2p_b[k])
        ia_, ib_ = p2p_if[k]
        if a == root:
            llsas.append((len(ifaces), rid(b), ib_, 1, 0, ll(b, ib_)))
            ifaces.append((ia_, 1000 - len(ifaces), IF_P2P, (0, 0, 0)))
        if b == root:
            llsas.append((len(ifaces), rid(a), ia_, 1, 0, ll(a, ia_)))
            ifaces.append((ib_, 1000 - len(ifaces), IF_P2P, (0, 0, 0)))
    for li, (members, costs) in enumerate(t.lans):
        if root in members:
            me = lan_if[li][members.index(root)]
            for m, i in zip(members, lan_if[li]):
                if m != root:
                    llsas.append((len(ifaces), rid(m), i, 1, 0, ll(m, i)))
            ifaces.append((me, 1000 - len(ifaces), IF_BROADCAST, (0, 0, 0)))
    area.ifaces = np.asarray(ifaces, dtype=IFACE_DT) if ifaces else np.zeros(0, IFACE_DT)
    la = np.zeros(len(llsas), LINK_LSA_DT)
    for i, x in enumerate(llsas):
        la[i] = x
    area.link_lsas = la
    area.ifnames = [f"if{int(x[0])}" for x in ifaces]
    return area


def inter_area_view(area: Ospfv3Area, seed: int, n_abr: int = 4, n_asbr: int = 3, n_inter: int = 60, n_ext: int = 50,
                    unreachable_abr: bool = True, n_overlap: int = 8, n_fresh: int = 10, n_ext_only: int = 8,
                    nu_fraction: float = 0.08):
    """The OSPFv3 twin of ospfv2.inter_area_view: a single-area LSDB as one area of a multi-area domain, returned as
    (area, inter-area LSAs, AS-external LSAs) for ospf_rib (ospf_rib.INTER_AREA_LSA_DT in LsaKey order,
    ospf_rib.EXTERNAL6_LSA_DT in LSDB order).  Seeded and independent of area.router_id.
      * n_abr routers get the B flag, n_asbr others the E flag (on every Router-LSA fragment of the router); with
        unreachable_abr a router with B|E and no links is added;
      * Inter-Area-Prefix LSAs from the ABRs (and from a router without the B flag and an unknown router) for
        intra-area prefixes, new prefixes, prefixes with host bits and the default route; Inter-Area-Router LSAs for
        in-area ASBRs and ASBRs outside the area, naming the ASBR in router_id (lsa_id is an unrelated number);
        AS-external LSAs of type 1 and 2 from those ASBRs, from routers without the E flag, from unknown routers and
        from ordinary routers;
      * a nu_fraction of the Inter-Area-Prefix, Inter-Area-Router and AS-external LSAs carry the NU option (only the
        first and last kinds are skipped for it);
      * metrics from small sets, so that ties are common; some LSAs at maxage or at LSInfinity."""
    from . import ospf_rib
    rng = np.random.default_rng(seed)
    a = Ospfv3Area(**{k: getattr(area, k) for k in area.__dataclass_fields__})
    rl = area.router_lsas.copy()
    rids = sorted({int(x) for x in rl["adv_rtr"]})
    pick = [int(x) for x in rng.permutation(rids)]
    abrs, asbrs, plain = pick[:n_abr], pick[n_abr:n_abr + n_asbr], pick[n_abr + n_asbr:]
    for i in range(len(rl)):
        r = int(rl["adv_rtr"][i])
        rl["flags"][i] |= (0x01 if r in abrs else 0) | (0x02 if r in asbrs else 0)
    lost = []
    if unreachable_abr:
        lost = [max(rids) + 0x100]
        rl = np.concatenate([rl, np.array([(lost[0], 0, 1, 0x03, OPT_R | OPT_V6, len(area.links), 0)], ROUTER_LSA_DT)])
    a.router_lsas = rl
    own = sorted({(bytes(int(b) for b in p["addr"]["bytes"]), int(p["len"])) for p in area.prefixes
                  if not int(p["options"]) & PFX_NU})
    six = lambda hi, lo=0: ipaddress.IPv6Address((0x20010DB8 << 96) | (hi << 64) | lo).packed
    intra = [own[int(i)] for i in rng.choice(len(own), min(len(own), n_overlap), replace=False)]
    fresh = [(six(0xC8_0000 + i), 64) for i in range(n_fresh)]
    pool = intra + fresh + [(six(0xC8_0000, 5), 64), (six(0xC8_0001, 5), 64), (bytes(16), 0)]
    metric = lambda: int(rng.choice([1, 10, 10, 20, 30])) if rng.random() > 0.05 else ospf_rib.LSA_INFINITY
    maxage = lambda: int(rng.random() < 0.06)
    nu = lambda: PFX_NU if rng.random() < nu_fraction else 0
    rec = lambda b: (tuple(b), 1, (0, 0, 0))
    sums, ids = [], {}
    next_id = lambda adv: ids.__setitem__(adv, ids.get(adv, 0) + 1) or ids[adv]
    advs3 = abrs + lost + plain[:1] + [0x7F000001]                # the last two: never an ABR of the area
    for _ in range(n_inter):
        p, ln = pool[int(rng.integers(0, len(pool)))]
        adv = int(rng.choice(advs3))
        sums.append((adv, next_id(adv), metric(), 0, rec(p), ln, nu(), 3, maxage()))
    outside = [0x0B000001 + i for i in range(3)]                  # ASBRs in other areas
    for asbr in asbrs[:2] + outside:
        for abr in rng.choice(abrs + lost, int(rng.integers(1, 4)), replace=False):
            sums.append((int(abr), next_id(int(abr)), metric(), asbr, rec(bytes(16)), 0, nu(), 4, maxage()))
    sums.sort(key=lambda x: (x[7], x[0], x[1]))
    summaries = np.zeros(len(sums), ospf_rib.INTER_AREA_LSA_DT)
    for i, x in enumerate(sums):
        summaries[i] = x
    ext = []
    advs5 = asbrs + outside + lost + plain[:3] + abrs[:1] + [0x7F000002]
    only5 = [(six(0xC0_0000 + i), 64) for i in range(n_ext_only)]  # prefixes only externals name
    pool5 = pool + only5
    for _ in range(n_ext):
        p, ln = pool5[int(rng.integers(0, len(pool5)))]
        e_bit = 1 if (p, ln) in only5[:4] else int(rng.integers(0, 2))   # four prefixes of type-2 LSAs only
        adv = int(rng.choice(advs5))
        ext.append((adv, next_id(adv), int(rng.choice([1, 5, 5, 20])) if rng.random() > 0.05 else ospf_rib.LSA_INFINITY,
                    int(rng.integers(0, 4)), rec(p), ln, nu(), e_bit, maxage()))
    ext.sort(key=lambda x: (x[0], x[1]))
    externals = np.zeros(len(ext), ospf_rib.EXTERNAL6_LSA_DT)
    for i, x in enumerate(ext):
        externals[i] = x
    return a, summaries, externals


ABR_ROUTER_ID = 0x0AFF0001   # the router abr_view roots every area at (ospfv2.ABR_ROUTER_ID)
ABR_TIE_ASBR = 0x0B0000F1    # an ASBR outside the domain that every non-backbone area of abr_view names
PFX_LA, PFX_P = 0x02, 0x08   # prefix options carried to the routing table unchanged (RFC 5340 A.4.1.1)


def _with_prefixes(area: Ospfv3Area, adds: dict) -> Ospfv3Area:
    """area with one more Intra-Area-Prefix-LSA per router of `adds` {router_id: [(addr bytes, len, options, metric)]},
    referencing the router's Router-LSA; LsaKey order kept."""
    a = Ospfv3Area(**{k: getattr(area, k) for k in area.__dataclass_fields__})
    iaps, prefixes = [tuple(x) for x in area.iap_lsas.tolist()], [tuple(x) for x in area.prefixes.tolist()]
    for rid, ps in adds.items():
        off = len(prefixes)
        prefixes += [((tuple(b), 1, (0, 0, 0)), ln, opt, metric) for (b, ln, opt, metric) in ps]
        iaps.append((rid, 0x7000_0000, 1, REF_ROUTER, 0, 0, rid, off, len(ps)))
    ia = np.zeros(len(iaps), IAP_LSA_DT)
    for i, x in enumerate(iaps):
        ia[i] = x
    pa = np.zeros(len(prefixes), PREFIX_DT)
    for i, x in enumerate(prefixes):
        pa[i] = x
    a.iap_lsas, a.prefixes = ia[np.lexsort((ia["lsa_id"], ia["adv_rtr"]))], pa
    return a


def abr_view(topos: list, seed: int, area_ids=None, roots=None, max_paths: int = 16, n_shared: int = 6,
             v_flag_area: int | None = 1, **inter_kw):
    """The OSPFv3 twin of ospfv2.abr_view: a multi-area domain as one ABR sees it, returned as (areas [Ospfv3Area],
    inter-area LSAs [ospf_rib.INTER_AREA_LSA_DT[] per area, LsaKey order], AS-external LSAs ospf_rib.EXTERNAL6_LSA_DT[]),
    the areas in instance order.  Area k is synth_area(topos[k], root=roots[k]) with router ids, prefixes and interface
    sort keys in ranges of its own; the root is router ABR_ROUTER_ID in every area, with the B flag.  Seeded.
      * area 0 (area_ids[0], 0 by default) carries inter_area_view's load (NU-option LSAs, Inter-Area-Router LSAs whose
        lsa_id is not the ASBR; those naming the root dropped); every other area gets Inter-Area-Prefix LSAs from two
        ABRs of its own, for some of area 0's prefixes and new ones, some with the NU option, and Inter-Area-Router
        LSAs (lsa_id a counter, never the ASBR);
      * shared prefixes: area 0's first LAN prefix is also area 1's (a transit network in both areas); n_shared
        router prefixes of area 0 are also advertised by a router of each other area, half at the metric that ties
        area 0's route and with other prefix options, half not;
      * an ASBR in each non-backbone area (its farthest router) with externals of its own, also named by a backbone
        Inter-Area-Router LSA at metric 1; an ASBR outside the domain named by every non-backbone area at one
        forwarding metric;
      * with v_flag_area, a router of that area (not the root) gets the V flag."""
    from . import ospf_rib
    from .ospfv2 import _dist_from
    rng = np.random.default_rng(seed)
    A = len(topos)
    area_ids = list(area_ids) if area_ids is not None else list(range(A))
    roots = list(roots) if roots is not None else [0] * A
    six = lambda hi, lo=0: ipaddress.IPv6Address((0x20010DB8 << 96) | (hi << 64) | lo).packed
    rec = lambda b: (tuple(b), 1, (0, 0, 0))
    areas = []
    for k, (t, r) in enumerate(zip(topos, roots)):
        rids = [ABR_ROUTER_ID if i == r else RID_BASE + i + (k << 20) for i in range(t.n_routers)]
        a = synth_area(t, root=r, max_paths=max_paths, rids=rids, area_id=area_ids[k])
        pb = a.prefixes["addr"]["bytes"]
        keep = np.zeros(len(pb), bool)
        if k == 1:                       # area 1's first LAN prefix is area 0's
            keep = (pb[:, 4] == 0x30) & (pb[:, 5] == 0) & (pb[:, 6] == 0) & (pb[:, 7] == 0)
        pb[:, 5] = np.where(keep, pb[:, 5], pb[:, 5] + k)
        a.prefixes["addr"]["bytes"] = pb
        ifs = a.ifaces.copy()
        ifs["sort_key"] += 1000 * k
        ifs["ifindex"] += 1000 * k
        a.ifaces = ifs
        a.router_lsas["flags"][a.router_lsas["adv_rtr"] == ABR_ROUTER_ID] |= 0x01
        areas.append(a)
    a0, sums0, ext = inter_area_view(areas[0], seed, **inter_kw)
    a0.router_lsas["flags"][a0.router_lsas["adv_rtr"] == ABR_ROUTER_ID] |= 0x01
    sums0 = sums0[~((sums0["lsa_type"] == 4) & (sums0["router_id"] == ABR_ROUTER_ID))]
    areas[0] = a0
    flat0 = Flat(a0)
    d0 = _dist_from(flat0, flat0.router_vertex(ABR_ROUTER_ID))
    stubs0 = []                           # (addr bytes, len, metric, router) of area 0's router prefixes
    for l in a0.iap_lsas:
        if int(l["ref_type"]) != REF_ROUTER or int(l["adv_rtr"]) == ABR_ROUTER_ID:
            continue
        for p in a0.prefixes[int(l["prefix_off"]): int(l["prefix_off"]) + int(l["n_prefixes"])]:
            stubs0.append((bytes(int(b) for b in p["addr"]["bytes"]), int(p["len"]), int(p["metric"]), int(l["adv_rtr"])))
    flags0 = {}
    for rr, f in zip(a0.router_lsas["adv_rtr"], a0.router_lsas["flags"]):
        flags0.setdefault(int(rr), int(f))
    bb_abrs = [rr for rr, f in flags0.items() if f & 0x01 and rr != ABR_ROUTER_ID and flat0.router_vertex(rr) != 0xFFFFFFFF
               and d0[flat0.router_vertex(rr)] < 1 << 40]
    inter_prefixes = sorted({(bytes(int(b) for b in s["prefix"]["bytes"]), int(s["len"])) for s in sums0
                             if s["lsa_type"] == 3})
    summaries, ext_rows, extra4 = [sums0], [tuple(x) for x in ext.tolist()], []
    ids = {}
    next_id = lambda adv: ids.__setitem__(adv, ids.get(adv, 0x100) + 1) or ids[adv]
    for k in range(1, A):
        a = areas[k]
        flat = Flat(a)
        dk = _dist_from(flat, flat.router_vertex(ABR_ROUTER_ID))
        reach = {int(flat.router_ids[v]): int(dk[v]) for v in range(len(flat.router_ids))
                 if flat.is_router[v] and dk[v] < 1 << 40}
        others = sorted({int(x) for x in a.router_lsas["adv_rtr"]} - {ABR_ROUTER_ID})
        pick = [int(x) for x in rng.permutation([rr for rr in others if rr in reach])]
        abrs, vrtr = pick[:2], pick[3]
        asbr = max((rr for rr in pick[2:] if rr != vrtr), key=lambda rr: (reach[rr], rr))     # the farthest router
        adds = {}
        shared = [stubs0[int(i)] for i in rng.choice(len(stubs0), min(n_shared, len(stubs0)), replace=False)]
        for j, (p, ln, metric, adv) in enumerate(shared):
            want = int(d0[flat0.router_vertex(adv)]) + metric
            cand = [(rid, d) for rid, d in reach.items() if rid != ABR_ROUTER_ID and d <= want - 1]
            if not cand or want > 0xFFFF:
                continue
            rid, d = cand[int(rng.integers(0, len(cand)))]
            m2 = want - d if j % 2 == 0 else want - d + int(rng.choice([-1, 5]))
            adds.setdefault(rid, []).append((p, ln, PFX_LA if j % 2 == 0 else PFX_P, max(int(m2), 1)))
        a = _with_prefixes(a, adds)
        rl = a.router_lsas
        for rid in abrs:
            rl["flags"][rl["adv_rtr"] == rid] |= 0x01
        rl["flags"][rl["adv_rtr"] == asbr] |= 0x02
        if v_flag_area is not None and k == v_flag_area:
            rl["flags"][rl["adv_rtr"] == vrtr] |= 0x04
        areas[k] = a
        pool = [(p, ln) for (p, ln, _, _) in shared] + inter_prefixes[:6] + [(six(0xD0_0000 + (k << 4) + i), 64)
                                                                              for i in range(4)]
        sums = []
        for n, (p, ln) in enumerate(pool):
            for abr in abrs[: int(rng.integers(1, 3))]:
                sums.append((abr, next_id(abr), int(rng.choice([1, 5, 10, 20])), 0, rec(p), ln,
                             PFX_NU if n % 7 == 3 else 0, 3, 0))
        sums.append((abrs[0], next_id(abrs[0]), 10, 0x0B000001, rec(bytes(16)), 0, 0, 4, 0))
        # the ASBR outside the domain every non-backbone area names at one forwarding metric: with one active area the
        # entries tie across areas and the higher area id wins
        sums.append((abrs[0], next_id(abrs[0]), max(1, 1000 - reach[abrs[0]]), ABR_TIE_ASBR, rec(bytes(16)), 0, 0, 4, 0))
        # this area's ASBR, also named by a backbone Inter-Area-Router LSA through the nearest backbone ABR at metric 1
        if bb_abrs:
            near = min(bb_abrs, key=lambda rr: (int(d0[flat0.router_vertex(rr)]), rr))
            extra4.append((near, next_id(near), 1, asbr, rec(bytes(16)), 0, 0, 4, 0))
        sums.sort(key=lambda x: (x[7], x[0], x[1]))
        s = np.zeros(len(sums), ospf_rib.INTER_AREA_LSA_DT)
        for i, x in enumerate(sums):
            s[i] = x
        summaries.append(s)
        for i in range(3):
            ext_rows.append((asbr, next_id(asbr), int(rng.choice([1, 5, 20])), k, rec(six(0xE0_0000 + (k << 8) + i)), 64,
                             PFX_P if i == 1 else 0, int(i % 2), 0))
        ext_rows.append((asbr, next_id(asbr), 5, k, rec(six(0xE0_0000 + (k << 8) + 9)), 64, PFX_NU, 0, 0))
        if inter_prefixes:                   # an ASBR of area 0's view seen from this area too
            ext_rows.append((0x0B000001, next_id(0x0B000001), 7, 0, rec(six(0xE0_0000 + (k << 8) + 0xF)), 64, 0, 1, 0))
    if A > 1:
        for i in range(2):
            ext_rows.append((ABR_TIE_ASBR, next_id(ABR_TIE_ASBR), 3, 9, rec(six(0xEF_0000 + i)), 64, 0, i, 0))
    if extra4:
        s0 = sorted([tuple(x) for x in summaries[0].tolist()] + extra4, key=lambda x: (x[7], x[0], x[1]))
        s = np.zeros(len(s0), ospf_rib.INTER_AREA_LSA_DT)
        for i, x in enumerate(s0):
            s[i] = x
        summaries[0] = s
    ext_rows.sort(key=lambda x: (x[0], x[1]))
    externals = np.zeros(len(ext_rows), ospf_rib.EXTERNAL6_LSA_DT)
    for i, x in enumerate(ext_rows):
        externals[i] = x
    return areas, summaries, externals


def backbone_view(t0: Topology, t1: Topology, seed: int, r: int = 0, borders=((1, 0), (2, 1), (3, 2)),
                  max_paths: int = 16, n_ext_keys: int = 3, t2: Topology | None = None, r1: int | None = None,
                  area1_asbrs: int = 0, area1_ext: int = 4):
    """The OSPFv3 twin of ospfv2.backbone_view: a backbone router R of area 0 and the area border routers ("borders")
    of one other area 1, each as its own image.  Seeded.  Area 0 is synth_area(t0) (router i is RID_BASE + i), area 1
    synth_area(t1) with router ids, prefixes and interface sort keys in ranges of its own, except that border (i0, i1)
    is router i0 of t0 and router i1 of t1, with one router id and the B flag in both areas.  The first border is also
    attached to a small area 2 (t2, or a seeded 12-router topology; its router 0 is the border).  Returns a dict:
      r_area        R's area-0 image (router r of t0);
      summaries0    area 0's Inter-Area-Prefix LSAs (LsaKey order): each border's for the prefixes of its other areas
                    it reaches, at its distance plus the prefix metric, with that prefix's options (what a job
                    replaces);
      externals     an ASBR of area 0 (the E flag) with AS-external LSAs for n_ext_keys area-1 loopbacks (prefixes
                    that are also keys) and for one prefix of its own;
      borders       per border (areas, area ids, inter-area LSAs per area): the first border lists area 1, area 0,
                    area 2; the others area 0, area 1;
      flip          (address bytes, length) of a /128 two routers of area 1 advertise, one with the LA option and
                    one with the P option, at metrics that tie at the first border: the first border's route takes the
                    lower router id's record, and a job that lengthens that router's path alone hands the route to
                    the other record at the same metric, with other options;
      shared        (address bytes, length) of a /64 that is intra-area in area 1 (LA) and area 2 (P) at metrics that
                    tie at the first border (its route there keeps area 1's options, the first of its areas);
      r1_area       with r1: the area-1 image of router r1 of t1, with area 1's prefixes as the borders see them.
    area1_asbrs = k > 0 (drawn from a generator of its own, so that every other part is as without it): k routers of
    area 1 get the E flag ("area1_asbrs" in the dict) and area1_ext AS-external /64s each, both E-bit values and a mix
    of prefix options, on prefixes the next ASBR shares in half, plus the area-0 ASBR's own /64 at one below its
    type-2 metric (so an area-1 ASBR's LSA wins it while R reaches one).
    summaries0 then also holds each border's Inter-Area-Router LSAs for those it reaches in area 1, at that distance
    (what hspf_ospfv3_rtr_summaries gives in the base job), numbered after its Inter-Area-Prefix LSAs.  With k >= 2,
    "flip_ext" is (address bytes, length, x1, x2) of a /64 that the first two ASBRs advertise as type-1, x1 with the LA
    and x2 with the P option, at costs that tie through the last border: R's route takes x1's LSA, and a job that cuts
    x1 off alone hands it to x2's at the same metric, with other options.  A border left out of a backbone table keeps
    its LSAs as another ABR's static ones."""
    from . import ospf_rib, synth
    from .ospfv2 import _dist_from
    rng = np.random.default_rng(seed)
    six = lambda hi, lo=0: ipaddress.IPv6Address((0x20010DB8 << 96) | (hi << 64) | lo).packed
    rec = lambda b: (tuple(b), 1, (0, 0, 0))
    if t2 is None:
        t2 = synth.random_topology(12, 30, synth.SEED_BASE + 4000 + seed, cost_choices=[5, 10, 20])
    rid0 = lambda i: RID_BASE + int(i)
    bids = [rid0(i0) for i0, _ in borders]
    cand = [i for i in range(t0.n_routers) if i != r and rid0(i) not in bids]
    asbr = rid0(cand[int(rng.integers(0, len(cand)))])

    def image(t, k, root, border_of):
        """area k of topology t seen by `root`; border_of {router index: border router id}"""
        rids = [border_of.get(i, RID_BASE + i + (k << 20)) for i in range(t.n_routers)]
        a = synth_area(t, root=root, max_paths=max_paths, rids=rids, area_id=k)
        pb = a.prefixes["addr"]["bytes"]
        pb[:, 5] = pb[:, 5] + k
        a.prefixes["addr"]["bytes"] = pb
        ifs = a.ifaces.copy()
        ifs["sort_key"] += 1000 * k
        ifs["ifindex"] += 1000 * k
        a.ifaces = ifs
        rl = a.router_lsas.copy()
        for b in border_of.values():
            rl["flags"][rl["adv_rtr"] == b] |= 0x01
        a.router_lsas = rl
        return a

    b0map = {i0: rid0(i0) for i0, _ in borders}
    b1map = {i1: rid0(i0) for i0, i1 in borders}
    b2map = {0: bids[0]}
    img0 = lambda i: image(t0, 0, i, b0map)
    r_area = img0(r)
    a0s = [img0(i0) for i0, _ in borders]
    a1s = [image(t1, 1, i1, b1map) for _, i1 in borders]
    a2 = image(t2, 2, 0, b2map)
    for a in [r_area] + a0s:
        a.router_lsas["flags"][a.router_lsas["adv_rtr"] == asbr] |= 0x02

    def dists(a):
        fl = Flat(a)
        d = _dist_from(fl, fl.router_vertex(a.router_id))
        return {int(fl.router_ids[v]): int(d[v]) for v in range(len(fl.router_ids)) if fl.is_router[v] and d[v] < 1 << 40}
    # the flip key: two area-1 routers tying at the first border, the lower id with LA
    d1 = dists(a1s[0])
    inner = sorted((d, rr) for rr, d in d1.items() if rr not in bids)
    y = inner[0][1]                                      # the first border's nearest: its path is one link
    xs = [rr for d, rr in inner if rr < y] or [rr for d, rr in inner[1:]]
    x = xs[int(rng.integers(0, len(xs)))]
    M = max(d1[x], d1[y]) + 5
    flip = (six(0xF1_0000, 1), 128)
    adds1 = {x: [(flip[0], 128, PFX_LA, M - d1[x])], y: [(flip[0], 128, PFX_P, M - d1[y])]}
    # the shared key: area 1 and area 2 tying at the first border
    d2 = dists(a2)
    n1 = min((d, rr) for rr, d in d1.items() if rr not in bids)
    n2 = min((d, rr) for rr, d in d2.items() if rr not in bids)
    shared = (six(0xF2_0000), 64)
    adds1.setdefault(n1[1], []).append((shared[0], 64, PFX_LA, 10 + max(0, n2[0] - n1[0])))
    adds2 = {n2[1]: [(shared[0], 64, PFX_P, 10 + max(0, n1[0] - n2[0]))]}
    a1s = [_with_prefixes(a, adds1) for a in a1s]
    a2 = _with_prefixes(a2, adds2)
    r1_area = _with_prefixes(image(t1, 1, r1, b1map), adds1) if r1 is not None else None
    asbrs1 = []
    if area1_asbrs:
        rng1 = np.random.default_rng([seed, 0x3A5B])
        cand1 = sorted({int(x["adv_rtr"]) for x in a1s[0].router_lsas} - set(bids))
        asbrs1 = sorted(cand1[int(i)] for i in rng1.choice(len(cand1), min(area1_asbrs, len(cand1)), replace=False))
        for a in a1s + ([r1_area] if r1_area is not None else []):
            rl = a.router_lsas.copy()
            for x in asbrs1:
                rl["flags"][rl["adv_rtr"] == x] |= 0x02
            a.router_lsas = rl
    # each border's Inter-Area-Prefix LSAs into area 0: its other areas' prefixes that are not area 0's
    own0 = {(bytes(int(b) for b in p["addr"]["bytes"]), int(p["len"])) for p in r_area.prefixes}
    sums0 = []
    for j, bid in enumerate(bids):
        best = {}
        for a in [a1s[j]] + ([a2] if j == 0 else []):
            fl = Flat(a)
            d = _dist_from(fl, fl.router_vertex(bid))
            for l in a.iap_lsas:
                v = fl.router_vertex(int(l["adv_rtr"])) if int(l["ref_type"]) == REF_ROUTER else 0xFFFFFFFF
                if v == 0xFFFFFFFF or d[v] >= 1 << 40:
                    continue
                for p in a.prefixes[int(l["prefix_off"]): int(l["prefix_off"]) + int(l["n_prefixes"])]:
                    key = (bytes(int(b) for b in p["addr"]["bytes"]), int(p["len"]))
                    m = int(d[v]) + int(p["metric"])
                    if key in own0 or int(p["options"]) & PFX_NU or (key in best and best[key][0] <= m):
                        continue
                    best[key] = (m, int(p["options"]))
        for n, (key, (m, opt)) in enumerate(sorted(best.items())):
            sums0.append((bid, n + 1, m, 0, rec(key[0]), key[1], opt, 3, 0))
    # each border's Inter-Area-Router LSAs into area 0: the area-1 ASBRs it reaches, at that distance
    n_iap = {bid: sum(1 for x in sums0 if x[0] == bid) for bid in bids}
    d_last = {}
    for bid, a in zip(bids, a1s) if asbrs1 else ():
        d = dists(a)
        reach = [x for x in asbrs1 if x in d]
        sums0 += [(bid, n_iap[bid] + k + 1, d[x], x, ((0,) * 16, 0, (0, 0, 0)), 0, 0, 4, 0) for k, x in enumerate(reach)]
        if bid == max(bids):
            d_last = d
    sums0.sort(key=lambda x: (x[7], x[0], x[1]))
    summaries0 = np.zeros(len(sums0), ospf_rib.INTER_AREA_LSA_DT)
    for i, x in enumerate(sums0):
        summaries0[i] = x
    loops = sorted({(bytes(int(b) for b in p["addr"]["bytes"]), int(p["len"])) for p in a1s[0].prefixes
                    if int(p["len"]) == 128 and (bytes(int(b) for b in p["addr"]["bytes"]), 128) != flip})
    keys = [loops[int(i)] for i in rng.choice(len(loops), min(n_ext_keys, len(loops)), replace=False)]
    ext = [(asbr, j + 1, int(rng.choice([5, 30])), 7, rec(k[0]), k[1], PFX_P if j == 1 else 0, int(j % 2), 0)
           for j, k in enumerate(keys)]
    ext.append((asbr, len(keys) + 1, 12, 8, rec(six(0xE0_0000)), 64, 0, 1, 0))
    opts = (0, PFX_P, PFX_LA, PFX_LA | PFX_P)
    for m, x in enumerate(asbrs1):
        ext.append((x, 1, 11, 9, rec(six(0xE0_0000)), 64, 0, 1, 0))
        for q in range(area1_ext):
            ext.append((x, q + 2, int(rng1.integers(1, 40)), 10 + m, rec(six(0xE9_0000 + m * area1_ext // 2 + q)), 64,
                        opts[int(rng1.integers(0, len(opts)))], (q + m) % 2, 0))
    flip_ext = None
    if len(asbrs1) >= 2 and all(x in d_last for x in asbrs1[:2]):
        x1, x2 = asbrs1[:2]
        M = max(d_last[x1], d_last[x2]) + 5
        flip_ext = (six(0xEA_0000), 64, x1, x2)
        ext += [(x1, area1_ext + 2, M - d_last[x1], 11, rec(flip_ext[0]), 64, PFX_LA, 0, 0),
                (x2, area1_ext + 2, M - d_last[x2], 11, rec(flip_ext[0]), 64, PFX_P, 0, 0)]
    externals = np.zeros(len(ext), ospf_rib.EXTERNAL6_LSA_DT)
    for i, x in enumerate(sorted(ext, key=lambda x: (x[0], x[1]))):
        externals[i] = x
    empty = np.zeros(0, ospf_rib.INTER_AREA_LSA_DT)
    out_borders = []
    for j, (a0, a1) in enumerate(zip(a0s, a1s)):
        s0 = summaries0[summaries0["adv_rtr"] != a0.router_id]
        if j == 0:
            out_borders.append(([a1, a0, a2], [1, 0, 2], [empty, s0, empty]))
        else:
            out_borders.append(([a0, a1], [0, 1], [s0, empty]))
    out = {"r_area": r_area, "summaries0": summaries0, "externals": externals, "borders": out_borders,
           "flip": flip, "shared": shared, "asbr": asbr}
    if area1_asbrs:
        out["area1_asbrs"], out["flip_ext"] = asbrs1, flip_ext
    if r1 is not None:
        out["r1_area"] = r1_area
    return out


def _lsa_array(rows, dt):
    out = np.zeros(len(rows), dt)
    for i, x in enumerate(rows):
        out[i] = x
    return out


def abr_backbone_view(t0: Topology, t1: Topology, t2: Topology, seed: int, r: int = 0, r2: int = 0,
                      borders=((1, 0), (2, 1), (3, 2)), max_paths: int = 16, n_ext_keys: int = 3, area1_asbrs: int = 0,
                      area1_ext: int = 4):
    """The OSPFv3 twin of ospfv2.abr_backbone_view: an area border router R of area 0 and of an area only R borders,
    and the borders of area 1, each as its own image: backbone_view's domain (areas 0 and 1, the three borders, the
    first also in area 2, the area-0 ASBR, with area1_asbrs / area1_ext its area-1 ASBRs, their AS-external LSAs and the
    borders' Inter-Area-Router LSAs), with R (router r of t0) also router r2 of synth_area(t2) as area 3 (area 2 is the
    first border's), in ranges of its own, and the B flag in both of R's areas.  Seeded; area 3 draws from a generator
    of its own.  Returns a dict:
      r_areas       R's images [area 0, area 3] (area ids `area_ids` [0, 3]), `summaries` per area: backbone_view's
                    summaries0 and none for area 3 (R is its only ABR);
      externals     backbone_view's, plus an area-3 ASBR's ("area3_asbr", the E flag) AS-external LSAs: the area-0 ASBR's
                    own /64, which every area-1 ASBR also advertises, and a /64 of its own ("area3_ext");
      area3_shared  (address bytes, length) of a prefix the borders advertise into area 0 that is also a prefix of an
                    area-3 router (intra-area at R);
      flip          backbone_view's option flip: a /128 two area-1 routers advertise with the LA and the P option, at
                    metrics that tie at the first border;
      borders, shared, asbr, area1_asbrs, flip_ext  as backbone_view's (R has the B flag in the borders' area-0 images)."""
    from . import ospf_rib
    from .ospfv2 import _dist_from
    v = backbone_view(t0, t1, seed, r=r, borders=borders, max_paths=max_paths, n_ext_keys=n_ext_keys,
                      area1_asbrs=area1_asbrs, area1_ext=area1_ext)
    rng = np.random.default_rng([seed, 0xAB3])
    six = lambda hi, lo=0: ipaddress.IPv6Address((0x20010DB8 << 96) | (hi << 64) | lo).packed
    rec = lambda b: (tuple(b), 1, (0, 0, 0))
    R = RID_BASE + int(r)

    def with_b(a, rids, bit=0x01):
        a = Ospfv3Area(**{k: getattr(a, k) for k in a.__dataclass_fields__})
        rl = a.router_lsas.copy()
        for x in rids:
            rl["flags"][rl["adv_rtr"] == x] |= bit
        a.router_lsas = rl
        return a
    rids = [R if i == r2 else RID_BASE + i + (3 << 20) for i in range(t2.n_routers)]
    a3 = synth_area(t2, root=r2, max_paths=max_paths, rids=rids, area_id=3)
    pb = a3.prefixes["addr"]["bytes"]
    pb[:, 5] = pb[:, 5] + 3
    a3.prefixes["addr"]["bytes"] = pb
    ifs = a3.ifaces.copy()
    ifs["sort_key"] += 3000
    ifs["ifindex"] += 3000
    a3.ifaces = ifs
    a3 = with_b(a3, [R])
    fl = Flat(a3)
    d = _dist_from(fl, fl.router_vertex(R))
    reach = sorted(int(fl.router_ids[x]) for x in range(len(fl.router_ids)) if fl.is_router[x] and 0 < d[x] < 1 << 40)
    t3 = v["summaries0"][v["summaries0"]["lsa_type"] == 3]
    pick = t3[int(rng.integers(0, len(t3)))]
    shared3 = (bytes(int(b) for b in pick["prefix"]["bytes"]), int(pick["len"]))
    a3 = _with_prefixes(a3, {reach[int(rng.integers(0, len(reach)))]: [(shared3[0], shared3[1], 0, 1)]})
    asbr3 = reach[int(rng.integers(0, len(reach)))]
    a3 = with_b(a3, [asbr3], 0x02)
    own3 = (six(0xE3_0000), 64)
    ext = [tuple(x) for x in v["externals"].tolist()]
    ext += [(asbr3, 1, 12, 12, rec(six(0xE0_0000)), 64, 0, 1, 0),
            (asbr3, 2, int(rng.integers(1, 40)), 12, rec(own3[0]), 64, PFX_P, 0, 0)]
    out_borders = [([with_b(a, [R]) if a.area_id == 0 else a for a in areas], ids, sums)
                   for areas, ids, sums in v["borders"]]
    return {"r_areas": [with_b(v["r_area"], [R]), a3], "area_ids": [0, 3],
            "summaries": [v["summaries0"], np.zeros(0, ospf_rib.INTER_AREA_LSA_DT)],
            "externals": _lsa_array(sorted(ext, key=lambda x: (x[0], x[1])), ospf_rib.EXTERNAL6_LSA_DT),
            "area3_shared": shared3, "area3_asbr": asbr3, "area3_ext": own3, "borders": out_borders,
            "shared": v["shared"], "flip": v["flip"], "asbr": v["asbr"], "area1_asbrs": v.get("area1_asbrs", []),
            "flip_ext": v.get("flip_ext")}


def nonbackbone_view(t0: Topology, t1: Topology, seed: int, spf, r: int | None = None,
                     borders=((1, 0), (2, 1), (3, 2)), max_paths: int = 16, n_ext_keys: int = 3, n_ext: int = 0):
    """The OSPFv3 twin of ospfv2.nonbackbone_view: an internal router R of area 1 and the area border routers
    ("borders") between area 0 and area 1, each as its own image: backbone_view's domain seen from area 1.  Seeded.
    Areas, borders (the first also in area 2), the area-0 ASBR (the E flag) with its AS-external LSAs are
    backbone_view(t0, t1, seed, ...)'s; R is router r of t1 (default: the first that is not a border).  Two area-0
    routers also get the B flag and advertise one /128 into area 0, one with the LA and one with the P option, at
    metrics that tie at the first border (the "inter-area flip": the first border's inter-area route takes the first
    LSA's record, and a job that lengthens that router's path alone hands the route to the other at the same metric,
    with other options).  `spf(csr, root_vertex, nh_words)` gives unperturbed planes, as area_from_planes takes them.
    Returns a dict:
      r_area        R's area-1 image;
      summaries1    area 1's Inter-Area-Prefix / Inter-Area-Router LSAs (LsaKey order): each border's
                    hspf_ospfv3_net_summaries and hspf_ospfv3_rtr_summaries into area 1 over its update_rib_full at the
                    unperturbed job, lsa_id numbered per border (nonbackbone_lsas);
      externals     backbone_view's, plus n_ext /64s of the area-0 ASBR, both E-bit values (drawn from a generator of
                    its own, so that every other part is as without them);
      borders       per border (areas, area ids, inter-area LSAs per area) as backbone_view's, the area-0 LSAs holding
                    the inter-area flip's two;
      flip          (address bytes, length) of the inter-area flip's /128, and its two advertisers (LA's first);
      shared        backbone_view's shared /64;
      asbr          the area-0 ASBR's router id."""
    from . import ospf_rib
    from .ospfv2 import _dist_from
    bids = {RID_BASE + int(i0) for i0, _ in borders}
    if r is None:
        r = next(i for i in range(t1.n_routers) if i not in {int(i1) for _, i1 in borders})
    v = backbone_view(t0, t1, seed, borders=borders, max_paths=max_paths, n_ext_keys=n_ext_keys, r1=r)
    rng = np.random.default_rng([seed, 0x1F1])
    # the inter-area flip: two area-0 routers, neither a border nor the ASBR, tying at the first border
    first = next(a for a in v["borders"][0][0] if a.area_id == 0)
    fl = Flat(first)
    d = _dist_from(fl, fl.router_vertex(first.router_id))
    dist = {int(fl.router_ids[u]): int(d[u]) for u in range(len(fl.router_ids)) if fl.is_router[u] and d[u] < 1 << 40}
    cand = sorted(x for x in dist if x not in bids and x != v["asbr"])
    x, y = sorted(int(q) for q in rng.choice(cand, 2, replace=False))
    M = max(dist[x], dist[y]) + 7
    key = (ipaddress.IPv6Address((0x20010DB8 << 96) | (0xF3_0000 << 64) | 1).packed, 128)
    rec = lambda b: (tuple(b), 1, (0, 0, 0))
    flip_lsas = [(x, 0x900, M - dist[x], 0, rec(key[0]), 128, PFX_LA, 3, 0),
                 (y, 0x900, M - dist[y], 0, rec(key[0]), 128, PFX_P, 3, 0)]
    out_borders = []
    for areas, ids, sums in v["borders"]:
        areas = list(areas)
        i0 = ids.index(0)
        a0 = Ospfv3Area(**{k: getattr(areas[i0], k) for k in areas[i0].__dataclass_fields__})
        rl = a0.router_lsas.copy()
        for q in (x, y):
            rl["flags"][rl["adv_rtr"] == q] |= 0x01
        a0.router_lsas = rl
        areas[i0] = a0
        s0 = sorted([tuple(z) for z in sums[i0].tolist()] + flip_lsas, key=lambda z: (z[7], z[0], z[1]))
        sums = list(sums)
        sums[i0] = _lsa_array(s0, ospf_rib.INTER_AREA_LSA_DT)
        out_borders.append((areas, ids, sums))
    ext = v["externals"]
    if n_ext:
        rng_e = np.random.default_rng([seed, 0x0E1])
        six = lambda hi, lo=0: ipaddress.IPv6Address((0x20010DB8 << 96) | (hi << 64) | lo).packed
        more = [(v["asbr"], 0x1000 + q, int(rng_e.integers(1, 40)), 11, rec(six(0xE8_0000 + q)), 64, 0, q % 2, 0)
                for q in range(n_ext)]
        ext = _lsa_array(sorted([tuple(z) for z in ext.tolist()] + more, key=lambda z: (z[0], z[1])),
                         ospf_rib.EXTERNAL6_LSA_DT)
    sums1 = []
    for areas, ids, bsums in out_borders:
        rib_areas = [ospf_rib.RibArea(a.area_id, area_from_planes(a, spf), a.ifaces, s, True)
                     for a, s in zip(areas, bsums)]
        sums1 += nonbackbone_lsas(areas[0].router_id, max_paths, rib_areas, ext, ids.index(1))
    return {"r_area": v["r1_area"], "summaries1": _lsa_array(sorted(sums1, key=lambda z: (z[7], z[0], z[1])),
                                                             ospf_rib.INTER_AREA_LSA_DT),
            "externals": ext, "borders": out_borders, "flip": (key[0], key[1], x, y), "shared": v["shared"],
            "asbr": v["asbr"]}


def nonbackbone_lsas(router_id: int, max_paths: int, rib_areas: list, externals, target: int, configs=None) -> list:
    """What an OSPFv3 border originates into rib_areas[target]: its update_rib_full over rib_areas, then
    hspf_ospfv3_net_summaries and hspf_ospfv3_rtr_summaries, as INTER_AREA_LSA_DT rows with lsa_id numbered from 1 in
    output order (Inter-Area-Prefix first)."""
    from . import ospf_rib
    cfg = configs if configs is not None else [ospf_rib.area_config()] * len(rib_areas)
    rib = ospf_rib.update_rib_full_v3(router_id, max_paths, rib_areas, externals)
    rows = [tuple(z) for z in ospf_rib.net_summaries_v3(router_id, rib, rib_areas, cfg, target).tolist()]
    rows += [tuple(z) for z in ospf_rib.rtr_summaries_v3(router_id, rib_areas, cfg, target).tolist()]
    return [(z[0], k + 1) + tuple(z[2:]) for k, z in enumerate(rows)]


def third_area_view(t0: Topology, t1: Topology, t3: Topology, seed: int, spf, n_c: int = 2, max_paths: int = 16,
                    n_ext_keys: int = 3, area1_asbrs: int = 0, area1_ext: int = 4):
    """The OSPFv3 twin of ospfv2.third_area_view: an internal router R of a non-backbone area, the area border routers
    C of that area and area 0 (n_c of them, 2 or 3), and the borders B of area 1, each as its own image.  Areas 0 and 1
    are backbone_view's (its three B's, the first also in area 2, the area-0 ASBR, area1_asbrs area-1 ASBRs with their
    AS-external and Inter-Area-Router LSAs); R's area is area 3, synth_area(t3) in ranges of its own, whose routers
    0 .. n_c - 1 are the C's (routers 0, then the first routers of t0 past the borders that are not the area-0 ASBR; the
    B flag in areas 0 and 3) and whose router n_c is R.  Area 3 also holds an ASBR ("area3_asbr", the E flag) with a
    /64 of its own, and a router that also advertises a prefix the B's advertise into area 0 ("area3_shared").  Seeded;
    area 3 draws from a generator of its own, so that every other generator's output stays as it was.
    `spf(csr, root_vertex, nh_words)` gives unperturbed planes, as area_from_planes takes them.  Returns a dict:
      r_area        R's area-3 image;
      summaries3    area 3's Inter-Area-Prefix / Inter-Area-Router LSAs (LsaKey order): each C's
                    hspf_ospfv3_net_summaries and hspf_ospfv3_rtr_summaries into area 3 over its update_rib_full at the
                    unperturbed job (nonbackbone_lsas);
      externals     backbone_view's plus the area-3 ASBR's;
      c_areas       per C (areas [area 0, area 3], area ids [0, 3], summaries per area: area 0's, none for area 3);
      borders       per B as backbone_view's (the C's have the B flag in its area-0 image);
      asbr, area1_asbrs, area3_asbr, area3_shared, flip, flip_ext, shared."""
    from . import ospf_rib
    from .ospfv2 import _dist_from
    if n_c not in (2, 3):
        raise ValueError("n_c is 2 or 3")
    v = backbone_view(t0, t1, seed, r=0, max_paths=max_paths, n_ext_keys=n_ext_keys, area1_asbrs=area1_asbrs,
                      area1_ext=area1_ext)
    rng = np.random.default_rng([seed, 0xC3B])
    six = lambda hi, lo=0: ipaddress.IPv6Address((0x20010DB8 << 96) | (hi << 64) | lo).packed
    rec = lambda b: (tuple(b), 1, (0, 0, 0))
    c0 = [0] + [i for i in range(4, t0.n_routers) if RID_BASE + i != v["asbr"]][:n_c - 1]
    cids = [RID_BASE + i for i in c0]

    def with_flags(a, bits):
        a = Ospfv3Area(**{k: getattr(a, k) for k in a.__dataclass_fields__})
        rl = a.router_lsas.copy()
        for x, b in bits.items():
            rl["flags"][rl["adv_rtr"] == x] |= b
        a.router_lsas = rl
        return a

    cflag = {c: 0x01 for c in cids}

    def img3(i):
        rids = [cids[k] if k < n_c else RID_BASE + k + (3 << 20) for k in range(t3.n_routers)]
        a = synth_area(t3, root=i, max_paths=max_paths, rids=rids, area_id=3)
        pb = a.prefixes["addr"]["bytes"]
        pb[:, 5] = pb[:, 5] + 3
        a.prefixes["addr"]["bytes"] = pb
        ifs = a.ifaces.copy()
        ifs["sort_key"] += 3000
        ifs["ifindex"] += 3000
        a.ifaces = ifs
        return with_flags(a, cflag)

    ra = img3(n_c)
    fl = Flat(ra)
    d = _dist_from(fl, fl.router_vertex(ra.router_id))
    reach = sorted(int(fl.router_ids[x]) for x in range(len(fl.router_ids))
                   if fl.is_router[x] and 0 < d[x] < 1 << 40 and int(fl.router_ids[x]) not in cids)
    t3s = v["summaries0"][v["summaries0"]["lsa_type"] == 3]
    pick = t3s[int(rng.integers(0, len(t3s)))]
    shared3 = (bytes(int(b) for b in pick["prefix"]["bytes"]), int(pick["len"]))
    adds = {reach[int(rng.integers(0, len(reach)))]: [(shared3[0], shared3[1], 0, 1)]}
    asbr3 = reach[int(rng.integers(0, len(reach)))]
    area3 = lambda i: with_flags(_with_prefixes(img3(i), adds), {asbr3: 0x02})
    own3 = (six(0xE3_0000), 64)
    ext = [tuple(x) for x in v["externals"].tolist()]
    ext += [(asbr3, 1, int(rng.integers(1, 40)), 12, rec(own3[0]), 64, PFX_P, 0, 0)]
    externals = _lsa_array(sorted(ext, key=lambda x: (x[0], x[1])), ospf_rib.EXTERNAL6_LSA_DT)
    bits0 = dict(cflag)
    bits0.update({RID_BASE + int(i0): 0x01 for i0 in (1, 2, 3)})
    bits0[v["asbr"]] = 0x02

    def area0(i):
        return with_flags(v["r_area"], cflag) if i == 0 else \
            with_flags(synth_area(t0, root=i, max_paths=max_paths, area_id=0), bits0)
    empty = np.zeros(0, ospf_rib.INTER_AREA_LSA_DT)
    c_areas = [([area0(i), area3(k)], [0, 3], [v["summaries0"], empty]) for k, i in enumerate(c0)]
    sums = []
    for areas, ids, csums in c_areas:
        rib_areas = [ospf_rib.RibArea(a.area_id, area_from_planes(a, spf), a.ifaces, s, True)
                     for a, s in zip(areas, csums)]
        sums += nonbackbone_lsas(areas[0].router_id, max_paths, rib_areas, externals, 1)
    borders = [([with_flags(a, cflag) if a.area_id == 0 else a for a in areas], ids, bs)
               for areas, ids, bs in v["borders"]]
    return {"r_area": area3(n_c), "summaries3": _lsa_array(sorted(sums, key=lambda z: (z[7], z[0], z[1])),
                                                           ospf_rib.INTER_AREA_LSA_DT),
            "externals": externals, "c_areas": c_areas, "borders": borders, "asbr": v["asbr"],
            "area1_asbrs": v.get("area1_asbrs", []), "area3_asbr": asbr3, "area3_shared": shared3,
            "flip": v["flip"], "flip_ext": v.get("flip_ext"), "shared": v["shared"]}
