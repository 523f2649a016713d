"""OSPFv2 routing-table stages after the per-area SPFs, from Python: ctypes/numpy twins of
hl_ospfv2_summary_lsa / hl_ospfv2_external_lsa / hl_ospfv2_rib_area / hl_rib_route /
hl_ospfv2_rib (include/holo_lsdb.h) and the `hspf_ospfv2_update_rib_full` call
(update_rib_full, holo-ospf/src/route.rs:146-193: inter-area networks and routers, transit
areas, AS-external routes)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import capi, ospfv2, route_table

PATH_INTRA, PATH_INTER, PATH_TYPE1, PATH_TYPE2 = 0, 1, 2, 3
PATH_NAMES = {PATH_INTRA: "intra-area", PATH_INTER: "inter-area", PATH_TYPE1: "external-1", PATH_TYPE2: "external-2"}
LSA_INFINITY = 0x00FFFFFF

SUMMARY_LSA_DT = np.dtype([("adv_rtr", "<u4"), ("lsa_id", "<u4"), ("mask", "<u4"), ("metric", "<u4"),
                           ("lsa_type", "u1"), ("maxage", "u1"), ("_pad", "u1", (2,))], align=True)
EXTERNAL_LSA_DT = np.dtype([("adv_rtr", "<u4"), ("lsa_id", "<u4"), ("mask", "<u4"), ("metric", "<u4"),
                            ("fwd_addr", "<u4"), ("tag", "<u4"), ("e_bit", "u1"), ("maxage", "u1"),
                            ("_pad", "u1", (2,))], align=True)
RIB_ROUTE_DT = np.dtype([("prefix", "<u4"), ("mask", "<u4"), ("metric", "<u4"), ("type2_metric", "<u4"),
                         ("tag", "<u4"), ("area_id", "<u4"), ("path_type", "u1"), ("flags", "u1"), ("has_area", "u1"),
                         ("has_type2", "u1"), ("nh_off", "<u4"), ("n_nh", "<u4"), ("sr_label", "<u4"),
                         ("has_sr_label", "u1"), ("_pad", "u1", (3,))], align=True)
ROUTE_CONNECTED, ROUTE_INSTALLED = 0x01, 0x02
RIB_INSTALL, RIB_UNINSTALL, RIB_UNINSTALL_OLD = 1, 2, 3
ACTION_DT = np.dtype([("route", "<u4"), ("old_sr_label", "<u4"), ("kind", "u1"), ("has_old_sr_label", "u1"),
                      ("_pad", "u1", (2,))], align=True)


# OSPFv3 twins (hl_ospfv3_inter_area_lsa, hl_ospfv3_external_lsa, hl_rib_route6)
def _ip_dt():
    from . import ospfv3
    return ospfv3.IP_DT


INTER_AREA_LSA_DT = np.dtype([("adv_rtr", "<u4"), ("lsa_id", "<u4"), ("metric", "<u4"), ("router_id", "<u4"),
                              ("prefix", _ip_dt()), ("len", "u1"), ("prefix_options", "u1"), ("lsa_type", "u1"),
                              ("maxage", "u1")], align=True)
EXTERNAL6_LSA_DT = np.dtype([("adv_rtr", "<u4"), ("lsa_id", "<u4"), ("metric", "<u4"), ("tag", "<u4"),
                             ("prefix", _ip_dt()), ("len", "u1"), ("prefix_options", "u1"), ("e_bit", "u1"),
                             ("maxage", "u1")], align=True)
RIB_ROUTE6_DT = np.dtype([("prefix", _ip_dt()), ("len", "u1"), ("path_type", "u1"), ("flags", "u1"),
                          ("prefix_options", "u1"), ("has_area", "u1"), ("has_type2", "u1"), ("_pad", "u1", (2,)),
                          ("metric", "<u4"), ("type2_metric", "<u4"), ("tag", "<u4"), ("area_id", "<u4"),
                          ("nh_off", "<u4"), ("n_nh", "<u4")], align=True)


class RibAreaStruct(C.Structure):
    _fields_ = [
        ("area_id", C.c_uint32), ("n_summaries", C.c_uint32),
        ("spf", C.c_void_p), ("ifaces", C.c_void_p), ("summaries", C.c_void_p),
        ("n_ifaces", C.c_uint32), ("active", C.c_uint8), ("_pad", C.c_uint8 * 3),
    ]


class RibStruct(C.Structure):
    _fields_ = [
        ("routes_cap", C.c_uint32), ("n_routes", C.c_uint32), ("routes", C.c_void_p),
        ("nexthops_cap", C.c_uint32), ("n_nexthops", C.c_uint32), ("nexthops", C.c_void_p),
    ]


# appended to hspf_abi_sizes() after the OSPFv3 block
ABI_SIZES = [SUMMARY_LSA_DT.itemsize, EXTERNAL_LSA_DT.itemsize, C.sizeof(RibAreaStruct), RIB_ROUTE_DT.itemsize,
             C.sizeof(RibStruct),
             INTER_AREA_LSA_DT.itemsize, EXTERNAL6_LSA_DT.itemsize, C.sizeof(RibAreaStruct), RIB_ROUTE6_DT.itemsize,
             C.sizeof(RibStruct),       # hl_ospfv3_rib_area / hl_ospfv3_rib have the layouts of the v2 structs
             ACTION_DT.itemsize]


@dataclass
class RibArea:
    """One attached area: the result of run_area, the area's interfaces and Summary-LSAs."""
    area_id: int
    result: ospfv2.Ospfv2Result
    ifaces: np.ndarray
    summaries: np.ndarray
    active: bool = True


@dataclass
class Rib:
    routes: np.ndarray
    nexthops: np.ndarray
    rc: int = 0

    def nh(self, rec):
        return [tuple(int(x[k]) for k in ("iface", "has_addr", "addr", "has_nbr", "nbr_router_id", "has_label", "sr_label"))
                for x in self.nexthops[int(rec["nh_off"]): int(rec["nh_off"]) + int(rec["n_nh"])]]


def _version(v3: bool):
    """(result struct class, result dtypes, iface dtype, summary dtype, external dtype, route dtype, nexthop dtype)"""
    if not v3:
        return (ospfv2.ResultStruct,
                (("vertices", ospfv2.SPT_VERTEX_DT), ("routers", ospfv2.ROUTE_RTR_DT), ("routes", ospfv2.ROUTE_NET_DT),
                 ("nexthops", ospfv2.NEXTHOP_DT)),
                ospfv2.IFACE_DT, SUMMARY_LSA_DT, EXTERNAL_LSA_DT, RIB_ROUTE_DT, ospfv2.NEXTHOP_DT)
    from . import ospfv3
    return (ospfv3.ResultStruct,
            (("vertices", ospfv3.SPT_VERTEX6_DT), ("routers", ospfv2.ROUTE_RTR_DT), ("routes", ospfv3.ROUTE_NET6_DT),
             ("nexthops", ospfv3.NEXTHOP6_DT)),
            ospfv3.IFACE_DT, INTER_AREA_LSA_DT, EXTERNAL6_LSA_DT, RIB_ROUTE6_DT, ospfv3.NEXTHOP6_DT)


def _result_struct(res, keep: list, v3: bool = False):
    cls, fields = _version(v3)[:2]
    r = cls()
    for name, dt in fields:
        a = np.ascontiguousarray(getattr(res, name), dtype=dt)
        keep.append(a)
        setattr(r, name + "_cap", len(a))
        setattr(r, "n_" + name, len(a))
        setattr(r, name, a.ctypes.data if len(a) else None)
    r.transit_capability = int(res.transit_capability)
    r.root_found = int(res.root_found)
    return r


def call_update_rib_full(fn, router_id: int, max_paths: int, areas: list, externals=None, v3: bool = False) -> Rib:
    """`fn` = hspf_ospfv{2,3}_update_rib_full of the product library or the oracle's twin."""
    _cls, _fields, IFACE_DT_, SUM_DT_, EXT_DT_, ROUTE_DT_, NH_DT_ = _version(v3)
    fn.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(RibAreaStruct), C.c_uint32, C.c_void_p, C.c_uint32,
                   C.POINTER(RibStruct)]
    keep = []
    arr = (RibAreaStruct * max(len(areas), 1))()
    for i, a in enumerate(areas):
        rs = _result_struct(a.result, keep, v3)
        keep.append(rs)
        ifs = np.ascontiguousarray(a.ifaces, dtype=IFACE_DT_)
        sm = np.ascontiguousarray(a.summaries, dtype=SUM_DT_)
        keep += [ifs, sm]
        arr[i].area_id, arr[i].n_summaries = a.area_id, len(sm)
        arr[i].spf = C.addressof(rs)
        arr[i].ifaces = ifs.ctypes.data if len(ifs) else None
        arr[i].summaries = sm.ctypes.data if len(sm) else None
        arr[i].n_ifaces, arr[i].active = len(ifs), int(a.active)
    ext = np.ascontiguousarray(externals if externals is not None else np.zeros(0, EXT_DT_), dtype=EXT_DT_)
    caps = [256, 1024]
    for _ in range(3):
        routes = np.zeros(caps[0], ROUTE_DT_)
        nhs = np.zeros(caps[1], NH_DT_)
        r = RibStruct()
        r.routes_cap, r.routes = caps[0], routes.ctypes.data
        r.nexthops_cap, r.nexthops = caps[1], nhs.ctypes.data
        rc = fn(router_id, max_paths, arr, len(areas), ext.ctypes.data if len(ext) else None, len(ext), C.byref(r))
        if rc == capi.HSPF_E_NOMEM:
            caps = [max(caps[0], r.n_routes), max(caps[1], r.n_nexthops)]
            continue
        break
    return Rib(routes[: r.n_routes].copy(), nhs[: r.n_nexthops].copy(), rc)


def update_rib_full(router_id: int, max_paths: int, areas: list, externals=None) -> Rib:
    """The product's host stage (libholo_spf.so); needs no device."""
    lib = capi.load_library()
    rib = call_update_rib_full(lib.hspf_ospfv2_update_rib_full, router_id, max_paths, areas, externals)
    if rib.rc != capi.HSPF_OK:
        raise capi.HspfError(rib.rc, "hspf_ospfv2_update_rib_full failed")
    return rib


def update_rib_full_v3(router_id: int, max_paths: int, areas: list, externals=None) -> Rib:
    """OSPFv3 twin (hspf_ospfv3_update_rib_full); host only."""
    lib = capi.load_library()
    rib = call_update_rib_full(lib.hspf_ospfv3_update_rib_full, router_id, max_paths, areas, externals, v3=True)
    if rib.rc != capi.HSPF_OK:
        raise capi.HspfError(rib.rc, "hspf_ospfv3_update_rib_full failed")
    return rib


def _rib_struct(rib: Rib, keep: list, route_dt, nh_dt) -> RibStruct:
    r = RibStruct()
    routes = np.ascontiguousarray(rib.routes, dtype=route_dt)
    nhs = np.ascontiguousarray(rib.nexthops, dtype=nh_dt)
    keep += [routes, nhs]
    r.routes_cap = r.n_routes = len(routes)
    r.nexthops_cap = r.n_nexthops = len(nhs)
    r.routes = routes.ctypes.data if len(routes) else None
    r.nexthops = nhs.ctypes.data if len(nhs) else None
    return r


def call_rib_diff(fn, old, new: Rib, v3: bool = False):
    """update_global_rib: returns (actions ACTION_DT[], new routes with HL_ROUTE_INSTALLED set as the
    reference would).  `fn` = hspf_ospfv{2,3}_rib_diff or the oracle's twin; `old` may be None."""
    ROUTE_DT_, NH_DT_ = _version(v3)[5:7]
    fn.argtypes = [C.c_void_p, C.POINTER(RibStruct), C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    keep = []
    ns = _rib_struct(new, keep, ROUTE_DT_, NH_DT_)
    new_routes = keep[0]
    if new_routes is new.routes:                  # never write into the caller's array
        new_routes = new_routes.copy()
        keep[0] = new_routes
        ns.routes = new_routes.ctypes.data if len(new_routes) else None
    os_ = _rib_struct(old, keep, ROUTE_DT_, NH_DT_) if old is not None else None
    cap = len(new.routes) + (len(old.routes) if old is not None else 0) + 1
    acts = np.zeros(cap, ACTION_DT)
    n = C.c_uint32()
    rc = fn(C.addressof(os_) if os_ is not None else None, C.byref(ns), acts.ctypes.data, cap, C.byref(n))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, "rib_diff failed")
    return acts[: n.value].copy(), new_routes


def rib_diff(old, new: Rib, v3: bool = False):
    lib = capi.load_library()
    return call_rib_diff(lib.hspf_ospfv3_rib_diff if v3 else lib.hspf_ospfv2_rib_diff, old, new, v3)


# ---- partial runs (update_rib_partial, holo-ospf/src/route.rs:196-340), OSPFv2 ---------------------------
RIB_RTR_DT = np.dtype([("area_id", "<u4"), ("router_id", "<u4"), ("metric", "<u4"), ("path_type", "u1"), ("flags", "u1"),
                       ("_pad", "u1", (2,)), ("nh_off", "<u4"), ("n_nh", "<u4")], align=True)


class RtrTablesStruct(C.Structure):
    _fields_ = [("rtrs_cap", C.c_uint32), ("n_rtrs", C.c_uint32), ("rtrs", C.c_void_p),
                ("nexthops_cap", C.c_uint32), ("n_nexthops", C.c_uint32), ("nexthops", C.c_void_p)]


@dataclass
class RtrTables:
    rtrs: np.ndarray
    nexthops: np.ndarray


def _area_array(areas: list, keep: list, with_results: bool, v3: bool = False):
    _cls, _fields, iface_dt, sum_dt = _version(v3)[:4]
    arr = (RibAreaStruct * max(len(areas), 1))()
    for i, a in enumerate(areas):
        ifs = np.ascontiguousarray(a.ifaces, dtype=iface_dt)
        sm = np.ascontiguousarray(a.summaries, dtype=sum_dt)
        keep += [ifs, sm]
        arr[i].area_id, arr[i].n_summaries = a.area_id, len(sm)
        if with_results:
            rs = _result_struct(a.result, keep, v3)
            keep.append(rs)
            arr[i].spf = C.addressof(rs)
        arr[i].ifaces = ifs.ctypes.data if len(ifs) else None
        arr[i].summaries = sm.ctypes.data if len(sm) else None
        arr[i].n_ifaces, arr[i].active = len(ifs), int(a.active)
    return arr


def _tables_out(cap_r, cap_h, keep):
    rt, nh = np.zeros(max(cap_r, 1), RIB_RTR_DT), np.zeros(max(cap_h, 1), ospfv2.NEXTHOP_DT)
    keep += [rt, nh]
    s = RtrTablesStruct(len(rt), 0, rt.ctypes.data, len(nh), 0, nh.ctypes.data)
    return s, rt, nh


def router_tables(router_id: int, areas: list, fn=None) -> RtrTables:
    """hspf_ospfv2_rib_router_tables: area.state.routers of every area after a full run."""
    if fn is None:
        fn = capi.load_library().hspf_ospfv2_rib_router_tables
    fn.argtypes = [C.c_uint32, C.POINTER(RibAreaStruct), C.c_uint32, C.POINTER(RtrTablesStruct)]
    keep = []
    arr = _area_array(areas, keep, True)
    caps = [64, 256]
    for _ in range(3):
        s, rt, nh = _tables_out(caps[0], caps[1], keep)
        rc = fn(router_id, arr, len(areas), C.byref(s))
        if rc == capi.HSPF_E_NOMEM:
            caps = [max(caps[0], s.n_rtrs), max(caps[1], s.n_nexthops)]
            continue
        break
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, "rib_router_tables failed")
    return RtrTables(rt[: s.n_rtrs].copy(), nh[: s.n_nexthops].copy())


def update_rib_partial(router_id: int, max_paths: int, areas: list, externals, triggers_or_sets, prev_rib: Rib,
                       prev_rtrs: RtrTables, fn=None):
    """hspf_ospfv2_update_rib_partial -> (new Rib, new RtrTables, actions).  `triggers_or_sets`: the
    (inter_network [(addr, mask)], inter_router [id], external [(addr, mask)]) sets of a PARTIAL computation."""
    if fn is None:
        fn = capi.load_library().hspf_ospfv2_update_rib_partial
    fn.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(RibAreaStruct), C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32,
                   C.POINTER(ospfv2.SpfComputationStruct), C.POINTER(RibStruct), C.POINTER(RtrTablesStruct),
                   C.POINTER(RibStruct), C.POINTER(RtrTablesStruct), C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    keep = []
    arr = _area_array(areas, keep, False)
    transit = np.asarray([int(a.result.transit_capability) for a in areas] or [0], np.uint8)
    ext = np.ascontiguousarray(externals if externals is not None else np.zeros(0, EXTERNAL_LSA_DT), dtype=EXTERNAL_LSA_DT)
    net, rtr, xt = triggers_or_sets
    netA = np.asarray(net or [(0, 0)], ospfv2.IPV4_NET_DT)
    rtrA = np.asarray(rtr or [0], np.uint32)
    xtA = np.asarray(xt or [(0, 0)], ospfv2.IPV4_NET_DT)
    pc = ospfv2.SpfComputationStruct(ospfv2.SPF_PARTIAL, len(net), len(rtr), len(xt), max(len(net), len(rtr), len(xt), 1),
                                     netA.ctypes.data, rtrA.ctypes.data, xtA.ctypes.data)
    prs = _rib_struct(prev_rib, keep, RIB_ROUTE_DT, ospfv2.NEXTHOP_DT)
    prt = np.ascontiguousarray(prev_rtrs.rtrs, RIB_RTR_DT)
    pnh = np.ascontiguousarray(prev_rtrs.nexthops, ospfv2.NEXTHOP_DT)
    pts = RtrTablesStruct(len(prt), len(prt), prt.ctypes.data if len(prt) else None, len(pnh), len(pnh),
                          pnh.ctypes.data if len(pnh) else None)
    caps = [len(prev_rib.routes) + 64, len(prev_rib.nexthops) + 512, len(prt) + 64, len(pnh) + 512, len(prev_rib.routes) + 128]
    for _ in range(3):
        routes, nhs = np.zeros(caps[0], RIB_ROUTE_DT), np.zeros(caps[1], ospfv2.NEXTHOP_DT)
        out = RibStruct(caps[0], 0, routes.ctypes.data, caps[1], 0, nhs.ctypes.data)
        ts, rt, tnh = _tables_out(caps[2], caps[3], keep)
        acts = np.zeros(caps[4], ACTION_DT)
        n = C.c_uint32()
        rc = fn(router_id, max_paths, arr, transit.ctypes.data, len(areas), ext.ctypes.data if len(ext) else None, len(ext),
                C.byref(pc), C.byref(prs), C.byref(pts), C.byref(out), C.byref(ts), acts.ctypes.data, caps[4], C.byref(n))
        if rc == capi.HSPF_E_NOMEM:
            caps = [max(caps[0], out.n_routes), max(caps[1], out.n_nexthops), max(caps[2], ts.n_rtrs), max(caps[3], ts.n_nexthops),
                    max(caps[4], n.value)]
            continue
        break
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, "update_rib_partial failed")
    return (Rib(routes[: out.n_routes].copy(), nhs[: out.n_nexthops].copy()), RtrTables(rt[: ts.n_rtrs].copy(), tnh[: ts.n_nexthops].copy()),
            acts[: n.value].copy())


# ---- batched routing-table stage for roots attached to one area (include/holo_spf_lsdb.h) ------------------
RIB_CELL_DT = np.dtype([("nh_mask", "<u8"), ("aux", "<u8"), ("winner", "<u4"), ("mpf", "<u4")])
RIB_RECORD_DT = np.dtype([("x", "<u4"), ("y", "<u4"), ("z", "<u4"), ("w", "<u4")])   # ospf_rib_cells.h: RibRec
JS_NOT_INTERNAL = 0x40            # HSPF_JS_NOT_INTERNAL: the job's root is an ABR
NO_RECORD = 0xFFFFFFFF


def cell_metric(cells):
    return cells["mpf"] & 0x03FFFFFF


def cell_path(cells):
    return (cells["mpf"] >> 26) & 0x3


def cell_flags(cells):
    return cells["mpf"] >> 28


class RibTable(route_table.RouteTable):
    """hspf_ospfv2_ribtable: the area's intra-area, type-3 and type-5 prefixes in prefix order and, per prefix,
    its intra-area advertisers, type-3 and type-5 records (host); `off` holds the three ranges per prefix
    ([3, P + 1]).  `upload(ctx)` copies it to the device for hspf_ospfv2_rib_cells.

    From an ospfv3.Flat the table is hspf_ospfv3_ribtable_create's (summaries: INTER_AREA_LSA_DT, externals:
    EXTERNAL6_LSA_DT); `prefix` then holds the IPv6 prefixes (ospfv3.IP_DT) and `v3` is set."""

    api, kind, contrib_dt = "hspf_ospfv2", "ribtable", RIB_RECORD_DT

    def __init__(self, flat, area_id: int, summaries=None, externals=None):
        from . import ospfv3
        self.flat = flat
        self.v3 = isinstance(flat, ospfv3.Flat)
        sum_dt, ext_dt = (INTER_AREA_LSA_DT, EXTERNAL6_LSA_DT) if self.v3 else (SUMMARY_LSA_DT, EXTERNAL_LSA_DT)
        sm = np.ascontiguousarray(summaries if summaries is not None else np.zeros(0, sum_dt), sum_dt)
        ext = np.ascontiguousarray(externals if externals is not None else np.zeros(0, ext_dt), ext_dt)
        self.area_id, self.summaries, self.externals = area_id, sm, ext
        lib = capi.load_library()
        super().__init__(lib.hspf_ospfv3_ribtable_create if self.v3 else lib.hspf_ospfv2_ribtable_create, flat.handle,
                         area_id, sm.ctypes.data if len(sm) else None, len(sm), ext.ctypes.data if len(ext) else None,
                         len(ext))
        pp, pl, po = C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint32)()
        self._call("arrays", C.byref(pp), C.byref(pl), C.byref(po), None)
        self.prefix = route_table.copy_records(pp, self.n_prefixes, np.uint32)
        self.plen = route_table.copy_records(pl, self.n_prefixes, np.uint32)
        self.off = route_table.copy_records(po, 3 * (self.n_prefixes + 1), np.uint32).reshape(3, self.n_prefixes + 1)
        if self.v3:
            p6 = C.c_void_p()
            rc = lib.hspf_ospfv3_ribtable_prefixes6(self.handle, C.byref(p6), None)
            if rc != capi.HSPF_OK:
                raise capi.HspfError(rc, "hspf_ospfv3_ribtable_prefixes6 failed")
            self.prefix = route_table.copy_records(p6, self.n_prefixes, ospfv3.IP_DT)


def rib_cells_device(ctx: capi.Context, rt: RibTable, n_jobs: int, rs, roots_ptr: int, cells_ptr: int,
                     status_out_ptr: int = 0, n_gather: int = 0, gather_job_ptr: int = 0, gather_v_ptr: int = 0,
                     gather_nh_ptr: int = 0):
    """hspf_ospfv2_rib_cells / _cells16 over DEVICE planes (rs: capi.ResultStruct or capi.Result16Struct holding
    device pointers); roots_ptr: device u32[n_jobs] root vertices; cells_ptr: device buffer of n_jobs * rt.n_prefixes
    RIB_CELL_DT; status_out_ptr: device u32[n_jobs] or 0.  Enqueued on the ctx stream; the table must have been
    uploaded."""
    route_table.call_stage(ctx, "hspf_ospfv2_rib_cells", rs, rt.handle, n_jobs, C.byref(rs), roots_ptr or None, cells_ptr,
                           status_out_ptr or None, n_gather, gather_job_ptr or None, gather_v_ptr or None,
                           gather_nh_ptr or None)


def rib_delta_device(ctx: capi.Context, rt: RibTable, n_jobs: int, rs, roots_ptr: int, base_ptr: int, n_base: int,
                     base_of_ptr: int, job_out_ptr: int, records_ptr: int, cap: int, n_records_ptr: int):
    """hspf_ospfv2_rib_delta / _delta16 over DEVICE planes (rs and roots_ptr as for rib_cells_device; rt an OSPFv2 or
    OSPFv3 RibTable): each job's cells compared with its base row of base_ptr ([n_base, rt.n_prefixes] RIB_CELL_DT, normally rib_cells_device over the
    unperturbed job of the same root; base_of_ptr: [n_jobs] u32 rows, 0 for row 0 of every job), without storing them.
    job_out_ptr: [n_jobs] route_table.DELTA_JOB_DT; records_ptr: [cap] route_table.DELTA_DT in (job, prefix) order
    (0 or cap 0: summaries only); n_records_ptr: u64 total.  All device pointers; enqueued on the ctx stream."""
    route_table.call_stage(ctx, "hspf_ospfv2_rib_delta", rs, rt.handle, n_jobs, C.byref(rs), roots_ptr or None,
                           base_ptr or None, n_base, base_of_ptr or None, job_out_ptr or None, records_ptr or None, cap,
                           n_records_ptr or None)


def _call_rib(fn, args, n_prefixes: int, route_dt, nh_dt) -> Rib:
    """fn(*args, &rib), the buffers grown once to the counts an HSPF_E_NOMEM reports."""
    caps = [max(n_prefixes, 1), max(4 * n_prefixes, 64)]
    for _ in range(2):
        routes, nhs = np.zeros(caps[0], route_dt), np.zeros(caps[1], nh_dt)
        r = RibStruct(caps[0], 0, routes.ctypes.data, caps[1], 0, nhs.ctypes.data)
        rc = fn(*args, C.byref(r))
        if rc == capi.HSPF_E_NOMEM:
            caps = [max(caps[0], r.n_routes), max(caps[1], r.n_nexthops)]
            continue
        break
    if rc not in (capi.HSPF_OK, capi.HSPF_E_UNSUPPORTED):
        raise capi.HspfError(rc, fn.__name__ + " failed")
    if rc != capi.HSPF_OK:
        return Rib(np.zeros(0, route_dt), np.zeros(0, nh_dt), rc)
    return Rib(routes[: r.n_routes].copy(), nhs[: r.n_nexthops].copy(), rc)


def _call_rib_from_cells(fn, area, rt: RibTable, cells: np.ndarray, gather_v, gather_nh, route_dt, nh_dt) -> Rib:
    cells = np.ascontiguousarray(cells, RIB_CELL_DT)
    assert cells.shape == (rt.n_prefixes,)
    gv = np.ascontiguousarray(gather_v, np.uint32)
    gn = np.ascontiguousarray(gather_nh, np.uint64)
    s = area.as_struct()
    return _call_rib(fn, (C.byref(s), rt.handle, cells.ctypes.data, gv.ctypes.data_as(C.POINTER(C.c_uint32)),
                          gn.ctypes.data_as(C.POINTER(C.c_uint64)), len(gv)), rt.n_prefixes, route_dt, nh_dt)


def rib_from_cells(area: ospfv2.Ospfv2Area, rt: RibTable, cells: np.ndarray, gather_v, gather_nh) -> Rib:
    """hspf_ospfv2_rib_from_cells (host): one job's cells -> the routing table update_rib_full gives for
    area.router_id over its one area.  rc HSPF_E_UNSUPPORTED is returned in the result (caller: the host
    stages over that job's planes)."""
    return _call_rib_from_cells(capi.load_library().hspf_ospfv2_rib_from_cells, area, rt, cells, gather_v, gather_nh,
                                RIB_ROUTE_DT, ospfv2.NEXTHOP_DT)


def rib_from_cells_v3(area, rt: RibTable, cells: np.ndarray, gather_v, gather_nh) -> Rib:
    """hspf_ospfv3_rib_from_cells (host): one job's cells over an OSPFv3 RibTable -> the routing table
    update_rib_full_v3 gives for area.router_id (an ospfv3.Ospfv3Area) over its one area (RIB_ROUTE6_DT routes,
    ospfv3.NEXTHOP6_DT next hops).  rc HSPF_E_UNSUPPORTED is returned in the result, as rib_from_cells."""
    from . import ospfv3
    return _call_rib_from_cells(capi.load_library().hspf_ospfv3_rib_from_cells, area, rt, cells, gather_v, gather_nh,
                                RIB_ROUTE6_DT, ospfv3.NEXTHOP6_DT)


# ---- batched routing-table stage for area border routers (include/holo_spf_lsdb.h) --------------------------
ABR_MAX_AREAS = 8                  # HSPF_ABR_MAX_AREAS


class AbrRibTable(route_table.RouteTable):
    """hspf_ospfv2_abr_ribtable: the routing-table records of one area border router over its attached areas, in
    the instance's area order.  `flats`: one ospfv2.Flat per area (each with the router as a router vertex);
    `summaries`: each area's SUMMARY_LSA_DT[] (LsaKey order); `active`: per area (default all); `externals`: the
    instance's EXTERNAL_LSA_DT[].  `off` is [2 n_areas + 1, P + 1] (intra-area ranges per area, type-3 ranges per
    area, type-5 ranges); per area `roots`, `n_vertices`, `atom_base`, `n_atoms`.

    From ospfv3.Flat areas the table is hspf_ospfv3_abr_ribtable_create's (summaries: INTER_AREA_LSA_DT, externals:
    EXTERNAL6_LSA_DT); `prefix` and `prefixes6` then hold the IPv6 prefixes (ospfv3.IP_DT) and `v3` is set."""

    api, kind, contrib_dt = "hspf_ospfv2", "abr_ribtable", RIB_RECORD_DT

    def __init__(self, router_id: int, flats: list, area_ids, summaries=None, active=None, externals=None):
        from . import ospfv3
        n = len(flats)
        self.router_id, self.flats, self.area_ids = router_id, list(flats), [int(a) for a in area_ids]
        self.v3 = bool(flats) and isinstance(flats[0], ospfv3.Flat)
        sum_dt, ext_dt = (INTER_AREA_LSA_DT, EXTERNAL6_LSA_DT) if self.v3 else (SUMMARY_LSA_DT, EXTERNAL_LSA_DT)
        sums = [np.ascontiguousarray(s if s is not None else np.zeros(0, sum_dt), sum_dt)
                for s in (summaries if summaries is not None else [None] * n)]
        ext = np.ascontiguousarray(externals if externals is not None else np.zeros(0, ext_dt), ext_dt)
        self.summaries, self.externals = sums, ext
        self.active = [True] * n if active is None else [bool(a) for a in active]
        fl = (C.c_void_p * max(n, 1))(*[f.handle.value for f in flats])
        ids = np.asarray(self.area_ids or [0], np.uint32)
        sp = (C.c_void_p * max(n, 1))(*[s.ctypes.data if len(s) else None for s in sums])
        ns = np.asarray([len(s) for s in sums] or [0], np.uint32)
        act = np.asarray([int(a) for a in self.active] or [0], np.uint8)
        self._keep = (fl, ids, sp, ns, act, sums, ext, flats)
        lib = capi.load_library()
        create = lib.hspf_ospfv3_abr_ribtable_create if self.v3 else lib.hspf_ospfv2_abr_ribtable_create
        super().__init__(create, router_id, n, fl, ids.ctypes.data, sp, ns.ctypes.data, act.ctypes.data,
                         ext.ctypes.data if len(ext) else None, len(ext))
        self.n_areas = n
        pp, pl, po = C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint32)()
        self._call("arrays", C.byref(pp), C.byref(pl), C.byref(po), None)
        self.prefix = route_table.copy_records(pp, self.n_prefixes, np.uint32)
        self.plen = route_table.copy_records(pl, self.n_prefixes, np.uint32)
        self.off = route_table.copy_records(po, (2 * n + 1) * (self.n_prefixes + 1), np.uint32).reshape(2 * n + 1, -1)
        info = [np.zeros(n, np.uint32) for _ in range(4)]
        self._call("areas", *[x.ctypes.data for x in info])
        self.roots, self.n_vertices, self.atom_base, self.n_atoms = [[int(v) for v in x] for x in info]
        if self.v3:
            p6 = C.c_void_p()
            rc = lib.hspf_ospfv3_abr_ribtable_prefixes6(self.handle, C.byref(p6), None)
            if rc != capi.HSPF_OK:
                raise capi.HspfError(rc, "hspf_ospfv3_abr_ribtable_prefixes6 failed")
            self.prefixes6 = route_table.copy_records(p6, self.n_prefixes, ospfv3.IP_DT)
            self.prefix = self.prefixes6


def _planes_array(planes: list):
    """Host array of capi.ResultStruct / capi.Result16Struct (one per area, device pointers)."""
    return (type(planes[0]) * len(planes))(*planes)


def abr_rib_cells_device(ctx: capi.Context, rt: AbrRibTable, n_jobs: int, planes: list, n_rows, rows_ptr: int,
                         cells_ptr: int, status_out_ptr: int = 0, n_gather: int = 0, gather_job_ptr: int = 0,
                         gather_area_ptr: int = 0, gather_v_ptr: int = 0, gather_nh_ptr: int = 0):
    """hspf_ospfv2_abr_rib_cells / _cells16 over DEVICE planes: `planes` one capi.ResultStruct (nh_words 1) or
    capi.Result16Struct per area, in the table's order; n_rows: rows of each area's planes; rows_ptr: device
    u32[n_jobs, n_areas]; cells_ptr: device [n_jobs, rt.n_prefixes] RIB_CELL_DT; gathers as (job, area, vertex)
    triples.  Enqueued on the ctx stream; the table must have been uploaded."""
    nr = np.ascontiguousarray(n_rows, np.uint32)
    route_table.call_stage(ctx, "hspf_ospfv2_abr_rib_cells", planes[0], rt.handle, n_jobs, _planes_array(planes),
                           nr.ctypes.data, rows_ptr or None, cells_ptr or None, status_out_ptr or None, n_gather,
                           gather_job_ptr or None, gather_area_ptr or None, gather_v_ptr or None, gather_nh_ptr or None)


def abr_rib_delta_device(ctx: capi.Context, rt: AbrRibTable, n_jobs: int, planes: list, n_rows, rows_ptr: int,
                         base_ptr: int, n_base: int, base_of_ptr: int, job_out_ptr: int, records_ptr: int, cap: int,
                         n_records_ptr: int):
    """hspf_ospfv2_abr_rib_delta / _delta16: each job's cells (as abr_rib_cells_device) compared with its base row of
    base_ptr on the device, as rib_delta_device."""
    nr = np.ascontiguousarray(n_rows, np.uint32)
    route_table.call_stage(ctx, "hspf_ospfv2_abr_rib_delta", planes[0], rt.handle, n_jobs, _planes_array(planes),
                           nr.ctypes.data, rows_ptr or None, base_ptr or None, n_base, base_of_ptr or None,
                           job_out_ptr or None, records_ptr or None, cap, n_records_ptr or None)


def _call_abr_rib_from_cells(fn, area_struct, areas: list, rt: AbrRibTable, cells: np.ndarray, gather_area, gather_v,
                             gather_nh, route_dt, nh_dt) -> Rib:
    cells = np.ascontiguousarray(cells, RIB_CELL_DT)
    assert cells.shape == (rt.n_prefixes,)
    ga = np.ascontiguousarray(gather_area, np.uint32)
    gv = np.ascontiguousarray(gather_v, np.uint32)
    gn = np.ascontiguousarray(gather_nh, np.uint64)
    structs = [a.as_struct() for a in areas]
    arr = (area_struct * max(len(areas), 1))(*structs)
    return _call_rib(fn, (rt.handle, arr, len(areas), cells.ctypes.data, ga.ctypes.data, gv.ctypes.data, gn.ctypes.data,
                          len(gv)), rt.n_prefixes, route_dt, nh_dt)


def abr_rib_from_cells(areas: list, rt: AbrRibTable, cells: np.ndarray, gather_area, gather_v, gather_nh) -> Rib:
    """hspf_ospfv2_abr_rib_from_cells (host): one job's cells -> the routing table update_rib_full gives for
    rt.router_id over its areas (ospfv2.Ospfv2Area images in the table's order).  rc HSPF_E_UNSUPPORTED is returned
    in the result, as rib_from_cells."""
    return _call_abr_rib_from_cells(capi.load_library().hspf_ospfv2_abr_rib_from_cells, ospfv2.AreaStruct, areas, rt,
                                    cells, gather_area, gather_v, gather_nh, RIB_ROUTE_DT, ospfv2.NEXTHOP_DT)


def abr_rib_from_cells_v3(areas: list, rt: AbrRibTable, cells: np.ndarray, gather_area, gather_v, gather_nh) -> Rib:
    """hspf_ospfv3_abr_rib_from_cells (host): one job's cells over an OSPFv3 AbrRibTable -> the routing table
    update_rib_full_v3 gives for rt.router_id over its areas (ospfv3.Ospfv3Area images in the table's order;
    RIB_ROUTE6_DT routes, ospfv3.NEXTHOP6_DT next hops).  rc HSPF_E_UNSUPPORTED is returned in the result, as
    rib_from_cells."""
    from . import ospfv3
    return _call_abr_rib_from_cells(capi.load_library().hspf_ospfv3_abr_rib_from_cells, ospfv3.AreaStruct, areas, rt,
                                    cells, gather_area, gather_v, gather_nh, RIB_ROUTE6_DT, ospfv3.NEXTHOP6_DT)


# ---- Summary-LSA origination of an area border router (include/holo_spf_lsdb.h) ----------------------------------
AREA_NORMAL, AREA_STUB, AREA_NSSA = 0, 1, 2
AREA_CONFIG_DT = np.dtype([("default_cost", "<u4"), ("area_type", "u1"), ("summary", "u1"), ("_pad", "u1", (2,))],
                          align=True)


def area_config(area_type: int = AREA_NORMAL, summary: bool = True, default_cost: int = 10):
    """One hl_ospf_area_config: the reference's defaults are a normal area with summaries and default cost 10."""
    return (default_cost, area_type, int(summary), (0, 0))


def net_summaries(router_id: int, rib: Rib, rtrs: RtrTables, areas: list, configs: list, target: int) -> np.ndarray:
    """hspf_ospfv2_net_summaries (host): the type-3 and type-4 contents the router originates into areas[target]
    (compute_net_summaries / compute_rtr_summaries), as SUMMARY_LSA_DT[] with adv_rtr = router_id and lsa_id the
    prefix address (type 3) or the ASBR id (type 4): type 3 in prefix order, then type 4 in router-id order.
    rib: update_rib_full's table; rtrs: router_tables' over the same areas (RibArea list); configs: one area_config()
    per area."""
    lib = capi.load_library()
    keep = []
    arr = _area_array(areas, keep, False)
    cfg = np.asarray(list(configs) or [area_config()], AREA_CONFIG_DT)
    rs = _rib_struct(rib, keep, RIB_ROUTE_DT, ospfv2.NEXTHOP_DT)
    prt = np.ascontiguousarray(rtrs.rtrs, RIB_RTR_DT)
    pnh = np.ascontiguousarray(rtrs.nexthops, ospfv2.NEXTHOP_DT)
    ts = RtrTablesStruct(len(prt), len(prt), prt.ctypes.data if len(prt) else None, len(pnh), len(pnh),
                         pnh.ctypes.data if len(pnh) else None)
    cap = len(rib.routes) + len(prt) + 1
    out = np.zeros(cap, SUMMARY_LSA_DT)
    n = C.c_uint32()
    rc = lib.hspf_ospfv2_net_summaries(router_id, C.byref(rs), C.byref(ts), arr, cfg.ctypes.data, len(areas), target,
                                       out.ctypes.data, cap, C.byref(n))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, "hspf_ospfv2_net_summaries failed")
    return out[: n.value].copy()


def net_summaries_v3(router_id: int, rib: Rib, areas: list, configs: list, target: int) -> np.ndarray:
    """hspf_ospfv3_net_summaries (host): the Inter-Area-Prefix contents the router originates into areas[target]
    (compute_net_summaries), as INTER_AREA_LSA_DT[] with adv_rtr = router_id, lsa_id 0, lsa_type 3 and each route's
    prefix options, in prefix order.  rib: update_rib_full_v3's table over `areas` (RibArea list); configs: one
    area_config() per area."""
    from . import ospfv3
    lib = capi.load_library()
    keep = []
    arr = _area_array(areas, keep, False, v3=True)
    cfg = np.asarray(list(configs) or [area_config()], AREA_CONFIG_DT)
    rs = _rib_struct(rib, keep, RIB_ROUTE6_DT, ospfv3.NEXTHOP6_DT)
    cap = len(rib.routes) + 1
    out = np.zeros(cap, INTER_AREA_LSA_DT)
    n = C.c_uint32()
    rc = lib.hspf_ospfv3_net_summaries(router_id, C.byref(rs), arr, cfg.ctypes.data, len(areas), target,
                                       out.ctypes.data, cap, C.byref(n))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, "hspf_ospfv3_net_summaries failed")
    return out[: n.value].copy()


def rtr_summaries_v3(router_id: int, areas: list, configs: list, target: int) -> np.ndarray:
    """hspf_ospfv3_rtr_summaries (host): the Inter-Area-Router contents the router originates into areas[target]
    (compute_rtr_summaries), as INTER_AREA_LSA_DT[] with adv_rtr = router_id, lsa_type 4, router_id the ASBR and its
    metric, in router-id order.  areas: the RibArea list given update_rib_full_v3; configs: one area_config() per
    area."""
    lib = capi.load_library()
    keep = []
    arr = _area_array(areas, keep, True, v3=True)
    cfg = np.asarray(list(configs) or [area_config()], AREA_CONFIG_DT)
    # one entry per id at most: every area's routers, and the ASBRs its Inter-Area-Router LSAs name
    cap = sum(len(a.result.routers) + int((np.asarray(a.summaries)["lsa_type"] == 4).sum()) for a in areas) + 1
    out = np.zeros(cap, INTER_AREA_LSA_DT)
    n = C.c_uint32()
    rc = lib.hspf_ospfv3_rtr_summaries(router_id, arr, cfg.ctypes.data, len(areas), target, out.ctypes.data, cap,
                                       C.byref(n))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, "hspf_ospfv3_rtr_summaries failed")
    return out[: n.value].copy()


# ---- backbone router over what-if jobs inside other areas (include/holo_spf_lsdb.h) -----------------------------
BACKBONE_MAX_BORDERS = 8           # HSPF_BACKBONE_MAX_BORDERS


class BackboneTable:
    """hspf_ospfv2_backbone_table of one internal backbone router R: its affected prefixes over what-if jobs inside
    the borders' other areas.  `flat`: R's area-0 ospfv2.Flat; `summaries`: area 0's SUMMARY_LSA_DT[] in LsaKey order;
    `externals`: EXTERNAL_LSA_DT[]; `borders`: the borders' AbrRibTable list (kept alive with this table).  `prefix`,
    `plen` [n_prefixes]: the affected prefixes in prefix order; a slot's winner is n_records + its slot index
    (n_slots in all).

    From an ospfv3.Flat the table is hspf_ospfv3_backbone_table_create's (summaries: INTER_AREA_LSA_DT, externals:
    EXTERNAL6_LSA_DT, borders: OSPFv3 AbrRibTables); `prefix` and `prefixes6` then hold the IPv6 prefixes
    (ospfv3.IP_DT), `v3` is set, and a slot's winner is n_records + (slot index << 8 | its prefix options).

    asbr=True: hspf_ospfv2_backbone_asbr_table_create (from an OSPFv3 area-0 flat without `config`:
    hspf_ospfv3_backbone_asbr_table_create), which re-originates the borders' type-4 / Inter-Area-Router LSAs per job
    too; `n_asbr_slots` type-4 slots read `n_asbr_sets` (border, area) plane sets, and a table with type-4 slots is
    read by backbone_asbr_cells_device / backbone_asbr_delta_device only.  An OSPFv3 table of area 0 made without
    asbr=True is refused by those two.

    config=area_config(...): hspf_ospfv2_nonbackbone_table_create (from an ospfv3.Flat:
    hspf_ospfv3_nonbackbone_table_create), the table of an internal router R of the non-backbone area of `flat` (the
    target area, `area_id`) over what-if jobs on the backbone; `summaries` are that area's type-3/4 (Inter-Area-Prefix
    / Inter-Area-Router) LSAs, `config` its configuration, and the borders' type-4 LSAs are re-originated per job as
    with asbr=True.  The device calls of both kinds take it; backbone_from_cells (backbone_from_cells_v3) decodes it
    over R's image of the area.

    config=area_config(...) with AbrBackboneTable borders: hspf_ospfv2_third_area_table_create, the table of an
    internal router R of a non-backbone area over what-if jobs inside another non-backbone area; the borders are R's
    area's ABRs attached to area 0, each over the perturbed area's ABRs.  `third_area` is set; `n_asbr_slots` are chain
    slots, which read the borders' abr_backbone_asbr_entries_device output through third_area_cells_device /
    third_area_delta_device; a table without them also runs through the backbone calls.  From an ospfv3.Flat with
    OSPFv3 AbrBackboneTable borders: hspf_ospfv3_third_area_table_create, whose cells only the third-area calls read
    (its borders' cells hold OSPFv3 slot winners); backbone_from_cells_v3 decodes it.  A flat and borders of different
    versions raise ValueError (a list that mixes versions is refused by the create, HSPF_E_INVAL)."""

    def __init__(self, flat, router_id: int, summaries=None, externals=None, borders=(), asbr: bool = False,
                 config=None):
        from . import ospfv3
        self.lib = capi.load_library()
        self.flat, self.router_id, self.borders = flat, router_id, list(borders)
        self.v3 = isinstance(flat, ospfv3.Flat)
        if asbr and self.v3 and (config is not None or int(flat.area.area_id) != 0):
            raise ValueError("asbr=True takes an OSPFv3 flat of area 0 and no config")
        sum_dt, ext_dt = (INTER_AREA_LSA_DT, EXTERNAL6_LSA_DT) if self.v3 else (SUMMARY_LSA_DT, EXTERNAL_LSA_DT)
        sm = np.ascontiguousarray(summaries if summaries is not None else np.zeros(0, sum_dt), sum_dt)
        ext = np.ascontiguousarray(externals if externals is not None else np.zeros(0, ext_dt), ext_dt)
        self.summaries, self.externals = sm, ext
        arr = (C.c_void_p * max(len(self.borders), 1))(*[b.handle.value for b in self.borders])
        h = C.c_void_p()
        self.area_id = int(flat.area.area_id) if config is not None else 0
        self.third_area = bool(self.borders) and all(isinstance(b, AbrBackboneTable) for b in self.borders)
        if not self.third_area and any(isinstance(b, AbrBackboneTable) for b in self.borders):
            raise ValueError("borders are all AbrBackboneTables (a third-area table) or none is")
        if self.third_area and all(b.v3 != self.v3 for b in self.borders):
            raise ValueError("a third-area table's flat and borders are of one OSPF version")
        create = ("hspf_ospfv3_third_area_table_create" if self.third_area and self.v3 else
                  "hspf_ospfv2_third_area_table_create" if self.third_area else
                  "hspf_ospfv3_nonbackbone_table_create" if self.v3 and config is not None else
                  "hspf_ospfv3_backbone_asbr_table_create" if self.v3 and asbr else
                  "hspf_ospfv3_backbone_table_create" if self.v3 else
                  "hspf_ospfv2_nonbackbone_table_create" if config is not None else
                  "hspf_ospfv2_backbone_asbr_table_create" if asbr else "hspf_ospfv2_backbone_table_create")
        args = (sm.ctypes.data if len(sm) else None, len(sm), ext.ctypes.data if len(ext) else None, len(ext), arr,
                len(self.borders), C.byref(h))
        if config is not None:
            self.config = np.array([config], AREA_CONFIG_DT)
            args = (self.config.ctypes.data,) + args
        elif self.third_area:
            args = (None,) + args
        rc = getattr(self.lib, create)(flat.handle, router_id, *args)
        if rc != capi.HSPF_OK:
            raise capi.HspfError(rc, create + " failed")
        self.handle = h
        n, pp, pl = C.c_uint32(), C.c_void_p(), C.c_void_p()
        assert self.lib.hspf_ospfv2_backbone_table_prefixes(h, C.byref(n), C.byref(pp), C.byref(pl)) == capi.HSPF_OK
        self.n_prefixes = n.value
        self.prefix = route_table.copy_records(pp, self.n_prefixes, np.uint32)
        self.plen = route_table.copy_records(pl, self.n_prefixes, np.uint32)
        nr, ns = C.c_uint32(), C.c_uint32()
        assert self.lib.hspf_ospfv2_backbone_table_records(h, C.byref(nr), C.byref(ns)) == capi.HSPF_OK
        self.n_records, self.n_slots = nr.value, ns.value
        na, nsets = C.c_uint32(), C.c_uint32()
        assert self.lib.hspf_ospfv2_backbone_table_asbr_slots(h, C.byref(na), C.byref(nsets)) == capi.HSPF_OK
        self.n_asbr_slots, self.n_asbr_sets = na.value, nsets.value
        if self.v3:
            p6 = C.c_void_p()
            rc = self.lib.hspf_ospfv3_backbone_table_prefixes6(h, None, C.byref(p6), None)
            if rc != capi.HSPF_OK:
                raise capi.HspfError(rc, "hspf_ospfv3_backbone_table_prefixes6 failed")
            self.prefixes6 = route_table.copy_records(p6, self.n_prefixes, ospfv3.IP_DT)
            self.prefix = self.prefixes6

    def upload(self, ctx: capi.Context):
        rc = self.lib.hspf_ospfv2_backbone_table_upload(ctx.handle, self.handle)
        if rc != capi.HSPF_OK:
            raise capi.HspfError(rc, ctx.last_error())

    def __del__(self):
        try:
            if self.handle:
                self.lib.hspf_ospfv2_backbone_table_free(self.handle)
                self.handle = None
        except Exception:
            pass


def _device_ptrs(ptrs):
    return (C.c_void_p * max(len(ptrs), 1))(*[int(p) or None for p in ptrs])


def backbone_cells_device(ctx: capi.Context, t: BackboneTable, n_jobs: int, rs, border_cells, border_status,
                          status_ptr: int, cells_ptr: int):
    """hspf_ospfv2_backbone_cells / _cells16 over DEVICE planes.  rs: R's area-0 capi.ResultStruct (nh_words 1) or
    capi.Result16Struct, only row 0 read; border_cells: per border a device pointer to its [n_jobs, K_b] RIB_CELL_DT
    ABR cells; border_status: per border a device u32 [n_jobs] pointer or 0 (None: none); status_ptr: device u32
    [n_jobs] or 0; cells_ptr: device [n_jobs, t.n_prefixes] RIB_CELL_DT.  Enqueued on the ctx stream; the table must
    have been uploaded."""
    st = _device_ptrs(border_status) if border_status is not None else None
    route_table.call_stage(ctx, "hspf_ospfv2_backbone_cells", rs, t.handle, n_jobs, C.byref(rs),
                           _device_ptrs(border_cells), st, status_ptr or None, cells_ptr or None)


def backbone_delta_device(ctx: capi.Context, t: BackboneTable, n_jobs: int, rs, border_cells, border_status,
                          base_ptr: int, n_base: int, base_of_ptr: int, job_out_ptr: int, records_ptr: int, cap: int,
                          n_records_ptr: int):
    """hspf_ospfv2_backbone_delta / _delta16: the route-delta stage over the same walk (arguments as
    backbone_cells_device and rib_delta_device)."""
    st = _device_ptrs(border_status) if border_status is not None else None
    route_table.call_stage(ctx, "hspf_ospfv2_backbone_delta", rs, t.handle, n_jobs, C.byref(rs),
                           _device_ptrs(border_cells), st, base_ptr or None, n_base, base_of_ptr or None,
                           job_out_ptr or None, records_ptr or None, cap, n_records_ptr or None)


def _border_plane_args(border_planes, border_n_rows, border_rows, keep: list):
    """The three per-border arrays of the asbr calls (None: NULL)."""
    if border_planes is None:
        return None, None, None
    pl = [_planes_array(p) for p in border_planes]
    nr = [np.ascontiguousarray(x, np.uint32) for x in border_n_rows]
    keep += [pl, nr]
    return (C.c_void_p * len(pl))(*[C.addressof(p) for p in pl]), (C.c_void_p * len(nr))(*[x.ctypes.data for x in nr]), \
        _device_ptrs(border_rows)


def backbone_asbr_cells_device(ctx: capi.Context, t: BackboneTable, n_jobs: int, rs, border_cells, border_status,
                               border_planes, border_n_rows, border_rows, status_ptr: int, cells_ptr: int):
    """hspf_ospfv2_backbone_asbr_cells / _cells16: backbone_cells_device over a table with type-4 / Inter-Area-Router
    slots (either version; an OSPFv3 table of area 0 from BackboneTable(..., asbr=True) only), plus per border its
    DEVICE planes (one capi.ResultStruct / Result16Struct per area, as given abr_rib_cells_device, of R's width), its
    row counts per area, and a device pointer to its rows u32 [n_jobs, n_areas].  The three may be None for a table
    without type-4 slots."""
    keep = []
    st = _device_ptrs(border_status) if border_status is not None else None
    bp, bn, br = _border_plane_args(border_planes, border_n_rows, border_rows, keep)
    route_table.call_stage(ctx, "hspf_ospfv2_backbone_asbr_cells", rs, t.handle, n_jobs, C.byref(rs),
                           _device_ptrs(border_cells), st, bp, bn, br, status_ptr or None, cells_ptr or None)


def backbone_asbr_delta_device(ctx: capi.Context, t: BackboneTable, n_jobs: int, rs, border_cells, border_status,
                               border_planes, border_n_rows, border_rows, base_ptr: int, n_base: int, base_of_ptr: int,
                               job_out_ptr: int, records_ptr: int, cap: int, n_records_ptr: int):
    """hspf_ospfv2_backbone_asbr_delta / _delta16: the route-delta stage over the same walk (arguments as
    backbone_asbr_cells_device and rib_delta_device)."""
    keep = []
    st = _device_ptrs(border_status) if border_status is not None else None
    bp, bn, br = _border_plane_args(border_planes, border_n_rows, border_rows, keep)
    route_table.call_stage(ctx, "hspf_ospfv2_backbone_asbr_delta", rs, t.handle, n_jobs, C.byref(rs),
                           _device_ptrs(border_cells), st, bp, bn, br, base_ptr or None, n_base, base_of_ptr or None,
                           job_out_ptr or None, records_ptr or None, cap, n_records_ptr or None)


def backbone_from_cells(area: ospfv2.Ospfv2Area, t: BackboneTable, cells: np.ndarray, gather_v, gather_nh) -> Rib:
    """hspf_ospfv2_backbone_from_cells (host): one job's cells -> R's routes for the affected prefixes.  area: R's
    image of the table's area (area 0, or the target area of a non-backbone table); gathers of R's row 0.  rc HSPF_E_UNSUPPORTED is returned in the result, as rib_from_cells."""
    cells = np.ascontiguousarray(cells, RIB_CELL_DT)
    assert cells.shape == (t.n_prefixes,)
    gv = np.ascontiguousarray(gather_v, np.uint32)
    gn = np.ascontiguousarray(gather_nh, np.uint64)
    s = area.as_struct()
    return _call_rib(capi.load_library().hspf_ospfv2_backbone_from_cells,
                     (t.handle, C.byref(s), cells.ctypes.data, gv.ctypes.data, gn.ctypes.data, len(gv)),
                     t.n_prefixes, RIB_ROUTE_DT, ospfv2.NEXTHOP_DT)


def backbone_from_cells_v3(area, t: BackboneTable, cells: np.ndarray, gather_v, gather_nh) -> Rib:
    """hspf_ospfv3_backbone_from_cells (host): one job's cells over an OSPFv3 BackboneTable -> R's routes for the
    affected prefixes, prefix options included (RIB_ROUTE6_DT routes, ospfv3.NEXTHOP6_DT next hops).  area: R's
    ospfv3.Ospfv3Area image of the table's area (area 0, or the target area of a non-backbone table); gathers of R's
    row 0.  rc HSPF_E_UNSUPPORTED is returned in the result."""
    from . import ospfv3
    cells = np.ascontiguousarray(cells, RIB_CELL_DT)
    assert cells.shape == (t.n_prefixes,)
    gv = np.ascontiguousarray(gather_v, np.uint32)
    gn = np.ascontiguousarray(gather_nh, np.uint64)
    s = area.as_struct()
    return _call_rib(capi.load_library().hspf_ospfv3_backbone_from_cells,
                     (t.handle, C.byref(s), cells.ctypes.data, gv.ctypes.data, gn.ctypes.data, len(gv)),
                     t.n_prefixes, RIB_ROUTE6_DT, ospfv3.NEXTHOP6_DT)


# ---- area border router over what-if jobs inside another area (include/holo_spf_lsdb.h) --------------------------
class AbrBackboneTable:
    """hspf_ospfv2_abr_backbone_table of an area border router R of area 0 and other areas: its affected prefixes over
    what-if jobs inside an area it is not attached to.  `router_id`, `flats`, `area_ids`, `summaries`, `active`,
    `externals` as for AbrRibTable (area 0's summaries as in R's LSDB); `borders`: the AbrRibTables of the perturbed
    area's ABRs attached to area 0 (kept alive with this table).  `prefix`, `plen` [n_prefixes]: the affected prefixes
    in prefix order; a slot's winner is n_records + its slot index (n_slots in all); `n_asbr_slots` type-4 slots read
    `n_asbr_sets` (border, area) plane sets.

    From ospfv3.Flat areas the table is hspf_ospfv3_abr_backbone_table_create's (summaries: INTER_AREA_LSA_DT,
    externals: EXTERNAL6_LSA_DT, borders: OSPFv3 AbrRibTables); `prefix` and `prefixes6` then hold the IPv6 prefixes
    (ospfv3.IP_DT), `v3` is set, and a slot's winner is n_records + (slot index << 8 | its prefix options)."""

    def __init__(self, router_id: int, flats: list, area_ids, summaries=None, active=None, externals=None, borders=()):
        from . import ospfv3
        n = len(flats)
        self.lib = capi.load_library()
        self.handle = None
        self.router_id, self.flats, self.area_ids = router_id, list(flats), [int(a) for a in area_ids]
        self.borders = list(borders)
        self.v3 = bool(flats) and isinstance(flats[0], ospfv3.Flat)
        sum_dt, ext_dt = (INTER_AREA_LSA_DT, EXTERNAL6_LSA_DT) if self.v3 else (SUMMARY_LSA_DT, EXTERNAL_LSA_DT)
        sums = [np.ascontiguousarray(s if s is not None else np.zeros(0, sum_dt), sum_dt)
                for s in (summaries if summaries is not None else [None] * n)]
        ext = np.ascontiguousarray(externals if externals is not None else np.zeros(0, ext_dt), ext_dt)
        self.summaries, self.externals = sums, ext
        self.active = [True] * n if active is None else [bool(a) for a in active]
        self.n_areas = n
        fl = (C.c_void_p * max(n, 1))(*[f.handle.value for f in flats])
        ids = np.asarray(self.area_ids or [0], np.uint32)
        sp = (C.c_void_p * max(n, 1))(*[s.ctypes.data if len(s) else None for s in sums])
        ns = np.asarray([len(s) for s in sums] or [0], np.uint32)
        act = np.asarray([int(a) for a in self.active] or [0], np.uint8)
        bt = (C.c_void_p * max(len(self.borders), 1))(*[b.handle.value for b in self.borders])
        self._keep = (fl, ids, sp, ns, act, sums, ext, flats)
        h = C.c_void_p()
        create = "hspf_ospfv3_abr_backbone_table_create" if self.v3 else "hspf_ospfv2_abr_backbone_table_create"
        rc = getattr(self.lib, create)(router_id, n, fl, ids.ctypes.data, sp, ns.ctypes.data, act.ctypes.data,
                                       ext.ctypes.data if len(ext) else None, len(ext), bt, len(self.borders),
                                       C.byref(h))
        if rc != capi.HSPF_OK:
            raise capi.HspfError(rc, create + " failed")
        self.handle = h
        np_, pp, pl = C.c_uint32(), C.c_void_p(), C.c_void_p()
        assert self.lib.hspf_ospfv2_abr_backbone_table_prefixes(h, C.byref(np_), C.byref(pp), C.byref(pl)) == capi.HSPF_OK
        self.n_prefixes = np_.value
        self.prefix = route_table.copy_records(pp, self.n_prefixes, np.uint32)
        self.plen = route_table.copy_records(pl, self.n_prefixes, np.uint32)
        c = [C.c_uint32() for _ in range(4)]
        assert self.lib.hspf_ospfv2_abr_backbone_table_records(h, *[C.byref(x) for x in c]) == capi.HSPF_OK
        self.n_records, self.n_slots, self.n_asbr_slots, self.n_asbr_sets = [x.value for x in c]
        ng, ids = C.c_uint32(), C.POINTER(C.c_uint32)()
        assert self.lib.hspf_ospfv2_abr_backbone_table_asbrs(h, C.byref(ng), C.byref(ids)) == capi.HSPF_OK
        # the ASBRs whose area-0 entry moves with the job (abr_backbone_asbr_entries_device's columns)
        self.asbr_ids = np.ctypeslib.as_array(ids, (ng.value,)).copy() if ng.value else np.zeros(0, np.uint32)
        if self.v3:
            p6 = C.c_void_p()
            rc = self.lib.hspf_ospfv3_abr_backbone_table_prefixes6(h, None, C.byref(p6), None)
            if rc != capi.HSPF_OK:
                raise capi.HspfError(rc, "hspf_ospfv3_abr_backbone_table_prefixes6 failed")
            self.prefixes6 = route_table.copy_records(p6, self.n_prefixes, ospfv3.IP_DT)
            self.prefix = self.prefixes6

    def upload(self, ctx: capi.Context):
        rc = self.lib.hspf_ospfv2_abr_backbone_table_upload(ctx.handle, self.handle)
        if rc != capi.HSPF_OK:
            raise capi.HspfError(rc, ctx.last_error())

    def __del__(self):
        try:
            if self.handle:
                self.lib.hspf_ospfv2_abr_backbone_table_free(self.handle)
                self.handle = None
        except Exception:
            pass


def abr_backbone_cells_device(ctx: capi.Context, t: AbrBackboneTable, n_jobs: int, planes: list, border_cells,
                              border_status, border_planes, border_n_rows, border_rows, status_ptr: int,
                              cells_ptr: int):
    """hspf_ospfv2_abr_backbone_cells / _cells16 over DEVICE planes.  planes: R's capi.ResultStruct (nh_words 1) or
    capi.Result16Struct per area, in the table's order, only row 0 read; border_cells / border_status as
    backbone_cells_device; border_planes / border_n_rows / border_rows as backbone_asbr_cells_device (None for a table
    without type-4 slots); status_ptr: device u32 [n_jobs] or 0; cells_ptr: device [n_jobs, t.n_prefixes]
    RIB_CELL_DT.  Enqueued on the ctx stream; the table must have been uploaded."""
    keep = []
    st = _device_ptrs(border_status) if border_status is not None else None
    bp, bn, br = _border_plane_args(border_planes, border_n_rows, border_rows, keep)
    route_table.call_stage(ctx, "hspf_ospfv2_abr_backbone_cells", planes[0], t.handle, n_jobs, _planes_array(planes),
                           _device_ptrs(border_cells), st, bp, bn, br, status_ptr or None, cells_ptr or None)


def abr_backbone_delta_device(ctx: capi.Context, t: AbrBackboneTable, n_jobs: int, planes: list, border_cells,
                              border_status, border_planes, border_n_rows, border_rows, base_ptr: int, n_base: int,
                              base_of_ptr: int, job_out_ptr: int, records_ptr: int, cap: int, n_records_ptr: int):
    """hspf_ospfv2_abr_backbone_delta / _delta16: the route-delta stage over the same walk (arguments as
    abr_backbone_cells_device and rib_delta_device)."""
    keep = []
    st = _device_ptrs(border_status) if border_status is not None else None
    bp, bn, br = _border_plane_args(border_planes, border_n_rows, border_rows, keep)
    route_table.call_stage(ctx, "hspf_ospfv2_abr_backbone_delta", planes[0], t.handle, n_jobs, _planes_array(planes),
                           _device_ptrs(border_cells), st, bp, bn, br, base_ptr or None, n_base, base_of_ptr or None,
                           job_out_ptr or None, records_ptr or None, cap, n_records_ptr or None)


def abr_backbone_asbr_entries_device(ctx: capi.Context, t: AbrBackboneTable, n_jobs: int, planes: list, border_planes,
                                     border_n_rows, border_rows, status_ptr: int, entries_ptr: int):
    """hspf_ospfv2_abr_backbone_asbr_entries / _entries16 (an OSPFv3 table: hspf_ospfv3_abr_backbone_asbr_entries /
    _entries16): per job and per ASBR of t.asbr_ids, the metric of the type-4 / Inter-Area-Router LSA the router
    originates for it into a normal area other than area 0 (0xFFFFFFFF: none), into device u32 [n_jobs,
    len(t.asbr_ids)] at entries_ptr.  planes / border_* as abr_backbone_cells_device."""
    keep = []
    bp, bn, br = _border_plane_args(border_planes, border_n_rows, border_rows, keep)
    name = "hspf_ospfv3_abr_backbone_asbr_entries" if t.v3 else "hspf_ospfv2_abr_backbone_asbr_entries"
    route_table.call_stage(ctx, name, planes[0], t.handle, n_jobs,
                           _planes_array(planes), bp, bn, br, status_ptr or None, entries_ptr or None)


def third_area_cells_device(ctx: capi.Context, t: BackboneTable, n_jobs: int, rs, border_cells, border_status,
                            border_entries, border_entry_status, status_ptr: int, cells_ptr: int):
    """hspf_ospfv2_third_area_cells / _cells16: backbone_cells_device's arguments over a third-area table (either
    version; the table's mark picks the walk), plus per
    border a device pointer to its [n_jobs, G_b] entries (0 allowed without chain slots; None: NULL) and per border
    the entries call's device u32 [n_jobs] status words or 0 (None: none)."""
    be = _device_ptrs(border_entries) if border_entries is not None else None
    es = _device_ptrs(border_entry_status) if border_entry_status is not None else None
    st = _device_ptrs(border_status) if border_status is not None else None
    route_table.call_stage(ctx, "hspf_ospfv2_third_area_cells", rs, t.handle, n_jobs, C.byref(rs),
                           _device_ptrs(border_cells), st, be, es, status_ptr or None, cells_ptr or None)


def third_area_delta_device(ctx: capi.Context, t: BackboneTable, n_jobs: int, rs, border_cells, border_status,
                            border_entries, border_entry_status, base_ptr: int, n_base: int, base_of_ptr: int,
                            job_out_ptr: int, records_ptr: int, cap: int, n_records_ptr: int):
    """hspf_ospfv2_third_area_delta / _delta16: the route-delta stage over the same walk (arguments as
    third_area_cells_device and rib_delta_device)."""
    be = _device_ptrs(border_entries) if border_entries is not None else None
    es = _device_ptrs(border_entry_status) if border_entry_status is not None else None
    st = _device_ptrs(border_status) if border_status is not None else None
    route_table.call_stage(ctx, "hspf_ospfv2_third_area_delta", rs, t.handle, n_jobs, C.byref(rs),
                           _device_ptrs(border_cells), st, be, es, base_ptr or None, n_base, base_of_ptr or None,
                           job_out_ptr or None, records_ptr or None, cap, n_records_ptr or None)


def abr_backbone_from_cells(areas: list, t: AbrBackboneTable, cells: np.ndarray, gather_area, gather_v,
                            gather_nh) -> Rib:
    """hspf_ospfv2_abr_backbone_from_cells (host): one job's cells -> R's routes for the affected prefixes.  areas:
    R's ospfv2.Ospfv2Area images in the table's order; gathers (area, vertex, nh_mask) of R's row 0.  rc
    HSPF_E_UNSUPPORTED is returned in the result, as rib_from_cells."""
    return _call_abr_rib_from_cells(capi.load_library().hspf_ospfv2_abr_backbone_from_cells, ospfv2.AreaStruct, areas,
                                    t, cells, gather_area, gather_v, gather_nh, RIB_ROUTE_DT, ospfv2.NEXTHOP_DT)


def abr_backbone_from_cells_v3(areas: list, t: AbrBackboneTable, cells: np.ndarray, gather_area, gather_v,
                               gather_nh) -> Rib:
    """hspf_ospfv3_abr_backbone_from_cells (host): one job's cells over an OSPFv3 AbrBackboneTable -> R's routes for
    the affected prefixes, prefix options included (RIB_ROUTE6_DT routes, ospfv3.NEXTHOP6_DT next hops).  areas: R's
    ospfv3.Ospfv3Area images in the table's order; gathers (area, vertex, nh_mask) of R's row 0.  rc
    HSPF_E_UNSUPPORTED is returned in the result, as rib_from_cells."""
    from . import ospfv3
    return _call_abr_rib_from_cells(capi.load_library().hspf_ospfv3_abr_backbone_from_cells, ospfv3.AreaStruct, areas,
                                    t, cells, gather_area, gather_v, gather_nh, RIB_ROUTE6_DT, ospfv3.NEXTHOP6_DT)
