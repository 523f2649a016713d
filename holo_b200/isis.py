"""IS-IS side of the engine from Python: level LSDB images (include/holo_lsdb.h), the
compute_spt call (holo-isis/src/spf.rs:525-707 replaced by hspf_isis_compute_spt), the
flattener for batched roots / perturbations, and a synthetic LSDB builder."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import capi, route_table
from .synth import Topology

REACH_LEGACY, REACH_EXT, REACH_MT = 0, 1, 2
LSPF_OL, LSPF_HAS_PROTOCOLS, LSPF_NLPID_IPV4, LSPF_NLPID_IPV6, LSPF_MT_IPV6_OL = 0x01, 0x02, 0x04, 0x08, 0x10
METRIC_STANDARD, METRIC_WIDE, METRIC_BOTH = 0, 1, 2
MT_NONE, MT_STANDARD, MT_IPV6 = 0xFF, 0, 2
MODE_NORMAL, MODE_HOPCOUNT = 0, 1

REACH_DT = np.dtype([("neighbor", "<u8"), ("metric", "<u4"), ("mt_id", "<u2"), ("kind", "u1"), ("_pad", "u1")], align=True)
LSP_DT = np.dtype([("lan_id", "<u8"), ("seqno", "<u4"), ("rem_lifetime", "<u2"), ("fragment", "u1"), ("flags", "u1"),
                   ("reach_off", "<u4"), ("n_reach", "<u4"), ("ipreach_off", "<u4"), ("n_ipreach", "<u4"),
                   ("srgb_off", "<u4"), ("n_srgb", "<u2"), ("sr_flags", "u1"), ("flood_algo", "u1")], align=True)
FLOOD_ZERO_PRUNER, FLOOD_MODIFIED_MANET = 1, 2
RNL_DT = np.dtype([("system_id", "<u8"), ("algo", "u1"), ("_pad", "u1", (7,))], align=True)
LSP_SR_HAS_CAP, LSP_SR_ALGO_SPF, LSP_SR_CAP_V, LSP_SR_CAP_I = 0x01, 0x02, 0x40, 0x80
PSID_R, PSID_N, PSID_P, PSID_E, PSID_V, PSID_L = 0x80, 0x40, 0x20, 0x10, 0x08, 0x04
SRGB_DT = np.dtype([("first", "<u4"), ("range", "<u4"), ("first_is_index", "u1"), ("_pad", "u1", (3,))], align=True)


def lsp_rec(lan_id, seqno, rem_lifetime, fragment, flags, reach_off, n_reach, ipreach_off=0, n_ipreach=0,
            srgb_off=0, n_srgb=0, sr_flags=0):
    """One LSP_DT record as a tuple."""
    return (lan_id, seqno, rem_lifetime, fragment, flags, reach_off, n_reach, ipreach_off, n_ipreach, srgb_off, n_srgb,
            sr_flags, 0)


def ipreach_rec(prefix, metric, mt_id, plen, kind, external=0, psid=None):
    """One IPREACH_DT record; psid = (flags, is_label, value) of a Prefix-SID sub-TLV for algorithm SPF."""
    has, fl, isl, val = (1, psid[0], int(psid[1]), psid[2]) if psid is not None else (0, 0, 0, 0)
    return (prefix, metric, mt_id, plen, kind, external, has, fl, isl, val)
IP_DT = np.dtype([("bytes", "u1", (16,)), ("is_v6", "u1"), ("_pad", "u1", (3,))], align=True)
IPREACH_DT = np.dtype([("prefix", IP_DT), ("metric", "<u4"), ("mt_id", "<u2"), ("len", "u1"), ("kind", "u1"),
                       ("external", "u1"), ("has_psid", "u1"), ("psid_flags", "u1"), ("psid_is_label", "u1"),
                       ("psid_value", "<u4")], align=True)
ADJ_DT = np.dtype([("system_id", "<u8"), ("snpa", "u1", (6,)), ("up", "u1"), ("level_usage", "u1"), ("topo_std", "u1"),
                   ("topo_ipv6", "u1"), ("has_ipv4", "u1"), ("has_ipv6", "u1"), ("area_disjoint", "u1"),
                   ("_pad", "u1", (3,)), ("ipv4", "<u4"), ("ipv6", IP_DT)], align=True)
IFACE_DT = np.dtype([("ifindex", "<u4"), ("metric", "<u4"), ("is_broadcast", "u1"), ("_pad", "u1", (3,)),
                     ("adj_off", "<u4"), ("n_adj", "<u4")], align=True)
NEXTHOP_DT = np.dtype([("system_id", "<u8"), ("iface", "<u4"), ("sr_label", "<u4"), ("addr", IP_DT), ("has_label", "<u4")],
                      align=True)
ROUTE_DT = np.dtype([("prefix", IP_DT), ("metric", "<u4"), ("len", "u1"), ("route_type", "u1"), ("flags", "u1"),
                     ("has_sr_label", "u1"), ("nh_off", "<u4"), ("n_nh", "<u4"), ("sr_label", "<u4")], align=True)
IP_V4_INTERNAL, IP_V4_EXTERNAL, IP_V4_EXT, IP_V6, IP_MT_V6 = range(5)
LSPF_ATT, LSPF_MT_IPV6_ATT = 0x20, 0x40
VERTEX_DT = np.dtype([("lan_id", "<u8"), ("distance", "<u4"), ("hops", "<u2"), ("_pad", "<u2"), ("par_off", "<u4"),
                      ("n_par", "<u4"), ("nh_off", "<u4"), ("n_nh", "<u4")], align=True)


class LevelStruct(C.Structure):
    _fields_ = [("metric_type", C.c_uint8), ("mt_id", C.c_uint8), ("metric_mode", C.c_uint8),
                ("ipv4_enabled", C.c_uint8), ("ipv6_enabled", C.c_uint8), ("_pad", C.c_uint8 * 3),
                ("n_lsps", C.c_uint32), ("lsps", C.c_void_p), ("n_reaches", C.c_uint32), ("reaches", C.c_void_p),
                ("n_ipreaches", C.c_uint32), ("ipreaches", C.c_void_p), ("n_srgbs", C.c_uint32), ("srgbs", C.c_void_p)]


class InstanceStruct(C.Structure):
    _fields_ = [("lvl", LevelStruct), ("system_id", C.c_uint64), ("max_paths", C.c_uint16), ("level", C.c_uint8),
                ("level_type", C.c_uint8), ("att_ignore", C.c_uint8), ("mt_ipv6_enabled", C.c_uint8),
                ("sr_enabled", C.c_uint8), ("_pad", C.c_uint8), ("n_ifaces", C.c_uint32), ("ifaces", C.c_void_p),
                ("n_adjs", C.c_uint32), ("adjs", C.c_void_p)]


class RibStruct(C.Structure):
    _fields_ = [("routes_cap", C.c_uint32), ("n_routes", C.c_uint32), ("routes", C.c_void_p),
                ("nexthops_cap", C.c_uint32), ("n_nexthops", C.c_uint32), ("nexthops", C.c_void_p)]


class SptStruct(C.Structure):
    _fields_ = [("vertices_cap", C.c_uint32), ("n_vertices", C.c_uint32), ("vertices", C.c_void_p),
                ("parents_cap", C.c_uint32), ("n_parents", C.c_uint32), ("parents", C.c_void_p),
                ("nexthops_cap", C.c_uint32), ("n_nexthops", C.c_uint32), ("nexthops", C.c_void_p),
                ("first_hops_cap", C.c_uint32), ("n_first_hops", C.c_uint32), ("first_hops", C.c_void_p),
                ("second_hops_cap", C.c_uint32), ("n_second_hops", C.c_uint32), ("second_hops", C.c_void_p)]


ABI_SIZES = [REACH_DT.itemsize, LSP_DT.itemsize, C.sizeof(LevelStruct), VERTEX_DT.itemsize, C.sizeof(SptStruct),
             IPREACH_DT.itemsize, ADJ_DT.itemsize, IFACE_DT.itemsize, C.sizeof(InstanceStruct), NEXTHOP_DT.itemsize,
             ROUTE_DT.itemsize, C.sizeof(RibStruct)]


@dataclass
class IsisLevel:
    metric_type: int = METRIC_WIDE
    mt_id: int = MT_STANDARD
    metric_mode: int = MODE_NORMAL
    ipv4_enabled: bool = True
    ipv6_enabled: bool = False
    lsps: np.ndarray = field(default_factory=lambda: np.zeros(0, LSP_DT))
    reaches: np.ndarray = field(default_factory=lambda: np.zeros(0, REACH_DT))
    ipreaches: np.ndarray = field(default_factory=lambda: np.zeros(0, IPREACH_DT))
    srgbs: np.ndarray = field(default_factory=lambda: np.zeros(0, SRGB_DT))

    def as_struct(self) -> LevelStruct:
        s = LevelStruct()
        s.metric_type, s.mt_id, s.metric_mode = self.metric_type, self.mt_id, self.metric_mode
        s.ipv4_enabled, s.ipv6_enabled = int(self.ipv4_enabled), int(self.ipv6_enabled)
        self.lsps = np.ascontiguousarray(self.lsps, dtype=LSP_DT)
        self.reaches = np.ascontiguousarray(self.reaches, dtype=REACH_DT)
        s.n_lsps, s.lsps = len(self.lsps), (self.lsps.ctypes.data if len(self.lsps) else None)
        s.n_reaches, s.reaches = len(self.reaches), (self.reaches.ctypes.data if len(self.reaches) else None)
        self.ipreaches = np.ascontiguousarray(self.ipreaches, dtype=IPREACH_DT)
        s.n_ipreaches = len(self.ipreaches)
        s.ipreaches = self.ipreaches.ctypes.data if len(self.ipreaches) else None
        self.srgbs = np.ascontiguousarray(self.srgbs, dtype=SRGB_DT)
        s.n_srgbs, s.srgbs = len(self.srgbs), (self.srgbs.ctypes.data if len(self.srgbs) else None)
        return s


@dataclass
class IsisSpt:
    vertices: np.ndarray
    parents: np.ndarray
    nexthops: np.ndarray
    first_hops: np.ndarray
    second_hops: np.ndarray
    rc: int = 0


def _call_spt(fn, n_vertices_hint: int, n_edges_hint: int, prefix_args):
    caps = [n_vertices_hint + 1, 2 * n_edges_hint + 16, 1 << 16]
    for _ in range(3):
        verts = np.zeros(caps[0], VERTEX_DT)
        par = np.zeros(caps[1], np.uint32)
        nh = np.zeros(caps[2], np.uint64)
        fh = np.zeros(caps[0], np.uint32)
        sh = np.zeros(caps[0], np.uint32)
        r = SptStruct()
        r.vertices_cap, r.vertices = caps[0], verts.ctypes.data
        r.parents_cap, r.parents = caps[1], par.ctypes.data
        r.nexthops_cap, r.nexthops = caps[2], nh.ctypes.data
        r.first_hops_cap, r.first_hops = caps[0], fh.ctypes.data
        r.second_hops_cap, r.second_hops = caps[0], sh.ctypes.data
        rc = fn(*prefix_args, C.byref(r))
        if rc == capi.HSPF_E_NOMEM:
            caps = [max(caps[0], r.n_vertices), max(caps[1], r.n_parents), max(caps[2], r.n_nexthops)]
            continue
        break
    return IsisSpt(verts[: r.n_vertices].copy(), par[: r.n_parents].copy(), nh[: r.n_nexthops].copy(),
                   fh[: r.n_first_hops].copy(), sh[: r.n_second_hops].copy(), rc)


def _bind(lib):
    lib.hspf_isis_flatten.argtypes = [C.POINTER(LevelStruct), C.POINTER(C.c_void_p)]
    lib.hspf_isis_flat_free.argtypes = [C.c_void_p]
    lib.hspf_isis_flat_free.restype = None
    lib.hspf_isis_flat_csr.argtypes = [C.c_void_p, C.POINTER(capi.CsrStruct)]
    lib.hspf_isis_flat_vertices.argtypes = [C.c_void_p, C.POINTER(C.POINTER(C.c_uint64)), C.POINTER(C.c_uint32)]
    lib.hspf_isis_flat_vertex.argtypes = [C.c_void_p, C.c_uint64]
    lib.hspf_isis_flat_vertex.restype = C.c_uint32
    lib.hspf_isis_spt_from_planes.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                              C.c_void_p, C.c_void_p, C.POINTER(SptStruct)]
    lib.hspf_isis_compute_spt.argtypes = [C.c_void_p, C.POINTER(LevelStruct), C.c_uint64, C.POINTER(SptStruct)]
    return lib


def compute_spt(ctx: capi.Context, level: IsisLevel, root_system_id: int) -> IsisSpt:
    lib = _bind(ctx.lib)
    s = level.as_struct()
    res = _call_spt(lib.hspf_isis_compute_spt, len(level.lsps), len(level.reaches),
                    (ctx.handle, C.byref(s), C.c_uint64(root_system_id)))
    if res.rc != capi.HSPF_OK:
        raise capi.HspfError(res.rc, ctx.last_error())
    return res


class Flat:
    def __init__(self, level: IsisLevel):
        self.lib = _bind(capi.load_library())
        self.level = level
        self._s = level.as_struct()
        h = C.c_void_p()
        rc = self.lib.hspf_isis_flatten(C.byref(self._s), C.byref(h))
        if rc != capi.HSPF_OK:
            raise capi.HspfError(rc, "hspf_isis_flatten failed")
        self.handle = h
        self._load()

    def _load(self):
        h = self.handle
        cs = capi.CsrStruct()
        self.lib.hspf_isis_flat_csr(h, C.byref(cs))
        V, E = cs.n_vertices, cs.n_edges
        as_np = lambda p, n, dt: np.ctypeslib.as_array(p, shape=(n,)).astype(dt).copy() if n else np.zeros(0, dt)
        self.csr = capi.Csr(as_np(cs.row_ptr, V + 1, np.uint32), as_np(cs.col, E, np.uint32),
                            as_np(cs.cost, E, np.uint32), as_np(cs.vflags, V, np.uint8),
                            reject_above=cs.reject_above, saturate_at=cs.saturate_at, flags=cs.flags, delta=cs.delta)
        ids, n = C.POINTER(C.c_uint64)(), C.c_uint32()
        self.lib.hspf_isis_flat_vertices(h, C.byref(ids), C.byref(n))
        self.ids = as_np(ids, n.value, np.uint64)

    def vertex(self, lan_id: int) -> int:
        return int(self.lib.hspf_isis_flat_vertex(self.handle, C.c_uint64(lan_id)))

    def spt_from_planes(self, root_vertex: int, dist: np.ndarray, hops: np.ndarray, overrides=()) -> IsisSpt:
        dist = np.ascontiguousarray(dist, np.uint32)
        hops = np.ascontiguousarray(hops, np.uint16)
        ove = np.asarray([e for e, _ in overrides] or [0], np.uint32)
        ovc = np.asarray([c for _, c in overrides] or [0], np.uint32)
        res = _call_spt(self.lib.hspf_isis_spt_from_planes, self.csr.n_vertices, self.csr.n_edges,
                        (self.handle, C.c_uint32(root_vertex), dist.ctypes.data, hops.ctypes.data,
                         C.c_uint32(len(overrides)), ove.ctypes.data, ovc.ctypes.data))
        if res.rc != capi.HSPF_OK:
            raise capi.HspfError(res.rc, "hspf_isis_spt_from_planes failed")
        return res

    def __del__(self):
        try:
            if self.handle:
                self.lib.hspf_isis_flat_free(self.handle)
                self.handle = None
        except Exception:
            pass


LSP_TRIGGER_DT = np.dtype([("lan_id", "<u8"), ("fragment", "u1"), ("_pad", "u1", (7,))], align=True)
SPF_FULL, SPF_ROUTE_ONLY = 1, 2
FLAT_UNCHANGED, FLAT_COSTS, FLAT_REBUILT = 0, 1, 2


def spf_type(old_level: IsisLevel, new_level: IsisLevel, triggers, lib=None, name="hspf_isis_spf_type") -> int:
    """hspf_isis_spf_type: SPF_FULL or SPF_ROUTE_ONLY for the LSPs [(lan_id, fragment)] that were just installed."""
    fn = getattr(lib or capi.load_library(), name)
    fn.argtypes = [C.POINTER(LevelStruct), C.POINTER(LevelStruct), C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    tr = np.zeros(len(triggers), LSP_TRIGGER_DT)
    for i, (lan_id, frag) in enumerate(triggers):
        tr[i]["lan_id"], tr[i]["fragment"] = lan_id, frag
    so, sn = old_level.as_struct(), new_level.as_struct()
    out = C.c_uint32()
    rc = fn(C.byref(so), C.byref(sn), tr.ctypes.data if len(tr) else None, len(tr), C.byref(out))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, name + " failed")
    return out.value


def flat_update(flat: "Flat", new_level: IsisLevel):
    """hspf_isis_flat_update -> (kind, edges, costs); the Flat's numpy views are refreshed."""
    lib = flat.lib
    lib.hspf_isis_flat_update.argtypes = [C.c_void_p, C.POINTER(LevelStruct), C.POINTER(C.c_uint32), C.c_void_p, C.c_void_p,
                                          C.c_uint32, C.POINTER(C.c_uint32)]
    cap = max(int(flat.csr.n_edges), 1)
    edges, costs = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
    kind, n = C.c_uint32(), C.c_uint32()
    s = new_level.as_struct()
    rc = lib.hspf_isis_flat_update(flat.handle, C.byref(s), C.byref(kind), edges.ctypes.data, costs.ctypes.data, cap, C.byref(n))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, "hspf_isis_flat_update failed")
    flat.level, flat._s = new_level, s
    flat._load()
    return kind.value, edges[: n.value].copy(), costs[: n.value].copy()


# ------------------------------------------------------------------------------ synthetic
SYSID_BASE = 0x000000000001


def sysid(i: int) -> int:
    return SYSID_BASE + int(i)


def synth_level(t: Topology, metric_type: int = METRIC_WIDE, mt_id: int = MT_STANDARD, metric_mode: int = MODE_NORMAL,
                max_reach_per_fragment: int = 0, overload=(), no_protocols=()) -> IsisLevel:
    """IS-IS level LSDB for topology `t`: router i has system id 1+i and one LSP (split
    into fragments of `max_reach_per_fragment` entries when > 0); LAN k is a pseudonode
    of its first member.  Wide metrics use TLV 22, standard TLV 2 (metric clipped to
    63), METRIC_BOTH advertises both (parallel edges, spf.rs:1005-1120)."""
    R = t.n_routers
    per = [[] for _ in range(R)]
    for k in range(t.n_p2p):
        a, b = int(t.p2p_a[k]), int(t.p2p_b[k])
        per[a].append((sysid(b) << 8, int(t.p2p_cost_ab[k])))
        per[b].append((sysid(a) << 8, int(t.p2p_cost_ba[k])))
    pn_lsps = []
    n_pn = [0] * R
    for members, costs in t.lans:
        dr = members[0]
        n_pn[dr] += 1
        assert n_pn[dr] < 256
        pn_id = (sysid(dr) << 8) | n_pn[dr]
        for m, c in zip(members, costs):
            per[m].append((pn_id, int(c)))
        pn_lsps.append((pn_id, [(sysid(m) << 8, 0) for m in members]))
    lsps, reaches = [], []

    def add_reach(nbr, metric):
        out = []
        if metric_type in (METRIC_STANDARD, METRIC_BOTH):
            out.append((nbr, min(metric, 63), 0, REACH_LEGACY, 0))
        if metric_type in (METRIC_WIDE, METRIC_BOTH):
            out.append((nbr, metric, 0, REACH_EXT, 0))
        if mt_id == MT_IPV6:
            out.append((nbr, metric, MT_IPV6, REACH_MT, 0))
        return out

    def emit(lan_id, entries, flags):
        chunks = [entries]
        if max_reach_per_fragment > 0:
            chunks = [entries[i:i + max_reach_per_fragment] for i in range(0, len(entries), max_reach_per_fragment)] or [[]]
        for frag, ch in enumerate(chunks):
            rr = [x for (nbr, m) in ch for x in add_reach(nbr, m)]
            lsps.append(lsp_rec(lan_id, 1, 1200, frag, flags if frag == 0 else 0, len(reaches), len(rr)))
            reaches.extend(rr)

    for i in range(R):
        fl = LSPF_HAS_PROTOCOLS | LSPF_NLPID_IPV4
        if i in overload:
            fl |= LSPF_OL | LSPF_MT_IPV6_OL
        if i in no_protocols:
            fl &= ~(LSPF_HAS_PROTOCOLS | LSPF_NLPID_IPV4)
        emit(sysid(i) << 8, per[i], fl)
    for pn_id, ent in pn_lsps:
        emit(pn_id, ent, 0)
    lv = IsisLevel(metric_type=metric_type, mt_id=mt_id, metric_mode=metric_mode)
    la = np.zeros(len(lsps), LSP_DT)
    for i, x in enumerate(lsps):
        la[i] = x
    order = np.lexsort((la["fragment"], la["lan_id"]))
    lv.lsps = la[order]
    ra = np.zeros(len(reaches), REACH_DT)
    for i, x in enumerate(reaches):
        ra[i] = x
    lv.reaches = ra
    return lv


# ------------------------------------------------------------------------------ route stage
def instance_struct(inst: dict) -> InstanceStruct:
    """hl_isis_instance from the dict produced by the image builders (keeps arrays alive
    through the dict)."""
    s = InstanceStruct()
    s.lvl = inst["level"].as_struct()
    s.system_id, s.max_paths = inst["system_id"], inst["max_paths"]
    s.level, s.level_type = inst["level_no"], inst["level_type"]
    s.att_ignore, s.mt_ipv6_enabled = inst["att_ignore"], inst["mt_ipv6"]
    s.sr_enabled = int(inst.get("sr_enabled", 0))
    inst["ifaces"] = np.ascontiguousarray(inst["ifaces"], dtype=IFACE_DT)
    inst["adjs"] = np.ascontiguousarray(inst["adjs"], dtype=ADJ_DT)
    s.n_ifaces, s.ifaces = len(inst["ifaces"]), (inst["ifaces"].ctypes.data if len(inst["ifaces"]) else None)
    s.n_adjs, s.adjs = len(inst["adjs"]), (inst["adjs"].ctypes.data if len(inst["adjs"]) else None)
    return s


@dataclass
class IsisRib:
    routes: np.ndarray
    nexthops: np.ndarray
    rc: int = 0

    def nh(self, rec):
        from .ospfv3 import ip_str
        return [(int(x["iface"]), ip_str(x["addr"]), int(x["system_id"]))
                for x in self.nexthops[int(rec["nh_off"]): int(rec["nh_off"]) + int(rec["n_nh"])]]


def _call_rib(fn, inst: dict, prefix_args=(), tail_args=()):
    s = instance_struct(inst)
    caps = [len(inst["level"].ipreaches) + 8, 16 * (len(inst["level"].ipreaches) + 8)]
    for _ in range(2):
        routes = np.zeros(caps[0], ROUTE_DT)
        nhs = np.zeros(caps[1], NEXTHOP_DT)
        r = RibStruct()
        r.routes_cap, r.routes = caps[0], routes.ctypes.data
        r.nexthops_cap, r.nexthops = caps[1], nhs.ctypes.data
        rc = fn(*prefix_args, C.byref(s), *tail_args, C.byref(r))
        if rc == capi.HSPF_E_NOMEM:
            caps = [max(caps[0], r.n_routes), max(caps[1], r.n_nexthops)]
            continue
        break
    return IsisRib(routes[: r.n_routes].copy(), nhs[: r.n_nexthops].copy(), rc)


def compute_routes(ctx: capi.Context, inst: dict) -> IsisRib:
    """compute_spt(local = true) per enabled topology + compute_routes on the GPU engine."""
    lib = ctx.lib
    lib.hspf_isis_compute_routes.argtypes = [C.c_void_p, C.POINTER(InstanceStruct), C.POINTER(RibStruct)]
    res = _call_rib(lib.hspf_isis_compute_routes, inst, (ctx.handle,))
    if res.rc != capi.HSPF_OK:
        raise capi.HspfError(res.rc, ctx.last_error())
    return res


def routes_from_planes(inst: dict, spf) -> IsisRib:
    """hspf_isis_routes_from_planes: the route stage over SPT planes supplied by `spf(csr, root_vertex)
    -> (dist u32[V], hops u16[V])`, called once per enabled topology on that topology's flattened
    CSR (host only; the planes may come from hspf_run_batch or, in tests, from the oracle)."""
    import copy
    lib = capi.load_library()
    u32p, u16p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint16)
    lib.hspf_isis_routes_from_planes.argtypes = [C.POINTER(InstanceStruct), u32p, u16p, u32p, u16p, C.POINTER(RibStruct)]
    planes = {}
    for mt in (MT_STANDARD, MT_IPV6):
        if mt == MT_IPV6 and not inst.get("mt_ipv6"):
            continue
        lv = copy.copy(inst["level"])
        lv.mt_id, lv.metric_mode = mt, MODE_NORMAL
        f = Flat(lv)
        root = f.vertex(inst["system_id"] << 8)
        if root == 0xFFFFFFFF:
            continue
        d, h = spf(f.csr, root)
        planes[mt] = (np.ascontiguousarray(d, np.uint32), np.ascontiguousarray(h, np.uint16))
    ptr = lambda a, ty: a.ctypes.data_as(ty) if a is not None else C.cast(None, ty)
    ds, hs = planes.get(MT_STANDARD, (None, None))
    d6, h6 = planes.get(MT_IPV6, (None, None))
    res = _call_rib(lib.hspf_isis_routes_from_planes, inst, (), tail_args=(ptr(ds, u32p), ptr(hs, u16p), ptr(d6, u32p), ptr(h6, u16p)))
    if res.rc != capi.HSPF_OK:
        raise capi.HspfError(res.rc, "hspf_isis_routes_from_planes failed")
    return res


# ---- batched route stage (include/holo_spf_lsdb.h: hspf_isis_rtable_*, hspf_isis_routes_batch*) --------
CELL_DT = np.dtype([("nh_mask", "<u8"), ("winner", "<u4"), ("metric", "<u4"), ("flags", "u1"), ("_pad", "u1", (7,))])
CONTRIB_DT = np.dtype([("vertex", "<u4"), ("metric", "<u4"), ("topology", "u1"), ("external", "u1"), ("has_psid", "u1"),
                       ("sr", "u1"), ("_pad", "<u4")])
CELL_PRESENT, CELL_CONNECTED, CELL_MIXED_SID = 1, 2, 4
TOPO_STD, TOPO_MT6 = 0, 1
NO_ROOT = 0xFFFFFFFF


class RouteTable(route_table.RouteTable):
    """hspf_isis_rtable: the instance's prefixes in NetKey order and their contributors (host);
    `upload(ctx)` copies it to the device for hspf_isis_routes_batch.  `n_vertices[t]` / `root[t]` per
    topology (TOPO_STD, TOPO_MT6; root NO_ROOT: the topology has no routes)."""

    api, contrib_dt = "hspf_isis", CONTRIB_DT

    def __init__(self, inst: dict):
        s = instance_struct(inst)
        super().__init__(capi.load_library().hspf_isis_rtable_create, C.byref(s))
        self.n_vertices, self.root = [], []
        for t in (TOPO_STD, TOPO_MT6):
            nv, r = C.c_uint32(), C.c_uint32()
            self._call("topology", t, C.byref(nv), C.byref(r))
            self.n_vertices.append(nv.value)
            self.root.append(r.value)
        pp, pl = C.c_void_p(), C.POINTER(C.c_uint32)()
        self._call("arrays", C.byref(pp), C.byref(pl), None, None)
        self.prefix = route_table.copy_records(pp, self.n_prefixes, IP_DT)
        self.len = route_table.copy_records(pl, self.n_prefixes, np.uint32)


def routes_batch_device(ctx: capi.Context, rt: RouteTable, n_jobs: int, rs_std, rs_mt6, cells_ptr: int):
    """hspf_isis_routes_batch / _batch16 over DEVICE planes (rs_*: capi.ResultStruct or capi.Result16Struct holding
    device pointers, one per topology; rs_mt6 may be None unless the table has an MT-IPv6 root); cells_ptr: device
    buffer of n_jobs * rt.n_prefixes cells.  Enqueued on the ctx stream; the table must have been uploaded."""
    route_table.call_stage(ctx, "hspf_isis_routes_batch", rs_std if rs_std is not None else rs_mt6, rt.handle, n_jobs,
                           C.byref(rs_std) if rs_std is not None else None,
                           C.byref(rs_mt6) if rs_mt6 is not None else None, cells_ptr)


def routes_delta_device(ctx: capi.Context, rt: RouteTable, n_jobs: int, rs_std, rs_mt6, base_ptr: int, n_base: int,
                        base_of_ptr: int, job_out_ptr: int, records_ptr: int, cap: int, n_records_ptr: int):
    """hspf_isis_routes_delta / _delta16 over DEVICE planes (rs_* as for routes_batch_device): each job's cells compared
    with its base row of base_ptr ([n_base, rt.n_prefixes] cells; base_of_ptr: [n_jobs] u32 rows, 0 for row 0 of
    every job), without storing them.  job_out_ptr: [n_jobs] route_table.DELTA_JOB_DT; records_ptr: [cap]
    route_table.DELTA_DT in (job, prefix) order (0 or cap 0: summaries only); n_records_ptr: u64 total.  All device
    pointers; enqueued on the ctx stream."""
    route_table.call_stage(ctx, "hspf_isis_routes_delta", rs_std if rs_std is not None else rs_mt6, rt.handle, n_jobs,
                           C.byref(rs_std) if rs_std is not None else None,
                           C.byref(rs_mt6) if rs_mt6 is not None else None, base_ptr or None, n_base,
                           base_of_ptr or None, job_out_ptr or None, records_ptr or None, cap, n_records_ptr or None)


def routes_from_cells(inst: dict, rt: RouteTable, cells: np.ndarray, std=None, mt6=None, ov_std=(), ov_mt6=()) -> IsisRib:
    """hspf_isis_routes_from_cells (host): one job's cells -> the table hspf_isis_routes_from_planes gives for the
    same planes.  std / mt6: that job's (dist u32[V], hops u16[V]) per topology; ov_*: its [(edge, cost), ...]
    overrides.  rc HSPF_E_UNSUPPORTED is returned in the result (caller: routes_from_planes)."""
    lib = capi.load_library()
    u32p, u16p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint16)
    cells = np.ascontiguousarray(cells, CELL_DT)
    assert cells.shape == (rt.n_prefixes,)
    keep = [cells]

    def arr(a, dt, ty):
        if a is None:
            return C.cast(None, ty)
        a = np.ascontiguousarray(a, dt)
        keep.append(a)
        return a.ctypes.data_as(ty)

    def planes(p):
        return (arr(None, None, u32p), arr(None, None, u16p)) if p is None else (arr(p[0], np.uint32, u32p), arr(p[1], np.uint16, u16p))

    def ov(o):
        o = list(o)
        return (len(o), arr([e for e, _ in o] or [0], np.uint32, u32p), arr([c for _, c in o] or [0], np.uint32, u32p))

    tail = (rt.handle, cells.ctypes.data, *planes(std), *planes(mt6), *ov(ov_std), *ov(ov_mt6))
    res = _call_rib(lib.hspf_isis_routes_from_cells, inst, (), tail_args=tail)
    if res.rc not in (capi.HSPF_OK, capi.HSPF_E_UNSUPPORTED):
        raise capi.HspfError(res.rc, "hspf_isis_routes_from_cells failed")
    return res


# ---- flooding reduction over hop-count SPTs (holo-isis/src/flooding/manet.rs) ------------------
def _spt_struct(spt: IsisSpt, keep: list) -> SptStruct:
    r = SptStruct()
    for name, dt in (("vertices", VERTEX_DT), ("parents", np.uint32), ("nexthops", np.uint64),
                     ("first_hops", np.uint32), ("second_hops", np.uint32)):
        a = np.ascontiguousarray(getattr(spt, name), dtype=dt)
        keep.append(a)
        setattr(r, name + "_cap", len(a))
        setattr(r, "n_" + name, len(a))
        setattr(r, name, a.ctypes.data if len(a) else None)
    return r


def flood_reduction_hash(system_id: int, pseudonode: int, fragment: int, lib=None, name="hspf_isis_flood_reduction_hash") -> int:
    lib = lib or capi.load_library()
    fn = getattr(lib, name)
    fn.argtypes, fn.restype = [C.c_uint64, C.c_uint8, C.c_uint8], C.c_uint16
    return int(fn(system_id, pseudonode, fragment))


def remote_neighbors(level: IsisLevel, spt: IsisSpt, lib=None, name="hspf_isis_remote_neighbors") -> np.ndarray:
    """Remote Neighbor List of the neighbour whose hop-count SPT `spt` is (manet.rs:72-88)."""
    lib = lib or capi.load_library()
    fn = getattr(lib, name)
    fn.argtypes = [C.POINTER(LevelStruct), C.POINTER(SptStruct), C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    keep = []
    ls, ss = level.as_struct(), _spt_struct(spt, keep)
    out = np.zeros(max(len(spt.first_hops), 1), RNL_DT)
    n = C.c_uint32()
    rc = fn(C.byref(ls), C.byref(ss), out.ctypes.data, len(out), C.byref(n))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, name + " failed")
    return out[: n.value].copy()


def reflood_list(spt: IsisSpt, rnl: np.ndarray, local_system_id: int, lsp_system_id: int, lsp_pseudonode: int,
                 lsp_fragment: int, lib=None, name="hspf_isis_reflood_list") -> list:
    """reflood_list (manet.rs:99-173): the two-hop neighbours this router must reflood the LSP to."""
    lib = lib or capi.load_library()
    fn = getattr(lib, name)
    fn.argtypes = [C.POINTER(SptStruct), C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint8, C.c_uint8,
                   C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    keep = []
    ss = _spt_struct(spt, keep)
    rnl = np.ascontiguousarray(rnl, dtype=RNL_DT)
    out = np.zeros(max(len(spt.second_hops), 1), np.uint64)
    n = C.c_uint32()
    rc = fn(C.byref(ss), rnl.ctypes.data if len(rnl) else None, len(rnl), local_system_id, lsp_system_id, lsp_pseudonode,
            lsp_fragment, out.ctypes.data, len(out), C.byref(n))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, name + " failed")
    return [int(x) for x in out[: n.value]]


# ---- end of update_rib: level merge + update_global_rib (holo-isis/src/route.rs:232-314) --------
ROUTE_CONNECTED, ROUTE_INSTALLED = 0x01, 0x02
ACTION_DT = np.dtype([("route", "<u4"), ("old_sr_label", "<u4"), ("kind", "u1"), ("has_old_sr_label", "u1"),
                      ("_pad", "u1", (2,))], align=True)


def _rib_struct(rib, keep: list) -> RibStruct:
    r = RibStruct()
    routes = np.ascontiguousarray(rib.routes, dtype=ROUTE_DT)
    nhs = np.ascontiguousarray(rib.nexthops, dtype=NEXTHOP_DT)
    keep += [routes, nhs]
    r.routes_cap = r.n_routes = len(routes)
    r.nexthops_cap = r.n_nexthops = len(nhs)
    r.routes = routes.ctypes.data if len(routes) else None
    r.nexthops = nhs.ctypes.data if len(nhs) else None
    return r


def rib_merge(l2, l1, lib=None, name="hspf_isis_rib_merge") -> IsisRib:
    """Merged local table of an L1/L2 router: L1 routes preferred (route.rs:236-242)."""
    lib = lib or capi.load_library()
    fn = getattr(lib, name)
    fn.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(RibStruct)]
    keep = []
    s2 = _rib_struct(l2, keep) if l2 is not None else None
    s1 = _rib_struct(l1, keep) if l1 is not None else None
    n_r = sum(len(x.routes) for x in (l2, l1) if x is not None)
    n_h = sum(len(x.nexthops) for x in (l2, l1) if x is not None)
    routes, nhs = np.zeros(max(n_r, 1), ROUTE_DT), np.zeros(max(n_h, 1), NEXTHOP_DT)
    r = RibStruct()
    r.routes_cap, r.routes = len(routes), routes.ctypes.data
    r.nexthops_cap, r.nexthops = len(nhs), nhs.ctypes.data
    rc = fn(C.addressof(s2) if s2 is not None else None, C.addressof(s1) if s1 is not None else None, C.byref(r))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, name + " failed")
    return IsisRib(routes[: r.n_routes].copy(), nhs[: r.n_nexthops].copy(), rc)


def rib_diff(old, new: IsisRib, lib=None, name="hspf_isis_rib_diff"):
    """update_global_rib: (actions ACTION_DT[], new routes with ROUTE_INSTALLED set as the reference would)."""
    lib = lib or capi.load_library()
    fn = getattr(lib, name)
    fn.argtypes = [C.c_void_p, C.POINTER(RibStruct), C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    keep = []
    ns = _rib_struct(IsisRib(new.routes.copy(), new.nexthops), keep)
    new_routes = keep[0]
    os_ = _rib_struct(old, keep) if old is not None else None
    cap = len(new.routes) + (len(old.routes) if old is not None else 0) + 1
    acts = np.zeros(cap, ACTION_DT)
    n = C.c_uint32()
    rc = fn(C.addressof(os_) if os_ is not None else None, C.byref(ns), acts.ctypes.data, cap, C.byref(n))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, name + " failed")
    return acts[: n.value].copy(), new_routes


# ---- L1/L2 routers: summary routes and L1 -> L2 propagation (holo-isis route.rs:189-231, lsdb.rs:1149-1357)
SUMMARY_DT = np.dtype([("prefix", IP_DT), ("cfg_metric", "<u4"), ("metric", "<u4"), ("len", "u1"),
                       ("has_cfg_metric", "u1"), ("_pad", "u1", (2,))], align=True)
ROUTE_SUMMARY = 0x04


def summary_cfg(entries) -> np.ndarray:
    """[(prefix string, metric or None), ...] -> SUMMARY_DT records in prefix order."""
    import ipaddress
    from . import ospfv3
    recs = []
    for p, m in entries:
        net = ipaddress.ip_network(p, strict=False)
        recs.append((ospfv3.ip_rec(net.network_address), 0 if m is None else int(m), 0, net.prefixlen, int(m is not None), (0, 0)))
    a = np.zeros(len(recs), SUMMARY_DT)
    for i, r in enumerate(recs):
        a[i] = r
    order = sorted(range(len(a)), key=lambda i: (int(a[i]["prefix"]["is_v6"]), bytes(a[i]["prefix"]["bytes"]), int(a[i]["len"])))
    return a[order] if len(a) else a


def summaries(l1_rib, cfg: np.ndarray, lib=None, name="hspf_isis_summaries") -> np.ndarray:
    """Active summaries of an L1 table (the L1 half of update_rib)."""
    lib = lib or capi.load_library()
    fn = getattr(lib, name)
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32)]
    keep = []
    s1 = _rib_struct(l1_rib, keep) if l1_rib is not None else None
    cfg = np.ascontiguousarray(cfg, dtype=SUMMARY_DT)
    out = np.zeros(max(len(cfg), 1), SUMMARY_DT)
    n = C.c_uint32()
    rc = fn(C.addressof(s1) if s1 is not None else None, cfg.ctypes.data if len(cfg) else None, len(cfg), out.ctypes.data,
            C.byref(n))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, name + " failed")
    return out[: n.value].copy()


def rib_add_summaries(l2_rib, active: np.ndarray, lib=None, name="hspf_isis_rib_add_summaries") -> IsisRib:
    """The L2 table with the active summaries as next-hop-less ROUTE_SUMMARY routes."""
    lib = lib or capi.load_library()
    fn = getattr(lib, name)
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(RibStruct)]
    keep = []
    s2 = _rib_struct(l2_rib, keep) if l2_rib is not None else None
    active = np.ascontiguousarray(active, dtype=SUMMARY_DT)
    n_r = (len(l2_rib.routes) if l2_rib is not None else 0) + len(active)
    n_h = len(l2_rib.nexthops) if l2_rib is not None else 0
    routes, nhs = np.zeros(max(n_r, 1), ROUTE_DT), np.zeros(max(n_h, 1), NEXTHOP_DT)
    r = RibStruct()
    r.routes_cap, r.routes = len(routes), routes.ctypes.data
    r.nexthops_cap, r.nexthops = len(nhs), nhs.ctypes.data
    rc = fn(C.addressof(s2) if s2 is not None else None, active.ctypes.data if len(active) else None, len(active), C.byref(r))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, name + " failed")
    return IsisRib(routes[: r.n_routes].copy(), nhs[: r.n_nexthops].copy(), rc)


def l1_to_l2(level: IsisLevel, local_system_id: int, spt_std: IsisSpt, spt_v6, l1_metric_type: int, l2_metric_type: int,
             cfg: np.ndarray, active: np.ndarray, up_down=None, lib=None, name="hspf_isis_l1_to_l2") -> np.ndarray:
    """lsp_propagate_l1_to_l2: the IP reachability entries an L1/L2 router adds to its L2 LSP."""
    lib = lib or capi.load_library()
    fn = getattr(lib, name)
    fn.argtypes = [C.POINTER(LevelStruct), C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint8, C.c_uint8,
                   C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    keep = []
    ls = level.as_struct()
    s_std = _spt_struct(spt_std, keep)
    s_v6 = _spt_struct(spt_v6, keep) if spt_v6 is not None else None
    cfg = np.ascontiguousarray(cfg, dtype=SUMMARY_DT)
    active = np.ascontiguousarray(active, dtype=SUMMARY_DT)
    ud = np.ascontiguousarray(up_down, dtype=np.uint8) if up_down is not None else None
    cap = len(level.ipreaches) + 3 * len(active) + 1
    out = np.zeros(cap, IPREACH_DT)
    n = C.c_uint32()
    rc = fn(C.byref(ls), ud.ctypes.data if ud is not None else None, local_system_id, C.addressof(s_std),
            C.addressof(s_v6) if s_v6 is not None else None, l1_metric_type, l2_metric_type,
            cfg.ctypes.data if len(cfg) else None, len(cfg), active.ctypes.data if len(active) else None, len(active),
            out.ctypes.data, cap, C.byref(n))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, name + " failed")
    return out[: n.value].copy()


# ---- routing table of an L1/L2 router (include/holo_spf_lsdb.h: hspf_isis_l1l2_*) ----------------
class JobPlanesStruct(C.Structure):
    _fields_ = [("dist", C.c_void_p), ("hops", C.c_void_p), ("n_ov", C.c_uint32), ("ov_edge", C.c_void_p),
                ("ov_cost", C.c_void_p)]


NO_SUMMARY = 0xFFFFFFFF
SUMMARY_ACTIVE = 1 << 32


class L1L2RibTable(route_table.RouteTable):
    """hspf_isis_l1l2_ribtable of one L1/L2 router: its level-1 and level-2 instances (`l1`, `l2`, dicts as for
    RouteTable), its configured summaries `cfg` (summary_cfg) and `l2_derived` (u8 per l2 IP reachability entry,
    or None).  `off` [2, n_prefixes + 1]: the L1 and L2 contributor ranges; contributors [0, n_l1) are L1's, the
    rest L2's, and winner n_contributors + s is summary s.  `sum_of`, `cov_off`, `cov`: each prefix's summary and
    the L1 prefixes each summary covers.  `n_vertices[level - 1][t]` / `root[level - 1][t]` per topology."""

    api, kind, contrib_dt = "hspf_isis", "l1l2_ribtable", CONTRIB_DT

    def __init__(self, l1: dict, l2: dict, cfg=None, l2_derived=None):
        s1, s2 = instance_struct(l1), instance_struct(l2)
        self.cfg = np.ascontiguousarray(cfg if cfg is not None else np.zeros(0, SUMMARY_DT), SUMMARY_DT)
        der = None if l2_derived is None else np.ascontiguousarray(l2_derived, np.uint8)
        super().__init__(capi.load_library().hspf_isis_l1l2_ribtable_create, C.byref(s1), C.byref(s2),
                         der.ctypes.data if der is not None and len(der) else None,
                         self.cfg.ctypes.data if len(self.cfg) else None, len(self.cfg))
        self.n_vertices = [[0, 0], [0, 0]]
        self.root = [[NO_ROOT, NO_ROOT], [NO_ROOT, NO_ROOT]]
        for level in (1, 2):
            for t in (TOPO_STD, TOPO_MT6):
                nv, r = C.c_uint32(), C.c_uint32()
                self._call("topology", level, t, C.byref(nv), C.byref(r))
                self.n_vertices[level - 1][t], self.root[level - 1][t] = nv.value, r.value
        pp, pl, po = C.c_void_p(), C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint32)()
        self._call("arrays", C.byref(pp), C.byref(pl), C.byref(po), None)
        P = self.n_prefixes
        self.prefix = route_table.copy_records(pp, P, IP_DT)
        self.len = route_table.copy_records(pl, P, np.uint32)
        self.off = route_table.copy_records(po, 2 * (P + 1), np.uint32).reshape(2, P + 1)
        n1, S = C.c_uint32(), C.c_uint32()
        so, co, cv = C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint32)()
        self._call("summaries", C.byref(n1), C.byref(S), C.byref(so), C.byref(co), C.byref(cv))
        self.n_l1, self.n_summaries = n1.value, S.value
        self.sum_of = route_table.copy_records(so, P, np.uint32)
        self.cov_off = route_table.copy_records(co, S.value + 1, np.uint32)
        self.cov = route_table.copy_records(cv, int(self.cov_off[-1]), np.uint32)


def _planes_pair(rs):
    return C.byref(rs) if rs is not None else None


def l1l2_rib_cells_device(ctx: capi.Context, t: L1L2RibTable, n_jobs: int, l1, l2, n_rows, rows_ptr: int,
                          summary_ptr: int, status_ptr: int, cells_ptr: int):
    """hspf_isis_l1l2_rib_cells / _cells16 over DEVICE planes.  l1, l2: (rs_std, rs_mt6) of the L1 and of the L2 batch
    (capi.ResultStruct or capi.Result16Struct holding device pointers; rs_mt6 may be None unless that level has an
    MT-IPv6 root); n_rows: (rows of the L1 batch, rows of the L2 batch); rows_ptr: device u32 [n_jobs, 2];
    summary_ptr: device u64 [n_jobs, t.n_summaries]; status_ptr: device u32 [n_jobs] or 0; cells_ptr: device
    [n_jobs, t.n_prefixes] cells.  Enqueued on the ctx stream; the table must have been uploaded."""
    nr = (C.c_uint32 * 2)(*[int(x) for x in n_rows])
    rs = next((x for x in (*l1, *l2) if x is not None), None)      # none at all: the call refuses the arguments
    route_table.call_stage(ctx, "hspf_isis_l1l2_rib_cells", rs, t.handle, n_jobs, *map(_planes_pair, (*l1, *l2)), nr,
                           rows_ptr or None, summary_ptr or None, status_ptr or None, cells_ptr or None)


def l1l2_rib_delta_device(ctx: capi.Context, t: L1L2RibTable, n_jobs: int, l1, l2, n_rows, rows_ptr: int,
                          summary_ptr: int, base_ptr: int, n_base: int, base_of_ptr: int, job_out_ptr: int,
                          records_ptr: int, cap: int, n_records_ptr: int):
    """hspf_isis_l1l2_rib_delta / _delta16: the summary pass, then the route-delta stage over the same walk (arguments
    as l1l2_rib_cells_device and routes_delta_device)."""
    nr = (C.c_uint32 * 2)(*[int(x) for x in n_rows])
    rs = next((x for x in (*l1, *l2) if x is not None), None)      # none at all: the call refuses the arguments
    route_table.call_stage(ctx, "hspf_isis_l1l2_rib_delta", rs, t.handle, n_jobs, *map(_planes_pair, (*l1, *l2)), nr,
                           rows_ptr or None, summary_ptr or None, base_ptr or None, n_base, base_of_ptr or None,
                           job_out_ptr or None, records_ptr or None, cap, n_records_ptr or None)


def l1l2_rib_from_cells(l1: dict, l2: dict, t: L1L2RibTable, cells: np.ndarray, words: np.ndarray, planes, ovs=None) -> IsisRib:
    """hspf_isis_l1l2_rib_from_cells (host): one job's cells and summary words -> its merged routing table.  planes:
    four (dist u32[V], hops u16[V]) or None, for L1 std, L1 MT-IPv6, L2 std, L2 MT-IPv6; ovs: four [(edge, cost)]
    lists.  rc HSPF_E_UNSUPPORTED is returned in the result."""
    lib = capi.load_library()
    cells = np.ascontiguousarray(cells, CELL_DT)
    words = np.ascontiguousarray(words, np.uint64)
    assert cells.shape == (t.n_prefixes,) and words.shape == (t.n_summaries,)
    keep = [cells, words]
    jp = (JobPlanesStruct * 4)()
    for k in range(4):
        p = planes[k]
        ov = list((ovs or [(), (), (), ()])[k])
        if p is not None:
            d, h = np.ascontiguousarray(p[0], np.uint32), np.ascontiguousarray(p[1], np.uint16)
            keep += [d, h]
            jp[k].dist, jp[k].hops = d.ctypes.data, h.ctypes.data
        e = np.asarray([x for x, _ in ov] or [0], np.uint32)
        c = np.asarray([x for _, x in ov] or [0], np.uint32)
        keep += [e, c]
        jp[k].n_ov, jp[k].ov_edge, jp[k].ov_cost = len(ov), e.ctypes.data, c.ctypes.data
    s1 = instance_struct(l1)
    tail = (t.handle, cells.ctypes.data if len(cells) else None, words.ctypes.data if len(words) else None, jp)
    res = _call_rib(lib.hspf_isis_l1l2_rib_from_cells, l2, (C.byref(s1),), tail_args=tail)
    if res.rc not in (capi.HSPF_OK, capi.HSPF_E_UNSUPPORTED):
        raise capi.HspfError(res.rc, "hspf_isis_l1l2_rib_from_cells failed")
    return res


# ---- L1 -> L2 propagation of an L1/L2 router (include/holo_spf_lsdb.h: hspf_isis_l1_to_l2_*) -------------
class L1ToL2Table:
    """hspf_isis_l1_to_l2_table of one L1/L2 router: what lsp_propagate_l1_to_l2 may put into its L2 LSP in any job.
    `l1`, `l2`: its instance images; `rib`: its L1L2RibTable (kept alive with this table; upload it before the
    device calls); `up_down`: u8 per l1 IP reachability entry, or None.  `kind`, `prefix`, `len` [n_keys]: the keys
    in hspf_isis_l1_to_l2's output order; a cell's winner < n_records is a record, n_records + s is summary s."""

    def __init__(self, l1: dict, l2: dict, rib: L1L2RibTable, up_down=None):
        self.lib = capi.load_library()
        self.rib = rib
        s1, s2 = instance_struct(l1), instance_struct(l2)
        ud = None if up_down is None else np.ascontiguousarray(up_down, np.uint8)
        h = C.c_void_p()
        rc = self.lib.hspf_isis_l1_to_l2_table_create(C.byref(s1), C.byref(s2),
                                                      ud.ctypes.data if ud is not None and len(ud) else None,
                                                      rib.handle, C.byref(h))
        if rc != capi.HSPF_OK:
            raise capi.HspfError(rc, "hspf_isis_l1_to_l2_table_create failed")
        self.handle = h
        nk, nr = C.c_uint32(), C.c_uint32()
        pk, pp, pl = C.c_void_p(), C.c_void_p(), C.c_void_p()
        assert self.lib.hspf_isis_l1_to_l2_table_keys(h, C.byref(nk), C.byref(nr), C.byref(pk), C.byref(pp),
                                                      C.byref(pl)) == capi.HSPF_OK
        self.n_keys, self.n_records = nk.value, nr.value
        self.kind = route_table.copy_records(pk, self.n_keys, np.uint8)
        self.prefix = route_table.copy_records(pp, self.n_keys, IP_DT)
        self.len = route_table.copy_records(pl, self.n_keys, np.uint8)
        self.n_summaries = rib.n_summaries

    def upload(self, ctx: capi.Context):
        rc = self.lib.hspf_isis_l1_to_l2_table_upload(ctx.handle, self.handle)
        if rc != capi.HSPF_OK:
            raise capi.HspfError(rc, ctx.last_error())

    def __del__(self):
        try:
            if self.handle:
                self.lib.hspf_isis_l1_to_l2_table_free(self.handle)
                self.handle = None
        except Exception:
            pass


def l1_to_l2_cells_device(ctx: capi.Context, t: L1ToL2Table, n_jobs: int, l1, n_rows: int, rows_ptr: int,
                          summary_ptr: int, status_ptr: int, cells_ptr: int):
    """hspf_isis_l1_to_l2_cells / _cells16 over DEVICE planes.  l1: (rs_std, rs_mt6) of the L1 batch
    (capi.ResultStruct or capi.Result16Struct holding device pointers; rs_mt6 may be None unless L1 has an MT-IPv6
    root); n_rows: rows of the L1 batch; rows_ptr: device u32 [n_jobs]; summary_ptr: device u64
    [n_jobs, t.n_summaries]; status_ptr: device u32 [n_jobs] or 0; cells_ptr: device [n_jobs, t.n_keys] cells.
    Enqueued on the ctx stream; both tables must have been uploaded."""
    rs = next((x for x in l1 if x is not None), None)      # none at all: the call refuses the arguments
    route_table.call_stage(ctx, "hspf_isis_l1_to_l2_cells", rs, t.handle, n_jobs, *map(_planes_pair, l1), n_rows,
                           rows_ptr or None, summary_ptr or None, status_ptr or None, cells_ptr or None)


def l1_to_l2_delta_device(ctx: capi.Context, t: L1ToL2Table, n_jobs: int, l1, n_rows: int, rows_ptr: int,
                          summary_ptr: int, base_ptr: int, n_base: int, base_of_ptr: int, job_out_ptr: int,
                          records_ptr: int, cap: int, n_records_ptr: int):
    """hspf_isis_l1_to_l2_delta / _delta16: the summary pass, then the route-delta stage over the same walk
    (arguments as l1_to_l2_cells_device and routes_delta_device)."""
    rs = next((x for x in l1 if x is not None), None)
    route_table.call_stage(ctx, "hspf_isis_l1_to_l2_delta", rs, t.handle, n_jobs, *map(_planes_pair, l1), n_rows,
                           rows_ptr or None, summary_ptr or None, base_ptr or None, n_base, base_of_ptr or None,
                           job_out_ptr or None, records_ptr or None, cap, n_records_ptr or None)


def l1_to_l2_from_cells(l1: dict, t: L1ToL2Table, cells: np.ndarray, words: np.ndarray) -> np.ndarray:
    """hspf_isis_l1_to_l2_from_cells (host): one job's cells and summary words -> the IPREACH_DT entries
    hspf_isis_l1_to_l2 gives over the job's L1 SPTs and active summaries."""
    lib = capi.load_library()
    cells = np.ascontiguousarray(cells, CELL_DT)
    words = np.ascontiguousarray(words, np.uint64)
    assert cells.shape == (t.n_keys,) and words.shape == (t.n_summaries,)
    s1 = instance_struct(l1)
    out = np.zeros(max(t.n_keys, 1), IPREACH_DT)
    n = C.c_uint32()
    rc = lib.hspf_isis_l1_to_l2_from_cells(C.byref(s1), t.handle, cells.ctypes.data if len(cells) else None,
                                           words.ctypes.data if len(words) else None, out.ctypes.data, len(out),
                                           C.byref(n))
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, "hspf_isis_l1_to_l2_from_cells failed")
    return out[: n.value].copy()


# ---- backbone routers over L1 what-if jobs (include/holo_spf_lsdb.h: hspf_isis_backbone_*) ------------------------
class BackboneTable:
    """hspf_isis_backbone_table of one backbone router R: its affected prefixes over an area's L1 jobs.  `l2`: R's
    level-2 instance image; `borders`: the area's L1ToL2Table list (kept alive with this table); `derived`: u8 per l2
    IP reachability entry marking the borders' propagated and summary entries, or None.  `prefix`, `len`
    [n_prefixes]: the affected prefixes in hl_isis_rib order."""

    def __init__(self, l2: dict, borders, derived=None):
        self.lib = capi.load_library()
        self.borders = list(borders)
        s2 = instance_struct(l2)
        der = None if derived is None else np.ascontiguousarray(derived, np.uint8)
        assert der is None or len(der) == len(l2["level"].ipreaches), "one derived byte per IP reachability entry"
        arr = (C.c_void_p * max(len(self.borders), 1))(*[b.handle.value for b in self.borders])
        h = C.c_void_p()
        rc = self.lib.hspf_isis_backbone_table_create(C.byref(s2), der.ctypes.data if der is not None and len(der) else None,
                                                      len(self.borders), arr, C.byref(h))
        if rc != capi.HSPF_OK:
            raise capi.HspfError(rc, "hspf_isis_backbone_table_create failed")
        self.handle = h
        n, pp, pl = C.c_uint32(), C.c_void_p(), C.c_void_p()
        assert self.lib.hspf_isis_backbone_table_prefixes(h, C.byref(n), C.byref(pp), C.byref(pl)) == capi.HSPF_OK
        self.n_prefixes = n.value
        self.prefix = route_table.copy_records(pp, self.n_prefixes, IP_DT)
        self.len = route_table.copy_records(pl, self.n_prefixes, np.uint8)

    def upload(self, ctx: capi.Context):
        rc = self.lib.hspf_isis_backbone_table_upload(ctx.handle, self.handle)
        if rc != capi.HSPF_OK:
            raise capi.HspfError(rc, ctx.last_error())

    def __del__(self):
        try:
            if self.handle:
                self.lib.hspf_isis_backbone_table_free(self.handle)
                self.handle = None
        except Exception:
            pass


def _device_ptrs(ptrs):
    return (C.c_void_p * max(len(ptrs), 1))(*[int(p) or None for p in ptrs])


def backbone_cells_device(ctx: capi.Context, t: BackboneTable, n_jobs: int, l2, border_cells, border_status,
                          status_ptr: int, cells_ptr: int):
    """hspf_isis_backbone_cells / _cells16 over DEVICE planes.  l2: (rs_std, rs_mt6) of R's L2 batch (only row 0 is
    read; rs_mt6 may be None unless R has an MT-IPv6 root); border_cells: per border a device pointer to its
    [n_jobs, K_b] L1 -> L2 cells; border_status: per border a device u32 [n_jobs] pointer or 0 (None: none);
    status_ptr: device u32 [n_jobs] or 0; cells_ptr: device [n_jobs, t.n_prefixes] cells.  Enqueued on the ctx
    stream; the table must have been uploaded."""
    rs = next((x for x in l2 if x is not None), None)      # none at all: the call refuses the arguments
    st = _device_ptrs(border_status) if border_status is not None else None
    route_table.call_stage(ctx, "hspf_isis_backbone_cells", rs, t.handle, n_jobs, *map(_planes_pair, l2),
                           _device_ptrs(border_cells), st, status_ptr or None, cells_ptr or None)


def backbone_delta_device(ctx: capi.Context, t: BackboneTable, n_jobs: int, l2, border_cells, border_status,
                          base_ptr: int, n_base: int, base_of_ptr: int, job_out_ptr: int, records_ptr: int, cap: int,
                          n_records_ptr: int):
    """hspf_isis_backbone_delta / _delta16: the route-delta stage over the same walk (arguments as
    backbone_cells_device and routes_delta_device)."""
    rs = next((x for x in l2 if x is not None), None)
    st = _device_ptrs(border_status) if border_status is not None else None
    route_table.call_stage(ctx, "hspf_isis_backbone_delta", rs, t.handle, n_jobs, *map(_planes_pair, l2),
                           _device_ptrs(border_cells), st, base_ptr or None, n_base, base_of_ptr or None,
                           job_out_ptr or None, records_ptr or None, cap, n_records_ptr or None)


def backbone_from_cells(l2: dict, t: BackboneTable, cells: np.ndarray, planes, entries) -> IsisRib:
    """hspf_isis_backbone_from_cells (host): one job's cells -> the routes of the affected prefixes.  planes: R's two
    (dist u32[V], hops u16[V]) or None (std, MT-IPv6; row 0); entries: per border the job's IPREACH_DT list
    (l1_to_l2_from_cells).  rc HSPF_E_UNSUPPORTED is returned in the result."""
    lib = capi.load_library()
    cells = np.ascontiguousarray(cells, CELL_DT)
    assert cells.shape == (t.n_prefixes,) and len(entries) == len(t.borders)
    keep = [cells]
    jp = (JobPlanesStruct * 2)()
    for k in range(2):
        if planes[k] is not None:
            d, h = np.ascontiguousarray(planes[k][0], np.uint32), np.ascontiguousarray(planes[k][1], np.uint16)
            keep += [d, h]
            jp[k].dist, jp[k].hops = d.ctypes.data, h.ctypes.data
    ents = [np.ascontiguousarray(e, IPREACH_DT) for e in entries]
    keep += ents
    ep = (C.c_void_p * len(ents))(*[e.ctypes.data if len(e) else None for e in ents])
    ne = (C.c_uint32 * len(ents))(*[len(e) for e in ents])
    tail = (t.handle, cells.ctypes.data if len(cells) else None, jp, ep, ne)
    res = _call_rib(lib.hspf_isis_backbone_from_cells, l2, (), tail_args=tail)
    if res.rc not in (capi.HSPF_OK, capi.HSPF_E_UNSUPPORTED):
        raise capi.HspfError(res.rc, "hspf_isis_backbone_from_cells failed")
    return res


def _adjacencies(t: Topology, root: int, sys_of, usage: int):
    """Local interfaces and adjacencies of router `root` of topology t (router i is system sys_of(i))."""
    from . import ospfv3
    ifaces, adjs = [], []
    for k in range(t.n_p2p):
        a, b = int(t.p2p_a[k]), int(t.p2p_b[k])
        for me, other, cost in ((a, b, int(t.p2p_cost_ab[k])), (b, a, int(t.p2p_cost_ba[k]))):
            if me == root:
                n = len(adjs) + 1
                adjs.append((sys_of(other), (2, 0, 0, 1, n >> 8, n & 255), 1, usage, 1, 1, 1, 1, 0, (0, 0, 0),
                             0xAC100000 + 4 * k + (2 if me == a else 1), ospfv3.ip_rec(f"fe80::{n:x}")))
                ifaces.append((len(ifaces) + 1, cost, 0, (0, 0, 0), len(adjs) - 1, 1))
    for members, costs in t.lans:
        if root in members:
            off = len(adjs)
            for m in sorted(members):
                if m != root:
                    n = len(adjs) + 1
                    adjs.append((sys_of(m), (2, 0, 0, 2, n >> 8, n & 255), 1, usage, 1, 1, 1, 1, 0, (0, 0, 0),
                                 0xC0A80000 + 256 * len(ifaces) + m % 250, ospfv3.ip_rec(f"fe80::1:{n:x}")))
            ifaces.append((len(ifaces) + 1, costs[members.index(root)], 1, (0, 0, 0), off, len(adjs) - off))
    return ifaces, adjs


def _with_ipreach(level: IsisLevel, entries: dict) -> IsisLevel:
    """`level` with entries[lan_id] (IPREACH_DT tuples) appended to each LAN id's zeroth fragment."""
    import copy
    lv = copy.copy(level)
    lsps, old = lv.lsps.copy(), lv.ipreaches
    new = []
    for i in range(len(lsps)):
        a, n = int(lsps["ipreach_off"][i]), int(lsps["n_ipreach"][i])
        ent = [tuple(x.tolist()) for x in old[a:a + n]]
        if int(lsps["fragment"][i]) == 0:
            ent += entries.get(int(lsps["lan_id"][i]), [])
        lsps["ipreach_off"][i], lsps["n_ipreach"][i] = len(new), len(ent)
        new += ent
    lv.lsps = lsps
    lv.ipreaches = np.array(new, IPREACH_DT) if new else np.zeros(0, IPREACH_DT)
    return lv


def _distances(flat: "Flat", root: int) -> np.ndarray:
    """Shortest distances from `root` over a flattened level (u32, 0xFFFFFFFF: unreached)."""
    import heapq
    row, col, cost, vf = flat.csr.row_ptr, flat.csr.col, flat.csr.cost, flat.csr.vflags
    V = flat.csr.n_vertices
    d = np.full(V, 0xFFFFFFFF, np.uint64)
    d[root] = 0
    heap, done = [(0, root)], np.zeros(V, bool)
    while heap:
        du, u = heapq.heappop(heap)
        if done[u]:
            continue
        done[u] = True
        if u != root and (vf[u] & 0x6):          # HSPF_VF_LEAF / LEAF_UNLESS_ROOT: a leaf relaxes nothing
            continue
        for e in range(int(row[u]), int(row[u + 1])):
            v, nd = int(col[e]), du + int(cost[e])
            if nd < d[v]:
                d[v] = nd
                heapq.heappush(heap, (nd, v))
    return d.astype(np.uint32)


def _spt_of(flat: "Flat", dist: np.ndarray) -> IsisSpt:
    """An IsisSpt holding only what hspf_isis_l1_to_l2 reads: the reached vertices' LAN ids and distances."""
    reached = np.nonzero(dist != 0xFFFFFFFF)[0]
    v = np.zeros(len(reached), VERTEX_DT)
    v["lan_id"], v["distance"] = flat.ids[reached], dist[reached]
    z = np.zeros(0, np.uint32)
    return IsisSpt(v, z, np.zeros(0, np.uint64), z, z)


def l1l2_view(seed: int, n_l1: int = 150, n_l2: int = 120, n_border: int = 3, root: int = 0,
              metric_type: int = METRIC_WIDE, mt6: bool = False, sr: bool = False, max_paths: int = 4,
              attached: bool = True, summaries=(("10.1.0.0/16", None),), cost_choices=None, l1_degree: int = 4,
              l2_topology=None) -> dict:
    """A seeded two-level domain: an L1 area of n_l1 routers (systems sysid(0 .. n_l1 - 1)) and an L2 backbone of n_l2
    routers joined by the L1/L2 routers 0 .. n_border - 1 (backbone router i >= n_border is sysid(n_l1 + i)).  L1
    router r advertises 10.1.r/32 (every third one also 10.2.(r % 16).0/24, and with mt6 an MT-IPv6 /128); backbone
    router i advertises 10.200.i/32.  `l2_topology` (a synth.Topology) replaces the generated backbone; n_l2 is then
    its router count.  The L1 area has l1_degree * n_l1 / 2 adjacencies (2: a tree and a few more).  Every L1/L2 router sets the ATT bit in its L1 LSP (the root only when
    `attached`) and carries in its own L2 LSP what lsp_propagate_l1_to_l2 puts there from its own L1 SPT with the
    configured `summaries`: the propagated entries and its active summaries.  Returns dict(l1, l2: the instance
    images of L1/L2 router `root`, cfg, l2_derived: the mask of root's derived L2 entries, borders, derived_all: the
    mask of every border's derived L2 entries).  l1l2_backbone gives a backbone router's L2 image."""
    from . import ospfv3, synth
    kw = dict(cost_choices=cost_choices) if cost_choices else dict(cost_lo=1, cost_hi=20)
    t1 = synth.random_topology(n_l1, l1_degree * n_l1, synth.SEED_BASE + 1000 + seed, lan_fraction=0.1, **kw)
    t2 = l2_topology or synth.random_topology(n_l2, 4 * n_l2, synth.SEED_BASE + 2000 + seed, lan_fraction=0.1, **kw)
    n_l2 = t2.n_routers
    sys2 = lambda i: sysid(i) if i < n_border else sysid(n_l1 + i)
    cfg = summary_cfg(list(summaries))
    narrow, wide = metric_type in (METRIC_STANDARD, METRIC_BOTH), metric_type in (METRIC_WIDE, METRIC_BOTH)

    def v4(net, plen, metric, psid=None):
        out = []
        if narrow:
            out.append(ipreach_rec(ospfv3.ip_rec(net), min(metric, 63), 0, plen, IP_V4_INTERNAL))
        if wide:
            out.append(ipreach_rec(ospfv3.ip_rec(net), metric, 0, plen, IP_V4_EXT, 0, psid if sr else None))
        return out

    def finish(lv):
        """SR capabilities, NLPIDs and ATT bits of a level"""
        lsps = lv.lsps.copy()
        lsps["flags"] |= np.where(lsps["fragment"] == 0, LSPF_NLPID_IPV6 if mt6 else 0, 0).astype(np.uint8)
        if sr:
            zero = (lsps["fragment"] == 0) & ((lsps["lan_id"] & 0xFF) == 0)
            lsps["sr_flags"] = np.where(zero, LSP_SR_HAS_CAP | LSP_SR_CAP_I | LSP_SR_CAP_V | LSP_SR_ALGO_SPF, 0)
            lsps["srgb_off"], lsps["n_srgb"] = 0, np.where(zero, 1, 0)
            lv.srgbs = np.array([(16000, 8000, 0, (0, 0, 0))], SRGB_DT)
        lv.lsps = lsps
        lv.ipv6_enabled = bool(mt6)
        return lv

    # level 1 (with mt6, synth_level's MT-IPv6 level carries the standard adjacencies beside the MT ones)
    lv1 = synth_level(t1, metric_type=metric_type, mt_id=MT_IPV6 if mt6 else MT_STANDARD)
    ent1 = {}
    for r in range(n_l1):
        e = v4(f"10.1.{r >> 8}.{r & 255}", 32, 1, (PSID_P, 0, r))
        if r % 3 == 0:
            e += v4(f"10.2.{r % 16}.0", 24, 5)
        if mt6:
            e.append(ipreach_rec(ospfv3.ip_rec(f"2001:db8:1::{r + 1:x}"), 2, MT_IPV6, 128, IP_MT_V6))
        ent1[sysid(r) << 8] = e
    lv1 = finish(_with_ipreach(lv1, ent1))
    lv1.mt_id = MT_STANDARD
    att = (lv1.lsps["fragment"] == 0) & np.isin(lv1.lsps["lan_id"], [sysid(b) << 8 for b in range(n_border)
                                                                      if attached or b != root])
    lv1.lsps["flags"] |= np.where(att, LSPF_ATT | (LSPF_MT_IPV6_ATT if mt6 else 0), 0).astype(np.uint8)
    # level 2: configured prefixes, then each L1/L2 router's propagated entries and active summaries
    lv2 = synth_level(t2, metric_type=metric_type, mt_id=MT_IPV6 if mt6 else MT_STANDARD)
    remap = lambda lid: (sys2(((int(lid) >> 8) - SYSID_BASE)) << 8) | (int(lid) & 0xFF)
    lsps = lv2.lsps.copy()
    lsps["lan_id"] = [remap(x) for x in lsps["lan_id"]]
    lv2.reaches = lv2.reaches.copy()
    lv2.reaches["neighbor"] = [remap(x) for x in lv2.reaches["neighbor"]]
    lv2.lsps = lsps[np.lexsort((lsps["fragment"], lsps["lan_id"]))]
    lv2.mt_id = MT_STANDARD
    ent2 = {}
    for i in range(n_l2):
        ent2[sys2(i) << 8] = v4(f"10.200.{i >> 8}.{i & 255}", 32, 1, (PSID_P, 0, 5000 + i))
    f1 = Flat(lv1)
    f6 = None
    if mt6:
        import copy
        l6 = copy.copy(lv1)
        l6.mt_id = MT_IPV6
        f6 = Flat(l6)
    derived = {}
    for b in range(n_border):
        d = _distances(f1, f1.vertex(sysid(b) << 8))
        d6 = _distances(f6, f6.vertex(sysid(b) << 8)) if mt6 else None
        spt6 = _spt_of(f6, d6) if mt6 else None
        # the router's L1 routes (contributions of reached vertices; ATT defaults only when not attached)
        low = {}
        for i in range(len(lv1.lsps)):
            lid, v = int(lv1.lsps["lan_id"][i]), f1.vertex(int(lv1.lsps["lan_id"][i]))
            a, n = int(lv1.lsps["ipreach_off"][i]), int(lv1.lsps["n_ipreach"][i])
            for r in lv1.ipreaches[a:a + n]:
                dv = d[v] if int(r["kind"]) != IP_MT_V6 else d6[f6.vertex(lid)]
                if dv == 0xFFFFFFFF:
                    continue
                key = (int(r["prefix"]["is_v6"]), bytes(r["prefix"]["bytes"]), int(r["len"]))
                low[key] = min(low.get(key, 1 << 40), int(dv) + int(r["metric"]))
        if not (attached or b != root):
            for i in np.nonzero(att)[0]:
                v = f1.vertex(int(lv1.lsps["lan_id"][i]))
                if d[v] != 0xFFFFFFFF:
                    key = (0, bytes(16), 0)
                    low[key] = min(low.get(key, 1 << 40), int(d[v]))
        rib = np.zeros(len(low), ROUTE_DT)
        for k, (key, m) in enumerate(sorted(low.items())):
            rib[k]["prefix"]["is_v6"], rib[k]["prefix"]["bytes"], rib[k]["len"], rib[k]["metric"] = key[0], list(key[1]), key[2], m
        act = summaries_of(rib, cfg)
        prop = l1_to_l2(lv1, sysid(b), _spt_of(f1, d), spt6, metric_type, metric_type, cfg, act)
        prop = [tuple(x.tolist()) for x in prop]
        derived[sysid(b) << 8] = len(prop)
        ent2[sysid(b) << 8] = ent2[sysid(b) << 8] + prop
    lv2 = finish(_with_ipreach(lv2, ent2))
    mask = np.zeros(len(lv2.ipreaches), np.uint8)
    mask_all = np.zeros(len(lv2.ipreaches), np.uint8)
    for i in range(len(lv2.lsps)):
        lid = int(lv2.lsps["lan_id"][i])
        if lid in derived and int(lv2.lsps["fragment"][i]) == 0:
            end = int(lv2.lsps["ipreach_off"][i]) + int(lv2.lsps["n_ipreach"][i])
            mask_all[end - derived[lid]: end] = 1
            if lid == sysid(root) << 8:
                mask[end - derived[lid]: end] = 1
    i1, a1 = _adjacencies(t1, root, sysid, 1)
    if attached:                  # an up L2 adjacency into another area: is_l2_attached_to_backbone
        a1.append((sys2(n_border), (2, 0, 0, 9, 0, 1), 1, 2, 1, 1, 1, 1, 1, (0, 0, 0), 0xAC1F0001,
                   ospfv3.ip_rec("fe80::9:1")))
        i1.append((len(i1) + 1, 10, 0, (0, 0, 0), len(a1) - 1, 1))
    r2 = next(i for i in range(n_l2) if sys2(i) == sysid(root))
    i2, a2 = _adjacencies(t2, r2, sys2, 2)
    base = dict(system_id=sysid(root), max_paths=max_paths, level_type=3, att_ignore=0, mt_ipv6=int(mt6), sr_enabled=int(sr))
    l1 = dict(base, level=lv1, level_no=1, ifaces=np.array(i1, IFACE_DT), adjs=np.array(a1, ADJ_DT))
    l2 = dict(base, level=lv2, level_no=2, ifaces=np.array(i2, IFACE_DT), adjs=np.array(a2, ADJ_DT))
    return dict(l1=l1, l2=l2, cfg=cfg, l2_derived=mask, borders=list(range(n_border)), t1=t1, t2=t2,
                derived_all=mask_all)


def l1l2_backbone(v: dict, i: int) -> dict:
    """The level-2 instance image of backbone router i (>= the view's border count) of an l1l2_view domain: the same
    L2 LSDB, level_type 2.  v["derived_all"] marks every border's derived entries in it."""
    n_border, n_l1 = len(v["borders"]), v["t1"].n_routers
    assert n_border <= i < v["t2"].n_routers
    sys2 = lambda k: sysid(k) if k < n_border else sysid(n_l1 + k)
    ifaces, adjs = _adjacencies(v["t2"], i, sys2, 2)
    return dict(v["l2"], system_id=sys2(i), level_type=2, ifaces=np.array(ifaces, IFACE_DT), adjs=np.array(adjs, ADJ_DT))


def summaries_of(l1_routes: np.ndarray, cfg: np.ndarray) -> np.ndarray:
    """hspf_isis_summaries over bare L1 routes (ROUTE_DT in prefix order, no next hops)."""
    return summaries(IsisRib(l1_routes, np.zeros(0, NEXTHOP_DT)), cfg)
