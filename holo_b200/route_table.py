"""The batched route stage's tables from Python (include/holo_spf_lsdb.h): the part the OSPFv2, OSPFv3 and IS-IS
`RouteTable` classes share, and the stage's ctypes signatures."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import capi


# route-delta stage (include/holo_lsdb.h: hl_route_delta, hl_route_delta_job, HL_DELTA_*)
DELTA_DT = np.dtype([("job", "<u4"), ("prefix", "<u4"), ("metric", "<u4"), ("kind", "u1"), ("_pad", "u1", (3,))])
DELTA_JOB_DT = np.dtype([("n_changed", "<u4"), ("n_lost", "<u4"), ("n_gained", "<u4"), ("n_metric", "<u4"),
                         ("n_nexthops", "<u4"), ("n_other", "<u4"), ("status", "<u4"), ("_pad", "<u4")])
DELTA_LOST, DELTA_GAINED, DELTA_METRIC, DELTA_NEXTHOPS, DELTA_OTHER = 0x01, 0x02, 0x04, 0x08, 0x10


def copy_records(ptr, n: int, dt) -> np.ndarray:
    """n records of dtype dt at a native pointer, copied out of the table that owns them."""
    dt = np.dtype(dt)
    return np.frombuffer(C.string_at(ptr, n * dt.itemsize), dt).copy() if n else np.zeros(0, dt)


def call_stage(ctx: capi.Context, name: str, rs, *args):
    """Calls route-stage entry point `name` (ctx first, then `args`), or its 16-bit twin `name`16 when the planes
    are 16-bit (`rs` a capi.Result16Struct); raises HspfError on a return code other than HSPF_OK."""
    fn = getattr(ctx.lib, name + "16" if isinstance(rs, capi.Result16Struct) else name)
    rc = fn(ctx.handle, *args)
    if rc != capi.HSPF_OK:
        raise capi.HspfError(rc, ctx.last_error())


class RouteTable:
    """A route table of the batched route stage: prefixes in route-table order, `off` [n_prefixes + 1] into the
    16-byte contributor records `contribs`, and `upload(ctx)`, which copies the table to the device.  Subclasses
    name the table type's functions (`api`), their record dtype, and read the prefixes."""

    api = ""                  # "hspf_ospfv2" or "hspf_isis": prefix of the table type's functions
    kind = "rtable"           # the table type's functions are {api}_{kind}_*
    contrib_dt = None

    def __init__(self, create, *args):
        self.lib = capi.load_library()
        h = C.c_void_p()
        rc = create(*args, C.byref(h))
        if rc != capi.HSPF_OK:
            raise capi.HspfError(rc, create.__name__ + " failed")
        self.handle = h
        self.n_prefixes = int(self._call("prefixes"))
        self.n_contributors = int(self._call("contributors"))
        po, pc = C.POINTER(C.c_uint32)(), C.c_void_p()
        self._call("arrays", None, None, C.byref(po), C.byref(pc))
        self.off = copy_records(po, self.n_prefixes + 1, np.uint32)
        self.contribs = copy_records(pc, self.n_contributors, self.contrib_dt)

    def _call(self, name, *args):
        return getattr(self.lib, f"{self.api}_{self.kind}_{name}")(self.handle, *args)

    def upload(self, ctx: capi.Context):
        rc = getattr(self.lib, f"{self.api}_{self.kind}_upload")(ctx.handle, self.handle)
        if rc != capi.HSPF_OK:
            raise capi.HspfError(rc, ctx.last_error())

    def __del__(self):
        try:
            if self.handle:
                self._call("free")
                self.handle = None
        except Exception:
            pass


def declare(lib: C.CDLL):
    """The route stage's C signatures, set once when the library is loaded.  Every caller shares one CDLL, so a
    signature set per call would change how the function is marshalled for all of them."""
    from . import isis, ospf_rib, ospfv2, ospfv3
    vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
    pvp, u16p, u32p, u64p = C.POINTER(vp), C.POINTER(C.c_uint16), C.POINTER(u32), C.POINTER(u64)
    res, res16 = C.POINTER(capi.ResultStruct), C.POINTER(capi.Result16Struct)
    sigs = {
        "hspf_ospfv2_rtable_create": [vp, pvp],
        "hspf_ospfv3_rtable_create": [vp, pvp],
        "hspf_ospfv2_rtable_arrays": [vp, C.POINTER(u32p), C.POINTER(u32p), C.POINTER(u32p), pvp],
        "hspf_ospfv3_rtable_prefixes6": [vp, pvp, C.POINTER(u32p)],
        "hspf_ospfv2_rtable_upload": [vp, vp],
        "hspf_ospfv2_routes_batch": [vp, vp, u32, res, vp, u32, vp, vp, vp],
        "hspf_ospfv2_routes_batch16": [vp, vp, u32, res16, vp, u32, vp, vp, vp],
        "hspf_ospfv2_run_area_batch": [vp, C.POINTER(ospfv2.AreaStruct), u32p, u32, vp, u64, u32p, u32p, u32p, u32p, u64p,
                                       u32, C.POINTER(C.c_double)],
        "hspf_ospfv2_routes_from_cells": [C.POINTER(ospfv2.AreaStruct), vp, vp, u32p, u64p, u32,
                                          C.POINTER(ospfv2.ResultStruct)],
        "hspf_ospfv3_routes_from_cells": [C.POINTER(ospfv3.AreaStruct), vp, vp, u32p, u64p, u32,
                                          C.POINTER(ospfv3.ResultStruct)],
        "hspf_isis_rtable_create": [C.POINTER(isis.InstanceStruct), pvp],
        "hspf_isis_rtable_topology": [vp, u32, u32p, u32p],
        "hspf_isis_rtable_arrays": [vp, pvp, C.POINTER(u32p), C.POINTER(u32p), pvp],
        "hspf_isis_rtable_upload": [vp, vp],
        "hspf_isis_routes_batch": [vp, vp, u32, res, res, vp],
        "hspf_isis_routes_batch16": [vp, vp, u32, res16, res16, vp],
        "hspf_ospfv2_routes_delta": [vp, vp, u32, res, vp, u32, vp, vp, vp, u64, vp],
        "hspf_ospfv2_routes_delta16": [vp, vp, u32, res16, vp, u32, vp, vp, vp, u64, vp],
        "hspf_isis_routes_delta": [vp, vp, u32, res, res, vp, u32, vp, vp, vp, u64, vp],
        "hspf_isis_routes_delta16": [vp, vp, u32, res16, res16, vp, u32, vp, vp, vp, u64, vp],
        "hspf_isis_routes_from_cells": [C.POINTER(isis.InstanceStruct), vp, vp, u32p, u16p, u32p, u16p, u32, u32p, u32p,
                                        u32, u32p, u32p, C.POINTER(isis.RibStruct)],
        "hspf_ospfv2_ribtable_create": [vp, u32, vp, u32, vp, u32, pvp],
        "hspf_ospfv2_ribtable_arrays": [vp, C.POINTER(u32p), C.POINTER(u32p), C.POINTER(u32p), pvp],
        "hspf_ospfv2_ribtable_upload": [vp, vp],
        "hspf_ospfv2_rib_cells": [vp, vp, u32, res, vp, vp, vp, u32, vp, vp, vp],
        "hspf_ospfv2_rib_cells16": [vp, vp, u32, res16, vp, vp, vp, u32, vp, vp, vp],
        "hspf_ospfv2_rib_delta": [vp, vp, u32, res, vp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_ospfv2_rib_delta16": [vp, vp, u32, res16, vp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_ospfv2_rib_from_cells": [C.POINTER(ospfv2.AreaStruct), vp, vp, u32p, u64p, u32, C.POINTER(ospf_rib.RibStruct)],
        "hspf_ospfv3_ribtable_create": [vp, u32, vp, u32, vp, u32, pvp],
        "hspf_ospfv3_ribtable_prefixes6": [vp, pvp, C.POINTER(u32p)],
        "hspf_ospfv3_rib_from_cells": [C.POINTER(ospfv3.AreaStruct), vp, vp, u32p, u64p, u32, C.POINTER(ospf_rib.RibStruct)],
        "hspf_ospfv2_abr_ribtable_create": [u32, u32, vp, vp, vp, vp, vp, vp, u32, pvp],
        "hspf_ospfv2_abr_ribtable_arrays": [vp, C.POINTER(u32p), C.POINTER(u32p), C.POINTER(u32p), pvp],
        "hspf_ospfv2_abr_ribtable_areas": [vp, vp, vp, vp, vp],
        "hspf_ospfv2_abr_ribtable_upload": [vp, vp],
        "hspf_ospfv2_abr_rib_cells": [vp, vp, u32, vp, vp, vp, vp, vp, u32, vp, vp, vp, vp],
        "hspf_ospfv2_abr_rib_cells16": [vp, vp, u32, vp, vp, vp, vp, vp, u32, vp, vp, vp, vp],
        "hspf_ospfv2_abr_rib_delta": [vp, vp, u32, vp, vp, vp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_ospfv2_abr_rib_delta16": [vp, vp, u32, vp, vp, vp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_ospfv2_abr_rib_from_cells": [vp, C.POINTER(ospfv2.AreaStruct), u32, vp, vp, vp, vp, u32,
                                           C.POINTER(ospf_rib.RibStruct)],
        "hspf_ospfv3_abr_ribtable_create": [u32, u32, vp, vp, vp, vp, vp, vp, u32, pvp],
        "hspf_ospfv3_abr_ribtable_prefixes6": [vp, pvp, C.POINTER(u32p)],
        "hspf_ospfv3_abr_rib_from_cells": [vp, C.POINTER(ospfv3.AreaStruct), u32, vp, vp, vp, vp, u32,
                                           C.POINTER(ospf_rib.RibStruct)],
        "hspf_isis_l1l2_ribtable_create": [C.POINTER(isis.InstanceStruct), C.POINTER(isis.InstanceStruct), vp, vp, u32,
                                           pvp],
        "hspf_isis_l1l2_ribtable_topology": [vp, u32, u32, u32p, u32p],
        "hspf_isis_l1l2_ribtable_arrays": [vp, pvp, C.POINTER(u32p), C.POINTER(u32p), pvp],
        "hspf_isis_l1l2_ribtable_summaries": [vp, u32p, u32p, C.POINTER(u32p), C.POINTER(u32p), C.POINTER(u32p)],
        "hspf_isis_l1l2_ribtable_upload": [vp, vp],
        "hspf_isis_l1l2_rib_cells": [vp, vp, u32, res, res, res, res, u32p, vp, vp, vp, vp],
        "hspf_isis_l1l2_rib_cells16": [vp, vp, u32, res16, res16, res16, res16, u32p, vp, vp, vp, vp],
        "hspf_isis_l1l2_rib_delta": [vp, vp, u32, res, res, res, res, u32p, vp, vp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_isis_l1l2_rib_delta16": [vp, vp, u32, res16, res16, res16, res16, u32p, vp, vp, vp, u32, vp, vp, vp, u64,
                                       vp],
        "hspf_isis_l1l2_rib_from_cells": [C.POINTER(isis.InstanceStruct), C.POINTER(isis.InstanceStruct), vp, vp, vp,
                                          C.POINTER(isis.JobPlanesStruct), C.POINTER(isis.RibStruct)],
        "hspf_isis_l1_to_l2_table_create": [C.POINTER(isis.InstanceStruct), C.POINTER(isis.InstanceStruct), vp, vp,
                                            pvp],
        "hspf_isis_l1_to_l2_table_keys": [vp, u32p, u32p, pvp, pvp, pvp],
        "hspf_isis_l1_to_l2_table_upload": [vp, vp],
        "hspf_isis_l1_to_l2_cells": [vp, vp, u32, res, res, u32, vp, vp, vp, vp],
        "hspf_isis_l1_to_l2_cells16": [vp, vp, u32, res16, res16, u32, vp, vp, vp, vp],
        "hspf_isis_l1_to_l2_delta": [vp, vp, u32, res, res, u32, vp, vp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_isis_l1_to_l2_delta16": [vp, vp, u32, res16, res16, u32, vp, vp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_isis_l1_to_l2_from_cells": [C.POINTER(isis.InstanceStruct), vp, vp, vp, vp, u32, u32p],
        "hspf_isis_backbone_table_create": [C.POINTER(isis.InstanceStruct), vp, u32, vp, pvp],
        "hspf_isis_backbone_table_prefixes": [vp, u32p, pvp, pvp],
        "hspf_isis_backbone_table_upload": [vp, vp],
        "hspf_isis_backbone_cells": [vp, vp, u32, res, res, vp, vp, vp, vp],
        "hspf_isis_backbone_cells16": [vp, vp, u32, res16, res16, vp, vp, vp, vp],
        "hspf_isis_backbone_delta": [vp, vp, u32, res, res, vp, vp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_isis_backbone_delta16": [vp, vp, u32, res16, res16, vp, vp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_ospfv2_net_summaries": [u32, C.POINTER(ospf_rib.RibStruct), C.POINTER(ospf_rib.RtrTablesStruct),
                                      C.POINTER(ospf_rib.RibAreaStruct), vp, u32, u32, vp, u32, u32p],
        "hspf_ospfv2_backbone_table_create": [vp, u32, vp, u32, vp, u32, pvp, u32, pvp],
        "hspf_ospfv2_backbone_table_prefixes": [vp, u32p, pvp, pvp],
        "hspf_ospfv2_backbone_table_records": [vp, u32p, u32p],
        "hspf_ospfv2_backbone_table_upload": [vp, vp],
        "hspf_ospfv2_backbone_cells": [vp, vp, u32, res, pvp, pvp, vp, vp],
        "hspf_ospfv2_backbone_cells16": [vp, vp, u32, res16, pvp, pvp, vp, vp],
        "hspf_ospfv2_backbone_delta": [vp, vp, u32, res, pvp, pvp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_ospfv2_backbone_delta16": [vp, vp, u32, res16, pvp, pvp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_ospfv2_backbone_from_cells": [vp, C.POINTER(ospfv2.AreaStruct), vp, vp, vp, u32,
                                            C.POINTER(ospf_rib.RibStruct)],
        "hspf_ospfv2_backbone_asbr_table_create": [vp, u32, vp, u32, vp, u32, pvp, u32, pvp],
        "hspf_ospfv2_backbone_table_asbr_slots": [vp, u32p, u32p],
        "hspf_ospfv2_nonbackbone_table_create": [vp, u32, vp, vp, u32, vp, u32, pvp, u32, pvp],
        "hspf_ospfv2_backbone_asbr_cells": [vp, vp, u32, res, pvp, pvp, pvp, pvp, pvp, vp, vp],
        "hspf_ospfv2_backbone_asbr_cells16": [vp, vp, u32, res16, pvp, pvp, pvp, pvp, pvp, vp, vp],
        "hspf_ospfv2_backbone_asbr_delta": [vp, vp, u32, res, pvp, pvp, pvp, pvp, pvp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_ospfv2_backbone_asbr_delta16": [vp, vp, u32, res16, pvp, pvp, pvp, pvp, pvp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_ospfv2_abr_backbone_table_create": [u32, u32, vp, vp, vp, vp, vp, vp, u32, pvp, u32, pvp],
        "hspf_ospfv2_abr_backbone_table_prefixes": [vp, u32p, pvp, pvp],
        "hspf_ospfv2_abr_backbone_table_records": [vp, u32p, u32p, u32p, u32p],
        "hspf_ospfv2_abr_backbone_table_upload": [vp, vp],
        "hspf_ospfv2_abr_backbone_cells": [vp, vp, u32, vp, pvp, pvp, pvp, pvp, pvp, vp, vp],
        "hspf_ospfv2_abr_backbone_cells16": [vp, vp, u32, vp, pvp, pvp, pvp, pvp, pvp, vp, vp],
        "hspf_ospfv2_abr_backbone_delta": [vp, vp, u32, vp, pvp, pvp, pvp, pvp, pvp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_ospfv2_abr_backbone_delta16": [vp, vp, u32, vp, pvp, pvp, pvp, pvp, pvp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_ospfv2_abr_backbone_from_cells": [vp, C.POINTER(ospfv2.AreaStruct), u32, vp, vp, vp, vp, u32,
                                                C.POINTER(ospf_rib.RibStruct)],
        "hspf_ospfv2_abr_backbone_table_asbrs": [vp, u32p, C.POINTER(u32p)],
        "hspf_ospfv2_abr_backbone_asbr_entries": [vp, vp, u32, vp, pvp, pvp, pvp, vp, vp],
        "hspf_ospfv2_abr_backbone_asbr_entries16": [vp, vp, u32, vp, pvp, pvp, pvp, vp, vp],
        "hspf_ospfv2_third_area_table_create": [vp, u32, vp, vp, u32, vp, u32, pvp, u32, pvp],
        "hspf_ospfv2_third_area_cells": [vp, vp, u32, res, pvp, pvp, pvp, pvp, vp, vp],
        "hspf_ospfv2_third_area_cells16": [vp, vp, u32, res16, pvp, pvp, pvp, pvp, vp, vp],
        "hspf_ospfv2_third_area_delta": [vp, vp, u32, res, pvp, pvp, pvp, pvp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_ospfv2_third_area_delta16": [vp, vp, u32, res16, pvp, pvp, pvp, pvp, vp, u32, vp, vp, vp, u64, vp],
        "hspf_ospfv3_net_summaries": [u32, C.POINTER(ospf_rib.RibStruct), C.POINTER(ospf_rib.RibAreaStruct), vp, u32,
                                      u32, vp, u32, u32p],
        "hspf_ospfv3_rtr_summaries": [u32, C.POINTER(ospf_rib.RibAreaStruct), vp, u32, u32, vp, u32, u32p],
        "hspf_ospfv3_backbone_table_create": [vp, u32, vp, u32, vp, u32, pvp, u32, pvp],
        "hspf_ospfv3_backbone_asbr_table_create": [vp, u32, vp, u32, vp, u32, pvp, u32, pvp],
        "hspf_ospfv3_nonbackbone_table_create": [vp, u32, vp, vp, u32, vp, u32, pvp, u32, pvp],
        "hspf_ospfv3_third_area_table_create": [vp, u32, vp, vp, u32, vp, u32, pvp, u32, pvp],
        "hspf_ospfv3_abr_backbone_asbr_entries": [vp, vp, u32, vp, pvp, pvp, pvp, vp, vp],
        "hspf_ospfv3_abr_backbone_asbr_entries16": [vp, vp, u32, vp, pvp, pvp, pvp, vp, vp],
        "hspf_ospfv3_backbone_table_prefixes6": [vp, u32p, pvp, C.POINTER(u32p)],
        "hspf_ospfv3_backbone_from_cells": [vp, C.POINTER(ospfv3.AreaStruct), vp, vp, vp, u32,
                                            C.POINTER(ospf_rib.RibStruct)],
        "hspf_ospfv3_abr_backbone_table_create": [u32, u32, vp, vp, vp, vp, vp, vp, u32, pvp, u32, pvp],
        "hspf_ospfv3_abr_backbone_table_prefixes6": [vp, u32p, pvp, C.POINTER(u32p)],
        "hspf_ospfv3_abr_backbone_from_cells": [vp, C.POINTER(ospfv3.AreaStruct), u32, vp, vp, vp, vp, u32,
                                                C.POINTER(ospf_rib.RibStruct)],
        "hspf_isis_backbone_from_cells": [C.POINTER(isis.InstanceStruct), vp, vp, C.POINTER(isis.JobPlanesStruct), vp,
                                          vp, C.POINTER(isis.RibStruct)],
    }
    for name, argtypes in sigs.items():
        getattr(lib, name).argtypes = argtypes
    for table in ("hspf_ospfv2_rtable", "hspf_isis_rtable", "hspf_ospfv2_ribtable", "hspf_ospfv2_abr_ribtable",
                  "hspf_isis_l1l2_ribtable"):
        getattr(lib, table + "_free").argtypes = [vp]
        getattr(lib, table + "_free").restype = None
        for name in ("prefixes", "contributors"):
            getattr(lib, f"{table}_{name}").argtypes = [vp]
            getattr(lib, f"{table}_{name}").restype = u32
    for table in ("hspf_isis_l1_to_l2_table", "hspf_isis_backbone_table", "hspf_ospfv2_backbone_table",
                  "hspf_ospfv2_abr_backbone_table"):
        getattr(lib, table + "_free").argtypes = [vp]
        getattr(lib, table + "_free").restype = None
