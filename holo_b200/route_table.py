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


class RouteTable:
    """A route table of the batched route stage: prefixes in route-table order, `off` [n_prefixes + 1] into the
    16-byte contributor records `contribs`, and `upload(ctx)`, which copies the table to the device.  Subclasses
    name the table type's functions (`api`), their record dtype, and read the prefixes."""

    api = ""                  # "hspf_ospfv2" or "hspf_isis": prefix of the table type's rtable_* functions
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
        return getattr(self.lib, f"{self.api}_rtable_{name}")(self.handle, *args)

    def upload(self, ctx: capi.Context):
        rc = getattr(self.lib, f"{self.api}_rtable_upload")(ctx.handle, self.handle)
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
    from . import isis, ospfv2, ospfv3
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
    }
    for name, argtypes in sigs.items():
        getattr(lib, name).argtypes = argtypes
    for api in ("hspf_ospfv2", "hspf_isis"):
        getattr(lib, api + "_rtable_free").argtypes = [vp]
        getattr(lib, api + "_rtable_free").restype = None
        for name in ("prefixes", "contributors"):
            getattr(lib, f"{api}_rtable_{name}").argtypes = [vp]
            getattr(lib, f"{api}_rtable_{name}").restype = u32
