"""GPU: the arguments every batched route-stage entry point refuses before it enqueues anything
(hspf_ospfv2_routes_batch[16] / _delta[16], hspf_isis_routes_batch[16] / _delta[16], hspf_ospfv2_rib_cells[16] /
_delta[16], hspf_ospfv2_abr_rib_cells[16] / _delta[16]): each returns HSPF_E_INVAL and counts no launch.  A call
with nothing to do returns HSPF_OK and counts no launch either, but the checks that come before that early return
still refuse.  Every pointer that is not the refused one points at a device buffer large enough for the call, so
nothing here reads an invalid address even if a check were missing."""
import ctypes as C

import pytest

from holo_b200 import capi, isis, ospf_rib, ospfv2, synth
from test_isis_route_cells import mt6_instance
from test_ospf_abr_rib_cells import domain
from test_ospf_rib_cells import view

pytestmark = pytest.mark.gpu

N = 3                    # jobs of a call
u16p, u32p, u64p = C.POINTER(C.c_uint16), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)

# the arguments of each entry point family, in order; "pl" is the result struct (an array of them for "abr")
ARGS = {
    "routes_batch": "ctx rt n pl cells n_gather gj gv gnh",
    "routes_delta": "ctx rt n pl base n_base base_of job_out records cap n_records",
    "isis_batch": "ctx rt n std mt6 cells",
    "isis_delta": "ctx rt n std mt6 base n_base base_of job_out records cap n_records",
    "rib_cells": "ctx rt n pl roots cells status_out n_gather gj gv gnh",
    "rib_delta": "ctx rt n pl roots base n_base base_of job_out records cap n_records",
    "abr_cells": "ctx rt n pl n_rows rows cells status_out n_gather gj ga gv gnh",
    "abr_delta": "ctx rt n pl n_rows rows base n_base base_of job_out records cap n_records",
}
ENTRY = {
    "hspf_ospfv2_routes_batch": ("routes", "routes_batch"), "hspf_ospfv2_routes_delta": ("routes", "routes_delta"),
    "hspf_isis_routes_batch": ("isis", "isis_batch"), "hspf_isis_routes_delta": ("isis", "isis_delta"),
    "hspf_ospfv2_rib_cells": ("rib", "rib_cells"), "hspf_ospfv2_rib_delta": ("rib", "rib_delta"),
    "hspf_ospfv2_abr_rib_cells": ("abr", "abr_cells"), "hspf_ospfv2_abr_rib_delta": ("abr", "abr_delta"),
}
ENTRY.update({k + "16": v for k, v in list(ENTRY.items())})


class Env:
    """One table of each type, uploaded, and a second copy that is not; device buffers for every pointer."""

    def __init__(self, ctx):
        import torch
        self.ctx = ctx
        t = synth.random_topology(60, 240, synth.SEED_BASE + 7, cost_choices=[5, 10], lan_fraction=0.1)
        flat = ospfv2.Flat(ospfv2.synth_area(t, root=2))
        area, sums, ext = view(t, 0, 5)
        rib_flat = ospfv2.Flat(area)
        dom = domain(3)
        make = {"routes": lambda: ospfv2.RouteTable(flat), "isis": lambda: isis.RouteTable(mt6_instance(t, 2)),
                "rib": lambda: ospf_rib.RibTable(rib_flat, area.area_id, sums, ext),
                "abr": lambda: ospf_rib.AbrRibTable(dom.rt.router_id, dom.flats, dom.rt.area_ids, dom.summaries, None,
                                                    dom.externals)}
        self.keep = (flat, rib_flat, dom)
        self.tables = {k: f() for k, f in make.items()}
        self.not_uploaded = {k: f() for k, f in make.items()}
        for rt in self.tables.values():
            rt.upload(ctx)
        assert isis.NO_ROOT not in self.tables["isis"].root
        V = max([flat.csr.n_vertices, rib_flat.csr.n_vertices] + list(self.tables["isis"].n_vertices) +
                list(self.tables["abr"].n_vertices))
        P = max(rt.n_prefixes for rt in self.tables.values())
        self.cap = N * P
        zeros = lambda nbytes: torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
        self.buf = {"dist": zeros(N * V * 4), "hops": zeros(N * V * 2), "nh": zeros(N * V * 8), "status": zeros(N * 4),
                    "cells": zeros(N * P * 24), "base": zeros(N * P * 24), "job_out": zeros(N * 32),
                    "records": zeros(self.cap * 16), "n_records": zeros(8), "roots": zeros(N * 4),
                    "rows": zeros(N * ospf_rib.ABR_MAX_AREAS * 4), "status_out": zeros(N * 4),
                    "gj": zeros(4), "ga": zeros(4), "gv": zeros(4), "gnh": zeros(8)}
        self.n_rows = (C.c_uint32 * ospf_rib.ABR_MAX_AREAS)(*[N] * ospf_rib.ABR_MAX_AREAS)
        torch.cuda.synchronize()

    def ptr(self, name):
        return self.buf[name].data_ptr()

    def result(self, narrow, **over):
        """A result struct over the plane buffers; `over` sets fields (None: NULL)."""
        rs = capi.Result16Struct() if narrow else capi.ResultStruct()
        d, n = (u16p, u16p) if narrow else (u32p, u64p)
        rs.dist, rs.hops, rs.nh_mask = C.cast(self.ptr("dist"), d), C.cast(self.ptr("hops"), u16p), C.cast(self.ptr("nh"), n)
        rs.job_status = C.cast(self.ptr("status"), u32p)
        if not narrow:
            rs.nh_words = 1
        for k, v in over.items():
            if v is None:
                setattr(rs, k, type(getattr(rs, k))())
            else:
                setattr(rs, k, v)
        return rs

    def defaults(self, kind, narrow):
        rt = self.tables[kind]
        a = {"ctx": self.ctx.handle, "rt": rt.handle, "n": N, "n_gather": 0, "gj": None, "ga": None, "gv": None,
             "gnh": None, "n_base": 1, "base_of": None, "cap": self.cap, "n_rows": C.addressof(self.n_rows)}
        for k in ("cells", "base", "job_out", "records", "n_records", "roots", "rows", "status_out"):
            a[k] = self.ptr(k)
        if kind == "abr":
            a["pl"] = self.planes_array(narrow, rt.n_areas)
        else:
            a["pl"] = a["std"] = a["mt6"] = C.byref(self.result(narrow))
        return a

    def planes_array(self, narrow, n_areas, area=None, **over):
        """One result struct per area; `over` applies to area `area` only."""
        cls = capi.Result16Struct if narrow else capi.ResultStruct
        return (cls * n_areas)(*[self.result(narrow, **(over if i == area else {})) for i in range(n_areas)])


@pytest.fixture(scope="module")
def env(ctx):
    return Env(ctx)


def cases(env, kind, family, narrow):
    """(label, argument overrides, expected return code) of one entry point."""
    rt = env.tables[kind]
    delta = family.endswith("delta")
    out = [("no ctx", {"ctx": None}, capi.HSPF_E_INVAL), ("no table", {"rt": None}, capi.HSPF_E_INVAL),
           ("table not uploaded", {"rt": env.not_uploaded[kind].handle}, capi.HSPF_E_INVAL),
           ("nothing to do", {"n": 0}, capi.HSPF_OK)]
    planes = [("dist", None), ("hops", None), ("nh_mask", None)] + ([] if narrow else [("nh_words", 2)])
    if kind == "isis":
        for topo in ("std", "mt6"):
            out.append((f"no {topo} planes", {topo: None}, capi.HSPF_E_INVAL))
            out += [(f"{topo} {f}={v}", {topo: C.byref(env.result(narrow, **{f: v}))}, capi.HSPF_E_INVAL)
                    for f, v in planes]
    elif kind == "abr":
        out.append(("no planes", {"pl": None}, capi.HSPF_E_INVAL))
        out += [(f"area 1 {f}={v}", {"pl": env.planes_array(narrow, rt.n_areas, 1, **{f: v})}, capi.HSPF_E_INVAL)
                for f, v in planes]
        out += [("no n_rows", {"n_rows": None}, capi.HSPF_E_INVAL), ("no rows", {"rows": None}, capi.HSPF_E_INVAL),
                ("no rows, no jobs", {"rows": None, "n": 0}, capi.HSPF_OK)]
    else:
        out.append(("no planes", {"pl": None}, capi.HSPF_E_INVAL))
        out += [(f"{f}={v}", {"pl": C.byref(env.result(narrow, **{f: v}))}, capi.HSPF_E_INVAL) for f, v in planes]
    if kind == "rib":
        out += [("no roots", {"roots": None}, capi.HSPF_E_INVAL), ("no roots, no jobs", {"roots": None, "n": 0}, capi.HSPF_OK)]
    if delta:
        out += [("no base", {"base": None}, capi.HSPF_E_INVAL), ("no base, no jobs", {"base": None, "n": 0}, capi.HSPF_E_INVAL),
                ("n_base 0", {"n_base": 0}, capi.HSPF_E_INVAL), ("no job_out", {"job_out": None}, capi.HSPF_E_INVAL),
                ("no n_records", {"n_records": None}, capi.HSPF_E_INVAL),
                ("base not 8-byte aligned", {"base": env.ptr("base") + 4}, capi.HSPF_E_INVAL)]
    else:
        out += [("no cells", {"cells": None}, capi.HSPF_E_INVAL),
                ("no cells, no jobs", {"cells": None, "n": 0}, capi.HSPF_E_INVAL)]
    if family in ("routes_batch", "rib_cells", "abr_cells"):
        gathers = ["gj", "gv", "gnh"] + (["ga"] if kind == "abr" else [])
        full = {g: env.ptr(g) for g in gathers}
        out += [(f"gathers without {g}", {**full, "n_gather": 1, g: None}, capi.HSPF_E_INVAL) for g in gathers]
        out.append(("gathers without pointers, no jobs", {"n_gather": 1, "n": 0}, capi.HSPF_E_INVAL))
    return out


@pytest.mark.parametrize("entry", sorted(ENTRY))
def test_refused_before_launch(env, entry):
    kind, family = ENTRY[entry]
    narrow = entry.endswith("16")
    fn = getattr(env.ctx.lib, entry)
    wrong = []
    for label, over, want in cases(env, kind, family, narrow):
        a = {**env.defaults(kind, narrow), **over}
        before = env.ctx.lib.hspf_launch_count(env.ctx.handle)
        rc = fn(*[a[k] for k in ARGS[family].split()])
        launched = env.ctx.lib.hspf_launch_count(env.ctx.handle) - before
        if rc != want or launched:
            wrong.append(f"{label}: rc {rc} (want {want}), {launched} launches")
    env.ctx.sync()
    assert not wrong, wrong
