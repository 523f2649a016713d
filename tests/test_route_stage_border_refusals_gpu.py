"""GPU: the arguments the route stages over borders' cells refuse before they enqueue anything, as
test_route_stage_refusals_gpu checks them for the one-table stages: the cells[16] / delta[16] calls of the OSPF
backbone, backbone_asbr and abr_backbone stages, of the IS-IS backbone stage, and of the IS-IS l1_to_l2 and l1l2_rib
stages (whose summary pass runs before the cells or the compare).  Each returns HSPF_E_INVAL and counts no launch; a
call with nothing to do returns HSPF_OK and counts no launch either, but the checks before that early return still
refuse.  An entry point that serves several table kinds (OSPFv2 and OSPFv3 tables, tables of area 0 and of a
non-backbone area) is tried on each.  Every pointer that is not the refused one points at a device buffer large
enough for the call, so nothing here reads an invalid address even if a check were missing."""
import ctypes as C

import pytest

import test_ospfv3_backbone_asbr_cells as v3asbr
import test_ospfv3_backbone_cells as v3bb
import test_ospfv3_nonbackbone_cells as v3nb
from holo_b200 import capi, isis, ospf_rib
from test_ospf_abr_backbone_cells import SynthAbrBackbone
from test_ospf_backbone_asbr_cells import AsbrBackbone
from test_ospf_backbone_cells import SynthBackbone
from test_ospf_nonbackbone_cells import SynthNonBackbone
from test_route_stage_refusals_gpu import N, Env

pytestmark = pytest.mark.gpu

# the arguments of each entry point family, in order; "pl" is R's result struct (an array of them, one per area, for
# the ABR-backbone stage); "b*" are the per-border arrays
BORDER = "bcells bstatus"
ASBR = "bcells bstatus bplanes bn_rows brows"
DELTA = "base n_base base_of job_out records cap n_records"
ARGS = {
    "backbone_cells": f"ctx rt n pl {BORDER} status_out cells",
    "backbone_delta": f"ctx rt n pl {BORDER} {DELTA}",
    "backbone_asbr_cells": f"ctx rt n pl {ASBR} status_out cells",
    "backbone_asbr_delta": f"ctx rt n pl {ASBR} {DELTA}",
    "isis_bb_cells": f"ctx rt n std mt6 {BORDER} status_out cells",
    "isis_bb_delta": f"ctx rt n std mt6 {BORDER} {DELTA}",
    "l1_to_l2_cells": "ctx rt n std mt6 n_l1 rows words status_out cells",
    "l1_to_l2_delta": f"ctx rt n std mt6 n_l1 rows words {DELTA}",
    "l1l2_cells": "ctx rt n std mt6 std mt6 n_rows rows words status_out cells",
    "l1l2_delta": f"ctx rt n std mt6 std mt6 n_rows rows words {DELTA}",
}
# entry point: (the table kinds it is tried on, its family)
ENTRY = {
    # a table of area 0 without type-4 slots, OSPFv2 and OSPFv3
    "hspf_ospfv2_backbone_cells": (["bb2", "bb3"], "backbone_cells"),
    "hspf_ospfv2_backbone_delta": (["bb2", "bb3"], "backbone_delta"),
    # tables with type-4 / Inter-Area-Router slots, and tables of a non-backbone area, OSPFv2 and OSPFv3
    "hspf_ospfv2_backbone_asbr_cells": (["asbr2", "asbr3", "nb2", "nb3"], "backbone_asbr_cells"),
    "hspf_ospfv2_backbone_asbr_delta": (["asbr2", "asbr3", "nb2", "nb3"], "backbone_asbr_delta"),
    "hspf_ospfv2_abr_backbone_cells": (["abr_bb"], "backbone_asbr_cells"),
    "hspf_ospfv2_abr_backbone_delta": (["abr_bb"], "backbone_asbr_delta"),
    "hspf_isis_backbone_cells": (["isis_bb"], "isis_bb_cells"), "hspf_isis_backbone_delta": (["isis_bb"], "isis_bb_delta"),
    "hspf_isis_l1_to_l2_cells": (["l1_to_l2"], "l1_to_l2_cells"), "hspf_isis_l1_to_l2_delta": (["l1_to_l2"], "l1_to_l2_delta"),
    "hspf_isis_l1l2_rib_cells": (["l1l2"], "l1l2_cells"), "hspf_isis_l1l2_rib_delta": (["l1l2"], "l1l2_delta"),
}
ENTRY.update({k + "16": v for k, v in list(ENTRY.items())})
OSPF_BB = ("bb2", "bb3", "asbr2", "asbr3", "nb2", "nb3")


class BorderEnv(Env):
    """One table of each kind, uploaded, and a second copy that is not; device buffers for every pointer (the
    result structs of Env)."""

    def __init__(self, ctx):
        import torch
        self.ctx = ctx
        # three borders of one IS-IS area (l1l2_view domains rooted at each) and backbone router 5 of its L2
        vs = [isis.l1l2_view(63, root=b, n_l1=50, n_l2=30, l1_degree=2, cost_choices=[10],
                             summaries=[("10.2.0.0/16", None), ("10.1.0.5/32", None)]) for b in range(3)]
        l1l2 = lambda v: isis.L1L2RibTable(v["l1"], v["l2"], v["cfg"], v["l2_derived"])
        l1_to_l2 = lambda v: isis.L1ToL2Table(v["l1"], v["l2"], l1l2(v))
        self.keep = []

        def table_of(b):
            self.keep.append(b)
            return b.table
        make = {"bb2": lambda: table_of(SynthBackbone(1)), "bb3": lambda: table_of(v3bb.SynthBackbone(1)),
                "asbr2": lambda: table_of(AsbrBackbone(1)), "asbr3": lambda: table_of(v3asbr.AsbrBackbone(1)),
                "nb2": lambda: table_of(SynthNonBackbone(1)), "nb3": lambda: table_of(v3nb.SynthNonBackbone(1)),
                "abr_bb": lambda: table_of(SynthAbrBackbone(1)),
                "isis_bb": lambda: isis.BackboneTable(isis.l1l2_backbone(vs[0], 5), [l1_to_l2(v) for v in vs],
                                                      vs[0]["derived_all"]),
                "l1_to_l2": lambda: l1_to_l2(vs[0]), "l1l2": lambda: l1l2(vs[0])}
        self.tables = {k: f() for k, f in make.items()}
        self.not_uploaded = {k: f() for k, f in make.items()}
        for rt in self.tables.values():
            rt.upload(ctx)
        self.tables["l1_to_l2"].rib.upload(ctx)
        tb = self.tables
        assert all(tb[k].n_asbr_slots for k in ("asbr2", "asbr3"))
        # vertices of every plane set a call may read, cells of a table's row and of a border's row, summary words
        ospf_borders = [b for k in OSPF_BB + ("abr_bb",) for b in tb[k].borders]
        isis_ribs = [tb["l1l2"], tb["l1_to_l2"].rib] + [b.rib for b in tb["isis_bb"].borders]
        V = max([tb[k].flat.csr.n_vertices for k in OSPF_BB] + [f.csr.n_vertices for f in tb["abr_bb"].flats] +
                [v for b in ospf_borders for v in b.n_vertices] + [v for r in isis_ribs for lv in r.n_vertices for v in lv])
        width = lambda rt: rt.n_keys if isinstance(rt, isis.L1ToL2Table) else rt.n_prefixes
        P = max(width(rt) for rt in tb.values())
        K = max(width(b) for b in ospf_borders + tb["isis_bb"].borders)
        S = max(r.n_summaries for r in isis_ribs)
        self.cap = N * P
        zeros = lambda nbytes: torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
        # 8 bytes over where a misaligned pointer is tried
        self.buf = {"dist": zeros(N * V * 4), "hops": zeros(N * V * 2), "nh": zeros(N * V * 8), "status": zeros(N * 4),
                    "cells": zeros(N * P * 24), "base": zeros(N * P * 24), "job_out": zeros(N * 32 + 8),
                    "records": zeros(self.cap * 16 + 8), "n_records": zeros(16),
                    "rows": zeros(N * ospf_rib.ABR_MAX_AREAS * 4), "status_out": zeros(N * 4),
                    "bcells": zeros(N * K * 24), "words": zeros(N * S * 8 + 8)}
        self.n_rows = (C.c_uint32 * ospf_rib.ABR_MAX_AREAS)(*[N] * ospf_rib.ABR_MAX_AREAS)
        torch.cuda.synchronize()

    def defaults(self, kind, narrow):
        rt = self.tables[kind]
        a = {"ctx": self.ctx.handle, "rt": rt.handle, "n": N, "n_base": 1, "base_of": None, "cap": self.cap,
             "n_rows": self.n_rows, "n_l1": N}
        for k in ("cells", "base", "job_out", "records", "n_records", "rows", "status_out", "words"):
            a[k] = self.ptr(k)
        if kind == "abr_bb":
            a["pl"] = self.planes_array(narrow, rt.n_areas)
        else:
            a["pl"] = a["std"] = a["mt6"] = C.byref(self.result(narrow))
        # every border reads the same cells and rows; an OSPF border's plane sets are one result struct per area
        borders = getattr(rt, "borders", [])
        arr = lambda ptrs: (C.c_void_p * max(len(ptrs), 1))(*ptrs)
        a["keep"] = [self.planes_array(narrow, b.n_areas) for b in borders if hasattr(b, "n_areas")]
        a["bcells"], a["bstatus"] = arr([self.ptr("bcells")] * len(borders)), None
        a["bplanes"] = arr([C.addressof(p) for p in a["keep"]])
        a["bn_rows"], a["brows"] = arr([C.addressof(self.n_rows)] * len(borders)), arr([self.ptr("rows")] * len(borders))
        return a


@pytest.fixture(scope="module")
def env(ctx):
    return BorderEnv(ctx)


def cases(env, kind, family):
    """(label, argument overrides, expected return code) of one entry point."""
    out = [("no ctx", {"ctx": None}, capi.HSPF_E_INVAL), ("no table", {"rt": None}, capi.HSPF_E_INVAL),
           ("table not uploaded", {"rt": env.not_uploaded[kind].handle}, capi.HSPF_E_INVAL),
           ("nothing to do", {"n": 0}, capi.HSPF_OK)]
    if family.endswith("delta"):
        out += [("no base", {"base": None}, capi.HSPF_E_INVAL), ("no base, no jobs", {"base": None, "n": 0}, capi.HSPF_E_INVAL),
                ("n_base 0", {"n_base": 0}, capi.HSPF_E_INVAL), ("no job_out", {"job_out": None}, capi.HSPF_E_INVAL),
                ("no n_records", {"n_records": None}, capi.HSPF_E_INVAL),
                ("base not 8-byte aligned", {"base": env.ptr("base") + 4}, capi.HSPF_E_INVAL),
                ("job_out not 4-byte aligned", {"job_out": env.ptr("job_out") + 2}, capi.HSPF_E_INVAL),
                ("n_records not 8-byte aligned", {"n_records": env.ptr("n_records") + 4}, capi.HSPF_E_INVAL),
                ("records not 4-byte aligned", {"records": env.ptr("records") + 2}, capi.HSPF_E_INVAL)]
    else:
        out += [("no cells", {"cells": None}, capi.HSPF_E_INVAL),
                ("no cells, no jobs", {"cells": None, "n": 0}, capi.HSPF_E_INVAL)]
    return out


@pytest.mark.parametrize("entry", sorted(ENTRY))
def test_refused_before_launch(env, entry):
    kinds, family = ENTRY[entry]
    narrow = entry.endswith("16")
    fn = getattr(env.ctx.lib, entry)
    wrong = []
    for kind in kinds:
        for label, over, want in cases(env, kind, family):
            a = {**env.defaults(kind, narrow), **over}
            before = env.ctx.lib.hspf_launch_count(env.ctx.handle)
            rc = fn(*[a[k] for k in ARGS[family].split()])
            launched = env.ctx.lib.hspf_launch_count(env.ctx.handle) - before
            if rc != want or launched:
                wrong.append(f"{kind} {label}: rc {rc} (want {want}), {launched} launches")
    env.ctx.sync()
    assert not wrong, wrong
