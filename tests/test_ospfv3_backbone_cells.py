"""CPU: Inter-Area-Prefix origination (hspf_ospfv3_net_summaries) and the backbone-router stage over what-if jobs
inside other areas for OSPFv3 (hspf_ospfv3_backbone_*).

The device kernel's body (ospf_backbone_cell_eval<true>, holo_b200/csrc/ospf_backbone_cells.h) is compiled into a test
harness and run on the CPU over the oracle's SPT planes.  Each job perturbs one link of a non-backbone area at every
border that has it.  The cells, decoded by hspf_ospfv3_backbone_from_cells, must equal byte for byte, prefix options
included, the host chain: each border's cells decoded (abr_rib_from_cells_v3), its net_summaries_v3 into area 0
spliced into R's LSDB in place of its Inter-Area-Prefix LSAs, and update_rib_full_v3 at R, restricted to the affected
prefixes."""
import ctypes as C
import ipaddress
import json
import subprocess
from pathlib import Path

import numpy as np
import pytest

import golden_util as gu
import test_ospfv3_abr_rib_cells as v3abr
from holo_b200 import capi, ospf_rib, ospfv3, synth
from holo_b200.route_table import DELTA_OTHER
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospf_abr_rib_cells import narrow, planes_of
from test_ospf_rib_cells import same_rib
from test_ospf_rib_delta import reference
from test_ospfv2_route_cells import gather_for
from test_ospfv3_rib_cells import rib_dict

ROOT = Path(__file__).resolve().parent.parent
SNAPS = gu.load_ospfv3()
MULTI = [s for s in SNAPS if len(s["areas"]) > 1]
SUMS = {(s["topo"], s["rt"]): s for s in json.loads((ROOT / "tests" / "golden" / "ospfv3_summaries.json").read_text())}
AREA_TYPE = {"normal": ospf_rib.AREA_NORMAL, "stub": ospf_rib.AREA_STUB, "nssa": ospf_rib.AREA_NSSA}
# prefix options by the names the reference records (RFC 5340 A.4.1.1)
OPT_BITS = {"nu-bit": ospfv3.PFX_NU, "la-bit": ospfv3.PFX_LA, "p-bit": ospfv3.PFX_P}


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    out = tmp_path_factory.mktemp("harness") / "libospfv3_backbone_cells_harness.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                    "-o", str(out), str(ROOT / "tests" / "native" / "ospfv3_backbone_cells_harness.cc")], check=True)
    lib = C.CDLL(str(out))
    for fn in (lib.harness_ospfv3_backbone_cells, lib.harness_ospfv3_backbone_cells16):
        fn.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 4
    return lib


def snap(topo, rt):
    return next(s for s in SNAPS if s["topo"] == topo and s["rt"] == rt)


def opt_bits(names):
    return sum(OPT_BITS[n] for n in names)


def opt_names(bits):
    return sorted(n for n, b in OPT_BITS.items() if int(bits) & b)


def full_image(s, area, keys):
    """gu.ospfv3_area_image with every recorded prefix option, not only NU: an ABR copies them into its LSAs."""
    img = gu.ospfv3_area_image(s, area, keys)
    il = sorted(area["iap_lsas"], key=lambda l: (gu.ip(l["adv"]), l["id"]))
    opts = [opt_bits(o) for l in il for (_p, _m, o) in l["prefixes"]]
    assert len(opts) == len(img.prefixes)
    px = img.prefixes.copy()
    px["options"] = opts
    img.prefixes = px
    return img


def full_inter_area_lsas(area):
    """gu.ospfv3_inter_area_lsas with every recorded prefix option."""
    out = gu.ospfv3_inter_area_lsas(area)
    ls = sorted(area.get("inter_area_lsas", []), key=lambda l: (l["type"], gu.ip(l["adv"]), l["id"]))
    out["prefix_options"] = [opt_bits(l.get("options", [])) if l["type"] == 3 else 0 for l in ls]
    return out


def golden_domain(s):
    """The ABR domain of a multi-area snapshot (as test_ospfv3_abr_rib_cells.golden_domain, with prefix options)."""
    keys = gu.global_sort_keys(s)
    areas, sums, active = [], [], []
    for area in s["areas"]:
        img = full_image(s, area, keys)
        if ospfv3.Flat(img).router_vertex(img.router_id) == 0xFFFFFFFF:
            continue
        areas.append(img)
        sums.append(full_inter_area_lsas(area))
        active.append(any((i.get("state") or "down") != "down" for i in area["interfaces"]))
    return v3abr.Domain(areas, sums, None, active), keys


def configs_of(s, dom):
    by_id = {a["area_id"]: a for a in SUMS[(s["topo"], s["rt"])]["areas"]}
    return [ospf_rib.area_config(AREA_TYPE[by_id[gu.ipstr(a.area_id)]["area_type"]], by_id[gu.ipstr(a.area_id)]["summary"],
                                 by_id[gu.ipstr(a.area_id)]["default_cost"]) for a in dom.areas]


def rib_areas(dom):
    return [ospf_rib.RibArea(a.area_id, None, a.ifaces, dom.summaries[i], dom.active[i]) for i, a in enumerate(dom.areas)]


def prefix_str(addr, ln):
    return str(ipaddress.IPv6Network((bytes(int(b) for b in addr["bytes"]), int(ln)), strict=False))


# ------------------------------------------------------------------------------------------ summary pin
@pytest.mark.parametrize("s", MULTI, ids=[f"{s['topo']}-{s['rt']}" for s in MULTI])
def test_net_summaries_equal_the_recorded_lsas(s):
    """The Inter-Area-Prefix LSAs the router originated into each attached area, as the reference recorded them:
    prefix, length, prefix options and metric."""
    dom, _ = golden_domain(s)
    cfg = configs_of(s, dom)
    rec = {a["area_id"]: a for a in SUMS[(s["topo"], s["rt"])]["areas"]}
    assert not any(a["ranges"] or a["type4"] for a in rec.values())
    assert len(dom.areas) == len(s["areas"])
    rib = dom.host(dom.planes())
    rid = dom.areas[0].router_id
    for i, a in enumerate(dom.areas):
        got = ospf_rib.net_summaries_v3(rid, rib, rib_areas(dom), cfg, i)
        assert (got["lsa_type"] == 3).all() and (got["adv_rtr"] == rid).all()
        mine = sorted([prefix_str(x["prefix"], x["len"]), opt_names(x["prefix_options"]), int(x["metric"])] for x in got)
        assert mine == rec[gu.ipstr(a.area_id)]["type3"], (s["topo"], s["rt"], gu.ipstr(a.area_id))


def test_summary_fixture_covers_every_multi_area_snapshot():
    assert len(MULTI) == 14 and len(SUMS) == 14
    assert {(s["topo"], s["rt"]) for s in MULTI} == set(SUMS)
    for s in MULTI:
        assert len(SUMS[(s["topo"], s["rt"])]["areas"]) == len(s["areas"])
    kinds = {a["area_type"] for s in SUMS.values() for a in s["areas"]}
    assert kinds == {"normal", "stub"}
    assert any(not a["summary"] for s in SUMS.values() for a in s["areas"])        # a totally stubby area
    la = [t for s in SUMS.values() for a in s["areas"] for t in a["type3"] if "la-bit" in t[1]]
    assert la and any(not t[1] for s in SUMS.values() for a in s["areas"] for t in a["type3"])


# -------------------------------------------------------------------------------------- backbone domains
def vertex_names(f):
    return [(int(r), int(i), int(k)) for r, i, k in zip(f.router_ids, f.iface_ids, f.is_router)]


class Backbone:
    """R's area-0 image and the borders' ABR domains (from their own snapshots), the table over them."""

    def __init__(self, topo, r, borders, externals=None):
        sr = snap(topo, r)
        keys = gu.global_sort_keys(sr)
        a0 = next(a for a in sr["areas"] if a["area_id"] == "0.0.0.0")
        self.area = full_image(sr, a0, keys)
        self.keys, self.snap = keys, sr
        self.flat = ospfv3.Flat(self.area)
        self.rv = self.flat.router_vertex(self.area.router_id)
        self.summaries = full_inter_area_lsas(a0)
        self.externals = externals
        self.bsnaps = [snap(topo, b) for b in borders]
        self.doms = [golden_domain(b)[0] for b in self.bsnaps]
        self.cfgs = [configs_of(b, d) for b, d in zip(self.bsnaps, self.doms)]
        self.make_table()
        self.planes = planes_of(self.flat.csr, self.rv)

    def make_table(self):
        self.table = ospf_rib.BackboneTable(self.flat, self.area.router_id, self.summaries, self.externals,
                                            [d.rt for d in self.doms])

    def job_overrides(self, link, cost):
        """Per border, per area: the overrides of link (vertex-name pair) at `cost` in the borders' non-backbone areas."""
        out = []
        for d in self.doms:
            ov = {}
            for i, (a, f) in enumerate(zip(d.areas, d.flats)):
                if a.area_id == 0:
                    continue
                names = vertex_names(f)
                src = np.repeat(np.arange(f.csr.n_vertices), np.diff(f.csr.row_ptr))
                e = [(int(k), cost) for k in range(f.csr.n_edges) if {names[src[k]], names[f.csr.col[k]]} == set(link)]
                if e:
                    ov[i] = e
            out.append(ov)
        return out

    def border_planes(self, jobs):
        return [[d.planes(ov[b]) for ov in jobs] for b, d in enumerate(self.doms)]

    def cells(self, abr, harness, bplanes, narrow_planes=False, status=None, root_status=0):
        bcells = [np.stack([d.cells(abr, p, narrow_planes)[0] for p in bp]) for d, bp in zip(self.doms, bplanes)]
        cells, out = self.cells_from(harness, bcells, narrow_planes, status, root_status)
        return cells, out, bcells

    def cells_from(self, harness, bcells, narrow_planes=False, status=None, root_status=0):
        J = len(bcells[0])
        pl = narrow(self.planes) if narrow_planes else self.planes
        keep = [np.ascontiguousarray(x) for x in pl] + [np.ascontiguousarray(c) for c in bcells]
        bc = (C.c_void_p * len(bcells))(*[c.ctypes.data for c in keep[3:]])
        st = None
        if status is not None:
            sk = [np.ascontiguousarray(x, np.uint32) for x in status]
            keep += sk
            st = (C.c_void_p * len(sk))(*[x.ctypes.data for x in sk])
        cells = np.zeros((J, self.table.n_prefixes), ospf_rib.RIB_CELL_DT)
        out = np.zeros(J, np.uint32)
        fn = harness.harness_ospfv3_backbone_cells16 if narrow_planes else harness.harness_ospfv3_backbone_cells
        assert fn(self.table.handle, J, keep[0].ctypes.data, keep[1].ctypes.data, keep[2].ctypes.data, root_status, bc,
                  st, cells.ctypes.data, out.ctypes.data) == 0
        return cells, out

    def decode(self, cells):
        v, n = gather_for(self.flat, self.rv, self.planes)
        return ospf_rib.backbone_from_cells_v3(self.area, self.table, cells, v, n)

    def affected(self, rib):
        keep = {(p.tobytes(), int(l)) for p, l in zip(self.table.prefixes6, self.table.plen)}
        sel = [k for k, r in enumerate(rib.routes) if (r["prefix"].tobytes(), int(r["len"])) in keep]
        routes, hops = [], []
        for k in sel:
            r = rib.routes[k].copy()
            h = rib.nexthops[int(r["nh_off"]): int(r["nh_off"]) + int(r["n_nh"])]
            r["nh_off"] = sum(len(x) for x in hops)
            routes.append(r)
            hops.append(h)
        return ospf_rib.Rib(np.array(routes, ospf_rib.RIB_ROUTE6_DT), np.concatenate(hops) if hops else
                            np.zeros(0, ospfv3.NEXTHOP6_DT))

    def host(self, bcells_of_job, bplanes_of_job):
        """The chain: each border's decoded cells, its net_summaries_v3 into area 0 in place of its Inter-Area-Prefix
        LSAs, update_rib_full_v3 at R."""
        bid = {d.areas[0].router_id for d in self.doms}
        new = [s for s in self.summaries if not (int(s["adv_rtr"]) in bid and s["lsa_type"] == 3)]
        for d, cfg, c, p in zip(self.doms, self.cfgs, bcells_of_job, bplanes_of_job):
            i0 = next(i for i, a in enumerate(d.areas) if a.area_id == 0)
            rib = d.decode(c, p)
            assert rib.rc == capi.HSPF_OK
            new += list(ospf_rib.net_summaries_v3(d.areas[0].router_id, rib, rib_areas(d), cfg, i0))
        s = np.array(new, ospf_rib.INTER_AREA_LSA_DT)
        s = s[np.lexsort((s["lsa_id"], s["adv_rtr"], s["lsa_type"]))]
        p = self.planes
        spf = ospfv3.area_from_planes(self.area, lambda csr, root, nhw: (p[0], p[1], np.pad(p[2][:, None], ((0, 0), (0, nhw - 1)))))
        ra = [ospf_rib.RibArea(0, spf, self.area.ifaces, s, True)]
        return self.affected(ospf_rib.update_rib_full_v3(self.area.router_id, self.area.max_paths, ra, self.externals))

    def check(self, abr, harness, jobs, narrow_planes=False):
        bp = self.border_planes(jobs)
        cells, st, bcells = self.cells(abr, harness, bp, narrow_planes)
        assert not st.any()
        for j in range(len(jobs)):
            same_rib(self.decode(cells[j]), self.host([c[j] for c in bcells], [bp[b][j] for b in range(len(self.doms))]))
        return cells, bcells


GOLDEN = [("topo1-1", "rt3", ["rt2", "rt4", "rt6"]), ("topo1-2", "rt3", ["rt2", "rt4", "rt6"]),
          ("topo2-2", "rt1", ["rt4", "rt5"]), ("topo2-2", "rt2", ["rt4", "rt5"]), ("topo2-2", "rt3", ["rt4", "rt5"]),
          ("topo3-1", "rt1", ["rt2", "rt5"])]
GIDS = [f"{t}-{r}" for t, r, _ in GOLDEN]


def non_backbone_links(bb):
    """Vertex-name pairs of the links of the borders' non-backbone areas: router to router, router to network."""
    out = set()
    for d in bb.doms:
        for a, f in zip(d.areas, d.flats):
            if a.area_id == 0:
                continue
            names = vertex_names(f)
            src = np.repeat(np.arange(f.csr.n_vertices), np.diff(f.csr.row_ptr))
            for e in range(f.csr.n_edges):
                if f.is_router[src[e]]:
                    out.add(tuple(sorted((names[src[e]], names[f.csr.col[e]]))))
    return sorted(out)


@pytest.mark.parametrize("g", GOLDEN, ids=GIDS)
def test_base_job_equals_the_recorded_local_rib(abr_harness, harness, g):
    """Job 0 (no perturbation) equals R's recorded local-rib, restricted to the affected prefixes: metric, route type
    and next hops.  None of the six is refused."""
    bb = Backbone(*g)
    cells, _ = bb.check(abr_harness, harness, [bb.job_overrides((), 0)])
    got = bb.decode(cells[0])
    mine = rib_dict(got, {v: k for k, v in bb.keys.items()})
    keys = {f"{ospfv3.ip_str(p)}/{int(l)}" for p, l in zip(bb.table.prefixes6, bb.table.plen)}
    want = {k: v for k, v in gu.golden_rib(bb.snap).items() if k in keys}
    norm = lambda d: {k: (v[0], v[1], [(a or "", b or "") for a, b in v[2]]) for k, v in d.items()}
    assert norm(mine) == norm(want)
    assert bb.table.n_prefixes > 0 and bb.table.v3


@pytest.mark.parametrize("g", GOLDEN, ids=GIDS)
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_chain_one_link_failed_or_recosted(abr_harness, harness, g, narrow_planes):
    """Every non-backbone link failed, then re-costed, one job each, all jobs in one batch."""
    bb = Backbone(*g)
    links = non_backbone_links(bb)
    assert links
    jobs = [bb.job_overrides((), 0)]
    for link in links:
        jobs.append(bb.job_overrides(link, capi.COST_DISABLED))
        jobs.append(bb.job_overrides(link, 35))
    cells, _ = bb.check(abr_harness, harness, jobs, narrow_planes)
    assert (cells != cells[0]).any()


def test_golden_slots_carry_the_la_option(abr_harness, harness):
    """The goldens' border loopbacks carry LA: R's inter-area routes through a slot keep it."""
    bb = Backbone("topo2-2", "rt1", ["rt4", "rt5"])
    cells, _ = bb.check(abr_harness, harness, [bb.job_overrides((), 0)])
    got = bb.decode(cells[0])
    inter = got.routes[got.routes["path_type"] == ospf_rib.PATH_INTER]
    assert (inter["prefix_options"] & ospfv3.PFX_LA).any()
    w = cells[0]["winner"][ospf_rib.cell_path(cells[0]) == ospf_rib.PATH_INTER].astype(np.int64)
    slot_w = w[w >= bb.table.n_records] - bb.table.n_records
    assert len(slot_w) and (slot_w >> 8 < bb.table.n_slots).all() and ((slot_w & 0xFF) == ospfv3.PFX_LA).any()


# ------------------------------------------------------------------------------------------- refusals
def test_table_refusals():
    bb = Backbone("topo2-2", "rt1", ["rt4", "rt5"])
    d4, d5 = bb.doms
    mk = lambda borders, flat=bb.flat, rid=bb.area.router_id, sums=bb.summaries: ospf_rib.BackboneTable(flat, rid, sums, None, borders)

    def refused(code, *args, **kw):
        with pytest.raises(capi.HspfError) as e:
            mk(*args, **kw)
        assert e.value.code == code

    for borders in ([], [d4.rt] * 2, [d4.rt] * 9):
        refused(capi.HSPF_E_INVAL, borders)
    # R with the B flag, or R one of the borders: rt4 as R
    s4 = snap("topo2-2", "rt4")
    k4 = gu.global_sort_keys(s4)
    a4 = full_image(s4, next(a for a in s4["areas"] if a["area_id"] == "0.0.0.0"), k4)
    refused(capi.HSPF_E_INVAL, [d5.rt], flat=ospfv3.Flat(a4), rid=a4.router_id)
    # R missing from the flat
    refused(capi.HSPF_E_INVAL, [d4.rt, d5.rt], rid=0x0909FFFF)
    # a border table without area 0
    no0 = ospf_rib.AbrRibTable(d4.areas[1].router_id, [d4.flats[1]], [d4.areas[1].area_id], [d4.summaries[1]])
    refused(capi.HSPF_E_INVAL, [no0])
    # a border that is not a B-flag router of R's flat
    a = ospfv3.Ospfv3Area(**{k: getattr(bb.area, k) for k in bb.area.__dataclass_fields__})
    rl = a.router_lsas.copy()
    rl["flags"][rl["adv_rtr"] == d5.areas[0].router_id] &= ~np.uint8(1)
    a.router_lsas = rl
    refused(capi.HSPF_E_INVAL, [d4.rt, d5.rt], flat=ospfv3.Flat(a), rid=a.router_id)
    # a border Inter-Area-Prefix LSA for a prefix that is not one of its keys
    row = lambda adv, ty, opts=0, rid=0: np.array([(adv, 0x777, 5, rid, ospfv3.ip_rec("2001:db8:9999::"), 64, opts, ty, 0)],
                                                  ospf_rib.INTER_AREA_LSA_DT)
    srt = lambda x: x[np.lexsort((x["lsa_id"], x["adv_rtr"], x["lsa_type"]))]
    bad = srt(np.concatenate([bb.summaries, row(d4.areas[0].router_id, 3)]))
    refused(capi.HSPF_E_INVAL, [d4.rt, d5.rt], sums=bad)
    # ... which is fine from another ABR, with the NU option, or dead
    mk([d4.rt], sums=srt(np.concatenate([bb.summaries, row(d5.areas[0].router_id, 3)])))
    mk([d4.rt, d5.rt], sums=srt(np.concatenate([bb.summaries, row(d4.areas[0].router_id, 3, ospfv3.PFX_NU)])))
    dead = bad.copy()
    dead["maxage"][dead["lsa_id"] == 0x777] = 1
    mk([d4.rt, d5.rt], sums=dead)
    # an OSPFv2 border table
    import test_ospf_abr_rib_cells as v2abr
    d2 = v2abr.domain(0)
    assert not d2.rt.__dict__.get("v3")
    refused(capi.HSPF_E_INVAL, [d4.rt, d2.rt])
    # a usable Inter-Area-Router LSA from a border (one with the NU option too: NU leaves only prefixes out)
    for opts in (0, ospfv3.PFX_NU):
        refused(capi.HSPF_E_UNSUPPORTED, [d4.rt, d5.rt],
                sums=srt(np.concatenate([bb.summaries, row(d4.areas[0].router_id, 4, opts, 0x09090909)])))
    # a V-flag router in R's area 0
    a = ospfv3.Ospfv3Area(**{k: getattr(bb.area, k) for k in bb.area.__dataclass_fields__})
    rl = a.router_lsas.copy()
    rl["flags"][rl["adv_rtr"] == d4.areas[0].router_id] |= np.uint8(0x04)
    a.router_lsas = rl
    refused(capi.HSPF_E_UNSUPPORTED, [d4.rt, d5.rt], flat=ospfv3.Flat(a), rid=a.router_id)


def test_versions_do_not_mix():
    """The OSPFv2 create refuses OSPFv3 borders, each decode refuses the other version's table, and the IPv6 prefix
    call refuses an OSPFv2 table."""
    import test_ospf_backbone_cells as v2bb
    lib = capi.load_library()
    bb3 = Backbone("topo2-2", "rt1", ["rt4", "rt5"])
    bb2 = v2bb.Backbone("topo2-2", "rt1", ["rt4", "rt5"])
    with pytest.raises(capi.HspfError) as e:
        ospf_rib.BackboneTable(bb2.flat, bb2.area.router_id, bb2.summaries, None, [bb3.doms[0].rt])
    assert e.value.code == capi.HSPF_E_INVAL
    P3, P2 = bb3.table.n_prefixes, bb2.table.n_prefixes
    out = lambda dt: (np.zeros(64, dt), np.zeros(256, dt))
    r6, h6 = out(ospf_rib.RIB_ROUTE6_DT)[0], np.zeros(256, ospfv3.NEXTHOP6_DT)
    rs = ospf_rib.RibStruct(64, 0, r6.ctypes.data, 256, 0, h6.ctypes.data)
    c2 = np.zeros(P2, ospf_rib.RIB_CELL_DT)
    s3 = bb3.area.as_struct()
    assert lib.hspf_ospfv3_backbone_from_cells(bb2.table.handle, C.byref(s3), c2.ctypes.data, None, None, 0,
                                               C.byref(rs)) == capi.HSPF_E_INVAL
    c3 = np.zeros(P3, ospf_rib.RIB_CELL_DT)
    s2 = bb2.area.as_struct()
    r4 = np.zeros(64, ospf_rib.RIB_ROUTE_DT)
    rs2 = ospf_rib.RibStruct(64, 0, r4.ctypes.data, 0, 0, None)
    assert lib.hspf_ospfv2_backbone_from_cells(bb3.table.handle, C.byref(s2), c3.ctypes.data, None, None, 0,
                                               C.byref(rs2)) == capi.HSPF_E_INVAL
    assert lib.hspf_ospfv3_backbone_table_prefixes6(bb2.table.handle, None, None, None) == capi.HSPF_E_INVAL


def test_job_refusals(abr_harness, harness):
    bb = Backbone("topo2-2", "rt1", ["rt4", "rt5"])
    bp = bb.border_planes([bb.job_overrides((), 0)] * 3)
    cells, st, _ = bb.cells(abr_harness, harness, bp, status=[np.array([0, 0x1, 0], np.uint32), np.array([0, 0, 0x4], np.uint32)])
    assert list(st) == [0, 0x1, 0x4]
    assert (cells["winner"][0] != ospf_rib.NO_RECORD).any()
    for j in (1, 2):
        assert (cells["winner"][j] == ospf_rib.NO_RECORD).all() and not cells["mpf"][j].any()
    cells, st, _ = bb.cells(abr_harness, harness, bp, root_status=0x2)
    assert list(st) == [0x2] * 3 and (cells["winner"] == ospf_rib.NO_RECORD).all()


def test_decode_refusals(abr_harness, harness):
    bb = Backbone("topo2-2", "rt1", ["rt4", "rt5"])
    cells, _, _ = bb.cells(abr_harness, harness, bb.border_planes([bb.job_overrides((), 0)]))
    k = int(np.nonzero(ospf_rib.cell_path(cells[0]) == ospf_rib.PATH_INTER)[0][0])
    for w in (0xFFFFFFF0, bb.table.n_records + (bb.table.n_slots << 8)):      # past every slot
        bad = cells[0].copy()
        bad["winner"][k] = w
        with pytest.raises(capi.HspfError):
            bb.decode(bad)
    wrong = ospfv3.Ospfv3Area(**{k: getattr(bb.area, k) for k in bb.area.__dataclass_fields__})
    wrong.area_id = 1
    v, n = gather_for(bb.flat, bb.rv, bb.planes)
    with pytest.raises(capi.HspfError):
        ospf_rib.backbone_from_cells_v3(wrong, bb.table, cells[0], v, n)


# ------------------------------------------------------------------------------------------- generated domains
class SynthBackbone(Backbone):
    """ospfv3.backbone_view: R and three borders of one area (the first also in area 2), with an ASBR in area 0, an
    options-flip key and a prefix shared by areas 1 and 2."""

    def __init__(self, seed, V0=30, E0=90, V1=25, E1=70, max_paths=16):
        t0 = synth.random_topology(V0, E0, synth.SEED_BASE + 950 + 2 * seed, cost_choices=[5, 10, 20])
        t1 = synth.random_topology(V1, E1, synth.SEED_BASE + 951 + 2 * seed, cost_choices=[5, 10, 20])
        v = ospfv3.backbone_view(t0, t1, seed, max_paths=max_paths)
        self.view = v
        self.area, self.summaries, self.externals = v["r_area"], v["summaries0"], v["externals"]
        self.flat = ospfv3.Flat(self.area)
        self.rv = self.flat.router_vertex(self.area.router_id)
        self.doms = [v3abr.Domain(areas, sums, self.externals) for areas, _ids, sums in v["borders"]]
        self.cfgs = [[ospf_rib.area_config()] * len(d.areas) for d in self.doms]
        self.make_table()
        self.planes = planes_of(self.flat.csr, self.rv)

    def key_index(self, key):
        b = np.frombuffer(key[0], np.uint8)
        u = [i for i in range(self.table.n_prefixes)
             if (self.table.prefixes6[i]["bytes"] == b).all() and int(self.table.plen[i]) == key[1]]
        return u[0] if u else None


def synth_jobs(bb, n, seed):
    links = non_backbone_links(bb)
    rng = np.random.default_rng(seed)
    jobs = [bb.job_overrides((), 0)]
    for k in rng.choice(len(links), min(n, len(links)), replace=False):
        jobs.append(bb.job_overrides(links[int(k)], capi.COST_DISABLED))
        jobs.append(bb.job_overrides(links[int(k)], int(rng.choice([1, 40]))))
    return jobs


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_generated_domains_chain(abr_harness, harness, seed, narrow_planes):
    """Every job's decode equals the host chain on backbone_view domains, prefix options included."""
    bb = SynthBackbone(seed)
    cells, _ = bb.check(abr_harness, harness, synth_jobs(bb, 12, seed), narrow_planes)
    present = (ospf_rib.cell_flags(cells) & 1) != 0
    assert (present & (ospf_rib.cell_path(cells) == ospf_rib.PATH_INTER)).any()
    assert bb.key_index(bb.view["flip"]) is not None and bb.key_index(bb.view["shared"]) is not None


def flip_cells(bb, abr_harness, harness):
    """Job 0's cells and the border cells of a second job in which one border's route for the flip key moves, at its
    metric, to the other advertiser's record (other options): that border's cell for the key takes the other record
    as its winner, nothing else changes.  The border is the one whose slot R's route takes."""
    jobs = [bb.job_overrides((), 0)]
    bp = bb.border_planes(jobs)
    cells, _, bcells = bb.cells(abr_harness, harness, bp)
    key = np.frombuffer(bb.view["flip"][0], np.uint8)
    u = bb.key_index(bb.view["flip"])
    for b, d in enumerate(bb.doms):
        k = next(i for i in range(d.rt.n_prefixes) if (d.rt.prefixes6[i]["bytes"] == key).all() and d.rt.plen[i] == 128)
        w = int(bcells[b][0][k]["winner"])
        i1 = d.rt.area_ids.index(1)
        lo, hi = int(d.rt.off[i1, k]), int(d.rt.off[i1, k + 1])
        assert hi - lo == 2 and lo <= w < hi
        flipped = [c.copy() for c in bcells]
        flipped[b][0][k]["winner"] = lo + hi - 1 - w
        got, _ = bb.cells_from(harness, flipped)
        if got[0][u]["winner"] != cells[0][u]["winner"]:
            return cells, bcells, flipped, bp
    raise AssertionError("no border's slot carries R's route to the flip key")


@pytest.mark.parametrize("seed", range(3))
def test_options_flip_at_an_equal_metric_is_other(abr_harness, harness, seed):
    """The flip key's two area-1 records tie at the first border with other options.  A job whose border cell takes
    the other record, at the same metric and atoms, changes R's route only in its prefix options: R's winner changes,
    the route-delta stage reports OTHER, and the decode gives the new options."""
    bb = SynthBackbone(seed)
    cells, bcells, flipped, bp = flip_cells(bb, abr_harness, harness)
    u = bb.key_index(bb.view["flip"])
    got, _ = bb.cells_from(harness, [np.concatenate([a, b]) for a, b in zip(bcells, flipped)])
    assert got[0].tobytes() == cells[0].tobytes()
    a, b = got[0][u], got[1][u]
    assert ospf_rib.cell_path(a) == ospf_rib.PATH_INTER
    assert int(a["mpf"]) == int(b["mpf"]) and int(a["nh_mask"]) == int(b["nh_mask"]) and int(a["winner"]) != int(b["winner"])
    assert (got[0] != got[1]).sum() == 1
    jobs, recs, total = reference(got, got[:1])
    assert total == 1 and int(recs[0]["prefix"]) == u and int(recs[0]["kind"]) == DELTA_OTHER
    assert int(jobs[1]["n_changed"]) == 1
    r0, r1 = bb.decode(got[0]), bb.decode(got[1])
    o = lambda rib: {(x["prefix"].tobytes(), int(x["len"])): int(x["prefix_options"]) for x in rib.routes}
    k = (bb.view["flip"][0] + b"\x01\x00\x00\x00", 128)
    assert {o(r0)[k], o(r1)[k]} == {ospfv3.PFX_LA, ospfv3.PFX_P}
    # the chain agrees with both jobs
    both = [np.concatenate([x, y]) for x, y in zip(bcells, flipped)]
    for j in range(2):
        same_rib(bb.decode(got[j]), bb.host([c[j] for c in both], [q[0] for q in bp]))


def test_options_flip_by_a_topology_change(abr_harness, harness):
    """The same through the SPT: cutting every link of the flip key's first advertiser hands the first border's route
    to the other one at the same metric.  Where R's route to the key goes through the first border only, R's winner
    changes while its metric and next hops stay, and the delta reports OTHER."""
    n = 0
    for seed in range(3):
        bb = SynthBackbone(seed)
        d = bb.doms[0]
        i1 = d.rt.area_ids.index(1)
        f1, a1 = d.flats[i1], d.areas[i1]
        key = bb.view["flip"][0]
        advs = sorted(int(l["adv_rtr"]) for l in a1.iap_lsas
                      for p in a1.prefixes[int(l["prefix_off"]): int(l["prefix_off"]) + int(l["n_prefixes"])]
                      if bytes(int(b) for b in p["addr"]["bytes"]) == key)
        first = advs[0]
        links = [l for l in non_backbone_links(bb) if any(x[0] == first and x[2] for x in l)]
        ovs = [bb.job_overrides(l, capi.COST_DISABLED) for l in links]
        merged = [{i: sum((o[b].get(i, []) for o in ovs), []) for i in range(len(bb.doms[b].areas))}
                  for b in range(len(bb.doms))]
        merged = [{i: e for i, e in m.items() if e} for m in merged]
        cells, _ = bb.check(abr_harness, harness, [bb.job_overrides((), 0), merged])
        u = bb.key_index(bb.view["flip"])
        a, b = cells[0][u], cells[1][u]
        if int(a["mpf"]) == int(b["mpf"]) and int(a["nh_mask"]) == int(b["nh_mask"]) and a["winner"] != b["winner"]:
            jobs, recs, _ = reference(cells, cells[:1])
            assert any(int(r["prefix"]) == u and int(r["kind"]) == DELTA_OTHER for r in recs if int(r["job"]) == 1)
            n += 1
    assert n > 0


def test_shared_prefix_keeps_the_first_areas_options(abr_harness, harness):
    """backbone_view's shared /64 is intra-area in areas 1 (LA) and 2 (P) of the first border at one metric: the
    border's route, and so R's, carries area 1's options (area 1 is the border's first area)."""
    for seed in range(3):
        bb = SynthBackbone(seed)
        cells, _ = bb.check(abr_harness, harness, [bb.job_overrides((), 0)])
        got = bb.decode(cells[0])
        key = (bb.view["shared"][0], 64)
        r = [x for x in got.routes if (x["prefix"].tobytes()[:16], int(x["len"])) == key]
        assert len(r) == 1 and int(r[0]["prefix_options"]) == ospfv3.PFX_LA and r[0]["path_type"] == ospf_rib.PATH_INTER


def test_nu_option_lsas_are_left_out():
    """An Inter-Area-Prefix LSA with the NU option from a border builds the same table as no LSA at all."""
    bb = SynthBackbone(0)
    s = bb.summaries.copy()
    assert len(s)
    nu = s.copy()
    nu["prefix_options"][0] |= ospfv3.PFX_NU
    t = ospf_rib.BackboneTable(bb.flat, bb.area.router_id, nu, bb.externals, [d.rt for d in bb.doms])
    t0 = ospf_rib.BackboneTable(bb.flat, bb.area.router_id, s[1:], bb.externals, [d.rt for d in bb.doms])
    assert (t.n_prefixes, t.n_records, t.n_slots) == (t0.n_prefixes, t0.n_records, t0.n_slots)
    assert t.prefixes6.tobytes() == t0.prefixes6.tobytes()
