"""CPU: the OSPFv3 area-border-router stage over what-if jobs inside an area the router is not attached to
(hspf_ospfv3_abr_backbone_*, abr_rib_cell_eval with kSlots over AbrBorderSlots<true>).

The walk is compiled into a test harness and run on the CPU over the oracle's SPT planes: R's row 0 of each of its
areas, each border's routing-table cells of the job and each border's area planes of the job, which the
Inter-Area-Router slots read.  Every job, decoded by hspf_ospfv3_abr_backbone_from_cells, must equal, prefix options
included, the host chain: each border's update_rib_full_v3 over its job planes, its net_summaries_v3 and
rtr_summaries_v3 into area 0 spliced into area 0's LSAs in LsaKey order in place of its own, then update_rib_full_v3 at
R over its areas' row-0 images, restricted to the affected prefixes."""
import ctypes as C
import ipaddress
import subprocess
import types
from pathlib import Path

import numpy as np
import pytest

import golden_util as gu
import test_ospfv3_abr_rib_cells as v3abr
from holo_b200 import capi, ospf_rib, ospfv3, synth
from holo_b200.route_table import DELTA_OTHER
from test_ospf_abr_backbone_cells import abr_backbone_cells
from test_ospf_abr_rib_cells import harness as abr_harness  # noqa: F401  (fixture)
from test_ospf_abr_rib_cells import planes_of
from test_ospf_backbone_asbr_cells import ext_path
from test_ospf_rib_cells import same_rib
from test_ospf_rib_delta import classify, reference
from test_ospfv2_route_cells import gather_for
from test_ospfv3_backbone_cells import Backbone, configs_of, golden_domain, non_backbone_links, snap, synth_jobs
from test_ospfv3_nonbackbone_cells import job_rib_areas, srt
from test_ospfv3_rib_cells import rib_dict

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    """The OSPFv3 walk, under the names abr_backbone_cells calls (its arguments are the OSPFv2 harness's)."""
    out = tmp_path_factory.mktemp("harness") / "libospfv3_abr_backbone_cells_harness.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-comment", "-I", str(ROOT / "include"),
                    "-o", str(out), str(ROOT / "tests" / "native" / "ospfv3_abr_backbone_cells_harness.cc")],
                   check=True)
    lib = C.CDLL(str(out))
    for fn in (lib.harness_ospfv3_abr_backbone_cells, lib.harness_ospfv3_abr_backbone_cells16):
        fn.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 12
        fn.restype = C.c_int
    lib.harness_abr_backbone_winners_fit.argtypes = [C.c_uint64, C.c_uint64, C.c_int]
    return types.SimpleNamespace(lib=lib, harness_ospf_abr_backbone_cells=lib.harness_ospfv3_abr_backbone_cells,
                                 harness_ospf_abr_backbone_cells16=lib.harness_ospfv3_abr_backbone_cells16)


def present(cells):
    return (ospf_rib.cell_flags(cells) & 1) != 0


class AbrBackbone(Backbone):
    """R's domain (its OSPFv3 areas, their LSAs and active flags), the borders' domains (each border's areas in its own
    order) and the table over them.  cut_border: R's area-0 row 0 with that border's area-0 links cut."""

    def __init__(self, r_dom, doms, cfgs=None, cut_border=None, keys=None):
        self.r, self.doms, self.keys = r_dom, doms, keys
        self.cfgs = cfgs if cfgs is not None else [[ospf_rib.area_config()] * len(d.areas) for d in doms]
        self.externals = r_dom.externals
        self.i0 = [a.area_id for a in r_dom.areas].index(0)
        self.table = self.table_of()
        self.planes = r_dom.planes()
        if cut_border is not None:
            f = r_dom.flats[self.i0]
            b, c = f.router_vertex(doms[cut_border].areas[0].router_id), f.csr
            ov = [(e, capi.COST_DISABLED) for e in range(c.n_edges) if c.col[e] == b or c.row_ptr[b] <= e < c.row_ptr[b + 1]]
            self.planes[self.i0] = planes_of(f.csr, r_dom.rv[self.i0], ov)

    def table_of(self, doms=None, summaries=None, flats=None, area_ids=None, active=None, router_id=None):
        r = self.r
        return ospf_rib.AbrBackboneTable(r.areas[0].router_id if router_id is None else router_id,
                                         r.flats if flats is None else flats,
                                         [a.area_id for a in r.areas] if area_ids is None else area_ids,
                                         r.summaries if summaries is None else summaries,
                                         r.active if active is None else active, r.externals,
                                         [d.rt for d in (self.doms if doms is None else doms)])

    def cells(self, abr, harness, bplanes, narrow_planes=False, **kw):
        bcells = [np.stack([d.cells(abr, p, narrow_planes)[0] for p in bp]) for d, bp in zip(self.doms, bplanes)]
        cells, out = abr_backbone_cells(harness, self.table, self.planes, bcells, bplanes, narrow_planes, **kw)
        return cells, out, bcells

    def decode(self, cells):
        ga, gv, gn = [], [], []
        for i, (f, r, p) in enumerate(zip(self.r.flats, self.r.rv, self.planes)):
            v, n = gather_for(f, r, p)
            ga += [i] * len(v); gv += list(v); gn += list(n)
        return ospf_rib.abr_backbone_from_cells_v3(self.r.areas, self.table, cells, ga, gv, gn)

    def lsdb(self, bplanes_of_job):
        """Area 0's LSDB of the job: each border's Inter-Area-Prefix / Inter-Area-Router LSAs re-originated."""
        bid = {d.areas[0].router_id for d in self.doms}
        new = [tuple(s) for s in self.r.summaries[self.i0].tolist() if int(s[0]) not in bid]
        for d, cfg, p in zip(self.doms, self.cfgs, bplanes_of_job):
            i0 = [a.area_id for a in d.areas].index(0)
            new += ospfv3.nonbackbone_lsas(d.areas[0].router_id, d.areas[0].max_paths, job_rib_areas(d, p),
                                           self.externals, i0, cfg)
        return srt(np.array(new, ospf_rib.INTER_AREA_LSA_DT))

    def host(self, bplanes_of_job):
        s0 = self.lsdb(bplanes_of_job)
        ra = []
        for i, (a, p) in enumerate(zip(self.r.areas, self.planes)):
            spf = ospfv3.area_from_planes(a, lambda csr, root, nhw, p=p: (p[0], p[1], np.pad(p[2][:, None], ((0, 0), (0, nhw - 1)))))
            ra.append(ospf_rib.RibArea(a.area_id, spf, a.ifaces, s0 if i == self.i0 else self.r.summaries[i],
                                       self.r.active[i]))
        r0 = self.r.areas[0]
        return self.affected(ospf_rib.update_rib_full_v3(r0.router_id, r0.max_paths, ra, self.externals))

    def check(self, abr, harness, jobs, narrow_planes=False):
        bp = self.border_planes(jobs)
        cells, st, _ = self.cells(abr, harness, bp, narrow_planes)
        assert not st.any()
        for j in range(len(jobs)):
            same_rib(self.decode(cells[j]), self.host([bp[b][j] for b in range(len(self.doms))]))
        return cells

    def key_index(self, key):
        b = np.frombuffer(key[0], np.uint8)
        u = [i for i in range(self.table.n_prefixes)
             if (self.table.prefixes6[i]["bytes"] == b).all() and int(self.table.plen[i]) == key[1]]
        return u[0] if u else None


class SynthAbrBackbone(AbrBackbone):
    """ospfv3.abr_backbone_view: R an ABR of areas 0 and 3, three borders of area 1 (those in `use`), k area-1
    ASBRs."""

    def __init__(self, seed, k=2, n_ext=4, use=(0, 1, 2), cut_border=None, max_paths=16):
        t0 = synth.random_topology(30, 90, synth.SEED_BASE + 950 + 3 * seed, cost_choices=[5, 10, 20])
        t1 = synth.random_topology(25, 70, synth.SEED_BASE + 951 + 3 * seed, cost_choices=[5, 10, 20])
        t2 = synth.random_topology(25, 70, synth.SEED_BASE + 952 + 3 * seed, cost_choices=[5, 10, 20])
        v = ospfv3.abr_backbone_view(t0, t1, t2, seed, max_paths=max_paths, area1_asbrs=k, area1_ext=n_ext)
        self.view = v
        r_dom = v3abr.Domain(v["r_areas"], v["summaries"], v["externals"])
        doms = [v3abr.Domain(areas, sums, v["externals"]) for b, (areas, _ids, sums) in enumerate(v["borders"])
                if b in use]
        super().__init__(r_dom, doms, cut_border=cut_border)

    def cut(self, x, borders=None):
        """A job: every area-1 link of router x disabled in the area planes of the borders in `borders` (all: None)."""
        ovs = [self.job_overrides(l, capi.COST_DISABLED) for l in non_backbone_links(self) if any(y[0] == x and y[2] for y in l)]
        return [{} if borders is not None and b not in borders else
                {i: e for i in range(len(d.areas)) if (e := sum((o[b].get(i, []) for o in ovs), []))}
                for b, d in enumerate(self.doms)]

    def ext_keys(self, x):
        e = self.externals[self.externals["adv_rtr"] == x]
        want = {(y["prefix"]["bytes"].tobytes(), int(y["len"])) for y in e}
        return [u for u in range(self.table.n_prefixes)
                if (self.table.prefixes6[u]["bytes"].tobytes(), int(self.table.plen[u])) in want]


# ------------------------------------------------------------------------------------------------ goldens
# topo1-1/1-2: each ABR among rt2, rt4 and rt6 as R, each other one as the single border of its area
GOLDEN = [(t, r, b) for t in ("topo1-1", "topo1-2") for r in ("rt2", "rt4", "rt6") for b in ("rt2", "rt4", "rt6")
          if b != r]
GIDS = [f"{t}-{r}-{b}" for t, r, b in GOLDEN]


def golden(topo, r, b):
    rs, bs = snap(topo, r), snap(topo, b)
    r_dom, keys = golden_domain(rs)
    bdom = golden_domain(bs)[0]
    return AbrBackbone(r_dom, [bdom], [configs_of(bs, bdom)], keys=keys), rs


@pytest.mark.parametrize("g", GOLDEN, ids=GIDS)
def test_base_job_equals_the_recorded_local_rib(abr_harness, harness, g):
    """Job 0 equals R's recorded local-rib, restricted to the affected prefixes: metric, route type and next hops,
    and the chain's prefix options."""
    bb, rs = golden(*g)
    assert bb.table.v3 and bb.table.n_prefixes > 0 and bb.table.n_slots > 0
    cells = bb.check(abr_harness, harness, [bb.job_overrides((), 0)])
    mine = rib_dict(bb.decode(cells[0]), {v: k for k, v in bb.keys.items()})
    affected = {f"{ospfv3.ip_str(p)}/{int(l)}" for p, l in zip(bb.table.prefixes6, bb.table.plen)}
    want = {k: v for k, v in gu.golden_rib(rs).items() if k in affected}
    norm = lambda d: {k: (v[0], v[1], [(a or "", b or "") for a, b in v[2]]) for k, v in d.items()}
    assert norm(mine) == norm(want)


@pytest.mark.parametrize("g", GOLDEN, ids=GIDS)
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_golden_chain_every_link_failed_and_recosted(abr_harness, harness, g, narrow_planes):
    bb, _ = golden(*g)
    jobs = [bb.job_overrides((), 0)]
    for link in non_backbone_links(bb):
        jobs += [bb.job_overrides(link, capi.COST_DISABLED), bb.job_overrides(link, 35)]
    assert len(jobs) > 1
    bb.check(abr_harness, harness, jobs, narrow_planes)


# ------------------------------------------------------------------------------------------- generated
@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("narrow_planes", [False, True], ids=["wide", "narrow"])
def test_generated_domains_chain(abr_harness, harness, seed, narrow_planes):
    """Every area-1 link failed and re-costed, one job each, all in one batch."""
    bb = SynthAbrBackbone(seed)
    assert bb.table.n_asbr_slots > 0 and 1 <= bb.table.n_asbr_sets <= 3
    jobs = [bb.job_overrides((), 0)]
    for link in non_backbone_links(bb):
        jobs += [bb.job_overrides(link, capi.COST_DISABLED), bb.job_overrides(link, 37)]
    cells = bb.check(abr_harness, harness, jobs, narrow_planes)
    assert (cells != cells[0]).any()
    assert bb.key_index(bb.view["flip"]) is not None


def test_option_flip_at_an_equal_metric_is_other(abr_harness, harness):
    """abr_backbone_view's flip /128: cutting the links of its lower-id advertiser hands the first border's route to
    the other advertiser's record at the same metric, with the other option (LA / P).  Where R's route stays at its
    metric and next hops, R's winner changes, the delta reports OTHER and the decode gives the other option."""
    n = 0
    for seed in range(4):
        bb = SynthAbrBackbone(seed)
        key = bb.view["flip"]
        a1 = next(a for a in bb.doms[0].areas if a.area_id == 1)
        advs = sorted(int(l["adv_rtr"]) for l in a1.iap_lsas
                      for p in a1.prefixes[int(l["prefix_off"]): int(l["prefix_off"]) + int(l["n_prefixes"])]
                      if bytes(int(b) for b in p["addr"]["bytes"]) == key[0])
        cells = bb.check(abr_harness, harness, [bb.job_overrides((), 0), bb.cut(advs[0])])
        u = bb.key_index(key)
        a, b = cells[0][u], cells[1][u]
        assert ospf_rib.cell_path(a) == ospf_rib.PATH_INTER and int(a["winner"]) >= bb.table.n_records
        if int(a["mpf"]) == int(b["mpf"]) and int(a["nh_mask"]) == int(b["nh_mask"]) and a["winner"] != b["winner"]:
            _, recs, _ = reference(cells, cells[:1])
            assert [int(r["kind"]) for r in recs if int(r["job"]) == 1 and int(r["prefix"]) == u] == [DELTA_OTHER]
            o = lambda rib: {(x["prefix"].tobytes()[:16], int(x["len"])): int(x["prefix_options"]) for x in rib.routes}
            assert {o(bb.decode(cells[0]))[key], o(bb.decode(cells[1]))[key]} == {ospfv3.PFX_LA, ospfv3.PFX_P}
            n += 1
    assert n > 0


def test_tied_borders_merge_atoms(abr_harness, harness):
    """Some inter-area route reaches R through two borders at one metric: its cell ORs their atoms."""
    n = 0
    for seed in range(3):
        bb = SynthAbrBackbone(seed)
        cells = bb.check(abr_harness, harness, synth_jobs(bb, 6, seed))
        inter = present(cells) & (ospf_rib.cell_path(cells) == ospf_rib.PATH_INTER)
        multi = np.vectorize(lambda m: bin(int(m)).count("1") > 1)(cells["nh_mask"])
        n += int((inter & multi & (cells["winner"] >= bb.table.n_records)).sum())
    assert n > 0


def test_lost_then_gained(abr_harness, harness):
    """A link cut that strands area-1 prefixes at every border makes them unreachable at R (LOST); the next job,
    unperturbed, has them back (GAINED)."""
    lost = 0
    for seed in range(3):
        bb = SynthAbrBackbone(seed)
        jobs = [bb.job_overrides((), 0)]
        for link in non_backbone_links(bb):
            jobs += [bb.job_overrides(link, capi.COST_DISABLED), bb.job_overrides((), 0)]
        cells = bb.check(abr_harness, harness, jobs)
        for j in range(1, len(jobs), 2):
            k = classify(cells[j], cells[0])
            if (k == 1).any():
                lost += 1
                assert (classify(cells[j + 1], cells[j])[k == 1] == 2).all()
    assert lost > 0


def test_externals_through_area1_asbrs_and_the_area3_asbr(abr_harness, harness):
    """The area-0 ASBR's own /64 is also advertised by each area-1 ASBR and by the area-3 ASBR, whose intra-area entry
    in area 3 keeps it routed in every job; the area-3 ASBR's own /64 is not affected.  Cutting an area-1 ASBR off from
    the last border in LsaKey order moves R's entry to an earlier border's Inter-Area-Router slot."""
    moved = 0
    six = lambda hi: ipaddress.IPv6Address((0x20010DB8 << 96) | (hi << 64)).packed
    for seed in range(3):
        bb = SynthAbrBackbone(seed)
        assert bb.key_index(bb.view["area3_ext"]) is None
        u = bb.key_index((six(0xE0_0000), 64))
        last = max(range(3), key=lambda b: bb.doms[b].areas[0].router_id)
        jobs = [bb.job_overrides((), 0)] + [bb.cut(x, {last}) for x in bb.view["area1_asbrs"]]
        jobs += synth_jobs(bb, 6, seed)[1:]
        cells = bb.check(abr_harness, harness, jobs)
        assert ext_path(cells[:, u]).all()
        for j, x in enumerate(bb.view["area1_asbrs"], start=1):
            us = [k for k in bb.ext_keys(x) if ext_path(cells[0][k:k + 1])[0]]
            moved += int(cells[j][us].tobytes() != cells[0][us].tobytes())
    assert moved > 0


def test_area3_intra_prefix_never_changes(abr_harness, harness):
    """A prefix the borders advertise into area 0 that is also an area-3 router's: affected, intra-area at R, the
    same cell in every job."""
    for seed in range(3):
        bb = SynthAbrBackbone(seed)
        u = bb.key_index(bb.view["area3_shared"])
        cells = bb.check(abr_harness, harness, synth_jobs(bb, 8, seed))
        assert ospf_rib.cell_path(cells[0][u:u + 1])[0] == ospf_rib.PATH_INTRA and present(cells[0][u:u + 1])[0]
        assert (cells[:, u] == cells[0, u]).all()


def test_border_unreachable_from_r(abr_harness, harness):
    """A border R cannot reach in area 0: its slots offer nothing, whatever its cells; the other borders' still do."""
    for seed in range(2):
        bb = SynthAbrBackbone(seed, cut_border=1)
        bb.check(abr_harness, harness, synth_jobs(bb, 6, seed))


def iap_row(adv, key, opts=0):
    return np.array([(adv, 0x777, 5, 0, ospfv3.ip_rec(key[0]), key[1], opts, 3, 0)], ospf_rib.INTER_AREA_LSA_DT)


def iar_row(adv, rid):
    return np.array([(adv, 0x778, 5, rid, ospfv3.ip_rec("::"), 0, 0, 4, 0)], ospf_rib.INTER_AREA_LSA_DT)


def test_nu_option_lsa_of_a_border_is_left_out(abr_harness, harness):
    """A border's Inter-Area-Prefix LSA with the NU option is left out: one for a prefix the border cannot advertise
    builds the table of the LSDB without it (without NU it is refused), and NU on one of its usable LSAs builds the
    table of the LSDB without that LSA."""
    bb = SynthAbrBackbone(0)
    s0 = bb.r.summaries[0]
    b0 = bb.doms[0].areas[0].router_id
    bogus = (bytes(16)[:15] + b"\x09", 128)
    sums = lambda s: [s, bb.r.summaries[1]]
    t = bb.table_of(summaries=sums(srt(np.concatenate([s0, iap_row(b0, bogus, ospfv3.PFX_NU)]))))
    assert (t.n_prefixes, t.n_records, t.n_slots) == (bb.table.n_prefixes, bb.table.n_records, bb.table.n_slots)
    with pytest.raises(capi.HspfError) as e:
        bb.table_of(summaries=sums(srt(np.concatenate([s0, iap_row(b0, bogus)]))))
    assert e.value.code == capi.HSPF_E_INVAL
    k = int(np.nonzero((s0["adv_rtr"] == b0) & (s0["lsa_type"] == 3))[0][0])
    nu = s0.copy()
    nu["prefix_options"][k] |= ospfv3.PFX_NU
    t = bb.table_of(summaries=sums(nu))
    assert t.prefixes6.tobytes() == bb.table.prefixes6.tobytes() and t.n_records == bb.table.n_records
    bb.table = t
    bb.check(abr_harness, harness, synth_jobs(bb, 4, 0))


# -------------------------------------------------------------------------------------------- refusals
def refused(code, fn):
    with pytest.raises(capi.HspfError) as e:
        fn()
    assert e.value.code == code


def with_b_cleared(a, rid):
    a = ospfv3.Ospfv3Area(**{k: getattr(a, k) for k in a.__dataclass_fields__})
    rl = a.router_lsas.copy()
    rl["flags"][rl["adv_rtr"] == rid] &= np.uint8(0xFE)
    a.router_lsas = rl
    return a


def with_flags(a, rid, bits):
    a = ospfv3.Ospfv3Area(**{k: getattr(a, k) for k in a.__dataclass_fields__})
    rl = a.router_lsas.copy()
    rl["flags"][rl["adv_rtr"] == rid] |= bits
    a.router_lsas = rl
    return a


def test_table_refusals():
    bb = SynthAbrBackbone(0)
    r = bb.r
    rid = r.areas[0].router_id
    refused(capi.HSPF_E_INVAL, lambda: bb.table_of(doms=[]))                          # no border
    refused(capi.HSPF_E_INVAL, lambda: bb.table_of(doms=[bb.doms[0]] * 2))           # a border twice
    refused(capi.HSPF_E_INVAL, lambda: bb.table_of(doms=[bb.doms[0]] * 9))           # more than 8 borders
    refused(capi.HSPF_E_INVAL, lambda: bb.table_of(area_ids=[5, 3]))                  # no area 0
    refused(capi.HSPF_E_INVAL, lambda: bb.table_of(active=[False, True]))             # area 0 inactive
    refused(capi.HSPF_E_INVAL, lambda: bb.table_of(active=[True, False]))             # one active area
    refused(capi.HSPF_E_INVAL,                                                        # R without the B flag
            lambda: bb.table_of(flats=[ospfv3.Flat(with_b_cleared(r.areas[0], rid)), r.flats[1]]))
    refused(capi.HSPF_E_INVAL, lambda: bb.table_of(doms=[bb.doms[0], r]))             # R one of the borders
    import test_ospf_abr_rib_cells as v2abr
    refused(capi.HSPF_E_INVAL, lambda: bb.table_of(doms=[bb.doms[0], v2abr.domain(0)]))   # an OSPFv2 border table
    # a border's Inter-Area-Prefix LSA for a prefix it cannot advertise, an Inter-Area-Router LSA for a router it
    # cannot originate for
    b0 = bb.doms[0].areas[0].router_id
    for row in (iap_row(b0, (bytes(15) + b"\x09", 128)), iar_row(b0, 0x09090909)):
        refused(capi.HSPF_E_INVAL,
                lambda: bb.table_of(summaries=[srt(np.concatenate([r.summaries[0], row])), r.summaries[1]]))
    # a V-flag router in R's area 3 (the transit-area step)
    a3 = with_flags(r.areas[1], bb.view["area3_asbr"], 0x04)
    refused(capi.HSPF_E_UNSUPPORTED, lambda: bb.table_of(flats=[r.flats[0], ospfv3.Flat(a3)]))
    # an E-flag router of a border's area with the B flag
    x = bb.view["area1_asbrs"][0]
    doms = [v3abr.Domain([with_flags(a, x, 0x01) if a.area_id != 0 else a for a in d.areas], d.summaries, d.externals)
            for d in bb.doms]
    refused(capi.HSPF_E_UNSUPPORTED, lambda: bb.table_of(doms=doms))


def test_more_than_8_plane_sets_are_refused():
    """Every Inter-Area-Router slot of a border reads the plane set of its (border, area): 4 + 2 + 2 sets build,
    4 + 2 + 3 are refused."""
    from test_ospfv3_backbone_asbr_cells import with_twins
    bb = SynthAbrBackbone(0)
    d0, d1, d2 = bb.doms
    t = bb.table_of(doms=[with_twins(d0, 3), with_twins(d1, 1), with_twins(d2, 1)])
    assert t.n_asbr_sets == 8 and t.n_asbr_slots > bb.table.n_asbr_slots
    refused(capi.HSPF_E_UNSUPPORTED, lambda: bb.table_of(doms=[with_twins(d0, 3), with_twins(d1, 1), with_twins(d2, 2)]))


def test_slot_winners_must_fit_32_bits(harness):
    """A table whose slot winners would not fit 32 bits is refused (HSPF_E_UNSUPPORTED).  A real one needs about 2^24
    OSPFv3 slots, so the rule the create applies with the OSPFv3 encoding is checked at its boundary: n_records +
    (slots << 8) must stay below 0xFFFFFFFF."""
    fit = harness.lib.harness_abr_backbone_winners_fit
    S = 0xFFFFFF
    assert fit(0xFE, S, 1) == 1 and fit(0xFF, S, 1) == 0 and fit(0, S + 1, 1) == 0
    assert fit(0xFF, S, 0) == 1
    bb = SynthAbrBackbone(0)
    assert fit(bb.table.n_records, bb.table.n_slots, 1) == 1


def test_versions_do_not_mix(abr_harness, harness):
    """Each version's create and decode refuse the other version's tables, and the OSPFv3 prefixes call refuses an
    OSPFv2 table."""
    import test_ospf_abr_backbone_cells as v2t
    bb = SynthAbrBackbone(0)
    v2 = v2t.SynthAbrBackbone(0)
    # the OSPFv2 create over OSPFv3 border tables, the OSPFv3 create over OSPFv2 ones
    refused(capi.HSPF_E_INVAL, lambda: ospf_rib.AbrBackboneTable(
        v2.r.areas[0].router_id, v2.r.flats, [a.area_id for a in v2.r.areas], v2.r.summaries, v2.r.active,
        v2.r.externals, [d.rt for d in bb.doms]))
    refused(capi.HSPF_E_INVAL, lambda: bb.table_of(doms=[v2t.SynthAbrBackbone(0).doms[0]]))
    cells, _, _ = bb.cells(abr_harness, harness, bb.border_planes([bb.job_overrides((), 0)]))
    ga, gv, gn = [], [], []
    refused(capi.HSPF_E_INVAL, lambda: ospf_rib.abr_backbone_from_cells(v2.r.areas, bb.table, cells[0], ga, gv, gn))
    v2cells = np.zeros(v2.table.n_prefixes, ospf_rib.RIB_CELL_DT)
    refused(capi.HSPF_E_INVAL, lambda: ospf_rib.abr_backbone_from_cells_v3(bb.r.areas, v2.table, v2cells, ga, gv, gn))
    p6 = C.c_void_p()
    assert v2.table.lib.hspf_ospfv3_abr_backbone_table_prefixes6(v2.table.handle, None, C.byref(p6), None) == \
        capi.HSPF_E_INVAL
    # the OSPFv3 walk's harness refuses an OSPFv2 table, as the device calls pick the walk from the mark
    assert harness.lib.harness_ospfv3_abr_backbone_cells(v2.table.handle, 0, *([None] * 12)) == -1


def test_job_status_rows(abr_harness, harness):
    """R's row-0 words, the borders' job words and the Inter-Area-Router rows' words are ORed into a job's word, a row
    out of range gives HSPF_JS_INVALID, and a refused job gets empty cells; the other jobs are unchanged."""
    bb = SynthAbrBackbone(1)
    jobs = synth_jobs(bb, 3, 1)
    bp = bb.border_planes(jobs)
    want, st, bcells = bb.cells(abr_harness, harness, bp)
    assert not st.any()
    J = len(jobs)
    rows = [np.repeat(np.arange(J, dtype=np.uint32)[:, None], len(d.areas), 1) for d in bb.doms]
    rows[1][2, :] = J                                                    # out of range
    ps = [[np.zeros(J, np.uint32) for _ in d.areas] for d in bb.doms]
    for i in range(len(bb.doms[0].areas)):
        ps[0][i][1] = 0x8
    bst = [np.zeros(J, np.uint32) for _ in bb.doms]
    bst[2][3] = 0x2
    got, st = abr_backbone_cells(harness, bb.table, bb.planes, bcells, bp, status=bst, rows=rows, pstatus=ps)
    assert st[2] & capi.JS_INVALID and st[1] == 0x8 and st[3] == 0x2
    for j in (1, 2, 3):
        assert (got["winner"][j] == ospf_rib.NO_RECORD).all() and not got["mpf"][j].any()
    keep = [j for j in range(J) if j not in (1, 2, 3)]
    assert got[keep].tobytes() == want[keep].tobytes()
    got, st = abr_backbone_cells(harness, bb.table, bb.planes, bcells, bp, root_status=[0, 0x4])
    assert (st == 0x4).all() and (got["winner"] == ospf_rib.NO_RECORD).all()
