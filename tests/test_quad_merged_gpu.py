"""Which phase-3 algorithm spf_quad_kernel runs, and that both agree with the oracle: jobs with at most
12 first-hop atoms whose ECMP vertices fit the layout's list run the merged hops / next-hop pass; jobs
with more ECMP vertices (unit costs), more atoms (a hub root) or a hop sum that overflows its share of
the aggregate (12 atoms and a 20-router chain) run the hop pass and the next-hop passes.
Phase-profile slot 13 counts rounds of the hop pass, which only the two-pass code runs."""
import ctypes as C

import numpy as np
import pytest

from holo_b200 import synth
from oracle import pyoracle

pytestmark = pytest.mark.gpu

PLANES = ["dist", "hops", "first_parent", "n_parents", "nh_mask"]


def run_profiled(ctx, csr, roots):
    g = ctx.upload(csr)
    ctx.lib.hspf_debug_phase_profile(ctx.handle, 1, None)
    try:
        res = ctx.run(g, np.asarray(roots, np.uint32))
    finally:
        out = (C.c_uint64 * 16)()
        ctx.lib.hspf_debug_phase_profile(ctx.handle, 0, out)
    g.free()
    for j, r in enumerate(roots):
        ref = pyoracle.csr_spf(csr, int(r))
        assert res.job_status[j] == ref["status"] == 0
        for k in PLANES:
            assert np.array_equal(getattr(res, k)[j], ref[k]), (int(r), k)
    return list(out)


def degree(csr, v):
    return int(csr.row_ptr[v + 1] - csr.row_ptr[v])


def test_c2_shape_runs_the_merged_pass(ctx):
    csr = synth.topology_csr(synth.random_topology(10000, 40000, synth.SEED_BASE + 2))
    roots = [r for r in range(0, 10000, 500) if degree(csr, r) <= 12]
    assert len(roots) >= 16
    prof = run_profiled(ctx, csr, roots)
    assert prof[13] == 0 and prof[14] > 0


def test_more_ecmp_vertices_than_the_list_holds_run_two_passes(ctx):
    csr = synth.topology_csr(synth.random_topology(20000, 80000, synth.SEED_BASE + 2, cost_choices=[1]))
    roots = [0, 4321, 19999]
    n_e = [int((pyoracle.csr_spf(csr, r)["n_parents"] >= 2).sum()) for r in roots]
    assert min(n_e) > 6500          # the merged list holds 6 464 entries at this size
    prof = run_profiled(ctx, csr, roots)
    assert prof[13] > 0


def hub_graph(leaves, chain):
    """1 990 routers at the C2 density (small enough for one 2 048-word jump pass, large enough for the
    merged layout), then a chain of `chain` routers below router 0 and `leaves` more routers on it."""
    t = synth.random_topology(1990, 4 * 1990, synth.SEED_BASE + 3)
    R = 1990 + chain + leaves
    a = [0] + list(range(1990, 1990 + chain - 1)) + [0] * leaves
    b = list(range(1990, 1990 + chain)) + list(range(1990 + chain, R))
    c = np.full(len(a), 3, np.uint32)
    return synth.topology_csr(synth.Topology(R, np.concatenate([t.p2p_a, np.asarray(a, np.uint32)]),
                                             np.concatenate([t.p2p_b, np.asarray(b, np.uint32)]),
                                             np.concatenate([t.p2p_cost_ab, c]), np.concatenate([t.p2p_cost_ba, c]), []))


def test_more_than_12_atoms_run_two_passes(ctx):
    csr = hub_graph(leaves=16, chain=2)
    assert degree(csr, 0) > 12 and degree(csr, 1989) <= 12
    assert run_profiled(ctx, csr, [0])[13] > 0
    assert run_profiled(ctx, csr, [1989])[13] == 0


def test_hop_sum_overflow_runs_two_passes(ctx):
    base = degree(hub_graph(leaves=0, chain=20), 0)
    csr = hub_graph(leaves=12 - base, chain=20)          # 12 atoms: 4 bits of hop sum, 20 routers in a row
    assert degree(csr, 0) == 12
    assert run_profiled(ctx, csr, [0])[13] > 0
    assert run_profiled(ctx, csr, [1989])[13] == 0
