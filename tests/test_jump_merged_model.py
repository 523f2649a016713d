"""CPU check of the merged hops / next-hop pointer-jumping pass of spf_quad_kernel (modelled step by
step in tests/jump_merged_model.py) against the reference-faithful oracle: LANs, ECMP ladders,
parallel links, unreached vertices, hops-0 vertices below a HOP vertex, and the jobs that run the
two-pass algorithm instead (more than 16 first-hop atoms, more ECMP vertices than the list holds)."""
import numpy as np
import pytest

from holo_b200 import synth
from holo_b200.capi import VF_HOP, Csr
from oracle import pyoracle

from jump_merged_model import merged_jump_phase
from jump_model import jump_phase

SHAPES = [
    dict(V=12, E=40, kw=dict(cost_choices=[1])),
    dict(V=30, E=100, kw=dict(cost_choices=[5])),
    dict(V=40, E=120, kw=dict(cost_choices=[10, 20], lan_fraction=0.3)),
    dict(V=60, E=260, kw=dict(cost_choices=[3], lan_fraction=0.2)),
    dict(V=80, E=300, kw=dict()),
    dict(V=80, E=400, kw=dict(cost_lo=1, cost_hi=3)),
    dict(V=150, E=700, kw=dict(cost_choices=[7, 14, 21], lan_fraction=0.1)),
]


def nh_int(row):
    x = 0
    for w, word in enumerate(row):
        x |= int(word) << (64 * w)
    return x


def check(csr, root, isis=False, ecap=1 << 30):
    """Model vs oracle for one root; returns the model's stats (None: the oracle refused the job)."""
    ref = pyoracle.csr_spf(csr, root, vec_mode=int(isis), nh_words=4)
    if ref["status"] != 0:
        return None
    hops, nh, _n, st = merged_jump_phase(csr, root, ref["dist"], ref["first_parent"], ref["n_parents"], ecap)
    assert np.array_equal(hops, ref["hops"]), (root, np.nonzero(hops != ref["hops"])[0][:5])
    exp = [nh_int(r) for r in ref["nh_mask"]]
    assert nh == exp, (root, [v for v in range(csr.n_vertices) if nh[v] != exp[v]][:5])
    return st


@pytest.mark.parametrize("shape", range(len(SHAPES)))
@pytest.mark.parametrize("isis", [False, True])
def test_merged_pass_matches_faithful_oracle(shape, isis):
    sh = SHAPES[shape]
    merged = ecmp_total = 0
    for seed in range(8):
        t = synth.random_topology(sh["V"], sh["E"], synth.SEED_BASE + 2000 + 17 * shape + seed, **sh["kw"])
        csr = synth.topology_csr(t, isis=isis)
        for root in range(csr.n_vertices):
            st = check(csr, root, isis)
            if st is not None and st["merged"]:
                merged += 1
                ecmp_total += st["n_ecmp"]
    assert merged > 50 and ecmp_total > 0


def ladder(n):
    """Equal-cost diamonds i -> i+1 -> i+2 and i -> i+2: every rung is an ECMP vertex below ECMP vertices."""
    a, b = [], []
    for i in range(n - 2):
        a += [i, i]
        b += [i + 1, i + 2]
    c = np.full(len(a), 4, np.uint32)
    c[1::2] = 8
    return synth.Topology(n, np.asarray(a, np.uint32), np.asarray(b, np.uint32), c, c.copy(), [])


def test_merged_pass_on_nested_ecmp_ladder_with_lans():
    """Deep chains of ECMP terminals, with LANs hung off the rungs (HOP vertices on the chains)."""
    t = ladder(24)
    t.lans = [([2, 3, 4], [4, 4, 4]), ([9, 10], [2, 2]), ([15, 16, 17], [4, 4, 4])]
    for isis in (False, True):
        csr = synth.topology_csr(t, isis=isis)
        resolved = 0
        for root in range(csr.n_vertices):
            st = check(csr, root, isis)
            if st is not None:
                assert st["merged"]
                resolved += st["n_ecmp"]
        assert resolved > 100


def test_merged_pass_with_parallel_links_lan_roots_and_unreached_vertices():
    """Parallel p2p links, roots on several LANs (atoms behind hops-0 networks) and routers that no
    link reaches."""
    rng = np.random.default_rng(11)
    merged = 0
    for trial in range(10):
        R = 16
        a = list(range(1, R - 2)) + [int(x) for x in rng.integers(0, R - 2, 10)]
        b = [int(rng.integers(0, i)) for i in range(1, R - 2)] + [int(x) for x in rng.integers(0, R - 2, 10)]
        keep = [(x, y) for x, y in zip(a, b) if x != y]
        keep += keep[:4]
        t = synth.Topology(R, np.asarray([x for x, _ in keep], np.uint32), np.asarray([y for _, y in keep], np.uint32),
                           rng.choice([5, 10], len(keep)).astype(np.uint32), rng.choice([5, 10], len(keep)).astype(np.uint32),
                           [([0, 3, 5, 7], [5, 5, 5, 5]), ([0, 2, 4], [10, 5, 5]), ([1, 2, 6, 8], [5, 5, 10, 5])])
        for isis in (False, True):
            csr = synth.topology_csr(t, isis=isis)
            for root in range(csr.n_vertices):
                st = check(csr, root, isis)
                merged += st is not None and st["merged"]
    assert merged > 100


def csr_of(V, edges, hop):
    """CSR of directed (tail, head, cost) edges; `hop`: the hop-counting (router) vertices."""
    edges = sorted(edges)
    row = np.zeros(V + 1, np.uint32)
    for u, _v, _c in edges:
        row[u + 1] += 1
    vflags = np.zeros(V, np.uint8)
    vflags[list(hop)] = VF_HOP
    return Csr(np.cumsum(row, dtype=np.uint32), np.asarray([v for _u, v, _c in edges], np.uint32),
               np.asarray([c for _u, _v, c in edges], np.uint32), vflags)


@pytest.mark.parametrize("p_first", [False, True])
def test_hops0_vertex_below_a_hop_vertex(p_first):
    """A network root R reaches router P at distance 0 and network F both directly and through P at the
    same distance, so F is a hops-0 vertex whose first parent is P.  The routers below F are cut (they
    point at the root), but their hop counts include P.  (A network-to-network edge is outside what the
    next-hop algorithm reproduces: its sets are compared with the two-pass algorithm's.)"""
    P, R = (0, 1) if p_first else (1, 0)
    F, A, B, C = 2, 3, 4, 5
    edges = [(R, P, 0), (R, F, 5), (P, F, 5), (P, R, 3), (F, A, 0), (F, P, 0), (A, F, 2), (A, B, 2), (B, A, 2),
             (B, C, 2), (C, B, 2)]
    csr = csr_of(6, edges, hop=[P, A, B, C])
    ref = pyoracle.csr_spf(csr, R, nh_words=4)
    assert ref["status"] == 0 and ref["first_parent"][F] == P
    args = (csr, R, ref["dist"], ref["first_parent"], ref["n_parents"])
    hops, nh, _n, st = merged_jump_phase(*args)
    assert st["merged"] and st["walked"] > 0
    assert np.array_equal(hops, ref["hops"]) and list(hops[[A, B, C]]) == [2, 3, 4]
    assert nh == jump_phase(*args)[1]


def test_jobs_past_the_merged_limits_run_the_two_pass_algorithm():
    t = ladder(30)
    csr = synth.topology_csr(t)
    root = 0
    ref = pyoracle.csr_spf(csr, root, nh_words=4)
    n_e = int((ref["n_parents"] >= 2).sum())
    assert n_e > 4
    assert check(csr, root, ecap=n_e)["merged"]
    assert not check(csr, root, ecap=n_e - 1)["merged"]
    # a hub with more than 12 first-hop atoms
    n = 40
    a = np.zeros(n - 1, np.uint32)
    b = np.arange(1, n, dtype=np.uint32)
    hub = synth.Topology(n, a, b, np.full(n - 1, 3, np.uint32), np.full(n - 1, 3, np.uint32), [])
    st = check(synth.topology_csr(hub), 0)
    assert not st["merged"] and st["why"] == "limits"


@pytest.mark.parametrize("chain", [14, 15, 40])
def test_hop_sum_overflow_runs_the_two_pass_algorithm(chain):
    """A root with 12 atoms leaves 4 bits of hop sum: a path of 16 or more routers below it overflows the
    field and the job runs the two-pass algorithm; 15 do not."""
    n = 13 + chain
    a = [0] * 12 + list(range(12, n - 1))
    b = list(range(1, 13)) + list(range(13, n))
    c = np.full(len(a), 3, np.uint32)
    t = synth.Topology(n, np.asarray(a, np.uint32), np.asarray(b, np.uint32), c, c.copy(), [])
    st = check(synth.topology_csr(t), 0)
    assert st["merged"] == (chain < 15)
    if not st["merged"]:
        assert st["why"] == "overflow"
