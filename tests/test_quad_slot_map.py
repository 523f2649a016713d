"""The slot -> vertex map of spf_quad_kernel's parents pass, restated on the quad-space image
(csrc/quad_layout.h) without a GPU.

The parents pass turns the best parent's slot into a vertex id from shared memory: the vertex of
the first slot of every 32-slot bitmap word, plus the number of chain starts (~fcont bits) below
the slot in its word.  That equals vert_of only if every in-quad record names a chain start and
no dummy quad sits between a word's first slot and a chain start; these tests pin both."""
import numpy as np
import pytest

from holo_b200 import synth
from holo_b200.capi import Csr, VF_HOP, quad_image


def shared_map(q, s: np.ndarray) -> np.ndarray:
    """vert_of[s & ~31] + popcount(~fcont[s >> 5] & ((1 << (s & 31)) - 1)), as the kernel computes it."""
    s = s.astype(np.int64)
    below = (~q.fcont[s >> 5].astype(np.int64)) & ((1 << (s & 31)) - 1)
    rank = np.array([bin(int(x)).count("1") for x in below], dtype=np.int64)
    return q.vert_of[s & ~31].astype(np.int64) + rank


def hub_csr() -> Csr:
    """Vertex 0 with 40 links both ways (a 10-quad chain), vertex 41 isolated."""
    V = 42
    src, dst = [], []
    for i in range(1, 41):
        src += [0, i]; dst += [i, 0]
    order = np.lexsort((np.arange(len(src)), np.asarray(src)))
    src, dst = np.asarray(src)[order], np.asarray(dst)[order]
    row = np.cumsum(np.bincount(src + 1, minlength=V + 1)).astype(np.uint32)
    return Csr(row, dst.astype(np.uint32), np.ones(len(src), np.uint32), np.full(V, VF_HOP, np.uint8))


@pytest.mark.parametrize("case", [
    (2, 2, 1, {}),
    (300, 1400, 5, dict(lan_fraction=0.1)),
    (120, 1400, 4, dict(cost_choices=[10, 20])),           # multi-quad chains, dummy quads at word tails
    (10000, 40000, 2, {}),                                  # C2
    "hub",
])
def test_shared_slot_map_equals_vert_of(built, case):
    if case == "hub":
        csr = hub_csr()
    else:
        V, E, seed, kw = case
        csr = synth.topology_csr(synth.random_topology(V, E, synth.SEED_BASE + seed, **kw))
    q = quad_image(csr)
    assert q.eligible
    V = csr.n_vertices
    # every vertex's chain start maps back to the vertex
    assert np.array_equal(shared_map(q, q.slot_of), np.arange(V))
    # every in-quad record (real, pad or dummy) names a chain start
    starts = np.zeros(q.NQ, bool)
    starts[q.slot_of] = True
    rec_slots = (q.iq & 0xFFFF).reshape(-1)
    assert starts[rec_slots].all()
