"""Executable model of the merged phase 3 of spf_quad_kernel (holo_b200/csrc/spf_quad.cuh): hops and
next-hop sets in ONE pointer-jumping pass over the next-hop tree, the tree cut at hops-0 vertices
and at ECMP vertices.

Per vertex the pass jumps one ancestor and carries one 16-bit aggregate of the segment (anc, v],
split per job: agg = hsum << n_atoms | atoms, where hsum is the number of HOP vertices on the segment
and atoms the first-hop atoms entering it.  An atom is seeded at one vertex, which a path crosses at
most once, so over disjoint segments the OR of the atoms is their sum and the whole aggregate is
added.  Every terminal (root, unreached and ECMP vertices) carries 0, so a terminal read twice in a
round adds nothing; an ECMP vertex's own seeds are kept aside until the ECMP vertices are resolved.
A vertex whose first parent f is a hops-0 vertex other than the root is cut (its ancestor is the
root) although its hop count along the first-parent chain is hops(f) + its own flag, and hops(f)
need not be 0 (a HOP vertex at distance 0 above f): that count is walked up the first-parent chain
when the vertex is set up.  After the rounds the ECMP vertices' next-hop sets are resolved by the
monotone sweeps of tests/jump_model.py, and their hop counts in the same sweeps:
hops(x) = flag(x) + hops(fp(x)), where hops(fp(x)) is hsum + hops(top) of an ordinary first parent,
or the resolved count of an ECMP one.

A job tries the merged pass when it has at most 12 first-hop atoms (at least 4 bits of hop sum) and
its ECMP vertices fit the list that shares shared memory with the jump words (`ecap`).  It runs the
two-pass algorithm (tests/jump_model.py) instead when it has more, when a segment's hop sum overflows
its field (a carry out of bit 15) or when the root itself is seeded.  The rounds are synchronous
here; the kernel runs them in place."""
from __future__ import annotations

import numpy as np

from jump_model import GF_NOHOP_TARGET_NO_NEXTHOP, INF, VF_HOP, jump_phase

UNRESOLVED = 0xFFFF


def merged_jump_phase(csr, root: int, dist: np.ndarray, first_parent: np.ndarray, n_parents: np.ndarray,
                      ecap: int = 1 << 30):
    """Returns (hops u16[V], nh python-int bitsets [V], n_atoms, stats); stats["merged"] tells which
    algorithm ran."""
    V = csr.n_vertices
    ecmp = n_parents >= 2
    row, col, cost = csr.row_ptr.astype(np.int64), csr.col.astype(np.int64), csr.cost.astype(np.int64)
    is_hop = (csr.vflags & VF_HOP) != 0
    rb, re_ = int(row[root]), int(row[root + 1])
    n_atoms = (re_ - rb) + sum(int(row[h + 1] - row[h]) for h in col[rb:re_] if not is_hop[h])
    def two_pass(why):
        hops, nh, n_atoms_, st = jump_phase(csr, root, dist, first_parent, n_parents)
        return hops, nh, n_atoms_, dict(st, merged=False, why=why)

    if n_atoms > 12 or int(ecmp.sum()) > ecap:
        return two_pass("limits")

    nohop_rule = bool(csr.flags & GF_NOHOP_TARGET_NO_NEXTHOP)
    d = dist.astype(np.int64)
    reached = dist != INF
    NONE = -1
    fp = np.where(first_parent == INF, NONE, first_parent.astype(np.int64))

    # ---- root edge table, hops-0 vertices and seeds: as in jump_model.jump_phase
    table = []
    nextbase = re_ - rb
    for e in range(rb, re_):
        h = int(col[e])
        if not is_hop[h]:
            table.append((h, nextbase, int(cost[e])))
            nextbase += int(row[h + 1] - row[h])
    hops0 = np.zeros(V, bool)
    for (h, _b, c) in table:
        if d[h] == c:
            hops0[h] = True
    hops0[root] = True
    seed = [0] * V
    for atom in range(n_atoms):
        u, e = root, None
        if atom < re_ - rb:
            e = rb + atom
        else:
            for k, (N, nb, _c) in enumerate(table):
                if not (nb <= atom < nb + int(row[N + 1] - row[N])):
                    continue
                first = all(t[0] != N for t in table[:k])
                if first and hops0[N]:
                    u, e = N, int(row[N]) + (atom - nb)
                break
        if e is None:
            continue
        v, c = int(col[e]), int(cost[e])
        if reached[u] and reached[v] and c != INF and d[u] + c == d[v] and not (nohop_rule and not is_hop[v]):
            seed[v] |= 1 << atom

    # ---- set-up: terminals (root, unreached, ECMP) point at themselves with aggregate 0
    anc = np.arange(V)
    hsum = np.zeros(V, np.int64)
    walked = 0
    for v in range(V):
        f = int(fp[v])
        if f == NONE or ecmp[v]:
            continue
        hsum[v] = int(is_hop[v])
        if hops0[f]:
            anc[v] = root
            u = f
            while u != root:           # hops(f): the first-parent chain above a cut hops-0 parent
                hsum[v] += int(is_hop[u])
                u = int(fp[u])
                walked += 1
        else:
            anc[v] = f
    if seed[root]:
        return two_pass("seeded root")
    terminal = anc == np.arange(V)
    agg = (hsum << n_atoms) + np.asarray([0 if terminal[v] else seed[v] for v in range(V)], np.int64)
    if (agg >> 16).any():
        return two_pass("overflow")

    # ---- rounds: two jumps per round (v -> A -> A2), until no ancestor moves
    rounds = 0
    while True:
        A = anc
        A2 = anc[A]
        new_anc = anc[A2]
        new_agg = agg + agg[A] + agg[A2]
        if (new_agg >> 16).any():
            return two_pass("overflow")
        moved = bool((new_anc != anc).any())
        anc, agg = new_anc, new_agg
        rounds += 1
        assert rounds <= 33
        if not moved:
            break
    top = anc.copy()
    amask = (1 << n_atoms) - 1
    hsum = agg >> n_atoms
    atoms = [int(x) & amask for x in agg]

    # ---- ECMP vertices: next-hop top and own segment through the first parent; hops unresolved
    elist = np.nonzero(ecmp)[0]
    hres = np.zeros(V, np.int64)
    for x in elist:
        f = int(fp[x])
        atoms[x] = seed[x]
        if hops0[f]:
            top[x] = root
        elif ecmp[f]:
            top[x] = f
        else:
            top[x] = anc[f]
            atoms[x] |= atoms[f]
        hres[x] = UNRESOLVED
    src = np.repeat(np.arange(V), np.diff(row))
    order = np.argsort(col, kind="stable")
    istart = np.searchsorted(col[order], np.arange(V + 1))
    sweeps = 0
    while True:
        changed = False
        for x in elist:
            need = atoms[int(top[x])] if top[x] != root else 0
            for j in range(istart[x], istart[x + 1]):
                e = order[j]
                u = int(src[e])
                if not reached[u] or cost[e] == INF or d[u] + cost[e] != d[x] or hops0[u]:
                    continue
                need |= atoms[u]
                if top[u] != root and top[u] != u:
                    need |= atoms[int(top[u])]
            need &= 0xFFFF & ~atoms[x]
            if need:
                atoms[x] |= need
                changed = True
            if hres[x] == UNRESOLVED:
                f = int(fp[x])
                w, t = int(is_hop[x]), root
                if ecmp[f]:
                    t = f
                elif f != root:
                    w, t = w + int(hsum[f]), int(top[f])
                if t == root:
                    hres[x] = w
                    changed = True
                elif hres[t] != UNRESOLVED:
                    hres[x] = w + hres[t]
                    changed = True
        sweeps += 1
        if not changed:
            break
        assert sweeps <= 2 * len(elist) + 2

    hops = np.zeros(V, np.uint16)
    nh = [0] * V
    for v in range(V):
        T = int(top[v])
        if ecmp[v]:
            hops[v] = hres[v]
        else:
            hops[v] = hsum[v] + (hres[T] if T != root and T != v else 0)
        nh[v] = atoms[v] | (atoms[T] if T != root and T != v else 0)
    return hops, nh, n_atoms, dict(merged=True, rounds=rounds, sweeps=sweeps, n_ecmp=len(elist), walked=walked)
