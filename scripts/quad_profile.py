#!/usr/bin/env python
"""Per-phase SM-cycle breakdown of spf_quad_kernel on the C2 workload (debug aid).

Counters (hspf_debug_phase_profile slots, thread 0 of every CTA, summed over CTAs):
0 init, 1 SSSP, 2 parents, 4 next hops, 5 hops, 7 SSSP rounds, 8 compaction (+ barrier),
9 expansion (thread 0's share), 10 barrier after the expansion, 12 queue entries,
13 hop jump rounds, 14 next-hop jump rounds, 15 ECMP sweeps.
A job that runs the merged phase-3 pass counts its set-up and rounds under "hops" and its
rounds in slot 14; the ECMP sweeps and the result writes fall under "next hops".  Slot 13
counts rounds of the hop pass, which only the two-pass code runs."""
import ctypes as C
import sys

import numpy as np

sys.path.insert(0, ".")
from holo_b200 import capi, synth  # noqa: E402

n_jobs = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
t = synth.random_topology(10000, 40000, synth.SEED_BASE + 2)
csr = synth.topology_csr(t)
ctx = capi.Context(0)
g = ctx.upload(csr)
lib = ctx.lib
roots = np.arange(n_jobs, dtype=np.uint32)
ctx.run(g, roots)
lib.hspf_debug_phase_profile(ctx.handle, 1, None)
ctx.run(g, roots)
out = (C.c_uint64 * 16)()
lib.hspf_debug_phase_profile(ctx.handle, 0, out)
names = {0: "init", 1: "sssp", 2: "parents", 5: "hops", 4: "nexthops"}
tot = sum(out[k] for k in names)
n = float(n_jobs)
print(f"jobs {n_jobs}: per job {tot / n / 1e3:.1f} kcycles of its CTA")
for k, nm in names.items():
    print(f"  {nm:9s} {100 * out[k] / tot:5.1f}%  {out[k] / n / 1e3:8.1f} kcycles/job")
print(f"  sssp: rounds/job {out[7] / n:.1f}  queue entries/job {out[12] / n:.0f}  kcycles/job: compaction {out[8] / n / 1e3:.1f}"
      f"  expansion {out[9] / n / 1e3:.1f}  barrier {out[10] / n / 1e3:.1f}")
print(f"  jump: hop rounds {out[13] / n:.1f}  next-hop rounds {out[14] / n:.1f}  ECMP sweeps {out[15] / n:.1f}")
