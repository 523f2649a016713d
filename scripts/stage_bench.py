"""What the route-stage measurement scripts (scripts/*_stage.py) share: the GPU check, a library built with another
launch bound, ptxas's register lines, the alternating CUDA-event loop, the card's name and power limit, the JSON
record, and the host SPF over one job's plane row.  Importing it puts the repository and its tests on sys.path, so
that the scripts can use the package, tests/test_isis_route_cells_gpu.py's DeviceTopology and the tests' references."""
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "holo_b200" / "csrc"
for _p in (ROOT / "tests", ROOT):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))


def require_gpu(script_name: str):
    """torch; exits when there is no CUDA device."""
    import torch
    if not torch.cuda.is_available():
        sys.exit(f"{script_name}: no CUDA device; this measurement runs on the GPU only")
    return torch


def _definition(const: str):
    return re.compile(rf"constexpr uint32_t {const} = (\d+);")


def launch_bound(cu_name: str, const: str) -> int:
    """The value of `constexpr uint32_t <const> = N;` in holo_b200/csrc/<cu_name>."""
    found = _definition(const).findall((CSRC / cu_name).read_text())
    assert len(found) == 1, (cu_name, const, found)
    return int(found[0])


def with_bound(text: str, const: str, bound: int) -> str:
    """`text` with its one definition of `const` set to `bound`."""
    new, n = _definition(const).subn(f"constexpr uint32_t {const} = {bound};", text)
    assert n == 1, (const, n)
    return new


def build_variant(cu_name: str, const: str, bound: int, prefix: str, ptxas: bool = False):
    """libholo_spf.so with `const` in `cu_name` set to `bound`, compiled from a copy of the sources in a new temporary
    directory named with `prefix`; with ptxas, the -Xptxas -v build, and (library, compiler log)."""
    from holo_b200 import build
    tmp = Path(tempfile.mkdtemp(prefix=prefix))
    src = tmp / "holo_b200" / "csrc"                 # the sources include ../../include
    shutil.copytree(build.CSRC, src)
    shutil.copytree(build.ROOT / "include", tmp / "include")
    cu = src / cu_name
    cu.write_text(with_bound(cu.read_text(), const, bound))
    out = tmp / "libholo_spf_variant.so"
    srcs = sorted(list(src.glob("*.cu")) + list(src.glob("*.cc")))
    p = subprocess.run([os.environ.get("NVCC", "nvcc"), *build.NVCC_FLAGS, *(["-Xptxas", "-v"] if ptxas else []),
                        "-o", str(out), *map(str, srcs)], check=True, capture_output=True, text=True)
    return (out, p.stdout + p.stderr) if ptxas else out


def ptxas_registers(log: str, keep) -> dict:
    """{kind_wide|kind_narrow: "N registers, S bytes spill stores, L bytes spill loads"} from an -Xptxas -v log, for
    the kernels whose mangled name passes `keep`; kind is the kernel's cell type."""
    out, cur, spill = {}, None, ""
    for line in log.splitlines():
        m = re.search(r"(?:Compiling entry function|Function properties for) '?([\w$]+)'?", line)
        if m:
            cur = m.group(1)
        if not cur or not keep(cur):
            continue
        if "spill" in line:
            spill = line.split(",", 1)[1].strip()
        m = re.search(r"Used (\d+) registers", line)
        if m:
            dm = subprocess.run(["c++filt", cur], capture_output=True, text=True).stdout.strip()
            kind = dm.split("<")[0].split("::")[-1] + ("_narrow" if "PlanesNarrow" in dm else "_wide")
            out[kind] = f"{m.group(1)} registers, {spill}"
    return out


def time_alternating(ctx, work: dict, reps: int, warmup: int) -> dict:
    """{name: [ms per rep]} of each launch in `work`: `warmup` passes over all of them, then `reps` passes, each launch
    between two CUDA events on the engine's stream, alternating so that clocks and heat are shared, and one
    synchronisation at the end."""
    import torch
    for _ in range(warmup):
        for fn in work.values():
            fn()
    ctx.sync()
    stream = torch.cuda.ExternalStream(ctx.stream)
    ev = {k: [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
          for k in work}
    for r in range(reps):
        for k, fn in work.items():
            ev[k][r][0].record(stream)
            fn()
            ev[k][r][1].record(stream)
    ctx.sync()
    return {k: [a.elapsed_time(b) for a, b in e] for k, e in ev.items()}


def card_and_power():
    """(name, power limit) of the first GPU, as nvidia-smi reports them (read, not set)."""
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    if q:
        return tuple((q[0].split(", ") + ["?"])[:2])
    import torch
    return torch.cuda.get_device_name(0), "?"


def write_json(out: dict, path: str = "") -> None:
    """Prints the record on one line; with a path, also writes it there, indented."""
    print(json.dumps(out))
    if path:
        Path(path).parent.mkdir(parents=True, exist_ok=True)
        Path(path).write_text(json.dumps(out, indent=1) + "\n")


def root_spf(ctx):
    """The `spf(csr, root_vertex, nh_words)` the domain views take for their base job: one unperturbed row of the
    engine, read back."""
    def spf(csr, root, nhw):
        g = ctx.upload(csr)
        r = ctx.run(g, np.array([root], np.uint32))
        g.free()
        return r.dist[0], r.hops[0], np.pad(r.nh_mask[0], ((0, 0), (0, nhw - r.nh_mask.shape[2])))
    return spf


def spf_from_planes(proto: str, area, planes):
    """area_from_planes of "ospfv2" or "ospfv3" over one job's (dist, hops, nh) row, nh widened to the words asked."""
    from holo_b200 import ospfv2, ospfv3
    d, h, m = planes
    mod = {"ospfv2": ospfv2, "ospfv3": ospfv3}[proto]
    return mod.area_from_planes(area, lambda csr, root, nhw: (d, h, np.pad(m[:, None], ((0, 0), (0, nhw - 1)))))
