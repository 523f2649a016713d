"""The route-stage measurement scripts (scripts/*_stage.py) on the CPU: each one's launch bound is found in the tree
and rewritten alone, and each imports, parses its default arguments and refuses to run without a GPU."""
import importlib.util
import os
import subprocess
import sys
from pathlib import Path

import pytest

SCRIPTS = Path(__file__).resolve().parent.parent / "scripts"
if str(SCRIPTS) not in sys.path:
    sys.path.insert(0, str(SCRIPTS))
import stage_bench  # noqa: E402

STAGES = sorted(SCRIPTS.glob("*_stage.py"))


def load(script: Path):
    spec = importlib.util.spec_from_file_location(script.stem, script)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


BOUNDED = [s for s in STAGES if hasattr(load(s), "BOUND")]


def test_every_script_that_builds_a_variant_names_its_bound():
    assert BOUNDED and all(s in BOUNDED for s in STAGES if "build_variant(" in s.read_text())


@pytest.mark.parametrize("script", BOUNDED, ids=lambda s: s.stem)
def test_launch_bound_is_read_and_rewritten_alone(script):
    cu, const = load(script).BOUND
    text = (stage_bench.CSRC / cu).read_text()
    cur = stage_bench.launch_bound(cu, const)
    line = f"constexpr uint32_t {const} = {cur};"
    assert text.count(line) == 1
    for bound in (4, 8):
        new = stage_bench.with_bound(text, const, bound)
        changed = [(a, b) for a, b in zip(text.splitlines(), new.splitlines()) if a != b]
        assert len(new.splitlines()) == len(text.splitlines())
        want = [] if bound == cur else [(a, a.replace(line, f"constexpr uint32_t {const} = {bound};"))
                                        for a in text.splitlines() if line in a]
        assert changed == want


@pytest.mark.parametrize("script", STAGES, ids=lambda s: s.stem)
def test_script_refuses_to_run_without_a_gpu(script):
    p = subprocess.run([sys.executable, str(script)], env=dict(os.environ, CUDA_VISIBLE_DEVICES=""),
                       capture_output=True, text=True, timeout=600)
    assert p.returncode != 0
    assert f"{script.name}: no CUDA device; this measurement runs on the GPU only" in p.stderr
