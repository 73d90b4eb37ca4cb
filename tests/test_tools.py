"""The timing tools under tools/, without a GPU: each imports and answers --help, the shared module's dump comparison and
spreads, and no tool imports another one except the shared measurement module (tools/timing.py)."""
import ast
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")
if TOOLS not in sys.path:
    sys.path.insert(0, TOOLS)

import timing as T  # noqa: E402

ENTRY_POINTS = ("colorize", "generate_points", "update_points", "select_patches", "retrieve_scan", "vmap_retrieve", "refpatch", "map_find", "map_mirror",
                "map_growth", "vmap")
MODULES = ("timing", "ab_timing", *(f"{e}_timing" for e in ENTRY_POINTS))


@pytest.mark.parametrize("module", MODULES)
def test_tool_imports_and_answers_help_without_a_gpu(module):
    r = subprocess.run([sys.executable, os.path.join(TOOLS, module + ".py"), "--help"], cwd=ROOT, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""),
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    if module != "timing":  # the shared module has no command line
        assert r.stdout.startswith("usage:"), r.stdout[:500]


@pytest.mark.parametrize("module", MODULES)
def test_tool_imports_no_other_tool(module):
    tools = {f[:-3] for f in os.listdir(TOOLS) if f.endswith(".py")} - {"timing"}
    with open(os.path.join(TOOLS, module + ".py")) as f:
        tree = ast.parse(f.read())
    imported = {a.name.split(".")[0] for n in ast.walk(tree) if isinstance(n, ast.Import) for a in n.names}
    imported |= {n.module.split(".")[0] for n in ast.walk(tree) if isinstance(n, ast.ImportFrom) and n.level == 0 and n.module}
    assert not imported & tools, f"{module} imports {sorted(imported & tools)}"


def _tree(root, files):
    for rel, data in files.items():
        path = root / rel
        path.parent.mkdir(parents=True, exist_ok=True)
        path.write_bytes(data)


def test_same_dumps_finds_identical_trees_identical(tmp_path):
    files = {"lio_state.npy": bytes(range(256)), "vio/state.npy": b"\x00" * 64, "vio/iters.npy": b"\x07"}
    _tree(tmp_path / "a", files)
    _tree(tmp_path / "b", files)
    assert T.same_dumps(tmp_path / "a", tmp_path / "b") == dict(files=3, differ=[])


def test_same_dumps_catches_one_byte_and_a_one_sided_file(tmp_path):
    files = {"lio_state.npy": bytes(range(256)), "vio/state.npy": b"\x00" * 64}
    _tree(tmp_path / "a", dict(files, **{"vio/only_a.npy": b"\x01"}))
    _tree(tmp_path / "b", dict(files, **{"vio/state.npy": b"\x00" * 63 + b"\x01"}))
    assert T.same_dumps(tmp_path / "a", tmp_path / "b") == dict(files=2, differ=[os.path.join("vio", "only_a.npy"), os.path.join("vio", "state.npy")])


def test_spread_skips_none_and_is_none_when_empty():
    assert T.spread([3.0, None, 1.0, 2.0]) == dict(min=1.0, median=2.0, max=3.0, n=3)
    assert T.spread([]) is None
    assert T.spread([None, None]) is None
