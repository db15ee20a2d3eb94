"""oracle/reference.py, the one locator and loader of the reference's own sources: every path a loader asks for is in
MANIFEST (so build() copies it), a built oracle/_ref serves every loader, and loading leaves sys.modules as it was."""
import ast
import os
import sys
import types

import pytest

from oracle import reference
from tests.common import ROOT

CALLS = {"reference.root", "reference.module", "reference.function"}


def requested_paths():
    """every path that a call of reference.root / module / function under oracle/, tests/, tools/ or bench.py names (of
    function(), the script), that oracle/reference.py itself looks up, and that a manifest file imports"""
    paths = {p for k, deps in reference.IMPORTS.items() for p in (k, *deps)}
    sources = [os.path.join(ROOT, "bench.py")] + [os.path.join(ROOT, d, f) for d in ("oracle", "tests", "tools")
                                                  for f in os.listdir(os.path.join(ROOT, d)) if f.endswith(".py")]
    for f in sources:
        calls = CALLS | {"root", "_need"} if f == reference.__file__ else CALLS
        for n in ast.walk(ast.parse(open(f).read())):
            if isinstance(n, ast.Call) and ast.unparse(n.func) in calls:
                for a in n.args[:1] if ast.unparse(n.func).endswith("function") else n.args:
                    if isinstance(a, ast.Constant):
                        paths.add(a.value)
                    elif ast.unparse(a) in ("CONFIG", "reference.CONFIG"):
                        paths.add(reference.CONFIG)
    return paths


def test_every_requested_path_is_in_the_manifest():
    paths = requested_paths()
    assert {"models", reference.CONFIG, "misc/fusion.py", "misc/gipuma.py", "datasets/general_eval.py",
            "datasets/data_io.py", "test.py", "test_tt.py"} <= paths, "the scan misses callers"
    assert paths <= set(reference.MANIFEST), sorted(paths - set(reference.MANIFEST))


@pytest.fixture
def built(monkeypatch):
    monkeypatch.delenv("MVSF_REFERENCE", raising=False)
    if not all(os.path.exists(os.path.join(reference.REF, p)) for p in reference.MANIFEST):
        pytest.skip("oracle/_ref is not built (build() makes it only where the reference is available)")


def test_built_copy_serves_every_loader(built):
    from oracle import ref_hotpath as RH
    for p in reference.MANIFEST:
        assert reference.root(p) == reference.REF, p
    for p, deps in reference.IMPORTS.items():
        assert reference.root(p, *deps) == reference.REF, p
    assert RH.reference_root() == reference.REF
    for p in reference.MANIFEST:
        if p.endswith(".py") and p.startswith(("misc/", "datasets/")):
            assert reference.module(p).__file__ == os.path.join(reference.REF, p)
    assert callable(reference.function("test.py", "write_cam")) and callable(reference.function("test_tt.py", "write_cam"))
    assert isinstance(reference.config(), dict)


ORDERS = [("datasets/data_io.py", "datasets/general_eval.py", "misc/gipuma.py") * 2,
          ("misc/gipuma.py", "datasets/general_eval.py", "datasets/data_io.py") * 2]


@pytest.mark.parametrize("order", ORDERS, ids=["datasets_first", "gipuma_first"])
@pytest.mark.parametrize("present", [False, True], ids=["no_datasets", "other_datasets"])
def test_loading_leaves_sys_modules_as_it_was(monkeypatch, order, present):
    if reference.root("misc/gipuma.py", "datasets/general_eval.py", "datasets/data_io.py") is None:
        pytest.skip("no reference sources")
    for k in [k for k in sys.modules if k.split(".")[0] in ("datasets", "misc")]:
        monkeypatch.delitem(sys.modules, k)
    if present:
        monkeypatch.setitem(sys.modules, "datasets", types.ModuleType("datasets"))
    before = {k: v for k, v in sys.modules.items() if k.split(".")[0] in ("datasets", "misc")}
    mods = [reference.module(p) for p in order]
    assert {k: v for k, v in sys.modules.items() if k.split(".")[0] in ("datasets", "misc")} == before
    gipuma = mods[order.index("misc/gipuma.py")]
    assert callable(gipuma.read_pfm) and callable(mods[order.index("datasets/general_eval.py")].MVSDataset)
