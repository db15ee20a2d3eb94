"""ORACLE - TEST INFRASTRUCTURE ONLY.  The one place that finds, copies and loads the reference's own sources.

MANIFEST lists every file of the reference that oracle/, tests/ and tools/ read.  root() finds them, in this order:
$MVSF_REFERENCE, oracle/_ref/ (the git-ignored copy build() makes where the reference is available; it travels with the
repository to machines without the reference), and the reference checkout at /root/reference.  Reference code is
loaded from there, never copied into tracked files.  root() is the probe; the loaders raise where the files are absent.

  python oracle/reference.py     # copies MANIFEST into oracle/_ref/; a no-op where the reference is absent
"""
import ast
import importlib.util
import json
import os
import shutil
import sys
import types

import numpy as np

REF = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")
CHECKOUT = "/root/reference"
CONFIG = "config/mvsformer++.json"
# relative paths; `models` is the reference's whole models/ package
MANIFEST = ("models", CONFIG, "misc/fusion.py", "misc/gipuma.py", "datasets/general_eval.py", "datasets/data_io.py",
            "test.py", "test_tt.py")
# files that import another file of the manifest when they load, so that both come from one root
IMPORTS = {"misc/gipuma.py": ("datasets/data_io.py",), "datasets/general_eval.py": ("datasets/data_io.py",)}


def _holds(d, relpaths):
    return all(os.path.exists(os.path.join(d, p)) for p in relpaths)


def _candidates():
    return [d for d in (os.environ.get("MVSF_REFERENCE"), REF, CHECKOUT) if d]


def root(*relpaths):
    """The first of $MVSF_REFERENCE, oracle/_ref and the checkout that holds every one of relpaths, or None."""
    return next((d for d in _candidates() if _holds(d, relpaths)), None)


def _need(*relpaths):
    r = root(*relpaths)
    if r is None:
        raise FileNotFoundError(f"reference sources not found: {', '.join(relpaths)} (oracle/_ref is made by "
                                "oracle/reference.py where the reference is available)")
    return r


def module(relpath):
    """One reference file loaded as a module named after its path (datasets/data_io.py -> datasets.data_io).  It loads
    under a bare `datasets` package of its root, so that `from datasets.data_io import ...` resolves without running the
    reference's datasets/__init__.py (its training loaders); sys.modules is left as it was."""
    r = _need(relpath, *IMPORTS.get(relpath, ()))
    name = relpath[:-len(".py")].replace("/", ".")
    tops = {"datasets", name.split(".")[0]}
    saved = {k: v for k, v in sys.modules.items() if k.split(".")[0] in tops}
    try:
        pkg = types.ModuleType("datasets")
        pkg.__path__ = [os.path.join(r, "datasets")]
        sys.modules["datasets"] = pkg
        spec = importlib.util.spec_from_file_location(name, os.path.join(r, relpath))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
    finally:
        for k in [k for k in sys.modules if k.split(".")[0] in tops]:
            del sys.modules[k]
        sys.modules.update(saved)
    return mod


def function(script, name):
    """A top-level function of one of the reference's scripts (test.py and test_tt.py parse the command line when
    imported), compiled alone from its source with numpy as `np`."""
    with open(os.path.join(_need(script), script)) as f:
        tree = ast.parse(f.read())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == name)
    ns = {"np": np}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), script, "exec"), ns)
    return ns[name]


def import_models(r=None):
    """Puts r (default: the root holding the reference's models/ package) on sys.path, so that `import models...` loads
    the reference's package, with its attention on the SDPA path a CPU runs (no flash-attn, no xFormers); -> r."""
    r = r or _need("models")
    if r not in sys.path:
        sys.path.insert(0, r)
    import models.dino.layers.attention as A
    A.FLASH_AVAILABLE = A.XFORMERS_AVAILABLE = False
    return r


def config():
    """arch.args of the reference's shipped config/mvsformer++.json (a new dict on every call)."""
    with open(os.path.join(_need(CONFIG), CONFIG)) as f:
        return json.load(f)["arch"]["args"]


def build():
    """Copies MANIFEST from $MVSF_REFERENCE or the checkout into a fresh oracle/_ref; a no-op where neither holds it.
    -> whether oracle/_ref holds the whole manifest."""
    src = next((d for d in _candidates() if d != REF and _holds(d, MANIFEST)), None)
    if src is not None:
        shutil.rmtree(REF, ignore_errors=True)
        for rel in MANIFEST:
            top = os.path.join(src, rel)
            files = [top] if os.path.isfile(top) else [os.path.join(dp, f) for dp, _, fs in os.walk(top)
                                                       if os.path.basename(dp) != "__pycache__" for f in fs]
            for s in files:   # into directories of our own: the checkout's may be read-only
                d = os.path.join(REF, os.path.relpath(s, src))
                os.makedirs(os.path.dirname(d), exist_ok=True)
                shutil.copy2(s, d)
    return _holds(REF, MANIFEST)


if __name__ == "__main__":
    print("oracle/_ref:", "complete" if build() else "absent")
