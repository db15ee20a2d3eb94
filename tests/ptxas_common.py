"""The harness of the compile-time guards (test_*_ptxas_cpu.py): the ptxas -v report of a CUDA source, compiled once per
test session with the library's flags, and its parsers.  No GPU needed."""
import functools
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from mvsformerplusplus_b200 import build as B


def _nvcc():
    try:
        nvcc = B._nvcc()
    except RuntimeError:
        return None
    return nvcc if shutil.which(nvcc) else None


@functools.lru_cache(maxsize=None)
def _compile(src):
    nvcc = _nvcc()
    if nvcc is None:
        return None
    with tempfile.TemporaryDirectory() as d:
        cmd = [nvcc] + B.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.CSRC, src), "-o", os.path.join(d, "t.o")]
        p = subprocess.run(cmd, capture_output=True, text=True)
    return p.returncode, p.stdout + p.stderr


def ptxas_report(src):
    """ptxas -v output of csrc/<src> (skips the test without nvcc)"""
    r = _compile(src)
    if r is None:
        pytest.skip("nvcc not available")
    rc, out = r
    assert rc == 0, out
    return out


def function_props(report):
    """(mangled name, spill store bytes, spill load bytes, registers or None) of every function in the report"""
    props = re.findall(r"Function properties for (\w+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes "
                       r"spill loads(?:\n[^\n]*Used (\d+) registers)?", report)
    return [(f, int(st), int(ld), int(r) if r else None) for f, st, ld, r in props]


def serialised(report, codes, pattern):
    """functions matching pattern whose wgmmas ptxas serialised with one of the warnings codes (a regex, e.g. C751[01])"""
    return sorted({m.group(2) for m in re.finditer(r"\((" + codes + r")\).*?function '(\w+)'", report)
                   if re.search(pattern, m.group(2))})
