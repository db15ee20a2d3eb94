"""Compile-time guard of the U-Net convolutions (csrc/conv3d_tc.cu): ptxas must keep every conv3d kernel's wgmma
products pipelined and in registers.  A kernel whose MMAs write overlapping parts of one accumulator with different N
gets its wgmmas serialised (ptxas C7510 / C7511: each one waits for the previous to retire), which costs several x
in the U-Nets and is easy to reintroduce; spills would put accumulators in local memory.  No GPU needed."""
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


@pytest.fixture(scope="module")
def ptxas_report():
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as d:
        cmd = [nvcc] + B.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.CSRC, "conv3d_tc.cu"), "-o", os.path.join(d, "c.o")]
        p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    return p.stdout + p.stderr


def test_conv3d_wgmma_not_serialised(ptxas_report):
    bad = sorted({m.group(2) for m in re.finditer(r"\((C751[01])\).*?function '(\w+)'", ptxas_report)
                  if "conv3d" in m.group(2)})
    assert not bad, "wgmma serialised by ptxas in:\n" + "\n".join(bad)


def test_conv3d_no_spills(ptxas_report):
    props = re.findall(r"Function properties for (\w+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                       ptxas_report)
    conv = [(f, int(st), int(ld)) for f, st, ld in props if "conv3d_tc_kernel" in f or "conv3d_col_kernel" in f]
    assert any("conv3d_col_kernel" in f for f, _, _ in conv) and any("conv3d_tc_kernelILi2E" in f for f, _, _ in conv), \
        "ptxas report lists no depth-streaming or transposed conv3d kernel"
    spilling = [f for f, st, ld in conv if st or ld]
    assert not spilling, "conv3d kernels spill:\n" + "\n".join(spilling)
