"""Compile-time guard of the U-Net convolutions (csrc/conv3d_tc.cu): ptxas must keep every conv3d kernel's wgmma
products pipelined and in registers.  A kernel whose MMAs write overlapping parts of one accumulator with different N
gets its wgmmas serialised (ptxas C7510 / C7511: each one waits for the previous to retire), which costs several x
in the U-Nets and is easy to reintroduce; spills would put accumulators in local memory.  No GPU needed."""
import pytest

from tests.ptxas_common import function_props, ptxas_report, serialised


@pytest.fixture(scope="module")
def report():
    return ptxas_report("conv3d_tc.cu")


def test_conv3d_wgmma_not_serialised(report):
    bad = serialised(report, "C751[01]", "conv3d")
    assert not bad, "wgmma serialised by ptxas in:\n" + "\n".join(bad)


def test_conv3d_no_spills(report):
    conv = [(f, st, ld) for f, st, ld, _ in function_props(report) if "conv3d_tc_kernel" in f or "conv3d_col_kernel" in f]
    assert any("conv3d_col_kernel" in f for f, _, _ in conv) and any("conv3d_tc_kernelILi2E" in f for f, _, _ in conv), \
        "ptxas report lists no depth-streaming or transposed conv3d kernel"
    spilling = [f for f, st, ld in conv if st or ld]
    assert not spilling, "conv3d kernels spill:\n" + "\n".join(spilling)
