"""Compile-time guard of the depth-map fusion kernels (csrc/fusion.cu): one thread per reference pixel keeps the whole
reprojection chain, and for dpcd its 15 vote counters, in registers; a spill or a stack frame would put them in local
memory.  No GPU needed."""
import re

import pytest

from tests.ptxas_common import function_props, ptxas_report

KERNELS = ("fusion_prepare_kernel", "fusion_pcd_kernel", "fusion_dpcd_kernel", "fusion_scan_kernel", "fusion_extract_kernel")
PER_PIXEL = ("fusion_pcd_kernel", "fusion_dpcd_kernel", "fusion_extract_kernel")


@pytest.fixture(scope="module")
def report():
    return ptxas_report("fusion.cu")


def test_fusion_kernels_compiled(report):
    names = [f for f, _, _, _ in function_props(report)]
    for k in KERNELS:
        assert any(k in f for f in names), k


def test_fusion_no_spills(report):
    spilling = [f for f, st, ld, _ in function_props(report) if st or ld]
    assert not spilling, "fusion kernels spill:\n" + "\n".join(spilling)


def test_fusion_per_pixel_kernels_keep_their_state_in_registers(report):
    # no stack frame (the source-view index list is read from the kernel parameters, the vote counters are unrolled), and
    # at most 64 registers, so that four 256-thread blocks fit an SM
    for k in PER_PIXEL:
        m = re.search(r"Function properties for (\w*" + k + r"\w*)\n\s*(\d+) bytes stack frame", report)
        assert m and int(m.group(2)) == 0, (k, m and m.group(2))
    regs = {f: r for f, _, _, r in function_props(report) if any(k in f for k in PER_PIXEL)}
    assert all(r is not None and r <= 64 for r in regs.values()), regs
