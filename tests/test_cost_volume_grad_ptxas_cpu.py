"""Compile-time guard of the cost-volume backward (csrc/warp_corr_bwd.cu): each lane keeps its 4 reference channels, their
gradient and the upstream gradient of its groups in registers; a spill or a stack frame would put them in local memory.
No GPU needed."""
import re

import pytest

from tests.ptxas_common import function_props, ptxas_report


@pytest.fixture(scope="module")
def report():
    return ptxas_report("warp_corr_bwd.cu")


def test_backward_kernels_compiled(report):
    names = [f for f, _, _, _ in function_props(report) if "warp_corr_aggregate_bwd_kernel" in f]
    # C = 8 / 16 / 32 / 64, each with the upstream gradient kept (D <= 2 C / 4) and reloaded per chunk
    assert len(names) == 8, names


def test_backward_no_spills_no_stack(report):
    spilling = [f for f, st, ld, _ in function_props(report) if st or ld]
    assert not spilling, "backward kernels spill:\n" + "\n".join(spilling)
    frames = re.findall(r"Function properties for (\w*warp_corr_aggregate_bwd_kernel\w*)\n\s*(\d+) bytes stack frame", report)
    assert frames and all(int(n) == 0 for _, n in frames), frames
