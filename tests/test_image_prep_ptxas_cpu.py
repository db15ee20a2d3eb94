"""Compile-time guard of the image preparation kernels (csrc/image_prep.cu): one thread per output pixel keeps its
coefficients and the 3 channels in registers; a spill or a stack frame would put them in local memory.  No GPU needed."""
import re

import pytest

from tests.ptxas_common import function_props, ptxas_report

KERNELS = ("image_resize_kernel", "image_normalize_kernel")


@pytest.fixture(scope="module")
def report():
    return ptxas_report("image_prep.cu")


def test_image_prep_kernels_compiled(report):
    names = [f for f, _, _, _ in function_props(report)]
    for k in KERNELS:
        assert any(k in f for f in names), k


def test_image_prep_no_spills_no_stack(report):
    for k in KERNELS:
        m = re.search(r"Function properties for (\w*" + k + r"\w*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                      r"(\d+) bytes spill loads", report)
        assert m and m.group(2) == m.group(3) == m.group(4) == "0", (k, m and m.groups())


def test_image_prep_register_budget(report):
    # at most 64 registers, so that eight 256-thread blocks fit an SM
    regs = {f: r for f, _, _, r in function_props(report) if any(k in f for k in KERNELS)}
    assert len(regs) == len(KERNELS) and all(r is not None and r <= 64 for r in regs.values()), regs
