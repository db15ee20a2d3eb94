"""Compile-time guard of the fused token MLP (csrc/linear_tc.cu: token_mlp_kernel<FORM>): a producer warpgroup and two
MMA warpgroups in one CTA per SM.  Each MMA warpgroup keeps FFN2's residual, the FFN1 input fragments, two FFN1 chunk
accumulators, the FFN2 accumulator and the GELU fragments in registers; a spill would put them in local memory, a
serialised wgmma (C7510 / C7511) would wait for the previous one to retire, and the 384 threads must fit the register
file.  No GPU needed."""
import re

import pytest

from tests.ptxas_common import function_props, ptxas_report, serialised

KERNEL = re.compile(r"token_mlp_kernelILi(\d+)E")


@pytest.fixture(scope="module")
def report():
    return ptxas_report("linear_tc.cu")


def _kernels(report):
    out = [(f, int(KERNEL.search(f).group(1)), st, ld, r) for f, st, ld, r in function_props(report) if KERNEL.search(f)]
    assert out, "ptxas report lists no token MLP kernel"
    return out


def test_token_mlp_all_forms_compiled(report):
    # pre-norm block, last pre-norm block, post-norm layer
    assert {form for _, form, _, _, _ in _kernels(report)} == {0, 1, 2}


def test_token_mlp_wgmma_not_serialised(report):
    bad = serialised(report, "C751[01]", KERNEL)
    assert not bad, "wgmma serialised by ptxas in:\n" + "\n".join(bad)


def test_token_mlp_no_spills(report):
    spilling = [f for f, _, st, ld, _ in _kernels(report) if st or ld]
    assert not spilling, "token MLP kernels spill:\n" + "\n".join(spilling)


def test_token_mlp_fits_register_file(report):
    # 384 threads, one CTA per SM; setmaxnreg then moves the producer's registers to the MMA warpgroups
    # (40 x 128 + 232 x 256 = 64 512 <= 65 536)
    too_big = [(f, r) for f, _, _, _, r in _kernels(report) if r is None or r * 384 > 65536]
    assert not too_big, "registers x 384 threads exceed the register file: " + repr(too_big)
