"""Compile-time guard of the stage-1 softmax attention (csrc/attention_fa.cuh on the body of csrc/softmax_attention.cuh,
built by costreg_tr.cu): attention_fa_kernel<NWG> runs NWG consumer warpgroups and a producer warpgroup in one CTA per
SM.  Its 64 fp32 scores, 20 P*V accumulators and 32 packed P registers per thread must stay in registers (spills put
them in local memory), ptxas must not serialise its wgmmas (C7510-C7512: each one waits for the previous to retire), and
the CTA must fit the register file.  No GPU needed."""
import re

import pytest

from tests.ptxas_common import function_props, ptxas_report, serialised

KERNEL = re.compile(r"attention_fa_kernelILi(\d+)E")


@pytest.fixture(scope="module")
def report():
    return ptxas_report("costreg_tr.cu")


def _kernels(report):
    """(mangled name, NWG, spill store bytes, spill load bytes, registers) of every stage-1 attention instance"""
    out = [(f, int(KERNEL.search(f).group(1)), st, ld, r) for f, st, ld, r in function_props(report) if KERNEL.search(f)]
    assert out, "ptxas report lists no stage-1 attention kernel"
    return out


def test_attention_wgmma_not_serialised(report):
    bad = serialised(report, "C751[012]", KERNEL)
    assert not bad, "wgmma serialised by ptxas in:\n" + "\n".join(bad)


def test_attention_no_spills(report):
    spilling = [f for f, _, st, ld, _ in _kernels(report) if st or ld]
    assert not spilling, "attention kernels spill:\n" + "\n".join(spilling)


def test_attention_one_cta_per_sm_fits_register_file(report):
    # NWG consumer warpgroups + one producer warpgroup; 65 536 registers per SM
    too_big = [(f, r, 128 * (nwg + 1)) for f, nwg, _, _, r in _kernels(report) if r * 128 * (nwg + 1) > 65536]
    assert not too_big, "registers x threads exceed the register file: " + repr(too_big)


def test_attention_ships_three_warpgroups(report):
    assert {nwg for _, nwg, _, _, _ in _kernels(report)} == {3}
