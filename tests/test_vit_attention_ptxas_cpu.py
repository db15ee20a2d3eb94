"""Compile-time guard of the ViT softmax attention (csrc/vit_attention.cuh on the body of csrc/softmax_attention.cuh,
built by vit.cu): two consumer warpgroups and a producer warpgroup in one CTA per SM.  Their 64 fp32 scores, 36 P*V
accumulators, 32 running outputs and 32 packed P registers per thread must stay in registers (spills put them in local
memory), ptxas must not serialise the wgmmas (C7510-C7512: each one waits for the previous to retire), and the register
count must fit the warpgroup layout: 384 threads at the compiled count fit the register file, and setmaxnreg 40 / 232
redistributes it.  No GPU needed."""
import re

import pytest

from tests.ptxas_common import function_props, ptxas_report, serialised

KERNEL = re.compile(r"vit_attention_kernel")


@pytest.fixture(scope="module")
def report():
    return ptxas_report("vit.cu")


def _kernels(report):
    """(mangled name, spill store bytes, spill load bytes, registers) of the attention kernel"""
    out = [p for p in function_props(report) if KERNEL.search(p[0])]
    assert len(out) == 1, "ptxas report should list the ViT attention kernel once"
    return out


def test_vit_attention_wgmma_not_serialised(report):
    bad = serialised(report, "C751[012]", KERNEL)
    assert not bad, "wgmma serialised by ptxas in:\n" + "\n".join(bad)


def test_vit_attention_no_spills(report):
    spilling = [f for f, st, ld, _ in _kernels(report) if st or ld]
    assert not spilling, "ViT attention spills:\n" + "\n".join(spilling)


def test_vit_attention_registers_fit_the_warpgroup_layout(report):
    # 2 consumer warpgroups + 1 producer warpgroup, one CTA per SM (65 536 registers); after setmaxnreg the producer
    # keeps 40 and each consumer thread may use up to 232
    for f, _, _, r in _kernels(report):
        assert r * 384 <= 65536, (f, r)
        assert 40 * 128 + 232 * 256 <= 65536


def test_no_spills_in_the_other_vit_kernels(report):
    props = [(f, st, ld) for f, st, ld, _ in function_props(report) if "vit" in f]
    assert props
    assert not [f for f, st, ld in props if st or ld]
