"""Compile-time guard of the ViT softmax attention (csrc/vit_attention.cuh, built by vit.cu): two consumer warpgroups and
a producer warpgroup in one CTA per SM.  Their 64 fp32 scores, 36 P*V accumulators, 32 running outputs and 32 packed P
registers per thread must stay in registers (spills put them in local memory), ptxas must not serialise the wgmmas
(C7510-C7512: each one waits for the previous to retire), and the register count must fit the warpgroup layout: 384
threads at the compiled count fit the register file, and setmaxnreg 40 / 232 redistributes it.  No GPU needed."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from mvsformerplusplus_b200 import build as B

KERNEL = re.compile(r"vit_attention_kernel")


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
        cmd = [nvcc] + B.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.CSRC, "vit.cu"), "-o", os.path.join(d, "t.o")]
        p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    return p.stdout + p.stderr


def _kernels(report):
    """(mangled name, spill store bytes, spill load bytes, registers) of the attention kernel"""
    props = re.findall(r"Function properties for (\w+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes "
                       r"spill loads\n[^\n]*Used (\d+) registers", report)
    out = [(f, int(st), int(ld), int(r)) for f, st, ld, r in props if KERNEL.search(f)]
    assert len(out) == 1, "ptxas report should list the ViT attention kernel once"
    return out


def test_vit_attention_wgmma_not_serialised(ptxas_report):
    bad = sorted({m.group(2) for m in re.finditer(r"\((C751[012])\).*?function '(\w+)'", ptxas_report)
                  if KERNEL.search(m.group(2))})
    assert not bad, "wgmma serialised by ptxas in:\n" + "\n".join(bad)


def test_vit_attention_no_spills(ptxas_report):
    spilling = [f for f, st, ld, _ in _kernels(ptxas_report) if st or ld]
    assert not spilling, "ViT attention spills:\n" + "\n".join(spilling)


def test_vit_attention_registers_fit_the_warpgroup_layout(ptxas_report):
    # 2 consumer warpgroups + 1 producer warpgroup, one CTA per SM (65 536 registers); after setmaxnreg the producer
    # keeps 40 and each consumer thread may use up to 232
    for f, _, _, r in _kernels(ptxas_report):
        assert r * 384 <= 65536, (f, r)
        assert 40 * 128 + 232 * 256 <= 65536


def test_no_spills_in_the_other_vit_kernels(ptxas_report):
    props = re.findall(r"Function properties for (\w*vit\w*)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) "
                       r"bytes spill loads", ptxas_report)
    assert props
    assert not [f for f, st, ld in props if int(st) or int(ld)]
