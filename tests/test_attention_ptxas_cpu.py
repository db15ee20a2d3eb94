"""Compile-time guard of the stage-1 softmax attention (csrc/attention_fa.cuh, built by costreg_tr.cu): the shipped
fp16-P kernel (attention_fa_kernel<false, NWG>) runs NWG consumer warpgroups and a producer warpgroup in one CTA per SM.
Its 64 fp32 scores, 20 P*V accumulators and 32 packed P registers per thread must stay in registers (spills put them in
local memory), ptxas must not serialise its wgmmas (C7510-C7512: each one waits for the previous to retire), and the CTA
must fit the register file.  The hi + lo kernel (attention_fa_kernel<true, 2>, opt-in through
mvsf_attention_set_precision(1)) spills and is serialised already and is not checked.  No GPU needed."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from mvsformerplusplus_b200 import build as B

FP16_P = re.compile(r"attention_fa_kernelILb0ELi(\d+)E")


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
        cmd = [nvcc] + B.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.CSRC, "costreg_tr.cu"), "-o", os.path.join(d, "t.o")]
        p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    return p.stdout + p.stderr


def _kernels(report):
    """(mangled name, NWG, spill store bytes, spill load bytes, registers) of every fp16-P attention instance"""
    props = re.findall(r"Function properties for (\w+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes "
                       r"spill loads\n[^\n]*Used (\d+) registers", report)
    out = [(f, int(FP16_P.search(f).group(1)), int(st), int(ld), int(r)) for f, st, ld, r in props if FP16_P.search(f)]
    assert out, "ptxas report lists no fp16-P attention kernel"
    return out


def test_attention_wgmma_not_serialised(ptxas_report):
    bad = sorted({m.group(2) for m in re.finditer(r"\((C751[012])\).*?function '(\w+)'", ptxas_report)
                  if FP16_P.search(m.group(2))})
    assert not bad, "wgmma serialised by ptxas in:\n" + "\n".join(bad)


def test_attention_no_spills(ptxas_report):
    spilling = [f for f, _, st, ld, _ in _kernels(ptxas_report) if st or ld]
    assert not spilling, "attention kernels spill:\n" + "\n".join(spilling)


def test_attention_one_cta_per_sm_fits_register_file(ptxas_report):
    # NWG consumer warpgroups + one producer warpgroup; 65 536 registers per SM
    too_big = [(f, r, 128 * (nwg + 1)) for f, nwg, _, _, r in _kernels(ptxas_report) if r * 128 * (nwg + 1) > 65536]
    assert not too_big, "registers x threads exceed the register file: " + repr(too_big)


def test_attention_ships_three_warpgroups(ptxas_report):
    assert {nwg for _, nwg, _, _, _ in _kernels(ptxas_report)} == {3}
