"""The exact-weight attention inputs of tests/attention_exact_common.py, checked without a GPU: every case the GPU module
builds meets the premise (members within 5e-5 of their level, non-members at least 44 below level 0, a level-0 member
first in every key range), softmax_tile's fp16 P reproduces the intended weights, the reference is a plain fp64 softmax
attention where the weights are all equal, and the constants the module restates are the ones in the sources."""
import math
import os

import numpy as np
import pytest

from tests import attention_exact_common as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGE1_N = [1, 64, 128, 129, 385, 4000, 27648, 32640]
VIT_N = [2, 13, 127, 128, 129, 1370, 1729, 2041]


@pytest.fixture(scope="module")
def lib():
    from mvsformerplusplus_b200.build import build
    build()


def _source(name):
    return " ".join(open(os.path.join(ROOT, "mvsformerplusplus_b200", "csrc", name)).read().split())


def test_constants_follow_the_sources():
    src = _source("softmax_attention.cuh")
    assert f"mb[h] = mx - {E.P_BIAS:.1f}f;" in src
    assert f"if (j * 128 + 8 * (i >> 2) + 2 * q + (i & 1) >= N) S[i] = {E.MASK:.0e}f;".replace("e+", "e") in src
    assert f"{E.VIT_SCALE}f * {E.LOG2E!r}f);" in _source("vit.cu")
    tr = _source("costreg_tr.cu")
    assert f"const float scale_log2e = softmax_scale * {E.LOG2E!r}f;" in tr
    assert f"N, softmax_scale * {E.LOG2E!r}f, (cudaStream_t)stream);" in tr
    assert E.VIT_SCALE == 64 ** -0.5


def _stage1_cases():
    """(N, SMs) of every stage-1 case of the GPU module on 132 and 114 SMs, the split-plan N included"""
    from tests import test_gpu_attention_split as SPLIT
    out = set()
    for sms in (132, 114):
        out |= {(N, sms) for N in STAGE1_N}
        for case in SPLIT.CASES:
            try:
                out.add((SPLIT.pick(sms, case), sms))
            except pytest.skip.Exception:
                pass
    return sorted(out)


def _check(case):
    E.premise(case)
    for h in range(case.geo.heads):
        S, w, *_ = E.intended_weights(case, h)
        want = (w * 2.0 ** E.P_BIAS).astype(np.float16)
        # the kernel's scores differ from these by its hi + lo split and fp32 sums, far below 2e-4
        for d in (0.0, 2e-4, -2e-4):
            assert np.array_equal(E.emulate_p(S + d * (w > 0)), want), (h, d)


def test_premise_and_fp16_weights_stage1(lib):
    cases = _stage1_cases()
    splits = {sms: 0 for sms in (132, 114)}
    for N, sms in cases:
        plan = E.split_plan(N, sms)
        splits[sms] += plan[0] > 0
        case = E.make_case(E.STAGE1, N, plan=plan, seed=N)
        _check(case)
        if plan[0]:
            # some part of the split holds no member of some group, so the merge's 2^(m_p - m) matters
            assert any(len(case.ranges) > 1 and not ((case.members(h, g) >= 128 * t0) & (case.members(h, g) < 128 * t1)).any()
                       for h in range(4) for g in range(16) if case.members(h, g).size for t0, t1 in case.ranges)
    assert splits[132] >= 3 and splits[114] >= 2, splits


@pytest.mark.parametrize("n", [1, 3, 5])
def test_premise_and_fp16_weights_vit(n):
    for N in VIT_N:
        case = E.make_case(E.VIT, N, n=n, scale=E.VIT_SCALE, ldq=2316, seed=n * 10000 + N)
        _check(case)
        kinds = {case.kinds[(h, g)] for h in range(12) for g in range(64)}
        assert kinds == ({"uniform", "ties", "levels"} if N > 2 else {"uniform", "ties", "levels"} & kinds)


def test_members_at_the_tiling_edges():
    for N in (129, 385, 4000, 1729):
        case = E.make_case(E.STAGE1, N, seed=N)
        for h in range(4):
            kg = case.kgroup[h]
            assert kg[0] >= 0 and kg[N - 1] >= 0
            if N % 128:   # the partial last tile's only member is key N - 1
                assert (kg[128 * (N // 128):] >= 0).sum() == 1
            for g in range(16):
                lv = case.klevel[h][case.members(h, g)]
                if case.kinds[(h, g)] == "ties":
                    assert lv.size >= 3 and (lv == 0).all()
                elif case.kinds[(h, g)] == "levels" and N > 129:
                    assert set(lv) == set(range(E.LEVELS))


@pytest.mark.parametrize("geo, N, n", [(E.STAGE1, 385, 1), (E.STAGE1, 32640, 1), (E.VIT, 1729, 3), (E.VIT, 13, 5)])
def test_reference_is_fp64_softmax_where_weights_are_equal(geo, N, n):
    """rows of uniform and tie groups: the reference equals softmax(q k^T scale) v in fp64 within 1e-12"""
    scale = E.VIT_SCALE if geo is E.VIT else E.STAGE1_SCALE
    case = E.make_case(geo, N, n=n, scale=scale, seed=N)
    want, terms = E.reference(case)
    checked = 0
    for h in range(geo.heads):
        for b in range(n):
            q = case.qkv[b * N:(b + 1) * N, case.cols("q", h)].astype(np.float64)
            k = case.qkv[b * N:(b + 1) * N, case.cols("k", h)].astype(np.float64)
            v = case.qkv[b * N:(b + 1) * N, case.cols("v", h)].astype(np.float64)
            for g in range(geo.hd):
                rows = np.nonzero(case.qgroup[h] == g)[0]
                if not rows.size or case.kinds[(h, g)] == "levels":
                    continue
                s = k @ q[rows[0]] * scale
                p = np.exp(s - s.max())
                got = p @ v / p.sum()
                r = b * N + rows[0]
                c = slice(h * geo.hd, (h + 1) * geo.hd)
                assert (np.abs(got - want[r, c]) / terms[r, c]).max() < 1e-12, (h, b, g)
                checked += 1
    assert checked > geo.heads


def test_error_sees_one_lost_lo_part():
    """the measure the GPU module uses: V rounded to fp16 in one head moves it far above the GPU bar"""
    case = E.make_case(E.STAGE1, 4000, seed=4000)
    want, terms = E.reference(case)
    assert E.error(want, case, want, terms) == 0.0
    bad = case.qkv.copy()
    c = case.cols("v", 1)
    bad[:, c] = bad[:, c].astype(np.float16).astype(np.float32)
    got, _ = E.reference(E.Case(**{**case.__dict__, "qkv": bad}))
    assert E.error(got, case, want, terms) > 1e-5
    assert math.isfinite(E.error(got, case, want, terms))
