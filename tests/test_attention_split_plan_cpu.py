"""The split plan of the stage-1 attention (mvsf_attention_split_plan, a host function): which items of the last,
partial wave run as key ranges, and into how many.  An item is one head's group of 192 query rows over ntiles = N / 128
key tiles, one CTA per SM; a part's partial takes 192 x 18 floats of the workspace beyond the tiled planes.  No GPU
needed."""
import ctypes

import pytest

ROWS, MIN_PART_TILES = 192, 16
PART_BYTES = ROWS * 18 * 4
TILE_BYTES = 106496   # tiled planes per 128-key tile


@pytest.fixture(scope="module")
def plan():
    from mvsformerplusplus_b200.build import build
    build()
    from mvsformerplusplus_b200 import _lib

    def f(N, sms):
        r, k = ctypes.c_int(-1), ctypes.c_int(-1)
        _lib.call("mvsf_attention_split_plan", N, sms, ctypes.byref(r), ctypes.byref(k))
        return r.value, k.value
    return f


def _shape(N):
    ntiles = -(-N // 128)
    return ntiles, 4 * -(-N // ROWS), (N + 128) * 896 - ntiles * TILE_BYTES   # key tiles, items, slack bytes


@pytest.mark.parametrize("N, sms, want", [
    (27648, 132, (48, 2)),    # DTU: 576 items, 4 full waves + 48
    (32640, 132, (20, 6)),    # Tanks and Temples: 680 items, 5 full waves + 20; 255 tiles in ranges of 42 and 43
    (25344, 132, (0, 1)),     # 528 items: exactly 4 waves
    (20000, 132, (24, 3)),    # the workspace holds 95 partials: 3 parts, not 132 // 24 = 5
    (27648, 114, (6, 13)),    # 5 waves + 6 items on an H100 PCIe; 216 tiles >= 13 x 16
    (32640, 114, (0, 1)),     # 110 items left over: no two parts of each fit
])
def test_plan_at_workload_sizes(plan, N, sms, want):
    assert plan(N, sms) == want


@pytest.mark.parametrize("sms", [132, 114])
@pytest.mark.parametrize("N", [1, 64, 128, 129, 200, 385, 1000, 4000])
def test_small_n_runs_whole(plan, N, sms):
    assert plan(N, sms) == (0, 1)


@pytest.mark.parametrize("sms", [132, 114])
def test_plan_fits_wave_and_workspace(plan, sms):
    """every N up to 40 000: a split takes the items of the last wave, at least two parts of at least MIN_PART_TILES
    tiles each, no more CTAs than the SMs left for them and no more partials than the workspace has room for, and as
    many parts as those limits allow"""
    splits = 0
    for N in range(1, 40001):
        r, k = plan(N, sms)
        ntiles, items, slack = _shape(N)
        left = items % sms
        best = min(sms // left, slack // (left * PART_BYTES), ntiles // MIN_PART_TILES) if left else 0
        if (r, k) == (0, 1):
            assert best < 2, N
            continue
        splits += 1
        assert r == left and k == best and k >= 2, N
        assert r * k <= sms and r * k * PART_BYTES <= slack and ntiles // k >= MIN_PART_TILES, N
    assert splits > 1000
