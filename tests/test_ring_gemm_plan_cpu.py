"""The plans of the shared ring GEMM's three ops, restated in tests/restate.py, against the library's workspace queries in modes 0
and 2; and the plan facts that tests/test_ring_gemm_gpu.py names its cases by.  No GPU needed."""
import itertools

import pytest

from scanobjectnn_b200 import _lib

from . import restate as R


@pytest.fixture(params=[0, 2], ids=["fp16x2", "bf16x3"])
def np_(request):
    lib = _lib.load()
    assert lib.psa_set_mlp_mode(request.param) == 0
    yield 2 if request.param == 0 else 3
    lib.psa_set_mlp_mode(0)


def test_conv3d_workspace_matches_the_plan(np_):
    lib = _lib.load()
    for b, r, k, c, co in itertools.product((1, 3, 32, 128, 300), (1, 2, 3, 5), (1, 3, 5), (64, 128, 256), (32, 64, 96, 128, 256)):
        assert lib.psa_conv3d_workspace_bytes(b, r, k, c, co) == R.conv_plan(b, r, k, c, co, np_)["total"], (b, r, k, c, co)
    # the shapes the FMA kernel takes ask for none
    assert lib.psa_conv3d_workspace_bytes(32, 5, 1, 20, 64) == 0 and lib.psa_conv3d_workspace_bytes(32, 5, 3, 64, 48) == 0


def test_dense_workspace_matches_the_plan(np_):
    lib = _lib.load()
    for rows, K, N in itertools.product((128, 255, 17025), (4, 60, 64, 100, 128, 480), (1, 63, 64, 65, 128, 129, 192, 384)):
        assert lib.psa_dense_elu_affine_workspace_bytes(rows, K, N) == R.pd_plan(rows, K, N, np_)["total"], (rows, K, N)
    assert lib.psa_dense_elu_affine_workspace_bytes(127, 64, 64) == 0          # rows < 128: the FMA kernel
    assert lib.psa_dense_elu_affine_workspace_bytes(1000, 62, 64) == 0         # K % 4 != 0


def test_spider_workspace_matches_the_plan(np_):
    lib = _lib.load()
    for (b, n), c, k, t, co in itertools.product([(1, 127), (1, 128), (3, 1000), (3, 5675)], (3, 32, 64, 96), (1, 3, 4, 20, 32),
                                                 (2, 3, 5), (32, 64, 128, 192, 256)):
        assert lib.psa_spider_conv_workspace_bytes(b, n, c, k, t, co) == R.spider_plan(b, n, c, k, t, co)["total"], (b, n, c, k, t, co)


def test_empty_units_need_one_channel_block():
    """A conv3d unit has no K blocks when its tile has fewer active blocks than the plan has splits.  Splits are at most 16, and
    for r >= 2, k >= 3 every tile has at least 8 active taps (each axis keeps the centre and one neighbour); at r = 1 or k = 1 the
    reach is one tap and the splits at most c / 128.  So only c = 64 (one 64-channel block per tap) makes empty units."""
    seen = set()
    for b, r, k, c in itertools.product((1, 16, 64, 128, 200), (1, 2, 3), (1, 3, 5), (64, 128, 192)):
        if any(0 in nb for nb in R.conv_unit_blocks(b, r, k, c, R.conv_plan(b, r, k, c, 64, 2)["splits"])):
            seen.add(c)
    assert seen == {64}


def test_the_gpu_cases_take_the_paths_they_are_named_for():
    # empty units: b = 128, r = 2, k = 3, c = 64 -> 8 one-voxel tiles with 8 active taps each and 13 splits
    p = R.conv_plan(128, 2, 3, 64, 64, 2)
    assert p["tiles"] == 8 and p["splits"] == 13 and p["Nt"] == 64
    assert all(sorted(nb) == [0] * 5 + [1] * 8 for nb in R.conv_unit_blocks(128, 2, 3, 64, 13))
    # c = 128: 16 splits over 16 active blocks, one block per unit
    p = R.conv_plan(128, 2, 3, 128, 64, 2)
    assert p["splits"] == 16 and all(nb == [1] * 16 for nb in R.conv_unit_blocks(128, 2, 3, 128, 16))
    # conv3d with c_out % 64 = 32: Np padding on 64-wide tiles, and on 128-wide tiles past 132 units (r = 1, 17025 rows)
    assert R.conv_plan(255, 1, 3, 64, 32, 2)["Np"] == 64
    p = R.conv_plan(17025, 1, 3, 64, 96, 2)
    assert p["Np"] == 128 and p["Nt"] == 128 and p["units"] > R.PLAN_SMS and p["splits"] == 1
    p = R.conv_plan(17023, 1, 5, 128, 32, 2)
    assert p["Nt"] == 64 and p["units"] > R.PLAN_SMS
    # dense: NC = 1 and NC = 2, the second chunk of N = 65 padded, more units than SMs for each
    assert R.pd_plan(17025, 60, 65, 2)["Nt"] == 128 and R.pd_plan(17025, 60, 65, 2)["units"] > R.PLAN_SMS
    assert R.pd_plan(6017, 100, 129, 2)["Nt"] == 64 and R.pd_plan(6017, 100, 129, 2)["units"] > R.PLAN_SMS
    assert R.pd_plan(255, 68, 192, 2)["Nt"] == 64 and R.pd_plan(255, 68, 192, 2)["Np"] == 192
    # spider, c = 32: 64-wide tiles on 134 units, 128-wide tiles on 134 units
    assert R.spider_plan(3, 5675, 32, 4, 3, 64)["units"] > R.PLAN_SMS
    p = R.spider_plan(3, 5675, 32, 4, 3, 128)
    assert p["Nt"] == 128 and p["units"] > R.PLAN_SMS
