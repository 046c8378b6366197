"""The routing of the training GEMM's launchers (csrc/train.cu), restated in tests/restate.py: its workspace formula against
psa_train_dense_workspace_bytes, and the paths the cases of tests/test_train_gemm_gpu.py take.  No GPU needed."""
import itertools

from scanobjectnn_b200 import _lib

from . import restate as R


def test_workspace_matches_the_plan():
    lib = _lib.load()
    for rows, K, N in itertools.product((1, 33, 127, 128, 200, 256, 257, 1024, 1025, 3000, 40009, 300000),
                                        (3, 40, 64, 65, 127, 128, 200, 512, 513, 1024), (1, 15, 48, 64, 65, 128, 192, 256, 1024)):
        assert lib.psa_train_dense_workspace_bytes(rows, K, N) == R.train_dense_workspace(rows, K, N), (rows, K, N)


def test_the_tensor_core_gate():
    assert R.tc_train_fwd_eligible(128, 128, 128) and R.tc_train_fwd_eligible(128, 512, 256)
    assert not R.tc_train_fwd_eligible(127, 128, 128) and not R.tc_train_fwd_eligible(128, 127, 128)
    assert not R.tc_train_fwd_eligible(128, 513, 128) and not R.tc_train_fwd_eligible(128, 128, 192)


def _fwd(case):
    _, rows, K, N, act, x, _, _ = case
    return R.train_fwd_plan(rows, K, N, ld={"slice": K + 8, "ld_odd": K + 3}.get(x, K), mask=act == "bn_mask")


def test_forward_cases_reach_every_path():
    plans = {c[0]: (_fwd(c), c) for c in R.FWD_CASES}
    paths = {(p["path"], p.get("bn"), c[7]) for p, c in plans.values()}
    # each path: the tensor cores, the small-M split (with and without statistics), one fp32 pass; both fp32 tile widths
    assert {("tc", None, True), ("tc", None, False), ("split", 128, True), ("split", 64, False), ("fp32", 64, True), ("fp32", 128, True)} <= paths
    # both sides of every bound of the tensor-core gate: rows 127 / 128, K 127 / 128 and 512 / 513, N 128 / 192
    assert plans["tc_gate_in"][0]["path"] == "tc" and plans["tc_k512"][0]["path"] == "tc"
    for case, (rows, K, N) in (("rows127", (127, 128, 128)), ("k127", (128, 127, 128)), ("k513", (256, 513, 256)), ("n192", (256, 200, 192))):
        assert plans[case][0]["path"] != "tc" and plans[case][1][1:4] == (rows, K, N)
    # K not a multiple of 64 (the padded K block) with the previous layer's batch norm on the tensor cores
    assert plans["tc_kpad"][0]["path"] == "tc" and plans["tc_kpad"][1][2] % 64 and plans["tc_kpad"][1][4] == "bn"
    # eligible shapes that leave the tensor cores: a dropout mask, a column slice
    for case in ("tc_shape_mask", "slice"):
        rows, K, N = plans[case][1][1:4]
        assert R.tc_train_fwd_eligible(rows, K, N) and plans[case][0]["path"] != "tc"
    # x through the scalar loads: ld % 4 != 0 and a 4-byte offset
    assert {c[5] for c in R.FWD_CASES} == {"dense", "slice", "ld_odd", "offset"}
    assert {c[6] for c in R.FWD_CASES} == {True, False}


def test_input_gradient_cases_reach_every_path():
    plans = [(R.train_bwd_input_plan(rows, K, N, R.train_dense_workspace(rows, K, N)), (rows, K, N, src, skip, ld))
             for _, rows, K, N, src, skip, ld in R.BWD_INPUT_CASES]
    assert {(p["path"], p["bn"]) for p, _ in plans} == {("split", 64), ("split", 128), ("fp32", 64), ("fp32", 128)}
    for p, (rows, K, N, src, skip, ld) in plans:
        # without a workspace the split cases run one split
        assert R.train_bwd_input_plan(rows, K, N, 0)["path"] == "fp32"
        if p["path"] == "split":
            assert p["splits"] > 1
    # col_skip into an odd ld_dx on both paths
    assert {p["path"] for p, c in plans if c[4] and c[5] % 2} == {"split", "fp32"}
    srcs = {f for c in R.BWD_INPUT_CASES for f in c[4].split("+")}
    assert srcs == {"plain", "mask", "gate", "coeffs", "pool20", "pool32", "scalar"}
    assert any(p["path"] == "split" and "pool20" in c[3] for p, c in plans)


def test_weight_gradient_cases_reach_every_path():
    plans = [(R.train_bwd_weight_plan(rows, K, N), (rows, K, N, act, x, src)) for _, rows, K, N, act, x, src in R.BWD_WEIGHT_CASES]
    assert {(p["bm"], p["bn"]) for p, _ in plans} == {(64, 64), (64, 128), (128, 64), (128, 128)}
    # one split, and the large case at two CTAs per SM over its two output tiles
    assert any(p["splits"] == 1 for p, _ in plans) and max(p["splits"] for p, _ in plans) == R.PLAN_SMS
    # many splits over rows that are a multiple of neither 16 nor the split length
    assert any(p["splits"] > 1 and c[0] % 16 and c[0] % p["kps"] for p, c in plans)
    assert any("pool" in c[5] for _, c in plans) and any("scalar" in c[5] for _, c in plans)
    assert {c[3] for _, c in plans} == {"raw", "bn", "bn_mask"} and {"ld_odd", "offset"} <= {c[4] for _, c in plans}
