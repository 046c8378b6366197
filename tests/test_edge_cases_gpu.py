"""Edge cases the reference's ops meet in practice (SURVEY 4/5): empty batches and query sets, shapes at and beyond the
compiled limits, argument errors mapped onto the reference's InvalidArgument behaviour -- never a silent fallback."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from scanobjectnn_b200 import _lib, ops
from scanobjectnn_b200.synthetic import make_clouds

from . import gpu_util as G

pytestmark = pytest.mark.gpu


def test_empty_batch_and_empty_queries_are_noops():
    z = torch.zeros((0, 16, 3), device="cuda")
    assert ops.farthest_point_sample(4, z).shape == (0, 4)
    xyz = G.cu(make_clouds("ball", 2, 64, seed=1))
    q0 = torch.zeros((2, 0, 3), device="cuda")
    idx, cnt = ops.query_ball_point(0.2, 8, xyz, q0)
    assert idx.shape == (2, 0, 8) and cnt.shape == (2, 0)
    d, i = ops.three_nn(q0, xyz)
    assert d.shape == (2, 0, 3)
    assert ops.group_point(torch.zeros((2, 64, 5), device="cuda"), torch.zeros((2, 0, 4), dtype=torch.int32, device="cuda")).shape == (2, 0, 4, 5)


def test_fps_beyond_register_limit_is_refused_not_degraded():
    big = torch.rand((1, 8193, 3), device="cuda")
    with pytest.raises(_lib.PsaError):
        ops.farthest_point_sample(16, big)
    ok = torch.rand((1, 8192, 3), device="cuda")
    assert np.array_equal(ops.farthest_point_sample(16, ok).cpu().numpy(), orc.fps(ok.cpu().numpy(), 16))


def test_ball_query_large_cloud_uses_scan_path_and_matches_oracle():
    # n > 4096: no spatial grid (shared-memory budget) -> ordered scan path
    xyz = make_clouds("ball", 1, 6000, seed=9)
    q = xyz[:, ::60].copy()
    idx, cnt = ops.query_ball_point(0.15, 24, G.cu(xyz), G.cu(q))
    oi, oc = orc.query_ball_point(0.15, 24, xyz, q, contract=True)
    assert np.array_equal(G.npy(idx), oi) and np.array_equal(G.npy(cnt), oc)


def test_ball_query_dense_neighbourhoods_overflow_to_scan():
    # 1500 of 2048 points inside every ball: > 128 hits per query -> grid path hands over to the early-exit scan
    rng = np.random.default_rng(0)
    xyz = (rng.standard_normal((2, 2048, 3)) * 0.02).astype(np.float32)
    xyz[:, 1500:] += 3.0
    q = xyz[:, :64].copy()
    idx, cnt = ops.query_ball_point(0.2, 32, G.cu(xyz), G.cu(q))
    oi, oc = orc.query_ball_point(0.2, 32, xyz, q, contract=True)
    assert np.array_equal(G.npy(idx), oi) and np.array_equal(G.npy(cnt), oc)
    assert (G.npy(cnt) == 32).all()


def test_ball_query_queries_outside_the_cloud():
    xyz = make_clouds("ball", 2, 1024, seed=4)
    q = np.concatenate([xyz[:, :8] * 1.5, xyz[:, :8] + 0.19, np.full((2, 4, 3), 7.0, np.float32)], axis=1).astype(np.float32)
    idx, cnt = ops.query_ball_point(0.2, 16, G.cu(xyz), G.cu(q))
    oi, oc = orc.query_ball_point(0.2, 16, xyz, q, contract=True, fill=0)
    assert np.array_equal(G.npy(idx), oi) and np.array_equal(G.npy(cnt), oc)


def test_knn_graph_k_limits_and_errors():
    x = torch.rand((1, 40, 3), device="cuda")
    assert ops.knn_graph(x, 32).shape == (1, 40, 32)
    with pytest.raises(_lib.PsaError):
        ops.knn_graph(x, 33)                      # a warp keeps at most 32 neighbours per row
    with pytest.raises(ValueError):
        ops.knn_graph(torch.rand((1, 10, 3), device="cuda"), 20)   # k > n: tf.nn.top_k rejects it too
    with pytest.raises(ValueError):
        ops.knn_graph(torch.rand((1, 0, 3), device="cuda"), 20)    # also for an empty cloud


def test_shared_mlp_argument_errors():
    w = torch.rand((8, 64), device="cuda")
    mlp = ops.MlpParams([(w, None, torch.zeros(64, device="cuda"), True)])
    with pytest.raises(ValueError):
        ops.shared_mlp(torch.rand((10, 7), device="cuda"), mlp)            # wrong input width
    with pytest.raises(ValueError):
        ops.shared_mlp(torch.rand((10, 8), device="cuda"), mlp, pool_k=4)  # rows not a multiple of pool_k
    with pytest.raises(ValueError):
        ops.MlpParams([(w, None, torch.zeros(64, device="cuda"), True), (torch.rand((32, 8), device="cuda"), None, torch.zeros(8, device="cuda"), True)])


def test_dtype_and_device_checks():
    xyz = torch.rand((1, 16, 3), device="cuda")
    with pytest.raises(TypeError):
        ops.farthest_point_sample(4, xyz.double())
    with pytest.raises(TypeError):
        ops.gather_point(xyz, torch.zeros((1, 4), dtype=torch.int64, device="cuda"))
    with pytest.raises(ValueError):
        ops.three_interpolate(torch.rand((1, 4, 2), device="cuda"), torch.zeros((1, 8, 2), dtype=torch.int32, device="cuda"),
                              torch.rand((1, 8, 2), device="cuda"))


def test_non_contiguous_inputs_are_accepted():
    base = torch.from_numpy(make_clouds("ball", 2, 256, seed=2)).cuda()
    strided = torch.empty((2, 256, 6), device="cuda")[:, :, :3]
    strided.copy_(base)
    assert not strided.is_contiguous()
    assert torch.equal(ops.farthest_point_sample(32, strided), ops.farthest_point_sample(32, base))
