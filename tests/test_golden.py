"""Golden vectors produced by the REFERENCE's own code (tests/golden/make_golden.py: its CUDA kernels run on the GPU,
its CPU ops run on x86-64).  CPU half: the oracle restatement must reproduce them bit for bit -- this is what pins
the oracle.  GPU half (-m gpu): this repo's kernels must reproduce them too."""
import os

import numpy as np
import pytest

from oracle import oracle as orc
from scanobjectnn_b200.synthetic import make_clouds

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = [("ball", 1001), ("shell", 1002), ("dup", 1003)]


def _load(name):
    return np.load(os.path.join(GOLD, name))


@pytest.mark.parametrize("kind,seed", CASES)
def test_oracle_reproduces_reference_gpu_kernels(kind, seed):
    g = _load(f"ref_gpu_{kind}.npz")
    xyz = make_clouds(kind, 4, 2048, seed=seed)
    fps1 = orc.fps(xyz, 512)
    assert np.array_equal(fps1, g["fps1"])
    l1 = orc.gather_point(xyz, fps1)
    bq1, cnt1 = orc.query_ball_point(0.2, 32, xyz, l1, contract=True)
    assert np.array_equal(bq1, g["bq1"]) and np.array_equal(cnt1, g["cnt1"])
    fps2 = orc.fps(l1, 128)
    assert np.array_equal(fps2, g["fps2"])
    l2 = orc.gather_point(l1, fps2)
    bq2, cnt2 = orc.query_ball_point(0.4, 64, l1, l2, contract=True)
    assert np.array_equal(bq2, g["bq2"]) and np.array_equal(cnt2, g["cnt2"])


def test_oracle_reproduces_reference_selection_sort():
    g = _load("ref_gpu_selection_sort.npz")
    rng = np.random.default_rng(77)
    d = rng.random((2, 8, 200), dtype=np.float32)
    d[0, 0, 10:40] = d[0, 0, 3]
    d[1, 1, :] = 0.25
    oi, ov = orc.selection_sort(16, d)
    assert np.array_equal(oi, g["outi"]) and np.array_equal(ov, g["out"])


def test_oracle_reproduces_reference_cpu_ops():
    g = _load("ref_cpu_three_nn.npz")
    xyz1 = make_clouds("shell", 2, 2048, seed=2001)
    xyz2 = make_clouds("ball", 2, 512, seed=2002)
    dist, idx = orc.three_nn(xyz1, xyz2)
    assert np.array_equal(idx, g["idx"]) and np.array_equal(dist, g["dist"])
    pts = np.random.default_rng(2003).standard_normal((2, 512, 16)).astype(np.float32)
    assert np.array_equal(orc.three_interpolate(pts, idx, orc.three_weights(dist)), g["interp"])
    qb, _ = orc.query_ball_point(0.2, 32, xyz2, xyz2[:, ::4].copy(), contract=False, fill=-1)
    assert np.array_equal(qb, _load("ref_cpu_ball_query.npz")["idx"])


@pytest.mark.gpu
@pytest.mark.parametrize("kind,seed", CASES)
def test_kernels_reproduce_reference_gpu_kernels(kind, seed):
    import torch

    from scanobjectnn_b200 import ops
    g = _load(f"ref_gpu_{kind}.npz")
    xyz = torch.from_numpy(make_clouds(kind, 4, 2048, seed=seed)).cuda()
    fps1, l1 = ops.farthest_point_sample_and_gather(512, xyz)
    assert np.array_equal(fps1.cpu().numpy(), g["fps1"])
    bq1, cnt1 = ops.query_ball_point(0.2, 32, xyz, l1)
    assert np.array_equal(bq1.cpu().numpy(), g["bq1"]) and np.array_equal(cnt1.cpu().numpy(), g["cnt1"])
    fps2, l2 = ops.farthest_point_sample_and_gather(128, l1)
    assert np.array_equal(fps2.cpu().numpy(), g["fps2"])
    bq2, cnt2 = ops.query_ball_point(0.4, 64, l1, l2)
    assert np.array_equal(bq2.cpu().numpy(), g["bq2"]) and np.array_equal(cnt2.cpu().numpy(), g["cnt2"])


@pytest.mark.gpu
def test_kernels_reproduce_reference_cpu_ops():
    import torch

    from scanobjectnn_b200 import ops
    g = _load("ref_cpu_three_nn.npz")
    xyz1 = torch.from_numpy(make_clouds("shell", 2, 2048, seed=2001)).cuda()
    xyz2 = torch.from_numpy(make_clouds("ball", 2, 512, seed=2002)).cuda()
    pts = torch.from_numpy(np.random.default_rng(2003).standard_normal((2, 512, 16)).astype(np.float32)).cuda()
    out, dist, idx, _ = ops.three_nn_interpolate(xyz1, xyz2, pts, return_aux=True)
    assert np.array_equal(idx.cpu().numpy(), g["idx"]) and np.array_equal(dist.cpu().numpy(), g["dist"])
    assert np.array_equal(out.cpu().numpy(), g["interp"])
