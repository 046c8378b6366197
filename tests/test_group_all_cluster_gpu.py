"""The group-all level as one cluster kernel per cloud (tc_group_all_kernel): parity against float64, the fp16 range guard
(any overflow gives bitwise the bf16x3 result), repeatability under CUDA-graph replay, and the shapes that keep the
one-launch-per-layer chain."""
import numpy as np
import pytest
import torch

from oracle import mlp_oracle as mo
from scanobjectnn_b200 import ops, pointnet2_cls_bga, pointnet2_cls_ssg
from scanobjectnn_b200.engine import InferenceEngine, pointnet2_cls_ssg_engine
from scanobjectnn_b200.pointnet_util import add_sa_module_params, pointnet_sa_module
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import VariableStore

from . import gpu_util as G

pytestmark = pytest.mark.gpu


@pytest.fixture(params=[0, 2], ids=["tensor", "tensor_bf16x3"])
def mlp_mode(request):
    ops.set_mlp_mode(request.param)
    try:
        yield request.param
    finally:
        ops.set_mlp_mode(0)


def _level(b, n, c, mlp, seed):
    p = VariableStore(device="cuda", seed=seed)
    add_sa_module_params(p, "sa", 3 + c, mlp, randomize_bn=True)
    rng = np.random.default_rng(seed)
    xyz = make_clouds("ball", b, n, seed=seed)
    pts = np.maximum(rng.standard_normal((b, n, c)), 0.0).astype(np.float32)
    return p, xyz, pts


def _run(p, xyz, pts, mlp):
    _, got, _ = pointnet_sa_module(G.cu(xyz), G.cu(pts), None, None, None, mlp, None, True, False, None, "sa", params=p)
    return got


def _kernels(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.key for e in prof.key_averages()]


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("mlp", [[256, 512, 1024], [256, 256, 512]], ids=["ssg", "narrow"])
@pytest.mark.parametrize("b", [1, 8, 32, 33, 200])
def test_group_all_matches_fp64(b, mlp, mlp_mode):
    """b = 8: 64-wide weight images for the inner layers; b = 200: more clusters than fit on the device at once"""
    n, c = 128, 256
    p, xyz, pts = _level(b, n, c, mlp, 70 + b)
    got = _run(p, xyz, pts, mlp)
    again = _run(p, xyz, pts, mlp)
    assert torch.equal(_bits(got), _bits(again)), "two calls differ"
    _, want, _ = mo.sa_module(xyz, pts, None, None, None, mlp, True, "sa", p)
    G.contract_close(G.npy(got).reshape(want.shape), want, f"sa_group_all b={b} {mlp} mode {mlp_mode}")


def test_group_all_runs_as_one_cluster_kernel():
    p, xyz, pts = _level(32, 128, 256, [256, 512, 1024], 5)
    names = _kernels(lambda: _run(p, xyz, pts, [256, 512, 1024]))
    assert sum("tc_group_all_kernel" in k for k in names) == 1, names


@pytest.mark.parametrize("n,c", [(256, 256), (128, 131)], ids=["n256", "c131"])
def test_ineligible_shapes_keep_the_chain(n, c):
    mlp = [256, 512, 1024]
    p, xyz, pts = _level(8, n, c, mlp, 90 + n + c)
    names = _kernels(lambda: _run(p, xyz, pts, mlp))
    assert not any("tc_group_all_kernel" in k for k in names), names
    got = _run(p, xyz, pts, mlp)
    _, want, _ = mo.sa_module(xyz, pts, None, None, None, mlp, True, "sa", p)
    G.contract_close(G.npy(got).reshape(want.shape), want, f"sa_group_all n={n} c={c}")


@pytest.mark.parametrize("case", ["features", "gamma", "nonfinite_weight"])
def test_range_guard_gives_the_bf16x3_result(case):
    """features x 3e5 overflow layer 0's operands, layer 1's gamma x 2e5 layer 2's, an infinite weight flags layer 2's image:
    the level's output is then bitwise what mode 2 computes"""
    b, n, c, mlp = 32, 128, 256, [256, 512, 1024]
    p, xyz, pts = _level(b, n, c, mlp, 17)
    if case == "features":
        pts = pts * np.float32(3e5)
    elif case == "gamma":
        p["sa/conv1/bn/gamma"] = p["sa/conv1/bn/gamma"] * 2e5
    else:
        w = p["sa/conv2/weights"].clone()
        w.view(-1)[1234] = float("inf")
        p["sa/conv2/weights"] = w
    p.invalidate()
    got = _run(p, xyz, pts, mlp).clone()
    ops.set_mlp_mode(2)
    try:
        want = _run(p, xyz, pts, mlp).clone()
    finally:
        ops.set_mlp_mode(0)
    assert torch.equal(_bits(got), _bits(want)), f"{case}: mode 0 differs from mode 2"
    assert torch.equal(torch.isfinite(got), torch.isfinite(want))
    if case != "nonfinite_weight":
        assert bool(torch.isfinite(got).all())


@pytest.mark.parametrize("model", ["ssg", "bga"])
def test_six_slot_engine_replay_matches_eager(model):
    b, npts = 32, 2048
    mod = {"ssg": pointnet2_cls_ssg, "bga": pointnet2_cls_bga}[model]
    params = mod.init_params(seed=8, randomize_bn=True)
    batches = [torch.from_numpy(make_clouds(kind, b, npts, seed=120 + i)).cuda()
               for i, kind in enumerate(["ball", "shell", "dup", "ball", "shell", "ball"])]
    want = [mod.get_model(x, False, params=params)[0].clone() for x in batches]
    if model == "ssg":
        eng = pointnet2_cls_ssg_engine(params, batch=b, npoints=npts, slots=6)
    else:
        eng = InferenceEngine(lambda x: mod.get_model(x, False, params=params)[0], (b, npts, 3), tuple(want[0].shape), slots=6)
    slots = [eng.submit(x) for x in batches]
    for s, w in zip(slots, want):
        assert torch.equal(_bits(eng.result(s)), _bits(w))
