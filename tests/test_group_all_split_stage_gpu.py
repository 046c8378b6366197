"""The group-all cluster kernel stores the slices of layers 0 and 1 once, already split into the next layer's fp16 A fragments,
and its readers load those pieces instead of splitting fp32 values themselves.  Its output must stay bitwise what the
one-launch-per-layer chain computes, around the one-wave boundary (30 clusters fit at once on an H100), for each of the three
slice shapes, and through the range guard when a layer-0 input leaves the fp16 range.

The chain is the same level on a copy of the features whose rows are not 16-byte aligned, which the cluster kernel does not take;
past the range guard it is the bf16x3 chain of psa_set_mlp_mode(2), which the kernel's reruns reproduce."""
import numpy as np
import pytest
import torch

from scanobjectnn_b200 import ops
from scanobjectnn_b200.pointnet_util import add_sa_module_params, pointnet_sa_module
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import VariableStore

pytestmark = pytest.mark.gpu

N, C = 128, 256
MLPS = {"1x1": [256, 256, 512], "1x2": [256, 512, 1024], "2x1": [512, 256, 512]}   # 64-column chunks of the two slices


def _level(b, mlp, seed):
    p = VariableStore(device="cuda", seed=seed)
    add_sa_module_params(p, "sa", 3 + C, mlp, randomize_bn=True)
    xyz = torch.from_numpy(make_clouds("ball", b, N, seed=seed)).cuda()
    rng = np.random.default_rng(seed)
    pts = torch.from_numpy(np.maximum(rng.standard_normal((b, N, C)), 0.0).astype(np.float32)).cuda()
    return p, xyz, pts


def _misaligned(t):
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    out = buf[1:].view(t.shape)
    out.copy_(t)
    assert out.data_ptr() % 16 != 0
    return out


def _run(p, xyz, pts, mlp):
    return pointnet_sa_module(xyz, pts, None, None, None, mlp, None, True, False, None, "sa", params=p)[1].clone()


def _device_kernels(fn):
    """The names of the device records (kernels, memsets) the profiler took while fn ran.  Now and then a window delivers no
    device record at all although all its host calls are there, cudaLaunchKernel included: such a window does not show which
    kernels ran, so fn is profiled again."""
    for _ in range(3):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if names:
            return names
    raise AssertionError("three profiler windows without a device record")


def _ran_cluster_kernel(fn):
    return any("tc_group_all_kernel" in k for k in _device_kernels(fn))


def _check(b, mlp, seed):
    p, xyz, pts = _level(b, mlp, seed)
    chain_pts = _misaligned(pts)
    assert _ran_cluster_kernel(lambda: _run(p, xyz, pts, mlp))
    assert not _ran_cluster_kernel(lambda: _run(p, xyz, chain_pts, mlp))
    got, want = _run(p, xyz, pts, mlp), _run(p, xyz, chain_pts, mlp)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32)), f"b={b} {mlp}: cluster kernel differs from the chain"


@pytest.mark.parametrize("shape", sorted(MLPS))
@pytest.mark.parametrize("b", [1, 29, 30, 31, 32, 33])
def test_split_stage_matches_the_chain(b, shape):
    _check(b, MLPS[shape], 300 + b)


@pytest.mark.parametrize("shape", sorted(MLPS))
def test_split_stage_range_guard_matches_the_bf16x3_chain(shape):
    """one layer-0 input of 1e6 leaves the fp16 range: the kernel's flag fires and the level is bitwise the bf16x3 chain's"""
    mlp = MLPS[shape]
    p, xyz, pts = _level(32, mlp, 77)
    pts[5, 17, 100] = 1e6
    assert _ran_cluster_kernel(lambda: _run(p, xyz, pts, mlp))
    got = _run(p, xyz, pts, mlp)
    ops.set_mlp_mode(2)
    try:
        want = _run(p, xyz, pts, mlp)
    finally:
        ops.set_mlp_mode(0)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32)), f"{mlp}: the range guard's result differs from mode 2"
    assert bool(torch.isfinite(got).all())
