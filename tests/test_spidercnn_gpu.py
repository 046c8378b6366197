"""SpiderCNN (spidercnn_cls_xyz) on the GPU against the float64 restatement oracle/spidercnn_oracle.py, on the run's own kNN
indices: the kNN order itself, each fused spiderConv shape in the three arithmetic modes, the group-norm affine, the whole model,
the fp16 range guard, determinism, CUDA-graph replay and the allocation peak."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import spidercnn_oracle as so
from scanobjectnn_b200 import ops
from scanobjectnn_b200 import spidercnn_cls_xyz as M
from scanobjectnn_b200.engine import InferenceEngine
from scanobjectnn_b200.synthetic import make_clouds

from . import gpu_util as G

pytestmark = pytest.mark.gpu
LAYERS = [(1, 3, 32), (2, 32, 64), (3, 64, 128), (4, 128, 256)]


@pytest.fixture(params=[0, 1, 2], ids=["tensor", "fma", "tensor_bf16x3"])
def mode(request):
    ops.set_mlp_mode(request.param)
    yield request.param
    ops.set_mlp_mode(0)


@pytest.fixture(scope="module")
def params():
    return M.init_params(seed=11, randomize_bn=True)


def _cloud(b, n, seed=0, kind="ball", scale=1.0):
    return torch.from_numpy(make_clouds(kind, b, n, seed) * np.float32(scale)).cuda()


@pytest.mark.parametrize("kind", ["ball", "shell", "dup"])
def test_knn_point_is_selection_sort_order(kind):
    xyz = _cloud(2, 1024, seed=4, kind=kind)
    _, idx = ops.knn_point(20, xyz, xyz)
    d = xyz[:, None, :, :] - xyz[:, :, None, :]                               # (b, query, dataset, 3)
    dist = ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).contiguous()
    oi, _ = ops.select_top_k(20, dist)
    assert torch.equal(idx, oi[..., :20])
    if orc.refgpu_available():
        ri, _ = G.ref_selection_sort(20, dist)
        assert torch.equal(idx, ri[..., :20])


def _layer_inputs(b, n, cin, seed, scale=1.0):
    xyz = _cloud(b, n, seed, scale=scale)
    _, idx = ops.knn_point(20, xyz, xyz)
    delta = (ops.group_point(xyz, idx) - xyz.unsqueeze(2)).contiguous()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    if cin == 3:
        return xyz, idx, delta, xyz, None, None
    feat = torch.randn((b, n, cin), generator=gen, device="cuda")
    s = torch.rand((b, cin), generator=gen, device="cuda") + 0.5
    u = torch.rand((b, cin), generator=gen, device="cuda") - 0.5
    return xyz, idx, delta, feat, s, u


def _layer64(p, l, idx, delta, feat, s, u):
    h = feat.double() if s is None else torch.relu(feat.double() * s.double()[:, None, :] + u.double()[:, None, :])
    return so.spider_conv_prenorm(h, idx, delta.double(), p, f"fanConv{l}/taylor")


@pytest.mark.parametrize("b,n", [(2, 1024), (2, 2048), (3, 1000), (1, 1024)])
@pytest.mark.parametrize("l,cin,cout", LAYERS)
def test_spider_conv_matches_float64(mode, params, b, n, l, cin, cout):
    _, idx, delta, feat, s, u = _layer_inputs(b, n, cin, seed=l + n)
    taylor, w, bias, _, _ = params.spider(f"fanConv{l}/taylor")
    y = ops.spider_conv(delta, idx, feat, taylor, w, bias, s, u)
    want = _layer64(params, l, idx, delta, feat, s, u)
    G.contract_close(G.npy(y), G.npy(want), f"fanConv{l} b={b} n={n} mode={mode}")


def test_group_norm_affine_matches_float64():
    gen = torch.Generator(device="cuda").manual_seed(1)
    b, n, c, groups = 3, 1000, 64, 16
    y = torch.randn((b, n, c), generator=gen, device="cuda") * 3 + 5
    y[1, :, 4:8] = 0.37                                                       # cloud 1, group 1: constant
    gamma = torch.rand(c, generator=gen, device="cuda") + 0.5
    beta = torch.rand(c, generator=gen, device="cuda") - 0.5
    out, s, u = ops.group_norm_affine(y, gamma, beta, groups, 1e-6, apply=True, relu=True)
    yg = y.double().reshape(b, n, groups, c // groups)
    mean = yg.mean(dim=(1, 3))
    var = ((yg - mean[:, None, :, None]) ** 2).mean(dim=(1, 3))
    s64 = gamma.double() / torch.sqrt(var.repeat_interleave(c // groups, dim=1) + 1e-6)
    u64 = beta.double() - mean.repeat_interleave(c // groups, dim=1) * s64
    assert float(var[1, 1]) == 0.0
    assert float(((s.double() - s64).abs() / s64.abs()).max()) < 1e-6
    assert float(((u.double() - u64).abs() / (beta.double().abs() + (mean.repeat_interleave(c // groups, dim=1) * s64).abs())).max()) < 1e-6
    G.contract_close(G.npy(out), G.npy(torch.relu(so.group_norm(y.double(), gamma, beta, groups))), "group norm + relu")


def test_topk_pool_matches_torch_topk():
    gen = torch.Generator(device="cuda").manual_seed(2)
    y = torch.randn((2, 1000, 96), generator=gen, device="cuda")
    y[0, 10:20, 3] = 7.0                                                      # a repeated maximum
    out = ops.topk_pool(y, 2)
    want = torch.topk(y.permute(0, 2, 1), 2, dim=-1).values
    assert torch.equal(out, want)
    assert float(out[0, 3, 0]) == float(out[0, 3, 1]) == 7.0


@pytest.mark.parametrize("b,n", [(4, 1024), (2, 1000)])
def test_model_matches_float64(mode, params, b, n):
    xyz = _cloud(b, n, seed=21)
    logits, ep = M.get_model(xyz, False, params=params, return_end_points=True)
    want_logits, want_pooled, _ = so.forward(xyz, ep["idx"], params)
    G.contract_close(G.npy(ep["pooled"]), G.npy(want_pooled), f"pooled mode={mode}")
    G.contract_close(G.npy(logits), G.npy(want_logits), f"logits mode={mode}")


def test_range_guard_reruns_on_bf16x3(params):
    """A cloud scaled x100 puts the cubic Taylor terms far past 65504: the fp16x2 pass must raise its flag, and what mode 0
    returns is then bit for bit what mode 2 computes."""
    for l, cin, cout in LAYERS[1:]:
        _, idx, delta, feat, s, u = _layer_inputs(2, 1024, cin, seed=5, scale=100.0)
        taylor, w, bias, _, _ = params.spider(f"fanConv{l}/taylor")
        got = {}
        for m in (0, 2):
            ops.set_mlp_mode(m)
            try:
                got[m] = ops.spider_conv(delta, idx, feat, taylor, w, bias, s, u)
            finally:
                ops.set_mlp_mode(0)
        assert torch.equal(got[0], got[2]), f"fanConv{l}: mode 0 is not the bf16x3 rerun"
        G.contract_close(G.npy(got[0]), G.npy(_layer64(params, l, idx, delta, feat, s, u)), f"fanConv{l} x100")
    xyz = _cloud(2, 1024, seed=6, scale=100.0)
    out = {}
    for m in (0, 2):
        ops.set_mlp_mode(m)
        try:
            out[m] = M.get_model(xyz, False, params=params, return_end_points=True)
        finally:
            ops.set_mlp_mode(0)
    assert torch.equal(out[0][0], out[2][0])
    want_logits, _, _ = so.forward(xyz, out[0][1]["idx"], params)
    G.contract_close(G.npy(out[0][0]), G.npy(want_logits), "logits x100")


def test_deterministic_and_graph_replay_is_bit_equal(params):
    xyz = _cloud(8, 1024, seed=8)
    a = M.get_model(xyz, False, params=params)
    b = M.get_model(xyz, False, params=params)
    assert torch.equal(a, b)
    eng = InferenceEngine(lambda x: M.get_model(x, False, params=params), (8, 1024, 3), (8, M.NUM_CLASSES), slots=1)
    slot = eng.submit(xyz)
    assert torch.equal(eng.result(slot), a)


def test_allocation_peak_rules_out_materialising():
    p = M.init_params(seed=3)
    xyz = _cloud(32, 1024, seed=9)
    M.get_model(xyz, False, params=p)                                         # warm-up: cached weights and taylor matrices
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    M.get_model(xyz, False, params=p)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print(f"[peak] B=32 N=1024 forward: {peak / 2**20:.1f} MiB above the inputs and weights")
    assert peak < 256 * 2**20
