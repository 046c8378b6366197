"""GPU parity of the fused grouped-MLP kernels and the SSG model against the fp64 restatement
(oracle/mlp_oracle.py).  Tolerance: 1e-5 absolute on O(1) activations (BASELINE.json north_star);
the plain-fp32 restatement's own distance from fp64 is printed beside it for scale."""
import numpy as np
import pytest
import torch

from oracle import mlp_oracle as mo
from oracle import oracle as orc
from scanobjectnn_b200 import ops, pointnet2_cls_ssg
from scanobjectnn_b200.pointnet_util import (add_fp_module_params, add_sa_module_msg_params, add_sa_module_params, pointnet_fp_module,
                                              pointnet_sa_module, pointnet_sa_module_msg)
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import VariableStore

from . import gpu_util as G

pytestmark = pytest.mark.gpu
TOL = G.CONTRACT_TOL


def _store(seed=0):
    return VariableStore(device="cuda", seed=seed)


@pytest.fixture(params=["tensor", "fma", "tensor_bf16x3"])
def mlp_mode(request):
    """0 = auto (tensor-core kernels where the shapes allow: fp16x2 operands + range guard), 1 = fp32 FMA kernels,
    2 = tensor-core kernels with bf16x3 operands (also what the range guard reruns on)"""
    ops.set_mlp_mode({"tensor": 0, "fma": 1, "tensor_bf16x3": 2}[request.param])
    yield request.param
    ops.set_mlp_mode(0)


@pytest.mark.parametrize("rows,pool_k,chans", [(256, 1, [7, 64]), (4096, 128, [259, 256, 512, 1024]), (32, 1, [1024, 512, 256, 15]),
                                               (300, 1, [131, 128, 40]), (640, 32, [64, 64]), (2 * 2048, 2048, [320, 1024]),
                                               (1280, 8, [6, 64, 128]),
                                               # dense tensor-core kernels, edge shapes: partial row tile + K tail; odd K (scalar x loads);
                                               # pool 32 / 64 / 256 (atomicMax path); K > 512 and N = 64; 8 K-blocks x 3 n-tiles
                                               (1000, 1, [100, 128]), (1000, 1, [99, 256]), (1024, 32, [64, 128, 256]), (1024, 64, [128, 128]),
                                               (512, 256, [200, 128]), (384, 1, [576, 128]), (384, 1, [64, 64]), (130, 1, [512, 384])])
def test_shared_mlp_matches_fp64(rows, pool_k, chans, mlp_mode):
    p = _store(rows)
    scopes = []
    for i in range(len(chans) - 1):
        p.add_conv2d(f"m/conv{i}", chans[i], chans[i + 1], bn=(i % 2 == 0), randomize_bn=True)
        scopes.append(f"m/conv{i}")
    relus = [True] * (len(scopes) - 1) + [pool_k > 1]
    rng = np.random.default_rng(rows)
    x = rng.standard_normal((rows, chans[0])).astype(np.float32)
    got = G.npy(ops.shared_mlp(G.cu(x), p.mlp(scopes, relus), pool_k=pool_k))
    want = mo.mlp_chain(x, p, scopes, relus)
    if pool_k > 1:
        want = want.reshape(rows // pool_k, pool_k, -1).max(1)
    G.contract_close(got, want, f"shared_mlp {chans} pool {pool_k}")


@pytest.mark.parametrize("kind", ["ball", "shell"])
@pytest.mark.parametrize("n,m,r,k,c,mlp", [(2048, 512, 0.2, 32, 0, [64, 64, 128]), (512, 128, 0.4, 64, 128, [128, 128, 256]),
                                           (2048, 512, 0.2, 64, 0, [64, 64, 128]), (300, 50, 0.3, 20, 5, [32, 48]),
                                           (256, 64, 0.3, 16, 64, [64]), (512, 100, 0.4, 32, 64, [128, 64, 128]),
                                           (512, 37, 0.5, 128, 16, [128, 256]), (1024, 333, 0.3, 32, 128, [128, 128, 128])])
def test_sa_module_infer_matches_fp64(kind, n, m, r, k, c, mlp, mlp_mode):
    p = _store(n + k)
    add_sa_module_params(p, "sa", 3 + c, mlp, randomize_bn=True)
    rng = np.random.default_rng(n)
    xyz = make_clouds(kind, 2, n, seed=n)
    pts = rng.standard_normal((2, n, c)).astype(np.float32) if c else None
    new_xyz, got, idx = pointnet_sa_module(G.cu(xyz), G.cu(pts) if c else None, m, r, k, mlp, None, False, False, None, "sa", params=p)
    oxyz, want, oidx = mo.sa_module(xyz, pts, m, r, k, mlp, False, "sa", p)
    assert np.array_equal(G.npy(new_xyz), oxyz)
    assert np.array_equal(G.npy(idx), oidx)
    err = np.abs(G.npy(got) - want).max()
    f32 = np.abs(mo.sa_module(xyz, pts, m, r, k, mlp, False, "sa", p, dtype=np.float32)[1] - want).max()
    print(f"sa_module[{mlp_mode}] max|err| cuda={err:.3e} numpy-fp32={f32:.3e} max|act|={np.abs(want).max():.3f}")
    G.contract_close(G.npy(got), want, f"sa_module[{mlp_mode}]")


@pytest.mark.parametrize("n,m,r,k,c,mlp", [(2048, 512, 0.2, 32, 0, [64, 64, 128]), (512, 128, 0.4, 64, 128, [128, 128, 256])])
def test_sa_module_unit_scale_absolute_bound(n, m, r, k, c, mlp, mlp_mode):
    """the contract's absolute form: weights scaled until every activation of the level is <= 1, then max|err| < 1e-5 flat"""
    p = _store(n + 1)
    add_sa_module_params(p, "sa", 3 + c, mlp, randomize_bn=True)
    rng = np.random.default_rng(n + 7)
    xyz = make_clouds("ball", 2, n, seed=n + 3)
    pts = (rng.standard_normal((2, n, c)) * 0.3).astype(np.float32) if c else None
    want = mo.sa_module(xyz, pts, m, r, k, mlp, False, "sa", p)[1]
    last = f"sa/conv{len(mlp) - 1}"
    shrink = 0.9 / max(1e-6, float(np.abs(want).max()))
    if shrink < 1.0:       # relu((x.W)*scale + shift) is positively homogeneous in (gamma, beta) of the last layer
        p[f"{last}/bn/gamma"] = p[f"{last}/bn/gamma"] * shrink
        p[f"{last}/bn/beta"] = p[f"{last}/bn/beta"] * shrink
    _, got, _ = pointnet_sa_module(G.cu(xyz), G.cu(pts) if c else None, m, r, k, mlp, None, False, False, None, "sa", params=p)
    want = mo.sa_module(xyz, pts, m, r, k, mlp, False, "sa", p)[1]
    assert np.abs(want).max() <= 1.0
    err = np.abs(G.npy(got) - want).max()
    print(f"unit-scale sa_module[{mlp_mode}] max|err|={err:.3e} (absolute bound 1e-5)")
    assert err < 1e-5


@pytest.mark.parametrize("pooling,mlp2", [("avg", None), ("weighted_avg", None), ("max_and_avg", [64]), ("max", [96, 32])])
def test_sa_module_pooling_modes_and_post_mlp(pooling, mlp2):
    """pointnet_sa_module's other pooling modes and the mlp2 post-MLP (pointnet_util.py:126-157)"""
    n, m, r, k, c, mlp = 512, 64, 0.35, 24, 16, [32, 64]
    p = _store(11)
    cl = add_sa_module_params(p, "sa", 3 + c, mlp, randomize_bn=True)
    if mlp2 is not None:
        cin = 2 * cl if pooling == "max_and_avg" else cl
        for i, co in enumerate(mlp2):
            p.add_conv2d(f"sa/conv_post_{i}", cin, co, bn=True, randomize_bn=True)
            cin = co
    rng = np.random.default_rng(5)
    xyz = make_clouds("ball", 2, n, seed=21)
    pts = rng.standard_normal((2, n, c)).astype(np.float32)
    new_xyz, got, idx = pointnet_sa_module(G.cu(xyz), G.cu(pts), m, r, k, mlp, mlp2, False, False, None, "sa", pooling=pooling, params=p)
    oxyz, want, oidx = mo.sa_module(xyz, pts, m, r, k, mlp, False, "sa", p, pooling=pooling, mlp2=mlp2)
    assert np.array_equal(G.npy(new_xyz), oxyz) and np.array_equal(G.npy(idx), oidx)
    G.contract_close(G.npy(got), want, f"sa_module pooling={pooling} mlp2={mlp2}")


@pytest.mark.parametrize("c", [0, 32])
def test_sa_module_msg_matches_fp64(c):
    """multi-scale grouping (pointnet_util.py:156-196): rows are [features, xyz] there; the fused kernel gets the rotated weights"""
    n, m = 1024, 128
    radii, ks, mlps = [0.1, 0.2, 0.4], [16, 32, 64], [[32, 32, 64], [64, 64, 128], [64, 96, 128]]
    p = _store(13 + c)
    total = add_sa_module_msg_params(p, "msg", 3 + c, mlps, randomize_bn=True)
    rng = np.random.default_rng(c)
    xyz = make_clouds("shell", 2, n, seed=31)
    pts = rng.standard_normal((2, n, c)).astype(np.float32) if c else None
    new_xyz, got = pointnet_sa_module_msg(G.cu(xyz), G.cu(pts) if c else None, m, radii, ks, mlps, False, None, "msg", params=p)
    oxyz, want = mo.sa_module_msg(xyz, pts, m, radii, ks, mlps, "msg", p)
    assert got.shape == (2, m, total) and np.array_equal(G.npy(new_xyz), oxyz)
    G.contract_close(G.npy(got), want, f"sa_module_msg c={c}")


def test_sa_module_unfused_paths_agree():
    """knn=True and group_all go through group_point + shared_mlp instead of the fused kernel."""
    p = _store(3)
    add_sa_module_params(p, "sa", 3 + 16, [32, 64], randomize_bn=True)
    rng = np.random.default_rng(0)
    xyz = make_clouds("ball", 2, 128, seed=9)
    pts = rng.standard_normal((2, 128, 16)).astype(np.float32)
    _, got, _ = pointnet_sa_module(G.cu(xyz), G.cu(pts), None, None, None, [32, 64], None, True, False, None, "sa", params=p)
    _, want, _ = mo.sa_module(xyz, pts, None, None, None, [32, 64], True, "sa", p)
    G.contract_close(G.npy(got), want, "activations")


@pytest.mark.parametrize("n,c,k,mlp", [(1024, 3, 20, [64]), (512, 64, 20, [64]), (256, 64, 20, [128]), (200, 3, 20, [64, 128]),
                                       (128, 8, 16, [32]), (2048, 3, 20, [64, 128]), (300, 3, 32, [64, 64, 128]), (256, 3, 7, [128, 128])])
def test_edgeconv_infer_matches_fp64(n, c, k, mlp):
    p = _store(n)
    scopes = []
    cin = 2 * c
    for i, co in enumerate(mlp):
        p.add_conv2d(f"e/conv{i}", cin, co, bn=True, randomize_bn=True)
        scopes.append(f"e/conv{i}")
        cin = co
    # negative BN scales on a third of the channels: the single-layer algebra path must switch from max_j to min_j there
    g = p["e/conv0/bn/gamma"]
    g[::3] = -g[::3]
    p.invalidate()
    rng = np.random.default_rng(n)
    x = rng.standard_normal((2, n, c)).astype(np.float32)
    idx = orc.dgcnn_knn(x, k)
    got = G.npy(ops.edgeconv_infer(G.cu(x), G.cu(idx), p.mlp(scopes)))
    want = mo.edgeconv(x, idx, p, scopes)
    G.contract_close(got, want, "activations")


def test_fp_module_matches_fp64():
    p = _store(5)
    add_fp_module_params(p, "fp", 256 + 128, [256, 128], randomize_bn=True)
    rng = np.random.default_rng(5)
    xyz1 = make_clouds("ball", 2, 512, seed=1)
    xyz2 = make_clouds("ball", 2, 128, seed=2)
    p1 = rng.standard_normal((2, 512, 128)).astype(np.float32)
    p2 = rng.standard_normal((2, 128, 256)).astype(np.float32)
    got = G.npy(pointnet_fp_module(G.cu(xyz1), G.cu(xyz2), G.cu(p1), G.cu(p2), [256, 128], False, None, "fp", params=p))
    want = mo.fp_module(xyz1, xyz2, p1, p2, [256, 128], "fp", p)
    G.contract_close(got, want, "activations")


@pytest.mark.parametrize("kind", ["ball", "shell", "dup"])
def test_pointnet2_cls_ssg_matches_oracle(kind, mlp_mode):
    p = pointnet2_cls_ssg.init_params(seed=1, randomize_bn=True)
    xyz = make_clouds(kind, 4, 2048, seed=1001)
    logits, ep = pointnet2_cls_ssg.get_model(G.cu(xyz), False, params=p)
    want, oep = mo.pointnet2_cls_ssg(xyz, p)
    assert np.array_equal(G.npy(ep["l1_indices"]), oep["l1_idx"])
    assert np.array_equal(G.npy(ep["l2_indices"]), oep["l2_idx"])
    assert np.array_equal(G.npy(ep["l1_xyz"]), oep["l1_xyz"])
    for name in ("l1_points", "l2_points", "l3_points"):
        w = oep[name].reshape(G.npy(ep[name]).shape)
        G.contract_close(G.npy(ep[name]), w, name)
    err = np.abs(G.npy(logits) - want).max()
    print(f"logits[{mlp_mode}] max|err|={err:.3e} max|logit|={np.abs(want).max():.3f}")
    G.contract_close(G.npy(logits), want, "logits")


@pytest.mark.parametrize("kind,n,m,r,k,c,c1,b", [("ball", 2048, 512, 0.2, 32, 0, 64, 3), ("shell", 2048, 512, 0.2, 64, 0, 64, 3),
                                                 ("ball", 512, 128, 0.4, 64, 128, 128, 3), ("dup", 300, 40, 0.3, 20, 5, 64, 3),
                                                 # CTA ranges that cross cloud boundaries (grid rebuilt mid-CTA), odd nsample
                                                 ("ball", 500, 37, 0.3, 13, 0, 64, 41), ("shell", 700, 333, 0.25, 32, 7, 128, 5),
                                                 # scan mode (cloud too small for the grid) and a 4096-point cloud (16 points per thread)
                                                 ("ball", 200, 20, 0.4, 16, 0, 64, 4), ("ball", 4096, 1024, 0.15, 32, 0, 64, 2),
                                                 # n % 4 != 0: the scalar cloud load (no 16-byte alignment per cloud); tail of a 16-point lane
                                                 ("ball", 301, 40, 0.3, 20, 0, 64, 3), ("shell", 1023, 100, 0.25, 32, 0, 64, 2),
                                                 # B = 32 clouds: nine CTAs per cloud, none crosses a cloud boundary
                                                 ("ball", 2048, 512, 0.2, 32, 0, 64, 32),
                                                 # beyond the streaming kernel's plan -> round-1 kernel: n > 4096 (scan mode), and
                                                 # nsample 128 at n = 4096 (> 110 KB of shared memory; grid mode, 16 points per thread)
                                                 ("ball", 8192, 256, 0.1, 32, 0, 64, 2), ("ball", 4096, 256, 0.2, 128, 0, 64, 2)])
def test_sa_conv1_prebn_training_front(kind, n, m, r, k, c, c1, b):
    """variant F1: pre-BN conv1 output + BN batch statistics vs the fp64 restatement of
    query_ball_point -> group_point -> centre -> concat -> conv2d + bias_add (pointnet_util.py:44-50,117-123)."""
    rng = np.random.default_rng(n + k)
    xyz = make_clouds(kind, b, n, seed=n)
    pts = rng.standard_normal((b, n, c)).astype(np.float32) if c else None
    w1 = (rng.uniform(-1, 1, (3 + c, c1)) * np.sqrt(6.0 / (3 + c + c1))).astype(np.float32)
    bias = rng.uniform(-0.1, 0.1, c1).astype(np.float32)
    new_xyz = orc.gather_point(xyz, orc.fps(xyz, m))
    pre, idx, cnt, stats = ops.sa_conv1_prebn(G.cu(xyz), G.cu(new_xyz), G.cu(pts) if c else None, r, k, G.cu(w1), G.cu(bias))
    oidx, ocnt = orc.query_ball_point(r, k, xyz, new_xyz, contract=True)
    assert np.array_equal(G.npy(idx), oidx) and np.array_equal(G.npy(cnt), ocnt)
    rows = orc.group_point(xyz, oidx) - new_xyz[:, :, None, :]
    if c:
        rows = np.concatenate([rows, orc.group_point(pts, oidx)], -1)
    want = rows.astype(np.float64) @ w1.astype(np.float64) + bias
    got = G.npy(pre)
    G.contract_close(got, want, "activations")
    s_want = np.stack([want.reshape(-1, c1).sum(0), (want.reshape(-1, c1) ** 2).sum(0)])
    np.testing.assert_allclose(G.npy(stats), s_want, rtol=2e-5, atol=1e-3)


def test_sa_conv1_prebn_nonfinite_inputs_keep_reference_indices():
    """NaN / inf coordinates: the reference's max(sqrtf(NaN),1e-20f) < r counts a NaN distance as inside.  The streaming
    kernel answers such queries (and whole clouds with a non-finite point) with the ordered scan: idx / pts_cnt exact."""
    n, m, k = 1024, 64, 32
    xyz = make_clouds("ball", 4, n, seed=77)
    xyz[1, 5, 1] = np.nan                      # cloud 1: grid unusable, every query scans
    xyz[2, 100, 0] = np.inf
    new_xyz = orc.gather_point(xyz, orc.fps(np.nan_to_num(xyz, nan=0.0, posinf=0.0), m))
    new_xyz[0, 3, 2] = np.nan                  # cloud 0: one NaN query on a finite cloud
    new_xyz[3, 7, 0] = -np.inf
    w1 = np.random.default_rng(5).uniform(-1, 1, (3, 64)).astype(np.float32)
    pre, idx, cnt, _ = ops.sa_conv1_prebn(G.cu(xyz), G.cu(new_xyz), None, 0.25, k, G.cu(w1), None)
    oidx, ocnt = orc.query_ball_point(0.25, k, xyz, new_xyz, contract=True)
    assert np.array_equal(G.npy(idx), oidx) and np.array_equal(G.npy(cnt), ocnt)
    # finite rows of the finite clouds still carry the conv output
    rows = orc.group_point(xyz, oidx) - new_xyz[:, :, None, :]
    want = rows.astype(np.float64) @ w1.astype(np.float64)
    ok = np.isfinite(want)
    assert ok[0].mean() > 0.9
    G.contract_close(G.npy(pre)[ok], want[ok], "pre-BN rows")


@pytest.mark.parametrize("where", ["features", "weights", "inner"])
def test_fp16_range_guard_reruns_on_bf16x3(where):
    """mode 0 splits operands into two fp16 pieces (|value| < 65504).  Features or an inner activation beyond that range raise the
    device-side flag and the op is rerun with bf16x3 operands inside the same call; weights beyond it are scaled into it per
    column.  The result still meets the contract (relative to its own magnitude); nothing is clamped, nothing becomes inf."""
    p = _store(91)
    mlp = [128, 128, 256]
    add_sa_module_params(p, "sa", 3 + 64, mlp, randomize_bn=True)
    rng = np.random.default_rng(5)
    xyz = make_clouds("ball", 2, 512, seed=12)
    pts = rng.standard_normal((2, 512, 64)).astype(np.float32)
    if where == "features":
        pts *= 3.0e5
    elif where == "weights":
        p["sa/conv1/weights"] = p["sa/conv1/weights"] * 1.0e6
    else:
        p["sa/conv0/bn/gamma"] = p["sa/conv0/bn/gamma"] * 2.0e5        # layer-1 activations ~1e5..1e6, inputs and weights ordinary
    assert ops.get_mlp_mode() == 0
    _, got, _ = pointnet_sa_module(G.cu(xyz), G.cu(pts), 128, 0.4, 64, mlp, None, False, False, None, "sa", params=p)
    want = mo.sa_module(xyz, pts, 128, 0.4, 64, mlp, False, "sa", p)[1]
    got = G.npy(got)
    assert np.isfinite(got).all() and np.abs(want).max() > 7e4
    G.contract_close(got, want, f"range guard ({where})")
    # dense chain (SA3 / PointNet shape): same guard, per layer
    q = _store(92)
    q.add_conv2d("m/conv0", 256, 256, bn=True, randomize_bn=True)
    q.add_conv2d("m/conv1", 256, 128, bn=True, randomize_bn=True)
    x = (rng.standard_normal((512, 256)) * (4.0e5 if where == "features" else 1.0)).astype(np.float32)
    if where == "weights":
        q["m/conv1/weights"] = q["m/conv1/weights"] * 1.0e6
    if where == "inner":
        q["m/conv0/bn/gamma"] = q["m/conv0/bn/gamma"] * 2.0e5
    d = G.npy(ops.shared_mlp(G.cu(x), q.mlp(["m/conv0", "m/conv1"], [True, False])))
    dw = mo.mlp_chain(x, q, ["m/conv0", "m/conv1"], [True, False])
    assert np.isfinite(d).all() and np.abs(dw).max() > 7e4
    G.contract_close(d, dw, f"range guard dense ({where})")
