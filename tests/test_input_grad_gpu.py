"""Gradients with respect to the input point coordinates (PointNet++), in training mode and in inference mode (batch norm on the
moving averages), against float64 restatements on the GPU's own sampling / grouping indices.  Bound: 1e-4 relative to the largest
entry (GTOL), as in test_train_gpu.py."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import train_oracle as T
from scanobjectnn_b200 import _lib, ops, pointnet2_cls_bga, pointnet2_cls_ssg
from scanobjectnn_b200._lib import ptr, stream
from scanobjectnn_b200.pointnet_util import add_sa_module_params, pointnet_sa_module
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import VariableStore
from scanobjectnn_b200.training import LevelSpec, _plain_grad

from . import gpu_util as G
from . import restate
from .restate import moving, rel

pytestmark = pytest.mark.gpu
GTOL = 1e-4


def _gather_grad(dnew, fps_idx, n):
    out = np.zeros((dnew.shape[0], n, 3))
    for b in range(dnew.shape[0]):
        np.add.at(out[b], fps_idx[b], dnew[b])
    return out


# ---------------------------------------------------------------------------------------------------------------------
# 1. the kernel, then one level through autograd
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c1,far", [(64, False), (128, True), (16, False)])
def test_conv1_bwd_xyz_kernel_against_numpy(c1, far):
    """psa_sa_conv1_bwd_xyz: row scatter and "- new_xyz" sums, with padding rows and (far=True) queries whose balls are empty"""
    lib = _lib.load()
    b, n, m, k = 3, 300, 40, 24
    rng = np.random.default_rng(c1)
    xyz = make_clouds("dup", b, n, seed=5)
    q = orc.gather_point(xyz, orc.fps(xyz, m))
    if far:
        q = q.copy()
        q[:, ::3] += 10.0                                            # every third query has an empty ball: idx = 0 throughout
    idx, cnt = orc.query_ball_point(0.3, k, xyz, q, contract=True)
    assert (cnt < k).any()                                           # padding rows
    if far:
        assert (cnt == 0).any()
    dy0 = rng.standard_normal((b, m, k, c1)).astype(np.float32)
    W = rng.standard_normal((3, c1)).astype(np.float32)
    dyd, Wd, idx_d = G.cu(dy0.reshape(-1, c1)), G.cu(W), G.cu(idx)
    g = _plain_grad(dyd)
    dxyz, dnew = torch.empty((b, n, 3), device="cuda"), torch.empty((b, m, 3), device="cuda")
    need = lib.psa_sa_conv1_bwd_xyz_workspace_bytes(b, n, m, k)
    ws = torch.empty(need // 4 + 16, device="cuda")
    args = (b, n, m, k, c1, ptr(Wd), ptr(idx_d), C.byref(g))
    assert lib.psa_sa_conv1_bwd_xyz(*args, ptr(dxyz), ptr(dnew), ptr(ws), C.c_size_t(need), stream()) == 0
    v = dy0.astype(np.float64) @ W.astype(np.float64).T             # (b, m, k, 3)
    want_dxyz = T.group_bwd(v, idx.astype(np.int64), n)
    assert rel(G.npy(dxyz), want_dxyz) < 1e-5
    assert rel(G.npy(dnew), -v.sum(axis=2)) < 1e-5
    dxyz2, dnew2 = torch.empty_like(dxyz), torch.empty_like(dnew)
    assert lib.psa_sa_conv1_bwd_xyz(*args, ptr(dxyz2), ptr(dnew2), ptr(ws), C.c_size_t(need), stream()) == 0
    assert torch.equal(dxyz, dxyz2) and torch.equal(dnew, dnew2), "coordinate gradient must be bit-reproducible"


def _level_layers(p, scope, mlp):
    layers = []
    for i in range(len(mlp)):
        w = G.npy(p[f"{scope}/conv{i}/weights"]).astype(np.float64)
        layers.append((w.reshape(-1, w.shape[-1]), G.npy(p[f"{scope}/conv{i}/biases"]).astype(np.float64),
                       G.npy(p[f"{scope}/conv{i}/bn/gamma"]).astype(np.float64), G.npy(p[f"{scope}/conv{i}/bn/beta"]).astype(np.float64)))
    return layers


def _oracle_level(xyz, pts, fps_idx, idx, layers, group_all):
    """-> (pooled, cache, fps) for the float64 level restatement; group_all as a centre at an appended origin point"""
    x64 = xyz.astype(np.float64)
    B, N = xyz.shape[:2]
    if group_all:
        x_aug = np.concatenate([x64, np.zeros((B, 1, 3))], axis=1)
        p_aug = None if pts is None else np.concatenate([pts.astype(np.float64), np.zeros((B, 1, pts.shape[-1]))], axis=1)
        return T.sa_level_train_fwd(x_aug, p_aug, np.full((B, 1), N, np.int64), idx, layers)
    return T.sa_level_train_fwd(x64, None if pts is None else pts.astype(np.float64), fps_idx, idx, layers)


@pytest.mark.parametrize("c,group_all,cloud,radius,k", [(0, False, "ball", 0.35, 16), (16, False, "ball", 0.35, 16), (24, True, "ball", None, None),
                                                        (0, False, "ball", 0.12, 48), (16, False, "dup", 0.3, 32)])
def test_one_level_training_xyz_grad(c, group_all, cloud, radius, k):
    """pointnet_sa_module(is_training=True): xyz.grad against sa_level_train_bwd's dxyz (GroupPointGrad + GatherPointGrad), including
    levels where nsample exceeds the neighbour count (padding rows) and the duplicated-points cloud"""
    B, N, m = 3, 256, 64
    mlp = [64, 32, 64]
    p = VariableStore(device="cuda", seed=5)
    add_sa_module_params(p, "lv", 3 + c, mlp)
    rng = np.random.default_rng(c + 3)
    xyz = make_clouds(cloud, B, N, seed=31)
    pts = rng.standard_normal((B, N, c)).astype(np.float32) if c else None
    xt = G.cu(xyz).requires_grad_(True)
    pt = G.cu(pts).requires_grad_(True) if c else None
    new_xyz, out, idx = pointnet_sa_module(xt, pt, None if group_all else m, radius, k, mlp, None, group_all, True, 0.5, "lv", params=p)
    assert out.requires_grad
    if not group_all:
        assert new_xyz.requires_grad
        _, fused = ops.farthest_point_sample_and_gather(m, xt.detach())
        assert torch.equal(new_xyz.detach(), fused), "gather_point must reproduce the fused gather bit for bit"
        cnt = (G.npy(idx) != G.npy(idx)[:, :, :1]).sum(-1) + 1
        if radius == 0.12:
            assert (cnt < k).any()
    R = rng.standard_normal(out.shape).astype(np.float32)
    (out * G.cu(R)).sum().backward()
    fps_idx = None if group_all else G.npy(ops.farthest_point_sample(m, xt.detach())).astype(np.int64)
    pooled, cache, _ = _oracle_level(xyz, pts, fps_idx, G.npy(idx).astype(np.int64), _level_layers(p, "lv", mlp), group_all)
    assert rel(G.npy(out), pooled) < 1e-5
    dxyz, dpts, _ = T.sa_level_train_bwd(R.astype(np.float64), cache)
    assert rel(G.npy(xt.grad), dxyz[:, :N]) < GTOL
    if c:
        assert rel(G.npy(pt.grad), dpts[:, :N]) < GTOL


def test_two_levels_chain_through_gather_point():
    """level 2's coordinate gradient reaches l1_xyz (= gather_point(xyz, fps)) and from there the input cloud"""
    B, N, m1, m2 = 3, 256, 64, 16
    mlp1, mlp2 = [64, 64], [64, 32]
    p = VariableStore(device="cuda", seed=8)
    add_sa_module_params(p, "l1", 3, mlp1)
    add_sa_module_params(p, "l2", 3 + mlp1[-1], mlp2)
    xyz = make_clouds("ball", B, N, seed=3)
    xt = G.cu(xyz).requires_grad_(True)
    l1_xyz, l1_pts, idx1 = pointnet_sa_module(xt, None, m1, 0.3, 16, mlp1, None, False, True, 0.5, "l1", params=p)
    l2_xyz, l2_pts, idx2 = pointnet_sa_module(l1_xyz, l1_pts, m2, 0.6, 16, mlp2, None, False, True, 0.5, "l2", params=p)
    rng = np.random.default_rng(4)
    R1, R2 = rng.standard_normal(l1_pts.shape).astype(np.float32), rng.standard_normal(l2_pts.shape).astype(np.float32)
    ((l1_pts * G.cu(R1)).sum() + (l2_pts * G.cu(R2)).sum()).backward()
    f1 = G.npy(ops.farthest_point_sample(m1, xt.detach())).astype(np.int64)
    f2 = G.npy(ops.farthest_point_sample(m2, l1_xyz.detach())).astype(np.int64)
    pooled1, c1, _ = T.sa_level_train_fwd(xyz.astype(np.float64), None, f1, G.npy(idx1).astype(np.int64), _level_layers(p, "l1", mlp1))
    new1 = xyz.astype(np.float64)[np.arange(B)[:, None], f1]
    pooled2, c2, _ = T.sa_level_train_fwd(new1, pooled1, f2, G.npy(idx2).astype(np.int64), _level_layers(p, "l2", mlp2))
    assert rel(G.npy(l2_pts), pooled2) < 1e-5
    d_new1, dpts1, _ = T.sa_level_train_bwd(R2.astype(np.float64), c2)
    dxyz1, _, _ = T.sa_level_train_bwd(R1.astype(np.float64) + dpts1, c1)
    want = dxyz1 + _gather_grad(d_new1, f1, N)
    assert rel(G.npy(xt.grad), want) < GTOL


# ---------------------------------------------------------------------------------------------------------------------
# whole models: restate.ssg on the trainer's own indices
# ---------------------------------------------------------------------------------------------------------------------
SMALL_LEVELS = [LevelSpec("layer1", 64, 0.3, 16, [64, 64, 128]), LevelSpec("layer2", 16, 0.6, 16, [128, 128, 256]),
                LevelSpec("layer3", None, None, None, [256, 512, 1024], group_all=True)]


def _trainer(p, frozen):
    return [t for k, t in p.__dict__["_trainers"].items() if (k[0] == "frozen") == frozen][0]


def _small_ssg_params(seed):
    return pointnet2_cls_ssg.init_params(seed=seed, randomize_bn=True)


def _get_model_small(xyz, is_training, p):
    """pointnet2_cls_ssg.get_model with the small level stack (same code path; smaller clouds)"""
    from scanobjectnn_b200.training import get_model_training, wants_input_grad
    frozen = not is_training and wants_input_grad(xyz)
    logits, tr = get_model_training(xyz, 0.5, 15, p, levels=SMALL_LEVELS, frozen=frozen)
    return logits, tr


def test_ssg_training_mode_xyz_grad_and_unchanged_results():
    B, N = 8, 256
    p = _small_ssg_params(3)
    xyz = G.cu(make_clouds("ball", B, N, seed=11))
    labels = G.cu(np.random.default_rng(0).integers(0, 15, B).astype(np.int64))
    _get_model_small(xyz, True, p)                                   # builds the trainer
    tr = _trainer(p, False)
    mov = moving(p)
    runs = []
    for want in (False, True):
        with torch.no_grad():
            for k, v in mov.items():
                p[k].copy_(v)
        x = xyz.clone().requires_grad_(want)
        tr._gen.manual_seed(7)
        tr.fp.flat.grad = None
        logits, _ = _get_model_small(x, True, p)
        torch.nn.functional.cross_entropy(logits, labels).backward()
        runs.append((logits.detach().clone(), tr.fp.flat.grad.clone(), {k: p[k].clone() for k in mov}, x, tr))
    (l0, g0, m0, _, _), (l1, g1, m1, x, tr) = runs
    assert torch.equal(l0, l1) and torch.equal(g0, g1), "asking for the coordinate gradient must not change logits or variable gradients"
    assert all(torch.equal(m0[k], m1[k]) for k in m0), "moving averages must update identically"
    assert x.grad is not None
    masks = {ly.scope: ly.mask for ly in tr.head if ly.mask is not None}
    x64 = x.detach().double().requires_grad_(True)
    # the moving averages moved during the run: the restatement uses batch statistics, so they do not enter
    lg64 = restate.ssg(x64, p, tr.levels, False, masks)
    assert rel(G.npy(l1), lg64.detach().cpu().numpy()) < 1e-4
    torch.nn.functional.cross_entropy(lg64, labels).backward()
    assert rel(G.npy(x.grad), x64.grad.cpu().numpy()) < GTOL


def test_ssg_inference_mode_xyz_grad():
    B, N = 8, 256
    p = _small_ssg_params(4)
    xyz = G.cu(make_clouds("ball", B, N, seed=12))
    labels = G.cu(np.random.default_rng(1).integers(0, 15, B).astype(np.int64))
    mov = moving(p)
    x = xyz.clone().requires_grad_(True)
    logits, _ = _get_model_small(x, False, p)
    tr = _trainer(p, True)
    bucket = tr.fp.grad.clone()
    torch.nn.functional.cross_entropy(logits, labels).backward()
    assert all(torch.equal(mov[k], p[k]) for k in mov), "inference mode must not move the moving averages"
    assert torch.equal(bucket, tr.fp.grad) and tr.fp.flat.grad is None, "inference mode leaves the gradient bucket alone"
    x64 = xyz.double().requires_grad_(True)
    lg64 = restate.ssg(x64, p, tr.levels, True, {})
    assert np.abs(G.npy(logits) - lg64.detach().cpu().numpy()).max() < 1e-5 * max(1.0, float(lg64.detach().abs().max()))
    torch.nn.functional.cross_entropy(lg64, labels).backward()
    assert rel(G.npy(x.grad), x64.grad.cpu().numpy()) < GTOL


def test_ssg_get_model_inference_routes_on_requires_grad():
    """the public get_model: with requires_grad the frozen path (same argmax as the fused kernels); without, the fused kernels and no
    trainer"""
    B, N = 4, 2048
    p = pointnet2_cls_ssg.init_params(seed=2, randomize_bn=True)
    xyz = G.cu(make_clouds("ball", B, N, seed=4))
    fused, _ = pointnet2_cls_ssg.get_model(xyz, False, params=p)
    assert not fused.requires_grad and "_trainers" not in p.__dict__ and getattr(p, "_flat", None) is None
    with torch.no_grad():
        fused2, _ = pointnet2_cls_ssg.get_model(xyz.clone().requires_grad_(True), False, params=p)
    assert torch.equal(fused, fused2) and "_trainers" not in p.__dict__
    x = xyz.clone().requires_grad_(True)
    logits, ep = pointnet2_cls_ssg.get_model(x, False, params=p)
    assert logits.requires_grad and ep["l1_indices"].shape == (B, 512, 32)
    assert torch.equal(logits.argmax(1), fused.argmax(1))
    assert rel(G.npy(logits), G.npy(fused)) < 1e-4
    logits[:, 0].sum().backward()
    assert x.grad is not None and torch.isfinite(x.grad).all() and float(x.grad.abs().max()) > 0


def test_reproducible_xyz_grad():
    B, N = 8, 256
    xyz = G.cu(make_clouds("shell", B, N, seed=2))
    labels = G.cu(np.arange(B, dtype=np.int64) % 15)
    for is_training in (True, False):
        grads = []
        for _ in range(2):
            p = _small_ssg_params(5)
            x = xyz.clone().requires_grad_(True)
            if is_training:
                _get_model_small(x, True, p)
                _trainer(p, False)._gen.manual_seed(9)
            logits, _ = _get_model_small(x, is_training, p)
            torch.nn.functional.cross_entropy(logits, labels).backward()
            grads.append(x.grad.clone())
        assert torch.equal(grads[0], grads[1]), f"is_training={is_training}: xyz.grad is not bit-reproducible"


@pytest.mark.parametrize("is_training", [True, False])
def test_bga_both_heads_reach_xyz(is_training):
    """pointnet2_cls_bga: the joint loss of both heads reaches the coordinates (through the levels, gather_point and the FP modules);
    inference mode does not move the moving averages.  In inference mode the classification head's logits and coordinate gradient are
    checked against the float64 restatement on the levels' own indices."""
    B, N = 4, 1024
    p = pointnet2_cls_bga.init_params(seed=3, randomize_bn=True)
    xyz = G.cu(make_clouds("ball", B, N, seed=8))
    labels = G.cu(np.array([1, 4, 7, 11], dtype=np.int64))
    mask = G.cu((np.random.default_rng(0).random((B, N)) > 0.5).astype(np.int64))
    mov = moving(p)
    x = xyz.clone().requires_grad_(True)
    cp, sp = pointnet2_cls_bga.get_model(x, is_training, bn_decay=0.5, params=p)
    assert cp.requires_grad and sp.requires_grad
    loss, _, _ = pointnet2_cls_bga.get_loss(cp, sp, labels, mask)
    loss.backward()
    g = x.grad
    assert torch.isfinite(g).all() and float(g.abs().max()) > 0
    if is_training:
        return
    assert all(torch.equal(mov[k], p[k]) for k in mov)
    x2 = xyz.clone().requires_grad_(True)
    cp2, _ = pointnet2_cls_bga.get_model(x2, False, params=p)
    torch.nn.functional.cross_entropy(cp2, labels).backward()
    assert not torch.equal(x2.grad, g)               # the segmentation head contributes
    trainers = p.__dict__["_trainers"]
    levels = [trainers[k].levels[0] for k in sorted(k for k in trainers if k[0] == "level_frozen")]
    assert [lv.spec.scope for lv in levels] == ["layer1", "layer2", "layer3"]
    x64 = xyz.double().requires_grad_(True)
    lg64 = restate.ssg(x64, p, levels, True, {})
    assert np.abs(G.npy(cp2) - lg64.detach().cpu().numpy()).max() < 1e-5 * max(1.0, float(lg64.detach().abs().max()))
    torch.nn.functional.cross_entropy(lg64, labels).backward()
    assert rel(G.npy(x2.grad), x64.grad.cpu().numpy()) < GTOL
