"""PointNet++ layers on the libpsa kernels: same names, argument order and return values as
pointnet2/utils/pointnet_util.py (plus a keyword-only ``params`` variable store, torch being stateless about
variable scopes).  Inference mode: batch norm uses the moving averages and is folded into the fused kernels."""
from __future__ import annotations

import torch

from . import ops
from .tf_grouping import group_point, knn_point, query_ball_point
from .tf_interpolate import three_interpolate, three_nn
from .tf_sampling import farthest_point_sample, gather_point
from .tf_util import VariableStore, _require_inference


def sample_and_group(npoint, radius, nsample, xyz, points, knn=False, use_xyz=True):
    """pointnet_util.sample_and_group (pointnet_util.py:22-56), materialising form.
    -> new_xyz (B,npoint,3), new_points (B,npoint,nsample,3+C), idx (B,npoint,nsample), grouped_xyz."""
    new_xyz = gather_point(xyz, farthest_point_sample(npoint, xyz))
    if knn:
        _, idx = knn_point(nsample, xyz, new_xyz)
    else:
        idx, _ = query_ball_point(radius, nsample, xyz, new_xyz)
    grouped_xyz = group_point(xyz, idx)
    grouped_xyz = grouped_xyz - new_xyz.unsqueeze(2)
    if points is not None:
        grouped_points = group_point(points, idx)
        new_points = torch.cat([grouped_xyz, grouped_points], dim=-1) if use_xyz else grouped_points
    else:
        new_points = grouped_xyz
    return new_xyz, new_points, idx, grouped_xyz


def sample_and_group_all(xyz, points, use_xyz=True):
    """pointnet_util.sample_and_group_all (pointnet_util.py:59-84)."""
    b, n, _ = xyz.shape
    new_xyz = torch.zeros((b, 1, 3), dtype=torch.float32, device=xyz.device)
    idx = torch.arange(n, dtype=torch.int32, device=xyz.device).reshape(1, 1, n).repeat(b, 1, 1)
    grouped_xyz = xyz.reshape(b, 1, n, 3)
    if points is not None:
        new_points = torch.cat([xyz, points], dim=2) if use_xyz else points
        new_points = new_points.unsqueeze(1)
    else:
        new_points = grouped_xyz
    return new_xyz, new_points, idx, grouped_xyz


def _mlp_scopes(scope, mlp, prefix="conv"):
    return [f"{scope}/{prefix}{i}" for i in range(len(mlp))]


def add_sa_module_params(params: VariableStore, scope, in_channels, mlp, mlp2=None, bn=True, randomize_bn=False):
    c = in_channels
    for s, cout in zip(_mlp_scopes(scope, mlp), mlp):
        params.add_conv2d(s, c, cout, bn=bn, randomize_bn=randomize_bn)
        c = cout
    for s, cout in zip(_mlp_scopes(scope, mlp2 or [], "conv_post_"), mlp2 or []):
        params.add_conv2d(s, c, cout, bn=bn, randomize_bn=randomize_bn)
        c = cout
    return c


def pointnet_sa_module(xyz, points, npoint, radius, nsample, mlp, mlp2, group_all, is_training, bn_decay, scope,
                       bn=True, pooling="max", knn=False, use_xyz=True, use_nchw=False, *, params: VariableStore,
                       new_xyz=None):
    """pointnet_util.pointnet_sa_module (pointnet_util.py:87-154) -> (new_xyz, new_points (B,npoint,C_out), idx).

    max-pooling / ball-query / use_xyz levels run as TWO launches: fused FPS+gather, then the fused
    ball-query -> group -> centre -> MLP -> max kernel pair (no (B,m,K,C) tensor is ever built).
    ``use_nchw`` only selected a cuDNN layout in the reference and has no effect on results.
    ``new_xyz`` (extension): centroids already sampled by the caller (= gather_point(xyz, farthest_point_sample(npoint,
    xyz))), e.g. on a side stream -- FPS of level l+1 only depends on level l's centroids, not on its features."""
    if pooling not in ("max", "avg", "weighted_avg", "max_and_avg"):
        raise ValueError(f"unknown pooling {pooling!r}")
    from .training import wants_input_grad
    frozen = not is_training and wants_input_grad(xyz, points)
    if is_training or frozen:
        # batch-statistics batch norm + autograd through the level (training.py); the configuration the in-scope models train with.
        # frozen: inference mode with an input gradient (saliency, adversarial perturbation) -- the same kernels with batch norm on the
        # moving averages; calls that need no gradient stay on the fused kernels below
        if not (pooling == "max" and mlp2 is None and use_xyz and not knn and bn and new_xyz is None):
            raise NotImplementedError("pointnet_sa_module(is_training=True) and input gradients of pointnet_sa_module(is_training=False) "
                                      "cover max pooling, use_xyz, ball query, bn=True, no mlp2 and no caller-sampled new_xyz (what "
                                      "pointnet2_cls_ssg / _bga train with); other configurations run in inference mode without gradients")
        from .training import LevelSpec, sa_module_training
        spec = LevelSpec(scope, None if group_all else npoint, None if group_all else radius, None if group_all else nsample, list(mlp),
                         group_all=bool(group_all))
        return sa_module_training(xyz, points, spec, bn_decay, params, frozen=frozen)
    scopes = _mlp_scopes(scope, mlp)
    if pooling != "max":
        # pointnet_util.py:128-146 -- unused by the in-scope models, so the grouped rows are materialised: group -> per-row
        # MLP (dense tensor-core kernels) -> row pooling kernel
        if group_all:
            new_xyz, new_points, idx, grouped_xyz = sample_and_group_all(xyz, points, use_xyz)
        else:
            new_xyz, new_points, idx, grouped_xyz = sample_and_group(npoint, radius, nsample, xyz, points, knn, use_xyz)
        b, m, k, c = new_points.shape
        rows = ops.shared_mlp(new_points.reshape(b * m * k, c).contiguous(), params.mlp(scopes))
        if pooling == "avg":
            pooled = ops.pool_rows(rows, k, "avg")
        elif pooling == "weighted_avg":
            dist = torch.linalg.vector_norm(grouped_xyz.reshape(b * m * k, 3), dim=-1)       # tf.norm(grouped_xyz, axis=-1)
            pooled = ops.pool_rows(rows, k, "weighted_avg", dist)
        else:
            pooled = torch.cat([ops.pool_rows(rows, k, "avg"), ops.pool_rows(rows, k, "max")], dim=-1)   # [avg, max] (:146)
        pooled = pooled.reshape(b, m, -1)
        if mlp2 is not None:
            pooled = ops.shared_mlp(pooled, params.mlp(_mlp_scopes(scope, mlp2, "conv_post_")))
        return new_xyz, pooled, idx
    if group_all:
        nsample = xyz.shape[1]
        b = xyz.shape[0]
        if points is not None and use_xyz:
            # sample_and_group_all without the concat: new_xyz = 0, idx = arange, rows = [xyz, points]
            new_xyz = torch.zeros((b, 1, 3), dtype=torch.float32, device=xyz.device)
            idx = torch.arange(nsample, dtype=torch.int32, device=xyz.device).reshape(1, 1, nsample).expand(b, 1, nsample)
            pooled = ops.sa_group_all_infer(xyz, points, params.mlp(scopes)).reshape(b, 1, -1)
        else:
            new_xyz, new_points, idx, _ = sample_and_group_all(xyz, points, use_xyz)
            rows = new_points.reshape(b * nsample, new_points.shape[-1])
            pooled = ops.shared_mlp(rows, params.mlp(scopes), pool_k=nsample).reshape(b, 1, -1)
    elif knn or not use_xyz:
        new_xyz, new_points, idx, _ = sample_and_group(npoint, radius, nsample, xyz, points, knn, use_xyz)
        b, m, k, c = new_points.shape
        pooled = ops.shared_mlp(new_points.reshape(b * m * k, c), params.mlp(scopes), pool_k=k).reshape(b, m, -1)
    else:
        if new_xyz is None:
            _, new_xyz = ops.farthest_point_sample_and_gather(npoint, xyz)
        pooled, idx, _ = ops.sa_module_infer(xyz, new_xyz, points, radius, nsample, params.mlp(scopes), return_idx=True)
    if mlp2 is not None:
        pooled = ops.shared_mlp(pooled, params.mlp(_mlp_scopes(scope, mlp2, "conv_post_")))
    return new_xyz, pooled, idx


def add_sa_module_msg_params(params: VariableStore, scope, in_channels, mlp_list, bn=True, randomize_bn=False):
    """variables of pointnet_sa_module_msg: scale i, layer j -> ``scope/conv{i}_{j}``; first-layer rows ordered
    [features, xyz] as the reference concatenates them (pointnet_util.py:184).  -> total output channels"""
    total = 0
    for i, mlp in enumerate(mlp_list):
        c = in_channels
        for j, cout in enumerate(mlp):
            params.add_conv2d(f"{scope}/conv{i}_{j}", c, cout, bn=bn, randomize_bn=randomize_bn)
            c = cout
        total += c
    return total


def pointnet_sa_module_msg(xyz, points, npoint, radius_list, nsample_list, mlp_list, is_training, bn_decay, scope, bn=True,
                           use_xyz=True, use_nchw=False, *, params: VariableStore):
    """pointnet_util.pointnet_sa_module_msg (pointnet_util.py:156-196): multi-scale grouping -> (new_xyz, new_points
    (B,npoint,sum_k mlp[k][-1])).  One FPS, then per scale the fused ball-query + group + MLP + max kernel
    (psa_sa_module_infer) and a concat of the pooled features; no (B,m,K,C) tensor is built."""
    _require_inference(is_training)
    _, new_xyz = ops.farthest_point_sample_and_gather(npoint, xyz)
    outs = []
    for i, (radius, nsample, mlp) in enumerate(zip(radius_list, nsample_list, mlp_list)):
        scopes = [f"{scope}/conv{i}_{j}" for j in range(len(mlp))]
        if points is not None and not use_xyz:
            idx, _ = query_ball_point(radius, nsample, xyz, new_xyz)
            g = group_point(points, idx)
            b, m, k, c = g.shape
            outs.append(ops.shared_mlp(g.reshape(b * m * k, c), params.mlp(scopes), pool_k=k).reshape(b, m, -1))
        else:
            # [grouped_points, grouped_xyz] (:184): coordinate rows last in the stored weights
            outs.append(ops.sa_module_infer(xyz, new_xyz, points, radius, nsample, params.mlp(scopes, xyz_last=points is not None)))
    return new_xyz, torch.cat(outs, dim=-1)


def add_fp_module_params(params: VariableStore, scope, in_channels, mlp, bn=True, randomize_bn=False):
    c = in_channels
    for i, cout in enumerate(mlp):
        params.add_conv2d(f"{scope}/conv_{i}", c, cout, bn=bn, randomize_bn=randomize_bn)
        c = cout
    return c


def pointnet_fp_module(xyz1, xyz2, points1, points2, mlp, is_training, bn_decay, scope, bn=True, *,
                       params: VariableStore):
    """pointnet_util.pointnet_fp_module (pointnet_util.py:199-229): three_nn + inverse-distance weights +
    three_interpolate in ONE launch (the reference runs them on the CPU), concat skip features, 1x1 convs."""
    scopes = [f"{scope}/conv_{i}" for i in range(len(mlp))]
    from .training import wants_input_grad
    frozen = not is_training and wants_input_grad(xyz1, xyz2, points1, points2)
    if is_training or frozen:
        # three_nn and the inverse-distance weights carry no gradient (they depend on coordinates only); three_interpolate is
        # differentiable in points2 (ThreeInterpolateGrad), the concat is autograd's, the MLP runs with batch-statistics batch norm
        # frozen (inference mode with an input gradient): the same, with batch norm on the moving averages; the three-NN weights are
        # constants (the reference's NoGradient('ThreeNN'))
        if not bn:
            raise NotImplementedError("pointnet_fp_module(is_training=True) needs bn=True (what the in-scope models use)")
        from .training import mlp_training
        with torch.no_grad():
            _, _, idx, weight = ops.three_nn_interpolate(xyz1, xyz2, points2.detach(), return_aux=True)
        interpolated = ops.three_interpolate(points2, idx, weight)
        new_points1 = torch.cat([interpolated, points1], dim=2) if points1 is not None else interpolated
        return mlp_training(new_points1, [(sc, True) for sc in scopes], bn_decay, params, frozen=frozen)
    interpolated = ops.three_nn_interpolate(xyz1, xyz2, points2)
    new_points1 = torch.cat([interpolated, points1], dim=2) if points1 is not None else interpolated
    return ops.shared_mlp(new_points1, params.mlp(scopes))


def pointnet_fp_module_broadcast(xyz1, xyz2, points1, points2, mlp, is_training, bn_decay, scope, bn=True, *, params: VariableStore):
    """pointnet_fp_module for a known level of ONE point (xyz2 (B,1,3), points2 (B,1,C2), e.g. after a group-all level), without
    building tile(points2) or its concatenation with points1.

    With one known point the reference's interpolation is a broadcast, exactly: three_nn leaves the two missing neighbours at their
    initial distance 1e40, inf in float (tf_interpolate.cpp:60-103), and index 0, so the weights (1/max(d,1e-10)) / sum
    (pointnet_util.py:211-216) are (1, 0, 0) and the interpolated rows are points2 itself.  The first layer's input is then
    concat([tile(points2), points1]), whose weight rows for points2 come first: those C2 rows run once per cloud (B rows) and the
    point layer adds the result per group of N1 rows (ops.shared_mlp_grouped; in training mode training.mlp_training(...,
    group=points2, group_first=True), differentiable in points1 and points2).  Results are those of pointnet_fp_module up to the order
    of the sums.  A non-finite coordinate makes the reference's weights NaN (inf / inf); this layer does not reproduce that."""
    if xyz2.shape[1] != 1 or points2.shape[1] != 1:
        raise ValueError(f"pointnet_fp_module_broadcast: the known level must have one point, got xyz2 {tuple(xyz2.shape)}, "
                         f"points2 {tuple(points2.shape)}")
    if points1 is None or not bn:
        raise NotImplementedError("pointnet_fp_module_broadcast needs skip features points1 and bn=True; use pointnet_fp_module")
    scopes = [f"{scope}/conv_{i}" for i in range(len(mlp))]
    b, c2 = points2.shape[0], points2.shape[-1]
    g = points2.reshape(b, c2)
    from .training import wants_input_grad
    frozen = not is_training and wants_input_grad(xyz1, xyz2, points1, points2)
    if is_training or frozen:
        from .training import mlp_training
        return mlp_training(points1, [(sc, True) for sc in scopes], bn_decay, params, frozen=frozen, group=g, group_first=True)
    rows_mlp, global_mlp = params.grouped_mlp(scopes, points1.shape[-1], group_first=True)
    return ops.shared_mlp_grouped(points1, rows_mlp, ops.shared_mlp(g, global_mlp))
