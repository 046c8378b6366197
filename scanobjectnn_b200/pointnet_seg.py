"""pointnet/models/pointnet_seg.py: PointNet's joint classification + background-mask model (train_seg.py).  The trunk is
pointnet_cls's; the segmentation head reads concat([point_feat (B,N,64), tile(global_feat, N) (B,N,1024)]), which is never built:
conv6's first 64 weight rows run over the points (K = 64) and its other 1024 rows over the B global features, one row per cloud
that the point layer adds before its batch norm (ops.shared_mlp_grouped; in training training.mlp_training(..., group=)).
get_model(point_cloud, is_training, bn_decay) -> (class_pred (B,15), seg_pred (B,N,2), end_points).  Inference, training
(is_training=True: batch-statistics batch norm, dropout after fc1 and fc2) and inference differentiable in the point cloud (batch
norm frozen on the moving averages) when the cloud requires a gradient."""
from __future__ import annotations

import torch

from . import ops, pointnet_cls
from .tf_util import VariableStore

NUM_CLASSES = 15
SEG_CLASSES = 2                      # background / object (the mask of train_seg.py)
HEAD = ["conv6", "conv7", "conv8", "conv9"]


def add_seg_head_params(p: VariableStore, num_seg: int, randomize_bn=False):
    """conv6 (1088 -> 512, the 64 point-feature rows first) ... conv9, and conv10 (128 -> num_seg, no batch norm)."""
    for scope, cin, cout in zip(HEAD, [1088, 512, 256, 128], [512, 256, 128, 128]):
        p.add_conv2d(scope, cin, cout, randomize_bn=randomize_bn)
    p.add_conv2d("conv10", 128, num_seg, bn=False)


def init_params(num_class=NUM_CLASSES, seed=0, device="cuda", randomize_bn=False) -> VariableStore:
    p = VariableStore(device=device, seed=seed)
    pointnet_cls.add_trunk_params(p, randomize_bn)
    pointnet_cls.add_fc_head_params(p, num_class, randomize_bn)
    add_seg_head_params(p, SEG_CLASSES, randomize_bn)
    return p


def seg_head(point_feat, global_feat, params: VariableStore):
    """conv6-conv10 over concat([point_feat, tile(global_feat)]) in inference mode: (B,N,64), (B,1024) -> (B,N,num_seg).
    conv6 and conv7 run as calls of their own: a chained call keeps two ping-pong buffers as wide as its widest layer, and at
    B=32, N=2048 two 512-wide ones would hold 256 MiB."""
    rows_mlp, global_mlp = params.grouped_mlp(HEAD[:1], point_feat.shape[-1])
    net = ops.shared_mlp_grouped(point_feat, rows_mlp, ops.shared_mlp(global_feat, global_mlp))
    net = ops.shared_mlp(net, params.mlp(HEAD[1:2]))
    return ops.shared_mlp(net, params.mlp(HEAD[2:] + ["conv10"], [True, True, False]))


def seg_head_training(point_feat, global_feat, bn_decay, params: VariableStore, frozen: bool = False):
    """seg_head in training mode (or frozen batch norm): one mlp_training node whose first layer takes the global feature per cloud."""
    from .training import mlp_training
    return mlp_training(point_feat, [(s, True) for s in HEAD] + [("conv10", False)], bn_decay, params, frozen=frozen, group=global_feat)


def _get_model_training(point_cloud, bn_decay, params: VariableStore, dropout: bool = True, frozen: bool = False):
    """get_model with is_training=True (dropout after fc1 and fc2), or frozen batch norm without dropout"""
    point_feat, global_feat, end_points = pointnet_cls.trunk_training(point_cloud, bn_decay, params, frozen)
    class_pred = pointnet_cls.fc_head_training(global_feat, bn_decay, params, dropout, frozen)
    return class_pred, seg_head_training(point_feat, global_feat, bn_decay, params, frozen), end_points


def get_model(point_cloud, is_training, bn_decay=None, *, params: VariableStore):
    from .training import wants_input_grad
    frozen = not is_training and wants_input_grad(point_cloud)
    if is_training or frozen:
        return _get_model_training(point_cloud, bn_decay, params, frozen=frozen)
    point_feat, global_feat, end_points = pointnet_cls.trunk(point_cloud, params)
    class_pred = ops.shared_mlp(global_feat, params.mlp(["fc1", "fc2", "fc3"], [True, True, False]))
    return class_pred, seg_head(point_feat, global_feat, params), end_points


def transform_regulariser(end_points):
    """tf.nn.l2_loss(T T^t - I) of the feature transform = || T T^t - I ||_F^2 / 2"""
    t = end_points["transform"]
    diff = torch.bmm(t, t.transpose(1, 2)) - torch.eye(t.shape[1], device=t.device)
    return 0.5 * (diff ** 2).sum()


def seg_cross_entropy(seg_pred, gt_seg):
    """mean over the clouds of the per-cloud mean point cross-entropy (pointnet_seg.py:122-123)"""
    return torch.nn.functional.cross_entropy(seg_pred.transpose(1, 2), gt_seg.long(), reduction="none").mean(dim=1).mean()


def get_loss(class_pred, seg_pred, gt_label, gt_mask, end_points, seg_weight=0.5, reg_weight=0.001):
    """pointnet_seg.py:111-134 -> (total, classify_loss, seg_loss): (1 - seg_weight) CE + seg_weight seg CE + reg_weight l2_loss(T T^t - I).
    gt_mask (B,N) holds the class of every point (0 background, 1 object: data_utils.convert_to_binary_mask)."""
    classify_loss = torch.nn.functional.cross_entropy(class_pred, gt_label.long())
    seg_loss = seg_cross_entropy(seg_pred, gt_mask)
    return (1 - seg_weight) * classify_loss + seg_weight * seg_loss + reg_weight * transform_regulariser(end_points), classify_loss, seg_loss
