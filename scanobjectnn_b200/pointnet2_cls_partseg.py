"""pointnet2/models/pointnet2_cls_partseg.py on the libpsa kernels: PointNet++ part segmentation (train_partseg.py).
get_model(point_cloud, is_training, bn_decay, num_class) -> seg_pred (B,N,num_class), the same layer hyper-parameters
(pointnet2_cls_partseg.py:20-45): pointnet2_cls_bga's set-abstraction levels and segmentation branch without its classification
head.  Its fa_layer1 interpolates from the single group-all point, an exact broadcast that pointnet_fp_module_broadcast folds into a
grouped first layer: the (B,128,1280) input of fa_layer1/conv_0 is never built.  Inference (fused kernels, batch norm folded),
training (is_training=True: batch-statistics batch norm, dropout after seg_fc1) and inference differentiable in the point cloud
(batch norm frozen on the moving averages) when the cloud requires a gradient.  The number of parts is that of the store
(init_params(num_class)); get_model's num_class is the reference's argument and must agree."""
from __future__ import annotations

import torch

from . import ops
from .pointnet_seg import seg_cross_entropy
from .pointnet_util import add_fp_module_params, add_sa_module_params, pointnet_fp_module, pointnet_fp_module_broadcast, pointnet_sa_module
from .tf_util import VariableStore

NUM_CLASSES = 6


def init_params(num_class=NUM_CLASSES, seed=0, device="cuda", randomize_bn=False) -> VariableStore:
    p = VariableStore(device=device, seed=seed)
    add_sa_module_params(p, "layer1", 3, [64, 64, 128], randomize_bn=randomize_bn)
    add_sa_module_params(p, "layer2", 3 + 128, [128, 128, 256], randomize_bn=randomize_bn)
    add_sa_module_params(p, "layer3", 3 + 256, [256, 512, 1024], randomize_bn=randomize_bn)
    add_fp_module_params(p, "fa_layer1", 1024 + 256, [256, 256], randomize_bn=randomize_bn)    # rows 0-1023 read l3_points
    add_fp_module_params(p, "fa_layer2", 256 + 128, [256, 128], randomize_bn=randomize_bn)
    add_fp_module_params(p, "fa_layer3", 128, [128, 128, 128], randomize_bn=randomize_bn)
    p.add_conv1d("seg_fc1", 128, 128, bn=True, randomize_bn=randomize_bn)
    p.add_conv1d("seg_fc2", 128, num_class, bn=False)
    return p


def get_model(point_cloud, is_training, bn_decay=None, num_class=NUM_CLASSES, *, params: VariableStore, return_end_points: bool = False):
    from .training import wants_input_grad
    if params["seg_fc2/weights"].shape[-1] != num_class:
        raise ValueError(f"num_class={num_class}, but the store's seg_fc2 has {params['seg_fc2/weights'].shape[-1]} outputs")
    frozen = not is_training and wants_input_grad(point_cloud)
    if is_training or frozen:
        # frozen: inference mode with an input gradient -- the training kernels with batch norm on the moving averages, no dropout
        return _get_model_training(point_cloud, bn_decay, params, return_end_points, dropout=not frozen, frozen=frozen)
    l0_xyz = point_cloud[:, :, 0:3].contiguous()
    sa = dict(mlp2=None, is_training=False, bn_decay=bn_decay, params=params)
    l1_xyz, l1_points, _ = pointnet_sa_module(l0_xyz, None, npoint=512, radius=0.2, nsample=64, mlp=[64, 64, 128], group_all=False, scope="layer1", **sa)
    l2_xyz, l2_points, _ = pointnet_sa_module(l1_xyz, l1_points, npoint=128, radius=0.4, nsample=64, mlp=[128, 128, 256], group_all=False, scope="layer2",
                                              **sa)
    l3_xyz, l3_points, _ = pointnet_sa_module(l2_xyz, l2_points, npoint=None, radius=None, nsample=None, mlp=[256, 512, 1024], group_all=True,
                                              scope="layer3", **sa)
    l2_points = pointnet_fp_module_broadcast(l2_xyz, l3_xyz, l2_points, l3_points, [256, 256], False, bn_decay, scope="fa_layer1", params=params)
    l1_points = pointnet_fp_module(l1_xyz, l2_xyz, l1_points, l2_points, [256, 128], False, bn_decay, scope="fa_layer2", params=params)
    l0_points = pointnet_fp_module(l0_xyz, l1_xyz, None, l1_points, [128, 128, 128], False, bn_decay, scope="fa_layer3", params=params)
    feats = ops.shared_mlp(l0_points, params.mlp(["seg_fc1"], [True]))
    seg_pred = ops.shared_mlp(feats, params.mlp(["seg_fc2"], [False]))
    end_points = dict(feats=feats, l1_xyz=l1_xyz, l2_xyz=l2_xyz, l1_points=l1_points, l2_points=l2_points, l3_points=l3_points)
    # reference arity (pointnet2_cls_partseg.py:45); the intermediate tensors only on request
    return (seg_pred, end_points) if return_end_points else seg_pred


def _get_model_training(point_cloud, bn_decay, params: VariableStore, return_end_points: bool = False, dropout: bool = True,
                        frozen: bool = False):
    """Training-mode forward (pointnet2_cls_partseg.py:20-45 with is_training=True): every layer with batch-statistics batch norm,
    dropout (keep 0.5) after seg_fc1 unless dropout=False, PyTorch autograd over the hand-written level / MLP / interpolation kernels.
    Gradients of the variables arrive on ``params._flat.flat.grad``.  frozen=True (with dropout=False): inference mode with batch norm
    on the moving averages, for a point cloud that requires grad -- input gradients only."""
    from .training import mlp_training
    l0_xyz = point_cloud[:, :, 0:3].contiguous()
    sa = dict(mlp2=None, is_training=not frozen, bn_decay=bn_decay, params=params)
    l1_xyz, l1_points, _ = pointnet_sa_module(l0_xyz, None, npoint=512, radius=0.2, nsample=64, mlp=[64, 64, 128], group_all=False, scope="layer1", **sa)
    l2_xyz, l2_points, _ = pointnet_sa_module(l1_xyz, l1_points, npoint=128, radius=0.4, nsample=64, mlp=[128, 128, 256], group_all=False, scope="layer2",
                                              **sa)
    l3_xyz, l3_points, _ = pointnet_sa_module(l2_xyz, l2_points, npoint=None, radius=None, nsample=None, mlp=[256, 512, 1024], group_all=True,
                                              scope="layer3", **sa)
    l2_points = pointnet_fp_module_broadcast(l2_xyz, l3_xyz, l2_points, l3_points, [256, 256], not frozen, bn_decay, scope="fa_layer1",
                                             params=params)
    l1_points = pointnet_fp_module(l1_xyz, l2_xyz, l1_points, l2_points, [256, 128], not frozen, bn_decay, scope="fa_layer2", params=params)
    l0_points = pointnet_fp_module(l0_xyz, l1_xyz, None, l1_points, [128, 128, 128], not frozen, bn_decay, scope="fa_layer3", params=params)
    feats = mlp_training(l0_points, [("seg_fc1", True)], bn_decay, params, frozen=frozen)
    net = torch.nn.functional.dropout(feats, 0.5, training=True) if dropout else feats
    seg_pred = mlp_training(net, [("seg_fc2", False)], bn_decay, params, frozen=frozen)
    end_points = dict(feats=feats, l1_xyz=l1_xyz, l2_xyz=l2_xyz, l1_points=l1_points, l2_points=l2_points, l3_points=l3_points)
    return (seg_pred, end_points) if return_end_points else seg_pred


def get_loss(seg_pred, gt_seg):
    """pointnet2_cls_partseg.py:54-87: the mean over the clouds of the per-cloud mean point cross-entropy"""
    return seg_cross_entropy(seg_pred, gt_seg)
