"""pointnet2/models/pointnet2_cls_bga.py on the libpsa kernels: joint classification + background-mask segmentation.
get_model(point_cloud, is_training, bn_decay, num_class) -> (class_pred (B,num_class), seg_pred (B,N,2)), same
layer hyper-parameters (pointnet2_cls_bga.py:30-66).  Inference (fused kernels, BN folded) and training (is_training=True:
batch-statistics BN, autograd over the hand-written level / MLP / interpolation kernels)."""
from __future__ import annotations

import torch

from . import ops
from .pointnet_util import add_fp_module_params, add_sa_module_params, pointnet_fp_module, pointnet_sa_module
from .tf_util import VariableStore

NUM_CLASSES = 15


def init_params(num_class=NUM_CLASSES, seed=0, device="cuda", randomize_bn=False) -> VariableStore:
    p = VariableStore(device=device, seed=seed)
    add_sa_module_params(p, "layer1", 3, [64, 64, 128], randomize_bn=randomize_bn)
    add_sa_module_params(p, "layer2", 3 + 128, [128, 128, 256], randomize_bn=randomize_bn)
    add_sa_module_params(p, "layer3", 3 + 256, [256, 512, 1024], randomize_bn=randomize_bn)
    p.add_fc("fc1", 1024, 512, bn=True, randomize_bn=randomize_bn)
    p.add_fc("fc2", 512, 256, bn=True, randomize_bn=randomize_bn)
    p.add_fc("fc3", 256, num_class, bn=False)
    add_fp_module_params(p, "fa_layer1", 256 + 256, [256, 256], randomize_bn=randomize_bn)
    add_fp_module_params(p, "fa_layer2", 256 + 128, [256, 128], randomize_bn=randomize_bn)
    add_fp_module_params(p, "fa_layer3", 128, [128, 128, 128], randomize_bn=randomize_bn)
    p.add_conv2d("seg_fc1", 128, 128, bn=True, randomize_bn=randomize_bn)      # conv1d k=1 == 1x1 conv
    p.add_conv2d("seg_fc2", 128, 2, bn=False)
    return p


def get_model(point_cloud, is_training, bn_decay=None, num_class=NUM_CLASSES, *, params: VariableStore, return_end_points: bool = False):
    from .training import wants_input_grad
    frozen = not is_training and wants_input_grad(point_cloud)
    if is_training or frozen:
        # frozen: inference mode with an input gradient -- the training kernels with batch norm on the moving averages, no dropout
        return _get_model_training(point_cloud, bn_decay, num_class, params, return_end_points, dropout=not frozen, frozen=frozen)
    batch_size = point_cloud.shape[0]
    end_points = {}
    l0_xyz = point_cloud[:, :, 0:3].contiguous()
    l0_points = None
    l1_xyz, l1_points, _ = pointnet_sa_module(l0_xyz, l0_points, npoint=512, radius=0.2, nsample=64, mlp=[64, 64, 128],
                                              mlp2=None, group_all=False, is_training=is_training, bn_decay=bn_decay,
                                              scope="layer1", params=params)
    l2_xyz, l2_points, _ = pointnet_sa_module(l1_xyz, l1_points, npoint=128, radius=0.4, nsample=64, mlp=[128, 128, 256],
                                              mlp2=None, group_all=False, is_training=is_training, bn_decay=bn_decay,
                                              scope="layer2", params=params)
    l3_xyz, l3_points, _ = pointnet_sa_module(l2_xyz, l2_points, npoint=None, radius=None, nsample=None,
                                              mlp=[256, 512, 1024], mlp2=None, group_all=True, is_training=is_training,
                                              bn_decay=bn_decay, scope="layer3", params=params)
    # classification branch
    net = l3_points.reshape(batch_size, -1)
    net = ops.shared_mlp(net, params.mlp(["fc1", "fc2"], [True, True]))
    class_vector = net.unsqueeze(1)                                          # (B,1,256)
    class_pred = ops.shared_mlp(net, params.mlp(["fc3"], [False]))
    # segmentation branch: three feature-propagation levels (three_nn + interpolation fused, on the GPU)
    l2_points = pointnet_fp_module(l2_xyz, l3_xyz, l2_points, class_vector, [256, 256], is_training, bn_decay,
                                   scope="fa_layer1", params=params)
    l1_points = pointnet_fp_module(l1_xyz, l2_xyz, l1_points, l2_points, [256, 128], is_training, bn_decay,
                                   scope="fa_layer2", params=params)
    l0_points = pointnet_fp_module(l0_xyz, l1_xyz, l0_points, l1_points, [128, 128, 128], is_training, bn_decay,
                                   scope="fa_layer3", params=params)
    feats = ops.shared_mlp(l0_points, params.mlp(["seg_fc1"], [True]))
    end_points["feats"] = feats
    seg_pred = ops.shared_mlp(feats, params.mlp(["seg_fc2"], [False]))
    end_points.update(l1_xyz=l1_xyz, l2_xyz=l2_xyz, l1_points=l1_points, l2_points=l2_points, l3_points=l3_points)
    # reference arity (pointnet2_cls_bga.py:75); the intermediate tensors only on request
    return (class_pred, seg_pred, end_points) if return_end_points else (class_pred, seg_pred)


def _get_model_training(point_cloud, bn_decay, num_class, params: VariableStore, return_end_points: bool, dropout: bool = True,
                        frozen: bool = False):
    """Training-mode forward (pointnet2_cls_bga.py:21-75 with is_training=True): every layer with batch-statistics batch norm, dropout
    (keep 0.5) after fc1 / fc2 / seg_fc1, PyTorch autograd over the hand-written level / MLP / interpolation kernels
    (training.py: sa_module_training, mlp_training; ops.three_interpolate).  Gradients of the variables arrive on
    ``params._flat.flat.grad`` (and per name through ``params._flat`` views).  frozen=True (with dropout=False): inference mode with
    batch norm on the moving averages, for a point cloud that requires grad -- input gradients only."""
    from .training import mlp_training
    f = torch.nn.functional
    b = point_cloud.shape[0]
    l0_xyz = point_cloud[:, :, 0:3].contiguous()
    sa = dict(mlp2=None, is_training=not frozen, bn_decay=bn_decay, params=params)
    mlp = lambda x, layers: mlp_training(x, layers, bn_decay, params, frozen=frozen)  # noqa: E731
    l1_xyz, l1_points, _ = pointnet_sa_module(l0_xyz, None, npoint=512, radius=0.2, nsample=64, mlp=[64, 64, 128], group_all=False, scope="layer1", **sa)
    l2_xyz, l2_points, _ = pointnet_sa_module(l1_xyz, l1_points, npoint=128, radius=0.4, nsample=64, mlp=[128, 128, 256], group_all=False, scope="layer2",
                                              **sa)
    l3_xyz, l3_points, _ = pointnet_sa_module(l2_xyz, l2_points, npoint=None, radius=None, nsample=None, mlp=[256, 512, 1024], group_all=True,
                                              scope="layer3", **sa)
    net = l3_points.reshape(b, -1)
    drop = (lambda t: f.dropout(t, 0.5, training=True)) if dropout else (lambda t: t)
    net = drop(mlp(net, [("fc1", True)]))                     # fc1 -> dp1
    net = mlp(net, [("fc2", True)])
    class_vector = net.unsqueeze(1)                                                      # taken BEFORE dp2 (pointnet2_cls_bga.py:45-48)
    class_pred = mlp(drop(net), [("fc3", False)])
    l2_points = pointnet_fp_module(l2_xyz, l3_xyz, l2_points, class_vector, [256, 256], not frozen, bn_decay, scope="fa_layer1", params=params)
    l1_points = pointnet_fp_module(l1_xyz, l2_xyz, l1_points, l2_points, [256, 128], not frozen, bn_decay, scope="fa_layer2", params=params)
    l0_points = pointnet_fp_module(l0_xyz, l1_xyz, None, l1_points, [128, 128, 128], not frozen, bn_decay, scope="fa_layer3", params=params)
    feats = mlp(l0_points, [("seg_fc1", True)])
    seg_pred = mlp(drop(feats), [("seg_fc2", False)])
    end_points = dict(feats=feats, l1_xyz=l1_xyz, l2_xyz=l2_xyz, l1_points=l1_points, l2_points=l2_points, l3_points=l3_points)
    return (class_pred, seg_pred, end_points) if return_end_points else (class_pred, seg_pred)


def get_loss(class_pred, seg_pred, gt_label, gt_mask, seg_weight=0.5):
    """(1-w)*mean CE(class) + w*mean over instances of mean per-point 2-way CE (pointnet2_cls_bga.py:78-93)."""
    f = torch.nn.functional
    classify_loss = f.cross_entropy(class_pred, gt_label.long())
    per_point = f.cross_entropy(seg_pred.reshape(-1, seg_pred.shape[-1]), gt_mask.reshape(-1).long(), reduction="none")
    seg_loss = per_point.reshape(gt_mask.shape).mean(dim=1).mean()
    return (1 - seg_weight) * classify_loss + seg_weight * seg_loss, classify_loss, seg_loss
