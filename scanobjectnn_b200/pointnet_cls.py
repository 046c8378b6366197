"""pointnet/models/pointnet_cls.py (vanilla PointNet, BASELINE.json configs[0]: the reference's plumbing case) on the same
dense kernels; its trunk (trunk / trunk_training) is shared with pointnet_seg and pointnet_partseg: every layer is a per-point shared MLP (`psa_shared_mlp`), the symmetric function is its fused max-pool.
get_model(point_cloud, is_training, bn_decay, num_class) -> (logits (B,num_class), end_points).  Inference, and training through
autograd over training.mlp_training (is_training=True), and inference differentiable in the point cloud (the same nodes with batch
norm frozen on the moving averages) when the cloud requires a gradient."""
from __future__ import annotations

from functools import partial

import torch

from . import ops
from .tf_util import VariableStore

NUM_CLASSES = 15


def _add_tnet(p: VariableStore, scope: str, cin: int, K: int, rb: bool):
    p.add_conv2d(f"{scope}/tconv1", cin, 64, randomize_bn=rb)        # conv [1,3] over (B,N,3,1) == 3 -> 64 per point
    p.add_conv2d(f"{scope}/tconv2", 64, 128, randomize_bn=rb)
    p.add_conv2d(f"{scope}/tconv3", 128, 1024, randomize_bn=rb)
    p.add_fc(f"{scope}/tfc1", 1024, 512, randomize_bn=rb)
    p.add_fc(f"{scope}/tfc2", 512, 256, randomize_bn=rb)
    name = "transform_XYZ" if K == 3 else "transform_feat"            # transform_nets.py:38,80
    p[f"{scope}/{name}/weights"] = torch.zeros((256, K * K), device=p.device)
    p[f"{scope}/{name}/biases"] = torch.zeros(K * K, device=p.device)


def add_trunk_params(p: VariableStore, randomize_bn=False):
    """The variables PointNet's classification and segmentation models share: both T-nets and conv1-conv5."""
    _add_tnet(p, "transform_net1", 3, 3, randomize_bn)
    p.add_conv2d("conv1", 3, 64, randomize_bn=randomize_bn)
    p.add_conv2d("conv2", 64, 64, randomize_bn=randomize_bn)
    _add_tnet(p, "transform_net2", 64, 64, randomize_bn)
    p.add_conv2d("conv3", 64, 64, randomize_bn=randomize_bn)
    p.add_conv2d("conv4", 64, 128, randomize_bn=randomize_bn)
    p.add_conv2d("conv5", 128, 1024, randomize_bn=randomize_bn)


def add_fc_head_params(p: VariableStore, num_class=NUM_CLASSES, randomize_bn=False):
    p.add_fc("fc1", 1024, 512, randomize_bn=randomize_bn)
    p.add_fc("fc2", 512, 256, randomize_bn=randomize_bn)
    p.add_fc("fc3", 256, num_class, bn=False)


def init_params(num_class=NUM_CLASSES, seed=0, device="cuda", randomize_bn=False) -> VariableStore:
    p = VariableStore(device=device, seed=seed)
    add_trunk_params(p, randomize_bn)
    add_fc_head_params(p, num_class, randomize_bn)
    return p


def transform_net(x, params: VariableStore, scope: str, K: int):
    """input_transform_net / feature_transform_net (pointnet/models/transform_nets.py:10-97): (B,N,C) -> (B,K,K)."""
    b, n, c = x.shape
    g = ops.shared_mlp(x.reshape(b * n, c), params.mlp([f"{scope}/tconv1", f"{scope}/tconv2", f"{scope}/tconv3"]), pool_k=n)
    g = ops.shared_mlp(g, params.mlp([f"{scope}/tfc1", f"{scope}/tfc2"]))
    name = "transform_XYZ" if K == 3 else "transform_feat"
    w = params[f"{scope}/{name}/weights"]
    bias = params[f"{scope}/{name}/biases"] + torch.eye(K, device=w.device).flatten()
    return (g @ w + bias).reshape(b, K, K)


def _transform_net_training(x, params: VariableStore, scope: str, K: int, bn_decay, frozen: bool = False):
    from .training import mlp_training as _mlp_training
    mlp_training = partial(_mlp_training, frozen=frozen)
    b = x.shape[0]
    g = mlp_training(x, [(f"{scope}/tconv1", True), (f"{scope}/tconv2", True), (f"{scope}/tconv3", True)], bn_decay, params).amax(dim=1)
    g = mlp_training(g, [(f"{scope}/tfc1", True), (f"{scope}/tfc2", True)], bn_decay, params)
    name = "transform_XYZ" if K == 3 else "transform_feat"
    names = (f"{scope}/{name}/weights", f"{scope}/{name}/biases")
    w, bias = (params[v].detach() for v in names) if frozen else (params._flat.live(v) for v in names)
    return (g @ w + bias + torch.eye(K, device=w.device).flatten()).reshape(b, K, K)


def trunk_training(point_cloud, bn_decay, params: VariableStore, frozen: bool = False):
    """trunk() with is_training=True: batch-statistics batch norm, autograd over training.mlp_training nodes; the T-nets' matrices
    are torch ops on live views of the flat parameter vector.  frozen=True: batch norm on the moving averages (never updated), the
    T-nets' matrices read detached."""
    from .training import mlp_training as _mlp_training
    mlp_training = partial(_mlp_training, frozen=frozen)
    end_points = {}
    t1 = _transform_net_training(point_cloud.contiguous(), params, "transform_net1", 3, bn_decay, frozen)
    x = torch.bmm(point_cloud, t1)
    net = mlp_training(x, [("conv1", True), ("conv2", True)], bn_decay, params)
    t2 = _transform_net_training(net, params, "transform_net2", 64, bn_decay, frozen)
    end_points["transform"] = t2
    point_feat = torch.bmm(net, t2)
    net = mlp_training(point_feat, [("conv3", True), ("conv4", True), ("conv5", True)], bn_decay, params).amax(dim=1)
    end_points["global"] = net
    return point_feat, net, end_points


def fc_head_training(net, bn_decay, params: VariableStore, dropout: bool = True, frozen: bool = False):
    """fc1-fc3 in training mode, dropout (keep 0.7) after fc1 and fc2 unless frozen (pointnet_cls.py:62-69)."""
    from .training import mlp_training as _mlp_training
    mlp_training = partial(_mlp_training, frozen=frozen)
    f = torch.nn.functional
    drop = (lambda t: f.dropout(t, 0.3, training=True)) if dropout and not frozen else (lambda t: t)
    net = drop(mlp_training(net, [("fc1", True)], bn_decay, params))
    net = drop(mlp_training(net, [("fc2", True)], bn_decay, params))
    return mlp_training(net, [("fc3", False)], bn_decay, params)


def _get_model_training(point_cloud, bn_decay, num_class, params: VariableStore, dropout: bool = True, frozen: bool = False):
    """pointnet_cls.get_model with is_training=True (pointnet_cls.py:21-75): batch-statistics batch norm in every layer, dropout
    (keep 0.7) after fc1 and fc2, autograd over training.mlp_training nodes.  frozen=True: inference mode differentiable in the
    point cloud -- batch norm on the moving averages (never updated), no dropout, the T-nets' matrices read detached: no variable
    receives a gradient."""
    _, net, end_points = trunk_training(point_cloud, bn_decay, params, frozen)
    return fc_head_training(net, bn_decay, params, dropout, frozen), end_points


def trunk(point_cloud, params: VariableStore):
    """The inference part PointNet's classification and segmentation models share (pointnet_cls.py:21-60, pointnet_seg.py:24-64):
    input T-net, conv1-conv2, feature T-net, conv3-conv5 and the max over the points.  -> (point_feat (B,N,64) = the transformed
    conv2 features, global feature (B,1024), end_points)."""
    b, n, _ = point_cloud.shape
    end_points = {}
    t1 = transform_net(point_cloud, params, "transform_net1", 3)
    x = torch.bmm(point_cloud, t1).contiguous()                                       # tf.matmul(point_cloud, transform)
    net = ops.shared_mlp(x.reshape(b * n, 3), params.mlp(["conv1", "conv2"])).reshape(b, n, 64)
    t2 = transform_net(net, params, "transform_net2", 64)
    end_points["transform"] = t2
    point_feat = torch.bmm(net, t2).contiguous()
    net = ops.shared_mlp(point_feat.reshape(b * n, 64), params.mlp(["conv3", "conv4", "conv5"]), pool_k=n)   # max over the N points
    end_points["global"] = net
    return point_feat, net, end_points


def get_model(point_cloud, is_training, bn_decay=None, num_class=NUM_CLASSES, *, params: VariableStore):
    from .training import wants_input_grad
    frozen = not is_training and wants_input_grad(point_cloud)
    if is_training or frozen:
        return _get_model_training(point_cloud, bn_decay, num_class, params, frozen=frozen)
    _, net, end_points = trunk(point_cloud, params)
    net = ops.shared_mlp(net, params.mlp(["fc1", "fc2", "fc3"], [True, True, False]))
    return net, end_points


def get_loss(pred, label, end_points, reg_weight=0.001):
    """classification CE + reg_weight * || I - T T^t ||_F^2 / 2 on the feature transform (pointnet_cls.py:78-95)."""
    ce = torch.nn.functional.cross_entropy(pred, label.long())
    t = end_points["transform"]
    k = t.shape[1]
    diff = torch.bmm(t, t.transpose(1, 2)) - torch.eye(k, device=t.device)
    return ce + reg_weight * 0.5 * (diff ** 2).sum()
