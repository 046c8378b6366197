"""dgcnn/models/dgcnn.py and dgcnn_bga.py on the libpsa kernels (inference, and training through autograd over the same kernels: is_training=True;
inference with a gradient w.r.t. the point cloud runs the training kernels with batch norm frozen on the moving averages).

Every `pairwise_distance -> knn -> get_edge_feature -> conv2d -> reduce_max` group of the reference
(dgcnn.py:31-80) is two launches here: the fused kNN graph (no (B,N,N) matrix) and the fused EdgeConv
(gather [x_i, x_j - x_i] + MLP + max over k, no (B,N,k,2C) tensor)."""
from __future__ import annotations

from functools import partial

import torch

from . import ops
from .tf_util import VariableStore

NUM_CLASSES = 15
K_NEIGHBORS = 20


def init_params(num_class=NUM_CLASSES, seed=0, device="cuda", randomize_bn=False, bga=False) -> VariableStore:
    p = VariableStore(device=device, seed=seed)
    rb = randomize_bn
    # transform_net1 (dgcnn/models/transform_nets.py:10-55)
    p.add_conv2d("transform_net1/tconv1", 6, 64, randomize_bn=rb)
    p.add_conv2d("transform_net1/tconv2", 64, 128, randomize_bn=rb)
    p.add_conv2d("transform_net1/tconv3", 128, 1024, randomize_bn=rb)
    p.add_fc("transform_net1/tfc1", 1024, 512, randomize_bn=rb)
    p.add_fc("transform_net1/tfc2", 512, 256, randomize_bn=rb)
    # transform_XYZ: weights 0, biases 0 (+ identity added at run time), transform_nets.py:38-50
    p["transform_net1/transform_XYZ/weights"] = torch.zeros((256, 9), device=p.device)
    p["transform_net1/transform_XYZ/biases"] = torch.zeros(9, device=p.device)
    p.add_conv2d("dgcnn1", 6, 64, randomize_bn=rb)
    p.add_conv2d("dgcnn2", 128, 64, randomize_bn=rb)
    p.add_conv2d("dgcnn3", 128, 64, randomize_bn=rb)
    p.add_conv2d("dgcnn4", 128, 128, randomize_bn=rb)
    p.add_conv2d("agg", 320, 1024, randomize_bn=rb)
    p.add_fc("fc1", 1024, 512, randomize_bn=rb)
    p.add_fc("fc2", 512, 256, randomize_bn=rb)
    p.add_fc("fc3", 256, num_class, bn=False)
    if bga:
        p.add_conv2d("seg/conv1", 256 + 1024 + 320, 512, randomize_bn=rb)
        p.add_conv2d("seg/conv2", 512, 256, randomize_bn=rb)
        p.add_conv2d("seg/conv3", 256, 2, bn=False)
    return p


def input_transform_net(point_cloud, nn_idx, params: VariableStore, scope="transform_net1", K=3):
    """transform_nets.input_transform_net on the fused EdgeConv: -> (B,K,K)."""
    b, n, _ = point_cloud.shape
    net = ops.edgeconv_infer(point_cloud, nn_idx, params.mlp([f"{scope}/tconv1", f"{scope}/tconv2"]))   # max over k
    net = ops.shared_mlp(net.reshape(b * n, -1), params.mlp([f"{scope}/tconv3"]), pool_k=n)               # max over N
    net = ops.shared_mlp(net, params.mlp([f"{scope}/tfc1", f"{scope}/tfc2"]))
    w = params[f"{scope}/transform_XYZ/weights"]
    bias = params[f"{scope}/transform_XYZ/biases"] + torch.eye(K, device=w.device).flatten()
    return (net @ w + bias).reshape(b, K, K)


def _backbone(point_cloud, params, end_points, k=K_NEIGHBORS):
    b, n, _ = point_cloud.shape
    nn_idx = ops.knn_graph(point_cloud, k)
    transform = input_transform_net(point_cloud, nn_idx, params)
    pct = torch.bmm(point_cloud, transform).contiguous()                      # tf.matmul(point_cloud, transform), dgcnn.py:38
    end_points.update(nn_idx0=nn_idx, transform=transform, point_cloud_transformed=pct)
    nets = []
    x = pct
    for i, scope in enumerate(["dgcnn1", "dgcnn2", "dgcnn3", "dgcnn4"]):
        idx = ops.knn_graph(x, k)
        y = ops.edgeconv_infer(x, idx, params.mlp([scope]))
        end_points[f"nn_idx{i + 1}"] = idx
        end_points[f"net{i + 1}"] = y
        nets.append(y)
        x = y
    cat = torch.cat(nets, dim=-1)                                             # (B,N,320)
    # agg conv (320 -> 1024) with the max over the N points folded into its epilogue: the (B,N,1024) tensor is never written
    glob = ops.shared_mlp(cat.reshape(b * n, 320), params.mlp(["agg"]), pool_k=n)        # (B,1024)
    return nets, glob


def _edge_conv_training(x, k, layers, bn_decay, params, idx=None, frozen=False):
    """pairwise_distance -> knn -> get_edge_feature -> conv2d(+BN+ReLU)... -> reduce_max over k (dgcnn.py:31-44) in training mode.
    The neighbour graph carries no gradient; batch statistics over all B*N*k edges.  The single-layer EdgeConvs (dgcnn1..4) and the
    T-net's two-layer one run as the fused edgeconv_training: no per-edge tensor."""
    from .training import edgeconv_training
    if idx is None:
        with torch.no_grad():
            idx = ops.knn_graph(x.detach().contiguous(), k)
    scopes = [scope for scope, _ in layers]
    return edgeconv_training(x, idx, scopes[0] if len(scopes) == 1 else scopes, bn_decay, params, frozen=frozen), idx


def _get_model_training(point_cloud, bn_decay, num_class, params: VariableStore, dropout: bool = True, k=K_NEIGHBORS, graphs=None, bga: bool = False,
                        frozen: bool = False):
    """dgcnn.get_model with is_training=True (dgcnn.py:24-102, transform_nets.py:10-55): batch-statistics batch norm everywhere,
    dropout (keep 0.5) after fc1 and fc2, PyTorch autograd over the hand-written kernels.  `graphs` (tests): the five neighbour
    graphs to use instead of recomputing them -- the graphs are piecewise-constant functions of the parameters, which a finite
    difference must not cross.  frozen=True: inference mode differentiable in the point cloud -- batch norm on the moving averages
    (never updated), no dropout, and no gradient for any variable (the T-net's transform_XYZ is read detached, so nothing reaches
    the flat parameter vector)."""
    from .training import mlp_training as _mlp_training
    f = torch.nn.functional
    b, n, _ = point_cloud.shape
    end_points = {}
    dropout = dropout and not frozen
    mlp_training = partial(_mlp_training, frozen=frozen)
    drop = (lambda t: f.dropout(t, 0.5, training=True)) if dropout else (lambda t: t)
    # input transform net on the raw cloud
    sc = "transform_net1"
    net, idx0 = _edge_conv_training(point_cloud, k, [(f"{sc}/tconv1", True), (f"{sc}/tconv2", True)], bn_decay, params,
                                    None if graphs is None else graphs[0], frozen)                                        # (B,N,128)
    end_points["nn_idx0"] = idx0
    net = mlp_training(net, [(f"{sc}/tconv3", True)], bn_decay, params).amax(dim=1)                                       # (B,1024)
    net = mlp_training(net, [(f"{sc}/tfc1", True), (f"{sc}/tfc2", True)], bn_decay, params)                               # (B,256)
    names = (f"{sc}/transform_XYZ/weights", f"{sc}/transform_XYZ/biases")
    w, bias = (params[v].detach() for v in names) if frozen else (params._flat.live(v) for v in names)
    transform = (net @ w + bias + torch.eye(3, device=w.device).flatten()).reshape(b, 3, 3)
    x = torch.bmm(point_cloud, transform)
    end_points.update(transform=transform, point_cloud_transformed=x)
    nets = []
    for i, scope in enumerate(["dgcnn1", "dgcnn2", "dgcnn3", "dgcnn4"]):
        x, idx = _edge_conv_training(x, k, [(scope, True)], bn_decay, params, None if graphs is None else graphs[i + 1], frozen)
        end_points[f"nn_idx{i + 1}"] = idx
        end_points[f"net{i + 1}"] = x
        nets.append(x)
    net = mlp_training(torch.cat(nets, dim=-1), [("agg", True)], bn_decay, params).amax(dim=1)                            # (B,1024)
    end_points["global"] = net
    if bga:
        # dgcnn_bga.py:95-134: class vector taken after fc2 (before dp2); per-point head on [class vector, global max, net1..net4]
        out_max = net
        net = drop(mlp_training(net, [("fc1", True)], bn_decay, params))
        net = mlp_training(net, [("fc2", True)], bn_decay, params)
        class_pred = mlp_training(drop(net), [("fc3", False)], bn_decay, params)
        concat = torch.cat([net.unsqueeze(1).expand(b, n, 256), out_max.unsqueeze(1).expand(b, n, 1024), *nets], dim=-1)
        # seg/conv1 and seg/conv2 are built without bn_decay (dgcnn_bga.py:125-128): their moving averages always decay at the default 0.9
        seg = mlp_training(concat, [("seg/conv1", True), ("seg/conv2", True)], None, params)
        if dropout:
            seg = f.dropout(seg, 0.3, training=True)                                                                      # keep_prob 0.7
        return class_pred, mlp_training(seg, [("seg/conv3", False)], bn_decay, params), end_points
    net = drop(mlp_training(net, [("fc1", True)], bn_decay, params))
    net = drop(mlp_training(net, [("fc2", True)], bn_decay, params))
    return mlp_training(net, [("fc3", False)], bn_decay, params), end_points


def get_model(point_cloud, is_training, bn_decay=None, num_class=NUM_CLASSES, *, params: VariableStore):
    """dgcnn.get_model (dgcnn.py:24-102): (B,N,3) -> (logits (B,num_class), end_points).  Inference mode with a point cloud that
    requires a gradient (and gradients enabled) runs the training kernels on frozen batch norm, so the logits differentiate in it."""
    from .training import wants_input_grad
    frozen = not is_training and wants_input_grad(point_cloud)
    if is_training or frozen:
        return _get_model_training(point_cloud, bn_decay, num_class, params, frozen=frozen)
    end_points = {}
    _, net = _backbone(point_cloud, params, end_points)                      # tf.reduce_max over N already applied
    end_points["global"] = net
    net = ops.shared_mlp(net, params.mlp(["fc1", "fc2", "fc3"], [True, True, False]))
    return net, end_points


def get_model_bga(point_cloud, is_training, bn_decay=None, num_class=NUM_CLASSES, *, params: VariableStore, return_end_points: bool = False):
    """dgcnn_bga.get_model (dgcnn_bga.py:27-134): -> (class_pred (B,num_class), seg_pred (B,N,2), end_points).  Differentiable in
    the point cloud in inference mode as get_model is."""
    from .training import wants_input_grad
    frozen = not is_training and wants_input_grad(point_cloud)
    if is_training or frozen:
        cp, sp, ep = _get_model_training(point_cloud, bn_decay, num_class, params, bga=True, frozen=frozen)
        return (cp, sp, ep) if return_end_points else (cp, sp)
    end_points = {}
    b, n, _ = point_cloud.shape
    nets, out_max = _backbone(point_cloud, params, end_points)               # (B,1024)
    net = ops.shared_mlp(out_max, params.mlp(["fc1", "fc2"], [True, True]))   # class vector (B,256)
    class_pred = ops.shared_mlp(net, params.mlp(["fc3"], [False]))
    concat = torch.cat([net.unsqueeze(1).expand(b, n, 256), out_max.unsqueeze(1).expand(b, n, 1024), *nets], dim=-1)
    seg = ops.shared_mlp(concat.reshape(b * n, -1).contiguous(), params.mlp(["seg/conv1", "seg/conv2", "seg/conv3"], [True, True, False]))
    # reference arity (dgcnn_bga.py:134); the intermediate tensors only on request
    return (class_pred, seg.reshape(b, n, 2), end_points) if return_end_points else (class_pred, seg.reshape(b, n, 2))


def get_loss(pred, label, end_points=None, num_class=NUM_CLASSES):
    """softmax cross-entropy with label smoothing 0.2 (dgcnn.py:105-111)."""
    return torch.nn.functional.cross_entropy(pred, label.long(), label_smoothing=0.2)


def get_loss_bga(class_pred, seg_pred, gt_label, gt_mask, seg_weight=0.5):
    """dgcnn_bga.get_loss (dgcnn_bga.py:137-152): (1-w)*mean CE(class) + w*mean over clouds of the mean per-point 2-way CE, without
    get_loss's label smoothing -> (total, classify, seg)"""
    f = torch.nn.functional
    classify_loss = f.cross_entropy(class_pred, gt_label.long())
    per_point = f.cross_entropy(seg_pred.reshape(-1, seg_pred.shape[-1]), gt_mask.reshape(-1).long(), reduction="none")
    seg_loss = per_point.reshape(gt_mask.shape).mean(dim=1).mean()
    return (1 - seg_weight) * classify_loss + seg_weight * seg_loss, classify_loss, seg_loss
