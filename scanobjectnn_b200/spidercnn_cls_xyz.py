"""SpiderCNN/models/spidercnn_cls_xyz.py on the libpsa kernels, inference mode.

The reference (spidercnn_cls_xyz.py:20-68): kNN (k = 20, SelectionSort order) -> delta = neighbour - point -> four spiderConv
layers 3->32->64->128->256 (Taylor filters, T = 5, group norm with G = 16, ReLU) -> concat (B,N,480) -> top-2 pooling over the
points -> (B,960) -> fc1 1024, fc2 512 (batch norm, ReLU; dropout is the identity at inference) -> fc3.

Here each layer is one fused spiderConv launch that writes its pre-norm output y (B,N,C) and nothing of size B*N*k*C; the group
norm becomes a per-cloud affine (scale, shift) that the next layer and the top-2 pooling apply while they read y, so no activated
(B,N,C) tensor and no (B,N,480) concatenation is built.  Training mode is not implemented.
"""
from __future__ import annotations

import torch

from . import ops
from .tf_util import GN_EPS, VariableStore

NUM_CLASSES = 15
NSAMPLE = 20
TAYLOR_CHANNEL = 5
GROUPS = 16
CHANNELS = (32, 64, 128, 256)
POOLED = 2 * sum(CHANNELS)          # 960


def init_params(num_class=NUM_CLASSES, seed=0, device="cuda", randomize_bn=False) -> VariableStore:
    """The reference's variables: fanConv{1..4}/taylor/... (spiderConv, gn=True) and fc1..fc3 (batch norm under fc1/bn, fc2/bn).
    randomize_bn: non-trivial batch-norm statistics and group-norm gamma / beta, so that parity tests exercise the folding."""
    p = VariableStore(device=device, seed=seed)
    cin = 3
    for l, cout in enumerate(CHANNELS, start=1):
        scope = f"fanConv{l}/taylor"
        p.add_spider_conv(scope, cin, cout, NSAMPLE, TAYLOR_CHANNEL)
        if randomize_bn:
            r = lambda lo, hi: (torch.rand(cout, generator=p._gen) * (hi - lo) + lo).to(p.device)
            p[f"{scope}/conv/gn/gamma"] = r(0.8, 1.2)
            p[f"{scope}/conv/gn/beta"] = r(-0.1, 0.1)
        cin = cout
    p.add_fc("fc1", POOLED, 1024, randomize_bn=randomize_bn)
    p.add_fc("fc2", 1024, 512, randomize_bn=randomize_bn)
    p.add_fc("fc3", 512, num_class, bn=False)
    return p


def get_model(xyz, is_training, bn_decay=None, num_class=NUM_CLASSES, *, params: VariableStore, return_end_points: bool = False):
    """spidercnn_cls_xyz.get_model: xyz (B,N,3) -> logits (B,num_class); with return_end_points also a dict holding the kNN
    indices ``idx``, the pooled features ``pooled`` (B,960) and each layer's pre-norm ``y{l}`` and group-norm ``scale{l}`` /
    ``shift{l}`` (l = 1..4)."""
    if is_training:
        raise NotImplementedError("spidercnn_cls_xyz: training mode is not implemented (inference only)")
    if isinstance(xyz, torch.Tensor) and xyz.requires_grad and torch.is_grad_enabled():
        raise NotImplementedError("spidercnn_cls_xyz: gradients with respect to the input points are not implemented")
    if params["fc3/biases"].numel() != num_class:
        raise ValueError(f"num_class={num_class} but the store's fc3 has {params['fc3/biases'].numel()} outputs")
    b, n, _ = xyz.shape
    _, idx = ops.knn_point(NSAMPLE, xyz, xyz)
    delta = ops.group_point(xyz, idx) - xyz.unsqueeze(2)                      # (B,N,k,3), the reference's `delta` scope
    pooled = torch.empty((b, POOLED // 2, 2), dtype=torch.float32, device=xyz.device)
    end_points = {"idx": idx}
    feat, scale, shift, off = xyz, None, None, 0
    for l, cout in enumerate(CHANNELS, start=1):
        taylor, w, bias, gamma, beta = params.spider(f"fanConv{l}/taylor")
        y = ops.spider_conv(delta, idx, feat, taylor, w, bias, scale, shift)
        scale, shift = ops.group_norm_affine(y, gamma, beta, min(GROUPS, cout), GN_EPS)
        ops.topk_pool(y, 2, scale, shift, relu=True, out=pooled, offset=off)   # channel c of layer l -> rows off + c
        end_points.update({f"y{l}": y, f"scale{l}": scale, f"shift{l}": shift})
        feat, off = y, off + cout
    net = pooled.reshape(b, POOLED)                                           # index c*2 + r, as tf.reshape of (B,480,2)
    end_points["pooled"] = net
    logits = ops.shared_mlp(net, params.mlp(["fc1", "fc2", "fc3"], [True, True, False]))
    return (logits, end_points) if return_end_points else logits


def get_loss(pred, label):
    """Mean sparse softmax cross-entropy (spidercnn_cls_xyz.py:71-80)."""
    return torch.nn.functional.cross_entropy(pred, label.long())
