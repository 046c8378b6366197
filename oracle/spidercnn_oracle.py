"""float64 torch restatement of SpiderCNN's classifier (SpiderCNN/models/spidercnn_cls_xyz.py:20-68, utils/tf_util.py:59-235,
363-377, 407-429) in inference mode, in the reference's own order: the 20 Taylor vectors tiled over (B,N,k), the filter summed as
g1 + ... + g6, the (B,N,k,C,T) product reshaped to channel index c*T + t, the [1,k] VALID conv as an einsum over (slot, channel),
group norm from the moments of contiguous channel groups, tf.nn.top_k over the points, and the FC head with inference batch norm.

The neighbour indices are an input (the run's own kNN), so the restatement checks the arithmetic, not the kNN.  CPU or CUDA."""
from __future__ import annotations

import torch

TAYLOR_TERMS = ("weight_x", "weight_y", "weight_z", "weight_xyz", "weight_xy", "weight_yz", "weight_xz", "biases", "weight_xx",
                "weight_yy", "weight_zz", "weight_xxy", "weight_xyy", "weight_xxz", "weight_xzz", "weight_yyz", "weight_yzz",
                "weight_xxx", "weight_yyy", "weight_zzz")
GN_EPS = 1e-6
BN_EPS = 1e-3


def _d(t):
    return torch.as_tensor(t).to(torch.float64)


def group_point(points, idx):
    """points (B,N,C), idx (B,M,k) -> (B,M,k,C)"""
    b = points.shape[0]
    return points[torch.arange(b, device=points.device)[:, None, None], idx.long()]


def delta_of(xyz, idx):
    xyz = _d(xyz)
    return group_point(xyz, idx) - xyz[:, :, None, :]


def taylor_filter(delta, p, scope):
    """g_d (B,N,k,T) of tf_util.py:207-213, every variable tiled to (B,N,k,T)"""
    b, n, k, _ = delta.shape
    w = {name.replace("weight_", ""): _d(p[f"{scope}/{name}"]).reshape(-1).to(delta.device).expand(b, n, k, -1) for name in TAYLOR_TERMS}
    X, Y, Z = (delta[..., i:i + 1] for i in range(3))
    g1 = w["x"] * X + w["y"] * Y + w["z"] * Z + w["xyz"] * X * Y * Z
    g2 = w["xy"] * X * Y + w["yz"] * Y * Z + w["xz"] * X * Z + w["biases"]
    g3 = w["xx"] * X * X + w["yy"] * Y * Y + w["zz"] * Z * Z
    g4 = w["xxy"] * X * X * Y + w["xyy"] * X * Y * Y + w["xxz"] * X * X * Z
    g5 = w["xzz"] * X * Z * Z + w["yyz"] * Y * Y * Z + w["yzz"] * Y * Z * Z
    g6 = w["xxx"] * X * X * X + w["yyy"] * Y * Y * Y + w["zzz"] * Z * Z * Z
    return g1 + g2 + g3 + g4 + g5 + g6


def spider_conv_prenorm(feat, idx, delta, p, scope):
    """grouped_points * g_d reshaped to (B,N,k,C*T), then the [1,k] VALID conv + bias -> (B,N,C_out), before the group norm"""
    feat = _d(feat)
    grouped = group_point(feat, idx)                                   # (B,N,k,C)
    b, n, k, c = grouped.shape
    g = taylor_filter(delta, p, scope)                                 # (B,N,k,T)
    t = g.shape[-1]
    prod = (grouped[..., None] * g[:, :, :, None, :]).reshape(b, n, k, c * t)
    w = _d(p[f"{scope}/conv/weights"]).to(feat.device)                 # (1,k,C*T,C_out)
    return torch.einsum("bnjq,jqo->bno", prod, w[0]) + _d(p[f"{scope}/conv/biases"]).to(feat.device)


def group_norm(x, gamma, beta, G, eps=GN_EPS):
    """group_norm_for_conv on (B,N,C) (H = N, W = 1): moments over (C/G channels, N points) per cloud and group"""
    b, n, c = x.shape
    G = min(G, c)
    xt = x.permute(0, 2, 1).reshape(b, G, c // G, n)
    mean = xt.mean(dim=(2, 3), keepdim=True)
    var = ((xt - mean) ** 2).mean(dim=(2, 3), keepdim=True)
    xn = ((xt - mean) / torch.sqrt(var + eps)).reshape(b, c, n)
    return (xn * _d(gamma).to(x.device)[None, :, None] + _d(beta).to(x.device)[None, :, None]).permute(0, 2, 1)


def spider_layer(feat, idx, delta, p, scope, G=16):
    """-> (pre-norm y, relu(group_norm(y)))"""
    y = spider_conv_prenorm(feat, idx, delta, p, scope)
    h = torch.relu(group_norm(y, p[f"{scope}/conv/gn/gamma"], p[f"{scope}/conv/gn/beta"], G))
    return y, h


def topk_pool(x, k=2):
    """(B,N,C) -> (B,C,k): tf.nn.top_k of the transpose, largest first"""
    return torch.topk(x.permute(0, 2, 1), k, dim=-1, sorted=True).values


def fc(x, p, scope, bn=True, relu=True):
    y = x @ _d(p[f"{scope}/weights"]).to(x.device) + _d(p[f"{scope}/biases"]).to(x.device)
    if bn:
        mm, mv = _d(p[f"{scope}/bn/moving_mean"]).to(x.device), _d(p[f"{scope}/bn/moving_variance"]).to(x.device)
        y = (y - mm) / torch.sqrt(mv + BN_EPS) * _d(p[f"{scope}/bn/gamma"]).to(x.device) + _d(p[f"{scope}/bn/beta"]).to(x.device)
    return torch.relu(y) if relu else y


def forward(xyz, idx, p, G=16):
    """-> (logits (B,num_class), pooled (B,960), [(y_l, h_l)] of the four layers), all float64"""
    xyz = _d(xyz)
    delta = delta_of(xyz, idx)
    feat, layers = xyz, []
    for l in range(1, 5):
        y, h = spider_layer(feat, idx, delta, p, f"fanConv{l}/taylor", G)
        layers.append((y, h))
        feat = h
    cat = torch.cat([h for _, h in layers], dim=2)                     # (B,N,480)
    pooled = topk_pool(cat, 2).reshape(xyz.shape[0], -1)               # (B,960), index c*2 + r
    net = fc(pooled, p, "fc1")
    net = fc(net, p, "fc2")
    return fc(net, p, "fc3", bn=False, relu=False), pooled, layers
