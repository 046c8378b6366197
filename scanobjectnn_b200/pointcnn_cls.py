"""PointCNN/pointcnn_cls.py with the setting pointcnn_cls/modelnet_x3_l4.py on the libpsa kernels, inference mode.

The reference (pointcnn.py:55-152, pointcnn_cls.py:10-17): four X-Conv layers on the points alone (no extra features, random
sampling = the first P points of the previous level, X-transformation on, no sorting, no links), the last with the global branch
of the query coordinates in front of its output -> fc0 384, fc1 192 per point (dropout is the identity at inference) -> the mean
over the points -> logits with a bias, (B, 1, num_class).  Every layer with batch norm has no bias and applies ELU before the
batch norm (pointfly.py:298-347).

Here each X-Conv layer is a kNN launch (every D-th of the K*D nearest), one core launch that writes only the (B*P, C_in*dm)
depthwise output, and one tensor-core GEMM for the pointwise conv with the ELU / batch-norm epilogue.  The last layer's global
branch and pointwise conv write their slices of the 480-wide row in place, so nothing is concatenated, and no (B,P,K,.) tensor
is built.  Training mode is not implemented.
"""
from __future__ import annotations

import math

import torch

from . import ops
from .tf_util import VariableStore

NUM_CLASSES = 15
MIN_POINTS = 384                 # tf.slice of layer 2's 384 queries fails on fewer points
# (K, D, P, C) of xconv_params, x = 3 (modelnet_x3_l4.py); P = -1: every point is a query
XCONV = ((8, 1, -1, 48), (12, 2, 384, 96), (16, 2, 128, 192), (16, 3, 128, 384))
FC = (384, 192)                  # fc_params: C of fc0, fc1
WITH_GLOBAL = True


def layer_table():
    """[(tag, K, D, P, C, C_pts_fts, C_prev, dm, global width)] as PointCNN.__init__ derives them (pointcnn.py:104-112)"""
    out = []
    for i, (k, d, p, c) in enumerate(XCONV):
        if i == 0:
            c_pts, c_prev, dm = c // 2, 0, 4
        else:
            c_prev = XCONV[i - 1][3]
            c_pts, dm = c_prev // 4, math.ceil(c / c_prev)
        glob = c // 4 if WITH_GLOBAL and i == len(XCONV) - 1 else 0
        out.append((f"xconv_{i + 1}_", k, d, p, c, c_pts, c_prev, dm, glob))
    return out


def init_params(num_class=NUM_CLASSES, seed=0, device="cuda", randomize_bn=False) -> VariableStore:
    """The reference's variables in the order it creates them, with TF's names and shapes: per layer ``xconv_<l>_nn_fts_from_pts_0``,
    ``_nn_fts_from_pts``, ``_X_0``, ``_X_1``, ``_X_2``, ``_fts_conv`` (and ``_fts_global_0``, ``_fts_global`` on the last), each
    with its ``_bn`` batch norm; then ``fc0``, ``fc1`` and ``logits/{kernel,bias}``.  randomize_bn: non-trivial batch-norm
    statistics, so that parity tests exercise the affine."""
    p = VariableStore(device=device, seed=seed)
    add = lambda name, shape, bn=True: p.add_pointfly(name, shape, bn=bn, randomize_bn=randomize_bn)
    for tag, k, _, _, c, c_pts, c_prev, dm, glob in layer_table():
        c_in = c_pts + c_prev
        add(f"{tag}nn_fts_from_pts_0/kernel", (3, c_pts))
        add(f"{tag}nn_fts_from_pts/kernel", (c_pts, c_pts))
        add(f"{tag}X_0/kernel", (1, k, 3, k * k))
        add(f"{tag}X_1/depthwise_weights", (1, k, k, k))
        add(f"{tag}X_2/depthwise_weights", (1, k, k, k))
        add(f"{tag}fts_conv/depthwise_kernel", (1, k, c_in, dm), bn=False)
        add(f"{tag}fts_conv/pointwise_kernel", (1, 1, c_in * dm, c))
        if glob:
            add(f"{tag}fts_global_0/kernel", (3, glob))
            add(f"{tag}fts_global/kernel", (glob, glob))
    cin = XCONV[-1][3] + layer_table()[-1][8]
    for i, c in enumerate(FC):
        add(f"fc{i}/kernel", (cin, c))
        cin = c
    add("logits/kernel", (cin, num_class), bn=False)
    p["logits/bias"] = torch.zeros(num_class, device=p.device)
    return p


def xconv_weights(params: VariableStore, tag: str) -> dict:
    """The core kernel's weights of layer ``tag`` (ops.XCONV_WEIGHTS), TF-shaped, with the batch norms as (s, t)"""
    key = ("xconv", tag)
    if key not in params._cache:
        w = {}
        for short, layer, var in (("pts0", "nn_fts_from_pts_0", "kernel"), ("pts1", "nn_fts_from_pts", "kernel"), ("x0", "X_0", "kernel"),
                                  ("x1", "X_1", "depthwise_weights"), ("x2", "X_2", "depthwise_weights")):
            w[f"w_{short}"] = params[f"{tag}{layer}/{var}"].float().contiguous()
            w[f"s_{short}"], w[f"t_{short}"] = params.elu_bn(f"{tag}{layer}")
        w["w_dw"] = params[f"{tag}fts_conv/depthwise_kernel"].float().contiguous()
        params._cache[key] = w
    return params._cache[key]


def _dense(params, layer, var, x, out=None, offset=0):
    s, t = params.elu_bn(layer)
    w = params[f"{layer}/{var}"]
    return ops.dense_elu_affine(x, w.reshape(-1, w.shape[-1]), s, t, out=out, offset=offset)


def get_model(points, is_training, num_class=NUM_CLASSES, *, params: VariableStore, return_end_points: bool = False):
    """Net(points, features=None, is_training=False, setting).logits: points (B,N,3), N >= 384 -> logits (B,1,num_class); with
    return_end_points also a dict holding each layer's kNN indices ``idx<l>`` (B,P,K) and output ``fts<l>`` (B,P,C) (l = 1..4),
    ``fc0``, ``fc1`` (B*128, C) and the mean ``fc_mean`` (B,192)."""
    if is_training:
        raise NotImplementedError("pointcnn_cls: training mode is not implemented (inference only)")
    if isinstance(points, torch.Tensor) and points.requires_grad and torch.is_grad_enabled():
        raise NotImplementedError("pointcnn_cls: gradients with respect to the input points are not implemented")
    if params["logits/bias"].numel() != num_class:
        raise ValueError(f"num_class={num_class} but the store's logits layer has {params['logits/bias'].numel()} outputs")
    if points.dim() != 3 or points.shape[-1] != 3:
        raise ValueError(f"pointcnn_cls: points must be (B, N, 3), got {tuple(points.shape)}")
    b, n, _ = points.shape
    if n < MIN_POINTS:
        raise ValueError(f"pointcnn_cls: N={n} points, fewer than the {MIN_POINTS} queries of layer 2 (tf.slice fails)")
    pts = ops._dev(points, torch.float32, "points", 3)
    fts, end_points = None, {}
    for l, (tag, k, d, p, c, _, _, dm, glob) in enumerate(layer_table(), start=1):
        p = n if p == -1 else p
        qrs = pts if p == pts.shape[1] else pts[:, :p].contiguous()          # random sampling: the first P points (pointcnn.py:101)
        idx = ops.knn_dilated(pts, qrs, k, d)
        out = torch.empty((b * p, glob + c), dtype=torch.float32, device=pts.device)
        if glob:                                                              # [global | conv] (pointcnn.py:47-50), before the core
            g0 = _dense(params, f"{tag}fts_global_0", "kernel", qrs.reshape(b * p, 3))      # allocates its depthwise output
            _dense(params, f"{tag}fts_global", "kernel", g0, out=out, offset=0)
            del g0
        dw = ops.xconv_core(pts, qrs, idx, fts, xconv_weights(params, tag), dm)
        _dense(params, f"{tag}fts_conv", "pointwise_kernel", dw, out=out, offset=glob)
        del dw                                                                # freed before the next layer's core allocates its own
        fts, pts = out.view(b, p, glob + c), qrs
        if return_end_points:
            end_points.update({f"idx{l}": idx, f"fts{l}": fts})
    net = fts.reshape(-1, fts.shape[-1])
    for i in range(len(FC)):
        net = _dense(params, f"fc{i}", "kernel", net)
        if return_end_points:
            end_points[f"fc{i}"] = net
    mean = ops.pool_rows(net, pts.shape[1], "avg")                             # fc_mean (pointcnn_cls.py:13-14)
    end_points["fc_mean"] = mean
    head = params._cache.get(("logits",))
    if head is None:
        head = params._cache[("logits",)] = ops.MlpParams([(params["logits/kernel"].float().contiguous(), None,
                                                            params["logits/bias"].float().contiguous(), False)])
    logits = ops.shared_mlp(mean, head).reshape(b, 1, num_class)
    return (logits, end_points) if return_end_points else logits

