"""SpiderCNN/models/spidercnn_cls_xyz.py on the libpsa kernels, in inference mode (get_model) and training mode (get_model_training).

The reference (spidercnn_cls_xyz.py:20-68): kNN (k = 20, SelectionSort order) -> delta = neighbour - point -> four spiderConv
layers 3->32->64->128->256 (Taylor filters, T = 5, group norm with G = 16, ReLU) -> concat (B,N,480) -> top-2 pooling over the
points -> (B,960) -> fc1 1024, fc2 512 (batch norm, ReLU; dropout is the identity at inference) -> fc3.

Here each layer is one fused spiderConv launch that writes its pre-norm output y (B,N,C) and nothing of size B*N*k*C; the group
norm becomes a per-cloud affine (scale, shift) that the next layer and the top-2 pooling apply while they read y, so no activated
(B,N,C) tensor and no (B,N,480) concatenation is built.

Training (get_model_training, SpiderCNN/train.py:127-157): group norm normalises per cloud, so the four spiderConv layers run the
inference forward and keep their pre-norm y; the backward (SpiderTrainer.backward, fp32 FMA kernels of csrc/spider.cu) runs per layer,
top down: group-norm + ReLU + top-2 backward -> dy, conv biases from sum dy, dW = A^T . dy with the gathered operand A recomputed, then
D = sum_t g Q and dg = sum_c h Q from Q = dy . W^T formed tile by tile, d taylor from dg, and the gradient of the layer below's
activation = GroupPointGrad(D).  The largest tensor is D (B,N,k,C_in), never the (B,N,k,C_in*T) conv input.  fc1 / fc2 train with
batch statistics (training.mlp_training).
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib, ops
from ._lib import check
from ._lib import ptr as _p
from ._lib import stream as _stream
from .tf_util import GN_EPS, TAYLOR_TERMS, VariableStore

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
        raise NotImplementedError("spidercnn_cls_xyz.get_model runs inference only: train through get_model_training")
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


class SpiderTrainer:
    """The four spiderConv layers and the top-2 pooling of one (B, N) shape in training mode: forward(xyz) -> pooled (B,960),
    backward(dpooled) -> every spiderConv variable's slice of the store's flat gradient.  Buffers are allocated once."""

    def __init__(self, params: VariableStore, b: int, n: int, device):
        from .training import FlatParams
        self.lib = _lib.load()
        self.fp = params._flat if getattr(params, "_flat", None) is not None else FlatParams(params)
        params._flat = self.fp
        self.b, self.n, k, t = b, n, NSAMPLE, TAYLOR_CHANNEL
        f32 = dict(dtype=torch.float32, device=device)
        fp, self.layers, cin = self.fp, [], 3
        for l, cout in enumerate(CHANNELS, start=1):
            sc = f"fanConv{l}/taylor"
            w = fp.views[f"{sc}/conv/weights"]
            if tuple(w.shape) != (1, k, cin * t, cout):
                raise ValueError(f"{sc}/conv/weights: shape {tuple(w.shape)}, want {(1, k, cin * t, cout)}")
            tv = [fp.views[f"{sc}/{m}"] for m in TAYLOR_TERMS]
            tg = [fp.gviews[f"{sc}/{m}"] for m in TAYLOR_TERMS]
            step = tg[1].data_ptr() - tg[0].data_ptr()
            # the 20 gradient vectors sit at one stride in the flat bucket: d taylor is written in place, row m at m * stride
            assert all(tg[m].data_ptr() - tg[0].data_ptr() == m * step for m in range(20)) and step % 4 == 0, sc
            self.layers.append(dict(
                c=cin, cout=cout, groups=min(GROUPS, cout), taylor_views=tv, taylor=torch.empty((20, t), **f32), dtaylor=tg[0],
                ld_taylor=step // 4, W=w, b=fp.views[f"{sc}/conv/biases"], gamma=fp.views[f"{sc}/conv/gn/gamma"],
                beta=fp.views[f"{sc}/conv/gn/beta"], dW=fp.gviews[f"{sc}/conv/weights"], db=fp.gviews[f"{sc}/conv/biases"],
                dgamma=fp.gviews[f"{sc}/conv/gn/gamma"], dbeta=fp.gviews[f"{sc}/conv/gn/beta"], y=torch.empty((b, n, cout), **f32),
                scale=torch.empty((b, cout), **f32), shift=torch.empty((b, cout), **f32)))
            cin = cout
        self.names = [nm for nm in fp.names if nm.startswith("fanConv")]
        self.pooled = torch.empty((b, POOLED // 2, 2), **f32)
        rows = b * n
        self.g = torch.empty((b, n, k, t), **f32)
        self.dg = torch.empty((b, n, k, t), **f32)
        self.D = torch.empty(rows * k * max(CHANNELS[:-1]), **f32)            # (B,N,k,C_in) of the layer being differentiated
        self.dh = torch.empty(rows * max(CHANNELS[:-1]), **f32)               # gradient of the layer below's activation
        self.dy = torch.empty(rows * max(CHANNELS), **f32)
        dims = [(ly["c"], ly["cout"]) for ly in self.layers]
        self.ws_inf_bytes = max(self.lib.psa_spider_conv_workspace_bytes(b, n, c, k, t, co) for c, co in dims)
        self.ws_bwd_bytes = max(self.lib.psa_spider_conv_bwd_workspace_bytes(b, n, c, k, t, co) for c, co in dims)
        self.ws_inf = torch.empty(self.ws_inf_bytes // 4 + 64, **f32)
        self.ws_bwd = torch.empty(self.ws_bwd_bytes // 4 + 64, **f32)
        self.sc_bytes = int(self.lib.psa_scatter_workspace_bytes(b, n, n * k))
        self.ws_scatter = torch.empty(max(self.sc_bytes, 4), dtype=torch.uint8, device=device)

    def forward(self, xyz: torch.Tensor) -> torch.Tensor:
        b, n, k, t, lib = self.b, self.n, NSAMPLE, TAYLOR_CHANNEL, self.lib
        _, idx = ops.knn_point(NSAMPLE, xyz, xyz)
        self.idx = idx
        self.delta = (ops.group_point(xyz, idx) - xyz.unsqueeze(2)).contiguous()
        feat, scale, shift, off = xyz, None, None, 0
        self.feats = []
        for ly in self.layers:
            with torch.no_grad():
                torch.cat([v.reshape(1, t) for v in ly["taylor_views"]], out=ly["taylor"])
            self.feats.append((feat, scale, shift))
            check(lib.psa_spider_conv_infer(b, n, ly["c"], k, t, ly["cout"], _p(self.delta), _p(idx), _p(feat), _p(scale), _p(shift),
                                            _p(ly["taylor"]), _p(ly["W"]), _p(ly["b"]), _p(ly["y"]), _p(self.ws_inf),
                                            C.c_size_t(self.ws_inf_bytes), _stream()), "spider_conv")
            check(lib.psa_group_norm_affine(b, n, ly["cout"], ly["groups"], C.c_float(GN_EPS), _p(ly["y"]), _p(ly["gamma"]), _p(ly["beta"]),
                                            _p(ly["scale"]), _p(ly["shift"]), None, 0, _stream()), "group_norm_affine")
            check(lib.psa_topk_pool(b, n, ly["cout"], 2, _p(ly["y"]), _p(ly["scale"]), _p(ly["shift"]), 1, _p(self.pooled), POOLED // 2, off,
                                    _stream()), "topk_pool")
            feat, scale, shift, off = ly["y"], ly["scale"], ly["shift"], off + ly["cout"]
        return self.pooled.view(b, POOLED)

    def backward(self, dpooled: torch.Tensor):
        """dpooled (B,960) -> the spiderConv variables' gradients in the flat bucket's views"""
        from .training import _plain_grad
        b, n, k, t, lib = self.b, self.n, NSAMPLE, TAYLOR_CHANNEL, self.lib
        dpool = dpooled.contiguous()
        wsb, wsn = _p(self.ws_bwd), C.c_size_t(self.ws_bwd_bytes)
        off = POOLED // 2
        for l in range(len(self.layers) - 1, -1, -1):
            ly = self.layers[l]
            c, cout = ly["c"], ly["cout"]
            feat, scale, shift = self.feats[l]
            off -= cout
            dy = self.dy[:b * n * cout]
            check(lib.psa_spider_gn_bwd(b, n, cout, ly["groups"], C.c_float(GN_EPS), _p(ly["y"]), _p(ly["scale"]), _p(ly["shift"]), _p(ly["gamma"]),
                                        _p(dpool), POOLED // 2, off, _p(self.dh) if l < len(self.layers) - 1 else None, _p(dy), _p(ly["dgamma"]),
                                        _p(ly["dbeta"]), wsb, wsn, _stream()), "spider_gn_bwd")
            g_in = _plain_grad(dy.view(b * n, cout))
            check(lib.psa_train_bias_grad(b * n, cout, C.byref(g_in), _p(ly["db"]), _stream()), "train_bias_grad")
            check(lib.psa_spider_taylor_filter(b, n, k, t, _p(self.delta), _p(ly["taylor"]), _p(self.g), _stream()), "spider_taylor_filter")
            check(lib.psa_spider_conv_bwd_weight(b, n, c, k, t, cout, _p(self.idx), _p(feat), _p(scale), _p(shift), _p(self.g), _p(dy),
                                                 _p(ly["dW"]), wsb, wsn, _stream()), "spider_conv_bwd_weight")
            D = self.D if l > 0 else None
            check(lib.psa_spider_conv_bwd_data(b, n, c, k, t, cout, _p(self.idx), _p(feat), _p(scale), _p(shift), _p(self.g), _p(ly["W"]),
                                               _p(dy), _p(D), _p(self.dg), _stream()), "spider_conv_bwd_data")
            check(lib.psa_spider_taylor_grad(b, n, k, t, _p(self.delta), _p(self.dg), _p(ly["dtaylor"]), ly["ld_taylor"], wsb, wsn, _stream()),
                  "spider_taylor_grad")
            if l > 0:
                check(lib.psa_group_point_grad(b, n, c, n, k, _p(self.D), _p(self.idx), _p(self.dh), _p(self.ws_scatter),
                                               C.c_size_t(self.sc_bytes), _stream()), "group_point_grad")

    def flat_grad(self) -> torch.Tensor:
        """a gradient bucket holding the spiderConv variables' gradients and zeros elsewhere"""
        g = torch.zeros_like(self.fp.grad)
        base = self.fp.grad.data_ptr()
        for nm in self.names:
            v = self.fp.gviews[nm]
            o = (v.data_ptr() - base) // 4
            g[o:o + v.numel()].copy_(v.reshape(-1))
        return g


class _SpiderFn(torch.autograd.Function):
    """SpiderTrainer as one autograd node over the store's flat parameter vector"""

    @staticmethod
    def forward(ctx, flat, xyz, trainer):
        ctx.trainer = trainer
        return trainer.forward(xyz).clone()

    @staticmethod
    def backward(ctx, dpooled):
        tr = ctx.trainer
        tr.backward(dpooled)
        return tr.flat_grad(), None, None


def get_model_training(xyz, bn_decay=None, num_class=NUM_CLASSES, *, params: VariableStore, dropout: bool = True,
                       return_end_points: bool = False):
    """spidercnn_cls_xyz.get_model with is_training=True: xyz (B,N,3) -> logits (B,num_class), differentiable in the store's variables
    (autograd over its flat parameter vector, training.FlatParams).  fc1 / fc2 use batch statistics and update their moving averages
    with bn_decay (0.9 for None); dropout keeps 0.3 after each (dropout=False: the identity).  With return_end_points also a dict
    holding ``idx``, ``pooled`` and each layer's ``y{l}``, ``scale{l}``, ``shift{l}``.  Gradients with respect to xyz are not
    implemented."""
    from .training import _cached, mlp_training
    if isinstance(xyz, torch.Tensor) and xyz.requires_grad:
        raise NotImplementedError("spidercnn_cls_xyz: gradients with respect to the input points are not implemented")
    if params["fc3/biases"].numel() != num_class:
        raise ValueError(f"num_class={num_class} but the store's fc3 has {params['fc3/biases'].numel()} outputs")
    xyz = ops._dev(xyz, torch.float32, "xyz", 3).contiguous()
    b, n, _ = xyz.shape
    tr = _cached(params, ("spidercnn", b, n), lambda: SpiderTrainer(params, b, n, xyz.device))
    net = _SpiderFn.apply(tr.fp.flat.requires_grad_(True), xyz, tr)
    drop = (lambda v: torch.nn.functional.dropout(v, 0.7, training=True)) if dropout else (lambda v: v)
    net = drop(mlp_training(net, [("fc1", True)], bn_decay, params))
    net = drop(mlp_training(net, [("fc2", True)], bn_decay, params))
    logits = mlp_training(net, [("fc3", False)], bn_decay, params)
    if not return_end_points:
        return logits
    ep = {"idx": tr.idx, "pooled": tr.pooled.view(b, POOLED).clone()}
    for l, ly in enumerate(tr.layers, start=1):
        ep.update({f"y{l}": ly["y"], f"scale{l}": ly["scale"], f"shift{l}": ly["shift"]})
    return logits, ep


def get_loss(pred, label):
    """Mean sparse softmax cross-entropy (spidercnn_cls_xyz.py:71-80)."""
    return torch.nn.functional.cross_entropy(pred, label.long())
