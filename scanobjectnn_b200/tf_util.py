"""The slice of the reference's tf_util.py files that sits on the hot path, on torch CUDA tensors.

* variable store with the reference's TF variable names (``layer1/conv0/weights``, ``.../bn/gamma`` ...), so a
  TF checkpoint name map is the identity;
* ``conv2d`` 1x1 / ``fully_connected`` (+bias +batch norm +ReLU) in inference mode, executed by the hand-written
  dense-layer kernel (pointnet2/utils/tf_util.py:120-185, 512-531; dgcnn/utils/tf_util.py:115-173, 462-499);
* DGCNN's graph functions (dgcnn/utils/tf_util.py:638-706);
* SpiderCNN's ``spiderConv``, ``group_norm_for_conv`` and ``topk_pool`` in inference mode (SpiderCNN/utils/tf_util.py:127-235,
  363-377, 407-429).
"""
from __future__ import annotations

import math

import torch

from . import ops
from .ops import get_edge_feature, knn, knn_graph, pairwise_distance  # noqa: F401

BN_EPS = 1e-3   # tf.contrib.layers.batch_norm default (pointnet2 tf_util.py:526-531); explicit in dgcnn tf_util.py:498
GN_EPS = 1e-6   # group_norm_for_conv's default (SpiderCNN/utils/tf_util.py:407)
# spiderConv's Taylor variables in the order the reference creates them (tf_util.py:181-205); "biases" is the constant term.
# This is also the row order of the (20, T) coefficient matrix of ops.spider_conv / psa_spider_conv_infer.
TAYLOR_TERMS = ("weight_x", "weight_y", "weight_z", "weight_xyz", "weight_xy", "weight_yz", "weight_xz", "biases", "weight_xx",
                "weight_yy", "weight_zz", "weight_xxy", "weight_xyy", "weight_xxz", "weight_xzz", "weight_yyz", "weight_yzz",
                "weight_xxx", "weight_yyy", "weight_zzz")


class VariableStore(dict):
    """name -> tensor, named exactly as the reference's TF variable scopes name them."""

    def __init__(self, device="cuda", seed: int = 0):
        super().__init__()
        self.device = torch.device(device)
        self._gen = torch.Generator(device="cpu")
        self._gen.manual_seed(seed)
        self._cache = {}

    # --- initialisers (tf_util._variable_with_weight_decay with use_xavier=True; biases 0; BN gamma 1 / beta 0) ---
    def _xavier(self, shape, fan_in, fan_out):
        limit = math.sqrt(6.0 / (fan_in + fan_out))
        w = (torch.rand(shape, generator=self._gen, dtype=torch.float32) * 2 - 1) * limit
        return w.to(self.device)

    def _bn(self, scope, c, randomize):
        if randomize:   # non-trivial statistics so parity tests exercise the folding
            r = lambda lo, hi: (torch.rand(c, generator=self._gen) * (hi - lo) + lo).to(self.device)
            self[f"{scope}/bn/beta"] = r(-0.1, 0.1)
            self[f"{scope}/bn/gamma"] = r(0.8, 1.2)
            self[f"{scope}/bn/moving_mean"] = r(-0.1, 0.1)
            self[f"{scope}/bn/moving_variance"] = r(0.5, 1.5)
        else:
            self[f"{scope}/bn/beta"] = torch.zeros(c, device=self.device)
            self[f"{scope}/bn/gamma"] = torch.ones(c, device=self.device)
            self[f"{scope}/bn/moving_mean"] = torch.zeros(c, device=self.device)
            self[f"{scope}/bn/moving_variance"] = torch.ones(c, device=self.device)

    def add_conv2d(self, scope, cin, cout, bn=True, randomize_bn=False):
        self[f"{scope}/weights"] = self._xavier((1, 1, cin, cout), cin, cout)
        self[f"{scope}/biases"] = torch.zeros(cout, device=self.device)
        if bn:
            self._bn(scope, cout, randomize_bn)

    def add_conv1d(self, scope, cin, cout, bn=True, randomize_bn=False):
        """tf_util.conv1d with kernel_size 1: the weights are (1, Cin, Cout), the same values add_conv2d would draw"""
        self[f"{scope}/weights"] = self._xavier((1, cin, cout), cin, cout)
        self[f"{scope}/biases"] = torch.zeros(cout, device=self.device)
        if bn:
            self._bn(scope, cout, randomize_bn)

    def add_fc(self, scope, cin, cout, bn=True, randomize_bn=False):
        self[f"{scope}/weights"] = self._xavier((cin, cout), cin, cout)
        self[f"{scope}/biases"] = torch.zeros(cout, device=self.device)
        if bn:
            self._bn(scope, cout, randomize_bn)

    def add_conv3d(self, scope, k, cin, cout, randomize_bn=False):
        """tf_util.conv3d with bn=True (3DmFV-Net/utils/tf_util.py:254-311): weights (k,k,k,cin,cout) with Xavier limits from TF's
        5-D fans k^3*cin and k^3*cout, zero biases, and the batch norm under ``scope/bn``."""
        self[f"{scope}/weights"] = self._xavier((k, k, k, cin, cout), k ** 3 * cin, k ** 3 * cout)
        self[f"{scope}/biases"] = torch.zeros(cout, device=self.device)
        self._bn(scope, cout, randomize_bn)

    def add_spider_conv(self, scope, cin, cout, k=20, taylor_channel=5):
        """spiderConv's variables under ``scope`` (e.g. ``fanConv1/taylor``) with gn=True, bn=False: the 20 Taylor vectors
        (1,1,1,T) (Xavier with TF's 4-D fans 1 and T; ``biases`` zero), the [1,k] conv (1,k,cin*T,cout) (fans k*cin*T and
        k*cout), its biases and the group norm's gamma / beta."""
        t = taylor_channel
        for name in TAYLOR_TERMS:
            shape = (1, 1, 1, t)
            self[f"{scope}/{name}"] = torch.zeros(shape, device=self.device) if name == "biases" else self._xavier(shape, 1, t)
        self[f"{scope}/conv/weights"] = self._xavier((1, k, cin * t, cout), k * cin * t, k * cout)
        self[f"{scope}/conv/biases"] = torch.zeros(cout, device=self.device)
        self[f"{scope}/conv/gn/gamma"] = torch.ones(cout, device=self.device)
        self[f"{scope}/conv/gn/beta"] = torch.zeros(cout, device=self.device)

    def spider(self, scope):
        """(taylor (20,T), conv weights (k, cin*T, cout), conv biases, gn gamma, gn beta) of a spiderConv ``scope``, as
        ops.spider_conv / ops.group_norm_affine take them; cached like ``folded``."""
        key = ("spider", scope)
        if key not in self._cache:
            taylor = torch.cat([self[f"{scope}/{name}"].reshape(1, -1).float() for name in TAYLOR_TERMS]).contiguous()
            w = self[f"{scope}/conv/weights"].float()
            self._cache[key] = (taylor, w.reshape(w.shape[-3:]).contiguous(), self[f"{scope}/conv/biases"].float().contiguous(),
                                self[f"{scope}/conv/gn/gamma"].float().contiguous(), self[f"{scope}/conv/gn/beta"].float().contiguous())
        return self._cache[key]

    # --- inference-mode folding: y = relu((x.W) * scale + shift) ---
    def folded(self, scope, relu=True):
        """(W (Cin,Cout), scale or None, shift, relu) for ``scope``; BN folded if ``scope/bn/gamma`` exists."""
        key = ("layer", scope, relu)
        if key not in self._cache:
            w = self[f"{scope}/weights"]
            w2 = w.reshape(-1, w.shape[-1]).contiguous().float()
            b = self[f"{scope}/biases"].float()
            if f"{scope}/bn/gamma" in self:
                inv = self[f"{scope}/bn/gamma"].float() * torch.rsqrt(self[f"{scope}/bn/moving_variance"].float() + BN_EPS)
                shift = (b - self[f"{scope}/bn/moving_mean"].float()) * inv + self[f"{scope}/bn/beta"].float()
                self._cache[key] = (w2, inv.contiguous(), shift.contiguous(), relu)
            else:
                self._cache[key] = (w2, None, b.contiguous(), relu)
        return self._cache[key]

    def mlp(self, scopes, relus=None, xyz_last: bool = False) -> ops.MlpParams:
        """``xyz_last``: the first layer's input is [features, xyz] (pointnet_sa_module_msg concatenates that way,
        pointnet_util.py:184) -- its last three weight rows are rotated to the front, which is where the fused kernels
        expect the coordinate rows."""
        relus = relus if relus is not None else [True] * len(scopes)
        key = ("mlp", tuple(scopes), tuple(relus), xyz_last)
        if key not in self._cache:
            layers = [self.folded(s, r) for s, r in zip(scopes, relus)]
            if xyz_last:
                w, sc, sh, r = layers[0]
                layers[0] = (torch.cat([w[-3:], w[:-3]], dim=0).contiguous(), sc, sh, r)
            self._cache[key] = ops.MlpParams(layers)
        return self._cache[key]

    def grouped_mlp(self, scopes, point_rows: int, group_first: bool = False):
        """The chain ``scopes`` (ReLU after every layer) whose first layer reads concat([point features (point_rows), global
        feature]), or concat([global feature, point features]) with group_first, split for ops.shared_mlp_grouped: (the chain with
        the first layer's point rows, the plain product over its global rows)."""
        key = ("grouped_mlp", tuple(scopes), point_rows, group_first)
        if key not in self._cache:
            layers = [self.folded(s) for s in scopes]
            w, sc, sh, r = layers[0]
            split = w.shape[0] - point_rows if group_first else point_rows
            w_pts, w_glob = (w[split:], w[:split]) if group_first else (w[:split], w[split:])
            glob = ops.MlpParams([(w_glob.contiguous(), None, torch.zeros_like(sh), False)])
            self._cache[key] = (ops.MlpParams([(w_pts.contiguous(), sc, sh, r)] + layers[1:]), glob)
        return self._cache[key]

    def invalidate(self):
        """Drop the folded conv+BN tensors / prepared weight images.  Called automatically when a variable is assigned,
        updated or deleted; call it yourself after an IN-PLACE edit of a weight tensor.  Inference engines / CUDA graphs
        captured earlier keep the old images: rebuild them after a weight change."""
        self._cache.clear()

    # assigning variables (e.g. loading a checkpoint after a forward) must not leave stale folded weights behind
    def __setitem__(self, key, value):
        if getattr(self, "_cache", None):
            self._cache.clear()
        super().__setitem__(key, value)

    def __delitem__(self, key):
        if getattr(self, "_cache", None):
            self._cache.clear()
        super().__delitem__(key)

    def update(self, *args, **kwargs):
        if getattr(self, "_cache", None):
            self._cache.clear()
        super().update(*args, **kwargs)


def _require_inference(is_training):
    if is_training:
        raise NotImplementedError(
            "is_training=True is not available for this configuration; training mode covers the models' own layer configurations "
            "(training.py: sa_module_training, mlp_training, PointNet2ClsTrainer) -- see INTEGRATION.md")


def _layer_training(inputs, scope, activation_fn, bn, bn_decay, params, frozen):
    """one conv / fully-connected layer in training mode (training.mlp_training): conv+BN+ReLU or a plain linear layer.
    frozen=True: inference mode with an input gradient (batch norm on the moving averages)."""
    if bn and activation_fn is not None:
        kind = True
    elif not bn and activation_fn is None:
        kind = False
    else:
        raise NotImplementedError("training mode covers conv/fc + batch norm + ReLU and plain linear layers (what the models use)")
    from .training import mlp_training
    return mlp_training(inputs, [(scope, kind)], bn_decay, params, frozen=frozen)


def conv2d(inputs, num_output_channels, kernel_size, scope, stride=(1, 1), padding="SAME", data_format="NHWC",
           activation_fn="relu", bn=False, bn_decay=None, is_training=False, *, params: VariableStore):
    """tf_util.conv2d restricted to what the hot path uses: 1x1 kernels, stride 1, NHWC, ReLU or None."""
    if tuple(kernel_size) != (1, 1) or tuple(stride) != (1, 1) or data_format != "NHWC":
        raise NotImplementedError("only 1x1 / stride-1 / NHWC convolutions are on the point-set-abstraction path")
    from .training import wants_input_grad
    frozen = not is_training and wants_input_grad(inputs)        # inference mode with an input gradient: frozen batch norm
    if is_training or frozen:
        return _layer_training(inputs, scope, activation_fn, bn, bn_decay, params, frozen)
    relu = activation_fn is not None
    mlp = params.mlp([scope], [relu])
    if mlp.channels[-1] != num_output_channels:
        raise ValueError(f"{scope}: stored weights have {mlp.channels[-1]} outputs, asked for {num_output_channels}")
    return ops.shared_mlp(inputs, mlp)


def fully_connected(inputs, num_outputs, scope, activation_fn="relu", bn=False, bn_decay=None, is_training=False, *,
                    params: VariableStore):
    from .training import wants_input_grad
    frozen = not is_training and wants_input_grad(inputs)        # inference mode with an input gradient: frozen batch norm
    if is_training or frozen:
        return _layer_training(inputs, scope, activation_fn, bn, bn_decay, params, frozen)
    relu = activation_fn is not None
    mlp = params.mlp([scope], [relu])
    if mlp.channels[-1] != num_outputs:
        raise ValueError(f"{scope}: stored weights have {mlp.channels[-1]} outputs, asked for {num_outputs}")
    return ops.shared_mlp(inputs, mlp)


def spiderConv(feat, idx, delta, num_conv, taylor_channel, bn=False, is_training=None, bn_decay=None, gn=False, G=32,
               is_multi_GPU=False, activation_fn="relu", scope="taylor", *, params: VariableStore):
    """tf_util.spiderConv (SpiderCNN/utils/tf_util.py:127-235) in inference mode, for the configuration SpiderCNN uses: gn=True,
    bn=False, ReLU.  feat (B,N,C), idx (B,N,k) int32, delta (B,N,k,3) -> (B,N,num_conv).  ``scope`` is the full variable scope
    (``fanConv1/taylor``).  The model itself chains ops.spider_conv on the pre-norm outputs and never builds this tensor."""
    _require_inference(is_training)
    if bn or not gn or activation_fn is None:
        raise NotImplementedError("spiderConv: only gn=True, bn=False with a ReLU (SpiderCNN's configuration) is implemented")
    taylor, w, bias, gamma, beta = params.spider(scope)
    if taylor.shape[1] != taylor_channel or w.shape[-1] != num_conv:
        raise ValueError(f"{scope}: stored variables have T={taylor.shape[1]}, {w.shape[-1]} outputs; asked for {taylor_channel}, {num_conv}")
    y = ops.spider_conv(delta, idx, feat, taylor, w, bias)
    out, _, _ = ops.group_norm_affine(y, gamma, beta, min(G, num_conv), GN_EPS, apply=True, relu=True)
    return out


def group_norm_for_conv(x, G=32, esp=GN_EPS, scope="gn", *, params: VariableStore):
    """tf_util.group_norm_for_conv (SpiderCNN/utils/tf_util.py:407-429) on x (B,N,C) or (B,N,1,C): G = min(G, C) contiguous
    channel groups, statistics per cloud, gamma / beta from ``scope/gamma``, ``scope/beta``."""
    shape = x.shape
    x3 = x.reshape(shape[0], -1, shape[-1])
    c = shape[-1]
    out, _, _ = ops.group_norm_affine(x3, params[f"{scope}/gamma"].float(), params[f"{scope}/beta"].float(), min(G, c), esp, apply=True)
    return out.reshape(shape)


def topk_pool(inputs, scope, k=2):
    """tf_util.topk_pool (SpiderCNN/utils/tf_util.py:363-377): (B,N,C) -> (B,C,k), the k largest values over the points."""
    if k != 2:
        raise NotImplementedError("topk_pool: only k = 2 (what SpiderCNN uses) is implemented")
    return ops.topk_pool(inputs, k)


def dropout(inputs, is_training, scope, keep_prob=0.5, noise_shape=None):
    """tf_util.dropout (tf_util.py:560-580): identity at inference, tf.nn.dropout(keep_prob) in training"""
    if is_training:
        if noise_shape is not None:
            raise NotImplementedError("dropout: noise_shape is not used by the in-scope models")
        return torch.nn.functional.dropout(inputs, 1.0 - keep_prob, training=True)
    return inputs
