"""Training mode of the PointNet++ classifier (pointnet2_cls_ssg) on the libpsa kernels: forward with batch-statistics
batch norm through every layer, backward of the fused set-abstraction levels and the FC head, Adam, and the
data-parallel gradient all-reduce.

Reference: pointnet2/train.py:139-171 (graph: get_model(is_training) -> get_loss -> AdamOptimizer.minimize), :246-252
(the per-batch feed: rotate + jitter, one sess.run of train_op), pointnet2/utils/tf_util.py:155-185,512-531 (conv2d /
batch norm in training mode), pointnet_util.py:87-154 (set-abstraction level), tf_grouping.py:43-47 (GroupPointGrad).

How a level is stored: ONE tensor per layer, the PRE-batch-norm activations y_l (B*m*K, C_l).  relu(BN(y_l)) is recomputed
inside the next layer's GEMM operand load, the batch-norm backward inside the backward GEMMs' operand loads
(csrc/train_gemm.cuh), the max-pool keeps the winning row per (group, channel).  The first layer of a level is the fused
ball-query + group + conv1 kernel (psa_sa_conv1_prebn); its backward is a coordinate reduction plus, for levels with
features, an ORDERED gather that replaces the reference's atomicAdd GroupPointGrad, and two dense products on the source
points instead of the grouped rows.

Everything numeric runs in libpsa.so; torch provides memory, streams and torch.distributed (one flat gradient bucket,
one NCCL all-reduce per step -- SURVEY 8e).  All buffers are allocated once, so a step can be captured in a CUDA graph.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import torch

from . import _lib, ops
from ._lib import PsaActIn, PsaGradIn, check
from ._lib import ptr as _p
from ._lib import stream as _stream
from .tf_util import BN_EPS, VariableStore

@dataclass
class LevelSpec:
    """One pointnet_sa_module call (pointnet2_cls_ssg.py:35-37)."""
    scope: str
    npoint: int | None
    radius: float | None
    nsample: int | None
    mlp: list
    group_all: bool = False


SSG_LEVELS = [LevelSpec("layer1", 512, 0.2, 32, [64, 64, 128]), LevelSpec("layer2", 128, 0.4, 64, [128, 128, 256]),
              LevelSpec("layer3", None, None, None, [256, 512, 1024], group_all=True)]
SSG_HEAD = [("fc1", 512, True, 0.5), ("fc2", 256, True, 0.5), ("fc3", None, False, None)]   # (scope, width, bn, keep_prob)
STATS_FROM_ROWS = 1024       # dense layers of at most this many rows take batch statistics from their output (psa_bn_finalize_rows)
DEFAULT_BN_DECAY = 0.9       # the moving averages' decay for bn_decay=None (tf_util.py's batch_norm_template / batch_norm_dist_template)


class FlatParams:
    """The trainable variables of a VariableStore re-homed as views of ONE flat fp32 tensor (same TF names), with a
    matching flat gradient tensor and Adam moments.  One bucket = one all-reduce, one Adam launch."""

    def __init__(self, params: VariableStore):
        self.params = params
        names = [k for k in params.keys() if not k.endswith(("/moving_mean", "/moving_variance"))]
        self.names = names
        dev = params[names[0]].device
        sizes = [params[k].numel() for k in names]
        pad = lambda n: (n + 63) // 64 * 64          # 256-byte aligned segments: float4 loads of the views stay legal  # noqa: E731
        offs, o = [], 0
        for n in sizes:
            offs.append(o)
            o += pad(n)
        self.total = o
        self.flat = torch.zeros(o, dtype=torch.float32, device=dev)
        self.grad = torch.zeros(o, dtype=torch.float32, device=dev)
        self.adam_m = torch.zeros(o, dtype=torch.float32, device=dev)
        self.adam_v = torch.zeros(o, dtype=torch.float32, device=dev)
        self.views, self.gviews = {}, {}
        for k, off, n in zip(names, offs, sizes):
            shape = params[k].shape
            v = self.flat[off:off + n].view(shape)
            v.copy_(params[k])
            dict.__setitem__(params, k, v)            # the store now aliases the flat buffer
            self.views[k] = v
            self.gviews[k] = self.grad[off:off + n].view(shape)
        params.invalidate()
        self.step_count = 0

    def grad_of(self, name):
        return self.gviews[name]

    def live(self, name) -> torch.Tensor:
        """a view of the flat parameter vector taken NOW (autograd-tracked when flat.requires_grad): for variables used directly in
        torch ops (e.g. the T-net's transform_XYZ matrix) rather than through the hand-written layers"""
        v = self.views[name]
        off = (v.data_ptr() - self.flat.data_ptr()) // 4
        return self.flat[off:off + v.numel()].view(v.shape)


class _Layer:
    """conv1x1 / fully_connected (+ batch norm + relu): parameter views, gradient views and per-step buffers."""

    def __init__(self, fp: FlatParams, scope: str, rows: int, bn: bool, dev):
        p = fp.params
        w = fp.views[f"{scope}/weights"]
        self.scope = scope
        self.W = w.view(-1, w.shape[-1])
        self.K, self.N = self.W.shape
        self.b = fp.views[f"{scope}/biases"]
        self.dW = fp.gviews[f"{scope}/weights"].view(self.K, self.N)
        self.db = fp.gviews[f"{scope}/biases"]
        self.bn = bn
        self.rows = rows
        f32 = dict(dtype=torch.float32, device=dev)
        self.y = torch.empty((rows, self.N), **f32)
        if bn:
            self.gamma, self.beta = fp.views[f"{scope}/bn/gamma"], fp.views[f"{scope}/bn/beta"]
            self.dgamma, self.dbeta = fp.gviews[f"{scope}/bn/gamma"], fp.gviews[f"{scope}/bn/beta"]
            self.mov_mean, self.mov_var = p[f"{scope}/bn/moving_mean"], p[f"{scope}/bn/moving_variance"]
            self.stats = torch.empty((2, self.N), **f32)
            self.scale = torch.empty(self.N, **f32)
            self.shift = torch.empty(self.N, **f32)
            self.mean_inv = torch.empty((2, self.N), **f32)
            self.ca = torch.empty(self.N, **f32)
            self.cb = torch.empty(self.N, **f32)
            self.cc = torch.empty(self.N, **f32)
        else:
            self.scale = self.shift = self.ca = self.cb = self.cc = None
        self.mask = None      # dropout mask applied to this layer's OUTPUT (rows, N), or None

    def act_in(self) -> PsaActIn:
        """this layer's output as the next layer's input"""
        return PsaActIn(x=_p(self.y), ld=self.N, scale=_p(self.scale), shift=_p(self.shift), mask=_p(self.mask), relu=int(self.bn))


# psa_act_in / psa_grad_in descriptors: fields not named are 0 / NULL
def _raw_in(x: torch.Tensor) -> PsaActIn:
    return PsaActIn(x=_p(x), ld=x.shape[-1])


def _grad_in(ly: _Layer, **dz) -> PsaGradIn:
    """dy of layer `ly` with its batch-norm coefficients (psa_bn_bwd_coeffs ignores them and fills them in); dz's source in `dz`"""
    return PsaGradIn(y=_p(ly.y), ld=ly.N, s=_p(ly.scale), t=_p(ly.shift), relu=int(ly.bn), ca=_p(ly.ca), cb=_p(ly.cb), cc=_p(ly.cc),
                     C=ly.N, **dz)


def _grad_dense(ly: _Layer, dh: torch.Tensor) -> PsaGradIn:
    return _grad_in(ly, dh=_p(dh), ld_dh=dh.shape[-1], mask=_p(ly.mask), pool_k=1)


def _grad_pooled(ly: _Layer, dp: torch.Tensor, pv: torch.Tensor, argk: torch.Tensor, pool_k: int) -> PsaGradIn:
    return _grad_in(ly, dp=_p(dp), pv=_p(pv), argk=_p(argk), pool_k=pool_k, mode=1)


def _plain_grad(dh: torch.Tensor) -> PsaGradIn:
    return PsaGradIn(dh=_p(dh), ld_dh=dh.shape[-1], pool_k=1, C=dh.shape[-1])


@dataclass
class _Level:
    spec: LevelSpec
    n: int
    m: int
    k: int
    c_in: int
    layers: list = field(default_factory=list)
    new_xyz: torch.Tensor = None
    idx: torch.Tensor = None
    cnt: torch.Tensor = None
    pooled: torch.Tensor = None
    argk: torch.Tensor = None
    dh: list = field(default_factory=list)      # dh[l] = gradient w.r.t. layer l's post-relu output (dense), l < L-1
    dU: torch.Tensor = None
    x_cat: torch.Tensor = None                  # group_all: [xyz, points] rows
    d_in: torch.Tensor = None                   # gradient w.r.t. the level's input features (B*n, c_in)
    fps_idx: torch.Tensor = None                # (B, m) int32: the sampled centroids (not group_all)
    dxyz: torch.Tensor = None                   # (B*n, 3): GroupPointGrad of the grouped coordinates (group_all: the xyz columns)
    dnew: torch.Tensor = None                   # (B*m, 3): gradient reaching new_xyz through "- new_xyz" inside this level
    dW_scratch: torch.Tensor = None             # frozen batch norm: psa_sa_conv1_bwd's dW_xyz, not a variable gradient


class _TrainOps:
    """Per-layer training operations shared by the trainers below (they provide self.ws, self.ws_bytes).

    frozen=True: inference-mode batch norm -- the moving averages (never updated) folded into every layer at the start of each
    forward, no batch statistics or psa_bn_finalize, and a backward of input products only that leaves the flat gradient
    bucket alone."""

    def __init__(self, params: VariableStore, device, frozen: bool):
        self.lib = _lib.load()
        self.params = params
        self.frozen = frozen
        self.dev = torch.device(device) if device is not None else params.device
        self.fp = params._flat if getattr(params, "_flat", None) is not None else FlatParams(params)
        params._flat = self.fp

    def _bn_finalize(self, ly: _Layer, count: int, decay: float):
        """batch statistics over `count` rows -> scale / shift, moving averages updated; nothing without batch statistics"""
        if ly.bn and not self.frozen:
            check(self.lib.psa_bn_finalize(ly.N, count, _p(ly.stats), _p(ly.gamma), _p(ly.beta), C.c_float(decay), _p(ly.mov_mean),
                                           _p(ly.mov_var), _p(ly.scale), _p(ly.shift), _p(ly.mean_inv), _stream()), "bn_finalize")

    def _layer_fwd(self, ly: _Layer, a: PsaActIn, decay: float):
        """y = a . W + b (+ batch statistics), then batch norm's scale / shift.  A layer of at most STATS_FROM_ROWS rows (the FC head,
        rows = batch) takes its statistics from y in two fp64 passes instead of the GEMM's sums: after a max over the points a column's
        mean can be ~60 times its spread, and E[y^2] - mean^2 from fp32 sums then loses the variance's digits."""
        from_rows = ly.bn and not self.frozen and ly.rows <= STATS_FROM_ROWS
        check(self.lib.psa_train_dense_fwd(ly.rows, ly.K, ly.N, C.byref(a), _p(ly.W), _p(ly.b), _p(ly.y),
                                           _p(ly.stats) if ly.bn and not self.frozen and not from_rows else None, _p(self.ws),
                                           C.c_size_t(self.ws_bytes), _stream()), "train_dense_fwd")
        if from_rows:
            check(self.lib.psa_bn_finalize_rows(ly.rows, ly.N, _p(ly.y), _p(ly.gamma), _p(ly.beta), C.c_float(decay), _p(ly.mov_mean),
                                                _p(ly.mov_var), _p(ly.scale), _p(ly.shift), _p(ly.mean_inv), _stream()), "bn_finalize_rows")
        else:
            self._bn_finalize(ly, ly.rows, decay)

    def _chain_fwd(self, layers, a: PsaActIn, decay: float):
        """a chain of dense layers on input `a`; the output is layers[-1].y"""
        for ly in layers:
            self._layer_fwd(ly, a, decay)
            a = ly.act_in()

    def _fold_frozen(self, layers):
        """inference-mode batch norm: the moving averages folded into scale / shift (VariableStore.folded's arithmetic), and the
        backward coefficients dy = scale * dz (ca = scale, cb = cc = 0).  The moving averages are read, never written."""
        if not self.frozen:
            return
        for ly in layers:
            if ly.bn:
                inv = ly.gamma * torch.rsqrt(ly.mov_var + BN_EPS)
                ly.scale.copy_(inv)
                ly.shift.copy_(ly.beta - ly.mov_mean * inv)
                ly.ca.copy_(inv)
                ly.cb.zero_()
                ly.cc.zero_()

    def _bn_bwd(self, ly: _Layer, g: PsaGradIn):
        """batch-norm sums and dy's coefficients, or the bias gradient of a layer without batch norm; nothing when frozen"""
        if self.frozen:
            return
        if ly.bn:
            check(self.lib.psa_bn_bwd_coeffs(ly.rows, ly.N, C.byref(g), _p(ly.gamma), _p(ly.mean_inv), _p(ly.dgamma), _p(ly.dbeta),
                                             _p(ly.ca), _p(ly.cb), _p(ly.cc), _p(self.ws), C.c_size_t(self.ws_bytes), _stream()), "bn_bwd_coeffs")
            ly.db.zero_()          # sum_r dy = 0 under batch norm
        else:
            check(self.lib.psa_train_bias_grad(ly.rows, ly.N, C.byref(g), _p(ly.db), _stream()), "train_bias_grad")

    def _products(self, g: PsaGradIn, rows: int, K: int, N: int, W, dW, a_in: PsaActIn | None, dx: torch.Tensor | None, col_skip: int = 0):
        """dW (K, N) = a_in^T . dy (not when frozen) and dx = dy . W^T over the input columns >= col_skip; None skips either"""
        if a_in is not None and not self.frozen:
            check(self.lib.psa_train_dense_bwd_weight(rows, K, N, C.byref(a_in), C.byref(g), _p(dW), _p(self.ws), C.c_size_t(self.ws_bytes),
                                                      _stream()), "train_dense_bwd_weight")
        if dx is not None:
            check(self.lib.psa_train_dense_bwd_input(rows, K, N, C.byref(g), _p(W), _p(dx), dx.shape[-1], col_skip, _p(self.ws),
                                                     C.c_size_t(self.ws_bytes), _stream()), "train_dense_bwd_input")

    def _layer_bwd(self, ly: _Layer, g: PsaGradIn, a_in: PsaActIn | None, dx: torch.Tensor | None, col_skip: int = 0):
        """gradients of one conv/fc(+BN+relu) layer: BN sums/coefficients or db, dW, dx."""
        self._bn_bwd(ly, g)
        self._products(g, ly.rows, ly.K, ly.N, ly.W, ly.dW, a_in, dx, col_skip)

    def _chain_bwd(self, layers, g: PsaGradIn, dh, a0: PsaActIn, dx: torch.Tensor):
        """backward of a chain of dense layers: g = the top layer's dy, dh[l] = buffer for the gradient w.r.t. layer l's output
        (l < L-1), a0 = the first layer's input, dx = where the gradient w.r.t. a0 goes"""
        for i in range(len(layers) - 1, -1, -1):
            if i < len(layers) - 1:
                g = _grad_dense(layers[i], dh[i])
            if i > 0:
                self._layer_bwd(layers[i], g, layers[i - 1].act_in(), dh[i - 1])
            else:
                self._layer_bwd(layers[i], g, a0, dx)


def _flat_grad_of_layers(fp: FlatParams, layers) -> torch.Tensor:
    """a gradient bucket that holds the given layers' gradients and zeros elsewhere (several autograd nodes share one bucket)"""
    g = torch.zeros_like(fp.grad)
    base = fp.grad.data_ptr()
    for ly in layers:
        for t in ([ly.dW, ly.db] + ([ly.dgamma, ly.dbeta] if ly.bn else [])):
            off = (t.data_ptr() - base) // 4
            g[off:off + t.numel()].copy_(t.reshape(-1))
    return g


class MlpTrainer(_TrainOps):
    """Training-mode shared MLP on dense rows -- tf_util.conv1d / conv2d(1x1) / fully_connected chains with batch-statistics batch
    norm + ReLU (tf_util.py:120-185,512-531): the FP modules' MLPs, FC heads, per-point heads.  layers = [(scope, bn), ...];
    a layer with bn=False has no activation (the reference's logits layers).  frozen=True: inference mode -- batch norm on the
    moving averages (never updated), and a backward that gives the input gradient only.

    group_channels > 0: the first layer reads concat([x, tile(g)]) with g (groups, group_channels) one row per group of
    rows / groups consecutive rows (PointNet's segmentation heads, pointnet/models/pointnet_seg.py:81-88).  The first
    in_channels rows of its weight multiply x, the others g, and the concatenation is never built: g . W_g is a product over the
    groups that psa_train_dense_fwd_grouped adds per row, and its gradient is the per-group sum of dy
    (psa_train_bias_grad_grouped).  group_first: the first layer reads concat([tile(g), x]) instead, so the first group_channels
    rows of its weight multiply g (a feature-propagation level whose known level is one point, pointnet2_cls_partseg's fa_layer1)."""

    def __init__(self, params: VariableStore, rows: int, in_channels: int, layers, device=None, frozen: bool = False, groups: int = 0,
                 group_channels: int = 0, group_first: bool = False):
        super().__init__(params, device, frozen)
        self.rows, self.in_channels, self.group_channels = rows, in_channels, group_channels
        f32 = dict(dtype=torch.float32, device=self.dev)
        self.layers: list[_Layer] = []
        cin, ws_bytes = in_channels + group_channels, 0
        for scope, bn in layers:
            ly = _Layer(self.fp, scope, rows, bn, self.dev)
            assert ly.K == cin, (scope, ly.W.shape, cin)
            ws_bytes = max(ws_bytes, self.lib.psa_train_dense_workspace_bytes(rows, ly.K, ly.N), self.lib.psa_bn_bwd_workspace_bytes(ly.N))
            self.layers.append(ly)
            cin = ly.N
        if group_channels:
            assert groups >= 1 and rows % groups == 0, (rows, groups)
            first = self.layers[0]
            self.groups = groups
            x_rows, g_rows = ((slice(group_channels, None), slice(0, group_channels)) if group_first else
                              (slice(0, in_channels), slice(in_channels, None)))
            self.W_x, self.W_g = first.W[x_rows], first.W[g_rows]
            self.dW_x, self.dW_g = first.dW[x_rows], first.dW[g_rows]
            self.g_add = torch.empty((groups, first.N), **f32)
            self.d_add = torch.empty((groups, first.N), **f32)
            self.d_g = torch.empty((groups, group_channels), **f32)
            ws_bytes = max(ws_bytes, self.lib.psa_train_dense_workspace_bytes(groups, group_channels, first.N))
        self.dh = [torch.empty((rows, ly.N), **f32) for ly in self.layers[:-1]]
        self.d_in = torch.empty((rows, in_channels), **f32)
        last = self.layers[-1]
        if last.bn:
            assert last.N % 4 == 0, "an activated last layer needs a width that is a multiple of 4"
            self.out = torch.empty((rows, last.N), **f32)
            self.argk = torch.empty((rows, last.N), dtype=torch.int32, device=self.dev)
        self.ws = torch.empty(ws_bytes // 4 + 64, **f32)
        self.ws_bytes = ws_bytes

    def forward(self, x: torch.Tensor, bn_decay: float = 0.5, g: torch.Tensor | None = None) -> torch.Tensor:
        assert x.shape == (self.rows, self.in_channels) and x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
        self.x = x
        self._fold_frozen(self.layers)
        if self.group_channels:
            assert g is not None and g.shape == (self.groups, self.group_channels) and g.is_contiguous()
            self.g = g
            first = self.layers[0]
            check(self.lib.psa_train_dense_fwd(self.groups, self.group_channels, first.N, C.byref(_raw_in(g)), _p(self.W_g), None,
                                               _p(self.g_add), None, _p(self.ws), C.c_size_t(self.ws_bytes), _stream()), "train_dense_fwd")
            check(self.lib.psa_train_dense_fwd_grouped(self.rows, self.rows // self.groups, self.in_channels, first.N, C.byref(_raw_in(x)),
                                                       _p(self.W_x), _p(first.b), _p(self.g_add),
                                                       _p(first.y), _p(first.stats) if first.bn and not self.frozen else None,
                                                       _p(self.ws), C.c_size_t(self.ws_bytes), _stream()), "train_dense_fwd_grouped")
            self._bn_finalize(first, self.rows, bn_decay)
            self._chain_fwd(self.layers[1:], first.act_in(), bn_decay)
        else:
            self._chain_fwd(self.layers, _raw_in(x), bn_decay)
        last = self.layers[-1]
        if not last.bn:
            return last.y
        # the stack's output is the activated tensor: relu(BN(y)) through the pooling kernel with runs of one row
        check(self.lib.psa_train_pool_fwd(self.rows, 1, last.N, _p(last.y), _p(last.scale), _p(last.shift), _p(self.out), _p(self.argk),
                                          _stream()), "train_pool_fwd")
        return self.out

    def backward(self, dout: torch.Tensor) -> torch.Tensor:
        """dout = gradient w.r.t. forward()'s return value -> gradient w.r.t. x; the layers' gradients go to the flat bucket"""
        dout = dout.contiguous()
        if not self.group_channels:
            self._chain_bwd(self.layers, _grad_dense(self.layers[-1], dout), self.dh, _raw_in(self.x), self.d_in)
            return self.d_in
        # grouped first layer: (gradient w.r.t. x, gradient w.r.t. g)
        first, top = self.layers[0], _grad_dense(self.layers[-1], dout)
        if len(self.layers) > 1:
            self._chain_bwd(self.layers[1:], top, self.dh[1:], first.act_in(), self.dh[0])
            top = _grad_dense(first, self.dh[0])
        self._bn_bwd(first, top)
        self._products(top, self.rows, self.in_channels, first.N, self.W_x, self.dW_x, _raw_in(self.x), self.d_in)
        check(self.lib.psa_train_bias_grad_grouped(self.rows, self.rows // self.groups, first.N, C.byref(top), _p(self.d_add), _stream()),
              "train_bias_grad_grouped")
        self._products(_plain_grad(self.d_add), self.groups, self.group_channels, first.N, self.W_g, self.dW_g, _raw_in(self.g), self.d_g)
        return self.d_in, self.d_g


class _NodeFn(torch.autograd.Function):
    """An MlpTrainer / EdgeConvTrainer / EdgeConv2Trainer as one autograd node: trainer.forward(x, *args, bn_decay), whose backward
    returns the gradient of x and of the trainer's variables (a flat bucket that is zero outside them: several nodes share one
    store; a frozen trainer is applied with flat=None and gives the input gradient only)."""

    @staticmethod
    def forward(ctx, flat, x, trainer, args, bn_decay):
        ctx.trainer, ctx.x_shape = trainer, x.shape
        return trainer.forward(x, *args, bn_decay).clone()

    @staticmethod
    def backward(ctx, dout):
        tr = ctx.trainer
        dx = tr.backward(dout)
        return (None if tr.frozen else _flat_grad_of_layers(tr.fp, tr.layers)), dx.view(ctx.x_shape).clone(), None, None, None


class _GroupedNodeFn(torch.autograd.Function):
    """A grouped MlpTrainer as one autograd node: trainer.forward(x, bn_decay, g), differentiable in x, g and the variables."""

    @staticmethod
    def forward(ctx, flat, x, g, trainer, bn_decay):
        ctx.trainer = trainer
        return trainer.forward(x, bn_decay, g).clone()

    @staticmethod
    def backward(ctx, dout):
        tr = ctx.trainer
        dx, dg = tr.backward(dout)
        return (None if tr.frozen else _flat_grad_of_layers(tr.fp, tr.layers)), dx.clone(), dg.clone(), None, None


def _cached(params: VariableStore, key, make):
    """the trainer cached on `params` under `key`, made on first use (its buffers are allocated once per configuration and shape)"""
    cache = params.__dict__.setdefault("_trainers", {})
    if key not in cache:
        cache[key] = make()
    return cache[key]


def _flat_and_decay(tr: _TrainOps, bn_decay):
    """the autograd input that carries the variables' gradients and the moving-average decay: 0.9 for None, the default of every
    reference tf_util's batch_norm_template and batch_norm_dist_template (`decay = bn_decay if bn_decay is not None else 0.9`);
    (None, 0.0) for a frozen trainer, which neither updates nor differentiates the variables"""
    if tr.frozen:
        return None, 0.0
    tr.fp.flat.requires_grad_(True)
    return tr.fp.flat, DEFAULT_BN_DECAY if bn_decay is None else float(bn_decay)


def mlp_training(x: torch.Tensor, layers, bn_decay, params: VariableStore, frozen: bool = False,
                 group: torch.Tensor | None = None, group_first: bool = False) -> torch.Tensor:
    """Training-mode shared MLP with autograd: x (..., C_in) -> (..., C_out); layers = [(scope, bn), ...].  Buffers are cached on
    `params` per (scopes, shape).  frozen=True: inference mode (moving averages, input gradient only).  group (G, C_g): the first
    layer reads concat([x, tile(group)]), one row of `group` per x.numel() / C_in / G consecutive rows (e.g. per cloud), without
    building the concatenation; its weight has C_in + C_g rows, x's first (group_first: group's first, concat([tile(group), x]))."""
    shape = x.shape
    rows = x.numel() // shape[-1]
    if group is None:
        tr = _cached(params, ("mlp_frozen" if frozen else "mlp", tuple(layers), rows, shape[-1]),
                     lambda: MlpTrainer(params, rows, shape[-1], list(layers), device=x.device, frozen=frozen))
        flat, decay = _flat_and_decay(tr, bn_decay)
        out = _NodeFn.apply(flat, x.reshape(rows, shape[-1]).contiguous(), tr, (), decay)
    else:
        gs = group.shape
        tr = _cached(params, ("mlp_frozen" if frozen else "mlp", tuple(layers), rows, shape[-1], "group", gs[0], gs[-1], group_first),
                     lambda: MlpTrainer(params, rows, shape[-1], list(layers), device=x.device, frozen=frozen, groups=gs[0],
                                        group_channels=gs[-1], group_first=group_first))
        flat, decay = _flat_and_decay(tr, bn_decay)
        out = _GroupedNodeFn.apply(flat, x.reshape(rows, shape[-1]).contiguous(), group.contiguous(), tr, decay)
    return out.view(*shape[:-1], out.shape[-1])


class EdgeConvTrainer(_TrainOps):
    """Training-mode single-layer EdgeConv (dgcnn.py:41-47: get_edge_feature -> conv2d + batch norm + ReLU -> reduce_max over k) on
    the fused kernels of csrc/edgeconv_train.cu: one product over the b*n points and gather passes; no (B,N,k,.) tensor is stored.
    Batch statistics over all b*n*k edges; the max's gradient is split evenly among tied edges, as torch.amax / TF reduce_max do.
    frozen=True: inference mode -- batch norm on the moving averages (never updated), and a backward that gives dx only."""

    def __init__(self, params: VariableStore, b: int, n: int, c: int, k: int, scope: str, device=None, frozen: bool = False):
        super().__init__(params, device, frozen)
        self.b, self.n, self.c, self.k = b, n, c, k
        ly = _Layer(self.fp, scope, 0, True, self.dev)       # rows = 0: the per-edge activations are never stored
        self.layers = [ly]
        if ly.K != 2 * c:
            raise ValueError(f"{scope}: weights of shape {tuple(ly.W.shape)}, an EdgeConv over {c} channels needs ({2 * c}, C_out)")
        rows, N = b * n, ly.N
        f32 = dict(dtype=torch.float32, device=self.dev)
        self.PQ = torch.empty((rows, 2 * N), **f32)
        self.pooled = torch.empty((rows, N), **f32)
        self.ties = torch.empty((rows, N), dtype=torch.uint8 if k <= 255 else torch.int32, device=self.dev)
        self.d_in = torch.empty((rows, c), **f32)
        self.ws_bytes = self.lib.psa_edgeconv_train_workspace_bytes(b, n, c, k, N)
        if self.ws_bytes == 0:
            raise _lib.PsaError(f"{scope}: EdgeConv training needs C_out a multiple of 32, at most 256 (got {N})")
        self.ws = torch.empty(self.ws_bytes // 4 + 64, **f32)

    def forward(self, x: torch.Tensor, nn_idx: torch.Tensor, bn_decay: float = 0.5) -> torch.Tensor:
        b, n, c, k, (ly,) = self.b, self.n, self.c, self.k, self.layers
        assert x.shape == (b, n, c) and x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
        assert nn_idx.shape == (b, n, k) and nn_idx.dtype == torch.int32 and nn_idx.is_contiguous()
        self.x, self.nn_idx = x, nn_idx
        self._fold_frozen(self.layers)
        check(self.lib.psa_edgeconv_train_fwd(b, n, c, k, ly.N, _p(x), _p(nn_idx), _p(ly.W), _p(ly.b), _p(self.PQ),
                                              None if self.frozen else _p(ly.stats), _p(self.ws), C.c_size_t(self.ws_bytes), _stream()),
              "edgeconv_train_fwd")
        self._bn_finalize(ly, b * n * k, bn_decay)
        check(self.lib.psa_edgeconv_train_pool(b, n, k, ly.N, _p(nn_idx), _p(self.PQ), _p(ly.scale), _p(ly.shift), _p(self.pooled), _p(self.ties),
                                               _stream()), "edgeconv_train_pool")
        return self.pooled

    def backward(self, dout: torch.Tensor) -> torch.Tensor:
        """dout = gradient w.r.t. forward()'s return value -> gradient w.r.t. x (b*n, c); the layer's gradients go to the flat bucket
        (not when frozen)"""
        b, n, c, k, (ly,) = self.b, self.n, self.c, self.k, self.layers
        dout = dout.contiguous()
        if self.frozen:
            check(self.lib.psa_edgeconv_frozen_bwd(b, n, c, k, ly.N, _p(self.x), _p(self.nn_idx), _p(ly.W), _p(self.PQ), _p(ly.scale), _p(ly.shift),
                                                   _p(self.pooled), _p(self.ties), _p(dout), _p(self.d_in), _p(self.ws), C.c_size_t(self.ws_bytes),
                                                   _stream()), "edgeconv_frozen_bwd")
            return self.d_in
        check(self.lib.psa_edgeconv_train_bwd(b, n, c, k, ly.N, _p(self.x), _p(self.nn_idx), _p(ly.W), _p(self.PQ), _p(ly.scale), _p(ly.shift),
                                              _p(ly.gamma), _p(ly.mean_inv), _p(self.pooled), _p(self.ties), _p(dout), _p(ly.dW), _p(ly.dgamma),
                                              _p(ly.dbeta), _p(self.d_in), _p(self.ws), C.c_size_t(self.ws_bytes), _stream()), "edgeconv_train_bwd")
        ly.db.zero_()          # sum over the edges of dy = 0 under batch norm
        return self.d_in


class EdgeConv2Trainer(_TrainOps):
    """Training-mode two-layer EdgeConv (transform_nets.py:18-27: get_edge_feature -> conv2d + BN + ReLU -> conv2d + BN + ReLU ->
    reduce_max over k) on csrc/edgeconv2_train.cu: layer 1 is the single-layer op's point product, the per-edge 64 -> 128 product runs
    on the tensor cores and is recomputed in every pass; no (B,N,k,.) tensor is stored in the forward.  Batch statistics over all
    b*n*k edges in both layers; the max's gradient is split evenly among tied edges.  frozen=True: inference mode -- batch norm on the
    moving averages (never updated) in both layers, and a backward that gives dx only."""

    def __init__(self, params: VariableStore, b: int, n: int, c: int, k: int, scopes, device=None, frozen: bool = False):
        super().__init__(params, device, frozen)
        self.b, self.n, self.c, self.k = b, n, c, k
        self.layers = [_Layer(self.fp, s, 0, True, self.dev) for s in scopes]     # rows = 0: the per-edge activations are never stored
        l1, l2 = self.layers
        if l1.K != 2 * c:
            raise ValueError(f"{l1.scope}: weights of shape {tuple(l1.W.shape)}, an EdgeConv over {c} channels needs ({2 * c}, C1)")
        if l2.K != l1.N:
            raise ValueError(f"{l2.scope}: weights of shape {tuple(l2.W.shape)}, the second layer needs ({l1.N}, C2)")
        rows, N = b * n, l2.N
        self.ws_bytes = self.lib.psa_edgeconv2_train_workspace_bytes(b, n, c, k, l1.N, N)
        if self.ws_bytes == 0:
            raise _lib.PsaError(f"{l1.scope}, {l2.scope}: two-layer EdgeConv training needs C1 = 64, C2 = 128 and k <= 32 "
                                f"(got C1 = {l1.N}, C2 = {N}, k = {k})")
        f32 = dict(dtype=torch.float32, device=self.dev)
        self.PQ = torch.empty((rows, 2 * l1.N), **f32)
        self.pooled = torch.empty((rows, N), **f32)
        self.mask = torch.empty((rows, N), dtype=torch.int32, device=self.dev)
        self.ywin = torch.empty((rows, N), **f32)
        self.d_in = torch.empty((rows, c), **f32)
        self.ws = torch.empty(self.ws_bytes // 4 + 64, **f32)

    def forward(self, x: torch.Tensor, nn_idx: torch.Tensor, bn_decay: float = 0.5) -> torch.Tensor:
        b, n, c, k = self.b, self.n, self.c, self.k
        l1, l2 = self.layers
        assert x.shape == (b, n, c) and x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
        assert nn_idx.shape == (b, n, k) and nn_idx.dtype == torch.int32 and nn_idx.is_contiguous()
        self.x, self.nn_idx = x, nn_idx
        lib, ws, wsb = self.lib, _p(self.ws), C.c_size_t(self.ws_bytes)
        self._fold_frozen(self.layers)
        check(lib.psa_edgeconv_train_fwd(b, n, c, k, l1.N, _p(x), _p(nn_idx), _p(l1.W), _p(l1.b), _p(self.PQ), None if self.frozen else _p(l1.stats),
                                         ws, wsb, _stream()), "edgeconv_train_fwd")
        if not self.frozen:            # frozen: layer 2's scale / shift are already folded, no statistics pass
            self._bn_finalize(l1, b * n * k, bn_decay)
            check(lib.psa_edgeconv2_train_fwd(b, n, c, k, l1.N, l2.N, _p(nn_idx), _p(self.PQ), _p(l1.scale), _p(l1.shift), _p(l2.W), _p(l2.b),
                                              _p(l2.stats), ws, wsb, _stream()), "edgeconv2_train_fwd")
            self._bn_finalize(l2, b * n * k, bn_decay)
        check(lib.psa_edgeconv2_train_pool(b, n, c, k, l1.N, l2.N, _p(nn_idx), _p(self.PQ), _p(l1.scale), _p(l1.shift), _p(l2.W), _p(l2.b),
                                           _p(l2.scale), _p(l2.shift), _p(self.pooled), _p(self.mask), _p(self.ywin), ws, wsb, _stream()),
              "edgeconv2_train_pool")
        return self.pooled

    def backward(self, dout: torch.Tensor) -> torch.Tensor:
        """dout = gradient w.r.t. forward()'s return value -> gradient w.r.t. x (b*n, c); both layers' gradients go to the flat bucket
        (not when frozen)"""
        b, n, c, k = self.b, self.n, self.c, self.k
        l1, l2 = self.layers
        dout = dout.contiguous()
        if self.frozen:
            check(self.lib.psa_edgeconv2_frozen_bwd(b, n, c, k, l1.N, l2.N, _p(self.x), _p(self.nn_idx), _p(l1.W), _p(self.PQ), _p(l1.scale),
                                                    _p(l1.shift), _p(l2.W), _p(l2.b), _p(l2.scale), _p(self.pooled), _p(self.mask), _p(self.ywin),
                                                    _p(dout), _p(self.d_in), _p(self.ws), C.c_size_t(self.ws_bytes), _stream()), "edgeconv2_frozen_bwd")
            return self.d_in
        check(self.lib.psa_edgeconv2_train_bwd(b, n, c, k, l1.N, l2.N, _p(self.x), _p(self.nn_idx), _p(l1.W), _p(self.PQ), _p(l1.scale),
                                               _p(l1.shift), _p(l1.gamma), _p(l1.mean_inv), _p(l2.W), _p(l2.b), _p(l2.gamma), _p(l2.mean_inv),
                                               _p(self.pooled), _p(self.mask), _p(self.ywin), _p(dout), _p(l1.dW), _p(l1.dgamma), _p(l1.dbeta),
                                               _p(l2.dW), _p(l2.dgamma), _p(l2.dbeta), _p(self.d_in), _p(self.ws), C.c_size_t(self.ws_bytes),
                                               _stream()), "edgeconv2_train_bwd")
        l1.db.zero_()          # sum over the edges of dy = 0 under batch norm, in both layers
        l2.db.zero_()
        return self.d_in


def edgeconv_training(x: torch.Tensor, nn_idx: torch.Tensor, scope, bn_decay, params: VariableStore, frozen: bool = False) -> torch.Tensor:
    """Training-mode EdgeConv with autograd: x (B, N, C), nn_idx (B, N, k) int32 -> (B, N, C_out) = max_j relu(BN([x_i, x_j - x_i] . W + b)),
    BN over all B*N*k edges.  `scope` is one scope, or a sequence of two for the two-layer EdgeConv (conv + BN + ReLU twice, then the
    max; C1 = 64, C2 = 128), which runs as one autograd node.  The graph carries no gradient.  Buffers are cached on `params` per
    (scopes, shape); the variables' gradients land in the flat bucket.  frozen=True: inference mode (batch norm on the moving averages,
    which stay put; the gradient of x only)."""
    b, n, c = x.shape
    k = nn_idx.shape[-1]
    scopes = (scope,) if isinstance(scope, str) else tuple(scope)
    if len(scopes) not in (1, 2):
        raise ValueError(f"edgeconv_training: one or two scopes, got {len(scopes)}")
    tag = "_frozen" if frozen else ""
    if len(scopes) == 1:
        tr = _cached(params, ("edgeconv" + tag, scopes[0], b, n, c, k),
                     lambda: EdgeConvTrainer(params, b, n, c, k, scopes[0], device=x.device, frozen=frozen))
    else:
        tr = _cached(params, ("edgeconv2" + tag, scopes, b, n, c, k),
                     lambda: EdgeConv2Trainer(params, b, n, c, k, scopes, device=x.device, frozen=frozen))
    flat, decay = _flat_and_decay(tr, bn_decay)
    out = _NodeFn.apply(flat, x.contiguous(), tr, (nn_idx.to(torch.int32).contiguous(),), decay)
    return out.view(b, n, -1)


class PointNet2ClsTrainer(_TrainOps):
    """Training engine of pointnet2_cls_ssg (or any stack of LevelSpec + FC head with the same structure).

    frozen=True: inference-mode differentiation -- batch norm on the moving averages (never updated), no dropout, the same
    forward kernels; the backward gives input gradients only (coordinates, features) and leaves the flat gradient bucket alone."""

    def __init__(self, params: VariableStore, batch: int, npoints: int, num_class: int = 15, levels=None, head=None,
                 device=None, process_group=None, in_channels: int = 0, frozen: bool = False):
        super().__init__(params, device, frozen)
        self.B, self.N0, self.num_class = batch, npoints, num_class
        self.pg = process_group
        self.world = torch.distributed.get_world_size(process_group) if (process_group is not None or
                                                                          (torch.distributed.is_available() and torch.distributed.is_initialized())) else 1
        dev = self.dev
        f32 = dict(dtype=torch.float32, device=dev)
        specs = levels if levels is not None else SSG_LEVELS
        self.levels: list[_Level] = []
        n, c = npoints, in_channels          # in_channels > 0: the first level takes per-point features (a level used on its own)
        self.in_channels = in_channels
        ws_bytes = 0
        lib = self.lib
        for sp in specs:
            if sp.group_all:
                m, k = 1, n
            else:
                m, k = sp.npoint, sp.nsample
            lv = _Level(sp, n, m, k, c)
            rows = batch * m * k
            cin = 3 + c
            for i, cout in enumerate(sp.mlp):
                lv.layers.append(_Layer(self.fp, f"{sp.scope}/conv{i}", rows, True, dev))
                assert lv.layers[-1].K == cin and lv.layers[-1].N == cout, (sp.scope, i, lv.layers[-1].W.shape, cin, cout)
                ws_bytes = max(ws_bytes, lib.psa_train_dense_workspace_bytes(rows, cin, cout), lib.psa_bn_bwd_workspace_bytes(cout))
                cin = cout
            L = len(sp.mlp)
            lv.pooled = torch.empty((batch * m, sp.mlp[-1]), **f32)
            lv.argk = torch.empty((batch * m, sp.mlp[-1]), dtype=torch.int32, device=dev)
            lv.dh = [torch.empty((rows, sp.mlp[i]), **f32) for i in range(L - 1)]
            lv.dxyz = torch.empty((batch * n, 3), **f32)
            if sp.group_all:
                lv.x_cat = torch.empty((batch * n, 3 + c), **f32)
                if c:
                    lv.d_in = torch.empty((batch * n, c), **f32)
            else:
                lv.dnew = torch.empty((batch * m, 3), **f32)
                ws_bytes = max(ws_bytes, lib.psa_sa_conv1_bwd_xyz_workspace_bytes(batch, n, m, k), lib.psa_scatter_workspace_bytes(batch, n, m))
                if frozen:
                    lv.dW_scratch = torch.empty((3, sp.mlp[0]), **f32)
                lv.idx = torch.empty((batch, m, k), dtype=torch.int32, device=dev)
                lv.cnt = torch.empty((batch, m), dtype=torch.int32, device=dev)
                c1 = sp.mlp[0]
                ws_bytes = max(ws_bytes, lib.psa_sa_conv1_prebn_workspace_bytes(batch, n, m, c, c1, 1), lib.psa_sa_conv1_bwd_workspace_bytes(batch, n, m, k, c1, 1 if c else 0))
                if c:
                    lv.dU = torch.empty((batch * n, c1), **f32)
                    lv.d_in = torch.empty((batch * n, c), **f32)
                    ws_bytes = max(ws_bytes, lib.psa_train_dense_workspace_bytes(batch * n, c, c1))
            self.levels.append(lv)
            n, c = m, sp.mlp[-1]
        # FC head on the (B, C) global feature
        self.head: list[_Layer] = []
        self.keep: list = []
        cin = c
        for scope, width, bn, keep in (head if head is not None else SSG_HEAD):
            width = width if width is not None else num_class
            ly = _Layer(self.fp, scope, batch, bn, dev)
            assert ly.K == cin and ly.N == width, (scope, ly.W.shape)
            if keep is not None and not frozen:          # no dropout in inference mode
                ly.mask = torch.ones((batch, width), **f32)
            self.head.append(ly)
            self.keep.append(keep)
            ws_bytes = max(ws_bytes, lib.psa_train_dense_workspace_bytes(batch, cin, width), lib.psa_bn_bwd_workspace_bytes(width))
            cin = width
        self.head_dh = [torch.empty((batch, ly.N), **f32) for ly in self.head[:-1]]
        self.d_feat = torch.empty_like(self.levels[-1].pooled)          # (B, C) under a head; (B*m, C) for a bare level stack
        self.dlogits = torch.empty((batch, num_class), **f32)
        self.loss = torch.zeros(1, **f32)
        self.ws = torch.empty(ws_bytes // 4 + 64, **f32)
        self.ws_bytes = ws_bytes
        self._gen = torch.Generator(device=dev)
        self._gen.manual_seed(1234)

    # ------------------------------------------------------------------------------------------------
    def draw_dropout(self):
        """tf.nn.dropout masks of the head (0 or 1/keep_prob), drawn on the device before the step."""
        for ly, keep in zip(self.head, self.keep):
            if keep is not None:
                r = torch.rand(ly.mask.shape, generator=self._gen, device=self.dev)
                ly.mask.copy_((r < keep).to(torch.float32) / keep)

    # ------------------------------------------------------------------------------------------------
    def forward(self, xyz: torch.Tensor, bn_decay: float = 0.5, points: torch.Tensor | None = None, sampled=None) -> torch.Tensor:
        """Training-mode forward (batch statistics, moving averages updated with `bn_decay`) -> logits (B, num_class); without a head
        -> the last level's pooled features (B*m, C).  `points` (B, N, in_channels): input features of the first level.  `sampled`:
        (fps_idx, new_xyz) of the first level, already sampled by the caller.  A frozen trainer ignores `bn_decay`."""
        B = self.B
        self._fold_frozen([ly for lv in self.levels for ly in lv.layers] + self.head)
        assert xyz.shape == (B, self.N0, 3) and xyz.is_cuda and xyz.dtype == torch.float32
        assert (points is None) == (self.in_channels == 0), "points must be given exactly when the trainer was built with in_channels > 0"
        cur_xyz, cur_pts = xyz.contiguous(), None
        if points is not None:
            assert points.shape == (B, self.N0, self.in_channels) and points.dtype == torch.float32
            cur_pts = points.contiguous()
        self.in_xyz = []
        for lv in self.levels:
            sp = lv.spec
            self.in_xyz.append((cur_xyz, cur_pts))
            L0 = lv.layers[0]
            if sp.group_all:
                # sample_and_group_all (pointnet_util.py:59-84): rows = [xyz, points], one group per cloud
                lv.x_cat[:, :3].copy_(cur_xyz.reshape(-1, 3))
                if cur_pts is not None:
                    lv.x_cat[:, 3:].copy_(cur_pts.reshape(B * lv.n, -1))
                self._layer_fwd(L0, _raw_in(lv.x_cat), bn_decay)
                lv.new_xyz = torch.zeros((B, 1, 3), dtype=torch.float32, device=self.dev)
            else:
                if sampled is not None and lv is self.levels[0]:
                    lv.fps_idx, lv.new_xyz = sampled
                else:
                    lv.fps_idx, lv.new_xyz = ops.farthest_point_sample_and_gather(lv.m, cur_xyz)
                check(self.lib.psa_sa_conv1_prebn(B, lv.n, lv.m, lv.c_in, C.c_float(sp.radius), lv.k, _p(cur_xyz), _p(lv.new_xyz), _p(cur_pts),
                                                  _p(L0.W), _p(L0.b), L0.N, _p(L0.y), _p(lv.idx), _p(lv.cnt), None if self.frozen else _p(L0.stats),
                                                  _p(self.ws), C.c_size_t(self.ws_bytes), _stream()), "sa_conv1_prebn")
                self._bn_finalize(L0, L0.rows, bn_decay)
            self._chain_fwd(lv.layers[1:], L0.act_in(), bn_decay)
            top = lv.layers[-1]
            check(self.lib.psa_train_pool_fwd(B * lv.m, lv.k, top.N, _p(top.y), _p(top.scale), _p(top.shift), _p(lv.pooled), _p(lv.argk),
                                              _stream()), "train_pool_fwd")
            cur_xyz, cur_pts = lv.new_xyz, lv.pooled.view(B, lv.m, -1)
        feat = self.levels[-1].pooled                                   # (B, C)
        if not self.head:
            return feat
        self._chain_fwd(self.head, _raw_in(feat), bn_decay)
        return self.head[-1].y

    # ------------------------------------------------------------------------------------------------
    def backward(self, dlogits: torch.Tensor, xyz_grad: bool = False):
        """Gradients of every trainable variable for d(loss)/d(logits) = dlogits, into the flat gradient bucket (a frozen trainer: input
        gradients only, the bucket is not touched).  xyz_grad: also each level's coordinate parts (lv.dxyz, lv.dnew; see
        input_xyz_grad); nothing else changes with it."""
        B = self.B
        # ---- head ----  (a bare level stack: dlogits is the gradient of the last level's pooled features)
        dh = dlogits.contiguous()
        if self.head:
            self._chain_bwd(self.head, _grad_dense(self.head[-1], dh), self.head_dh, _raw_in(self.levels[-1].pooled), self.d_feat)
        else:
            self.d_feat.copy_(dh.reshape(self.d_feat.shape))
        # ---- set-abstraction levels, last to first ----
        dpool = self.d_feat
        for li in range(len(self.levels) - 1, -1, -1):
            lv = self.levels[li]
            cur_xyz, cur_pts = self.in_xyz[li]
            L0 = lv.layers[0]
            g = _grad_pooled(lv.layers[-1], dpool, lv.pooled, lv.argk, lv.k)
            if len(lv.layers) > 1:
                self._chain_bwd(lv.layers[1:], g, lv.dh[1:], L0.act_in(), lv.dh[0])
                g = _grad_dense(L0, lv.dh[0])
            if lv.spec.group_all:
                self._layer_bwd(L0, g, _raw_in(lv.x_cat), lv.d_in, col_skip=3)
                if xyz_grad:
                    # the coordinate columns of dx: a second product over the first three rows of W (the feature columns above are unchanged)
                    self._products(g, L0.rows, 3, L0.N, L0.W, None, None, lv.dxyz)
            else:
                self._bn_bwd(L0, g)
                if not self.frozen or lv.c_in:
                    # frozen: only for dU (the dW_xyz it also writes goes to scratch)
                    check(self.lib.psa_sa_conv1_bwd(B, lv.n, lv.m, lv.k, L0.N, _p(cur_xyz), _p(lv.new_xyz), _p(lv.idx), C.byref(g),
                                                    _p(lv.dW_scratch if self.frozen else L0.dW[:3]), _p(lv.dU), _p(self.ws),
                                                    C.c_size_t(self.ws_bytes), _stream()), "sa_conv1_bwd")
                if lv.c_in:
                    # the feature rows of W: two dense products on the source points, dU = GroupPointGrad of dy
                    self._products(_plain_grad(lv.dU), B * lv.n, lv.c_in, L0.N, L0.W[3:], L0.dW[3:], _raw_in(cur_pts.reshape(B * lv.n, lv.c_in)),
                                   lv.d_in)
                if xyz_grad:
                    check(self.lib.psa_sa_conv1_bwd_xyz(B, lv.n, lv.m, lv.k, L0.N, _p(L0.W), _p(lv.idx), C.byref(g), _p(lv.dxyz), _p(lv.dnew),
                                                        _p(self.ws), C.c_size_t(self.ws_bytes), _stream()), "sa_conv1_bwd_xyz")
            dpool = lv.d_in

    def input_xyz_grad(self) -> torch.Tensor:
        """After backward(..., xyz_grad=True): the gradient w.r.t. the input cloud (B, N0, 3).  Levels last to first:
        d new_xyz = this level's -sum term + the next level's input-coordinate gradient, then d xyz_in = the rows' GroupPointGrad +
        GatherPointGrad(d new_xyz, fps_idx).  The group-all level's new_xyz is the constant origin."""
        B = self.B
        dnext = None
        for lv in reversed(self.levels):
            if lv.spec.group_all:
                d = lv.dxyz
            else:
                dn = lv.dnew if dnext is None else lv.dnew + dnext.view(-1, 3)
                gp = torch.empty_like(lv.dxyz)
                check(self.lib.psa_gather_point_grad(B, lv.n, lv.m, _p(dn), _p(lv.fps_idx), _p(gp), _p(self.ws), C.c_size_t(self.ws_bytes),
                                                     _stream()), "gather_point_grad")
                d = gp.add_(lv.dxyz)
            dnext = d
        return dnext.view(B, self.N0, 3)

    # ------------------------------------------------------------------------------------------------
    def loss_and_grad(self, logits: torch.Tensor, labels: torch.Tensor):
        """mean sparse softmax cross-entropy (pointnet2_cls_ssg.py:50-57) -> loss (1,) and d loss / d logits."""
        check(self.lib.psa_softmax_xent(self.B, self.num_class, _p(logits), _p(labels), _p(self.loss), _p(self.dlogits), _stream()), "softmax_xent")
        return self.loss, self.dlogits

    def allreduce_grads(self):
        """data parallelism: ONE all-reduce (sum) of the flat gradient bucket; averaged inside the Adam kernel"""
        if self.world > 1:
            torch.distributed.all_reduce(self.fp.grad, group=self.pg)

    def adam(self, lr: float, beta1=0.9, beta2=0.999, eps=1e-8):
        fp = self.fp
        fp.step_count += 1
        check(self.lib.psa_adam_step(fp.total, _p(fp.flat), _p(fp.grad), _p(fp.adam_m), _p(fp.adam_v), C.c_float(lr), C.c_float(beta1),
                                     C.c_float(beta2), C.c_float(eps), fp.step_count, C.c_float(1.0 / self.world), _stream()), "adam_step")
        self.params.invalidate()

    def train_step(self, xyz: torch.Tensor, labels: torch.Tensor, lr: float = 1e-3, bn_decay: float = 0.5, dropout: bool = True):
        """one sess.run(train_op) of pointnet2/train.py:246-252: forward, loss, backward, (all-reduce), Adam.  -> loss (1,)"""
        if dropout:
            self.draw_dropout()
        logits = self.forward(xyz, bn_decay)
        loss, dl = self.loss_and_grad(logits, labels)
        self.backward(dl)
        self.allreduce_grads()
        self.adam(lr)
        return loss


class _TrainFn(torch.autograd.Function):
    """get_model(is_training=True) for autograd users: logits whose backward fills the flat gradient bucket, and gives the gradient
    of the input cloud when it requires one.  A frozen trainer (inference mode) is applied with flat=None: input gradient only."""

    @staticmethod
    def forward(ctx, flat, trainer, xyz, bn_decay):
        ctx.trainer = trainer
        return trainer.forward(xyz, bn_decay).clone()

    @staticmethod
    def backward(ctx, dlogits):
        tr = ctx.trainer
        want_xyz = ctx.needs_input_grad[2]
        tr.backward(dlogits.contiguous(), xyz_grad=want_xyz)
        dxyz = tr.input_xyz_grad().clone() if want_xyz else None
        return (None if tr.frozen else tr.fp.grad.clone()), None, dxyz, None


class _LevelFn(torch.autograd.Function):
    """One pointnet_sa_module(is_training=True): pooled features whose backward returns the gradient of the input features and
    of this level's variables (a flat bucket that is zero outside the level -- several levels may share one store), and, when
    asked for, the level's coordinate parts: the rows' GroupPointGrad for xyz and the "- new_xyz" term for new_xyz (new_xyz itself
    comes from the differentiable gather_point, so autograd adds GatherPointGrad and whatever later levels send).  A frozen
    trainer (inference mode) gives input gradients only (flat=None)."""

    @staticmethod
    def forward(ctx, flat, points, xyz, new_xyz, trainer, bn_decay, fps_idx):
        ctx.trainer = trainer
        ctx.has_points = points is not None
        sampled = None if fps_idx is None else (fps_idx, new_xyz.detach().contiguous())
        out = trainer.forward(xyz.contiguous(), bn_decay, points, sampled=sampled)
        lv = trainer.levels[-1]
        return out.clone().view(trainer.B, lv.m, -1)

    @staticmethod
    def backward(ctx, dout):
        tr = ctx.trainer
        need = ctx.needs_input_grad
        want_xyz = need[2] or need[3]
        tr.backward(dout.contiguous(), xyz_grad=want_xyz)
        g = None if tr.frozen else _flat_grad_of_layers(tr.fp, [ly for lv in tr.levels for ly in lv.layers])
        lv = tr.levels[0]
        dp = lv.d_in.view(tr.B, tr.N0, tr.in_channels).clone() if ctx.has_points and need[1] else None
        dxyz = lv.dxyz.view(tr.B, tr.N0, 3).clone() if need[2] else None
        dnew = lv.dnew.view(tr.B, lv.m, 3).clone() if need[3] and not lv.spec.group_all else None
        return g, dp, dxyz, dnew, None, None, None


def wants_input_grad(*tensors) -> bool:
    """inference-mode calls take the frozen-batch-norm autograd path when gradients are being recorded and an input asks for one"""
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


def sa_module_training(xyz, points, spec: LevelSpec, bn_decay, params: VariableStore, frozen: bool = False):
    """Training-mode pointnet_sa_module (max pooling, use_xyz): -> (new_xyz, new_points (B,m,C) with a grad_fn, idx).  The level's
    buffers are cached on `params` per (scope, shape); gradients of its variables arrive in `params._flat.grad_of(name)` /
    through autograd on `params._flat.flat`, the gradients of `points` and `xyz` through autograd.  frozen=True: inference mode
    (batch norm on the moving averages, which stay put; input gradients only)."""
    b, n, _ = xyz.shape
    c = 0 if points is None else points.shape[-1]
    key = ("level_frozen" if frozen else "level", spec.scope, b, n, c, spec.npoint, spec.radius, spec.nsample, tuple(spec.mlp), spec.group_all)
    tr = _cached(params, key, lambda: PointNet2ClsTrainer(params, b, n, levels=[spec], head=[], device=xyz.device, in_channels=c, frozen=frozen))
    flat, decay = _flat_and_decay(tr, bn_decay)
    if spec.group_all:
        fps_idx, new_xyz = None, None
    else:
        fps_idx, new_xyz = ops.farthest_point_sample_and_gather(spec.npoint, xyz)
        if wants_input_grad(xyz):
            new_xyz = ops.gather_point(xyz, fps_idx)       # same values as the fused gather, differentiable (GatherPointGrad)
    out = _LevelFn.apply(flat, points, xyz, new_xyz, tr, decay, fps_idx)
    lv = tr.levels[0]
    idx = lv.idx
    if spec.group_all:            # sample_and_group_all: one group holding every point in order (pointnet_util.py:75-77)
        idx = torch.arange(n, dtype=torch.int32, device=xyz.device).view(1, 1, n).repeat(b, 1, 1)
        new_xyz = lv.new_xyz
    return new_xyz, out, idx


def get_model_training(point_cloud, bn_decay, num_class, params: VariableStore, levels=None, head=None, frozen: bool = False):
    """Training-mode forward of the classifier; the trainer (buffers, flat parameter bucket) is cached on `params`.  frozen=True:
    inference-mode forward (moving averages, no dropout) whose backward gives the gradient of the input cloud only."""
    key = (tuple(point_cloud.shape), num_class) if not frozen else ("frozen", tuple(point_cloud.shape), num_class)
    tr = _cached(params, key, lambda: PointNet2ClsTrainer(params, point_cloud.shape[0], point_cloud.shape[1], num_class, levels=levels,
                                                          head=head, device=point_cloud.device, frozen=frozen))
    flat, decay = _flat_and_decay(tr, bn_decay)
    if not frozen:
        tr.draw_dropout()
    return _TrainFn.apply(flat, tr, point_cloud, decay), tr
