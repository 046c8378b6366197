"""PointCNN/pointcnn_cls.py with the setting pointcnn_cls/modelnet_x3_l4.py on the libpsa kernels, inference and training mode.

The reference (pointcnn.py:55-152, pointcnn_cls.py:10-17): four X-Conv layers on the points alone (no extra features, random
sampling = the first P points of the previous level, X-transformation on, no sorting, no links), the last with the global branch
of the query coordinates in front of its output -> fc0 384, fc1 192 per point (dropout is the identity at inference) -> the mean
over the points -> logits with a bias, (B, 1, num_class).  Every layer with batch norm has no bias and applies ELU before the
batch norm (pointfly.py:298-347).

Here each X-Conv layer is a kNN launch (every D-th of the K*D nearest), one core launch that writes only the (B*P, C_in*dm)
depthwise output, and one tensor-core GEMM for the pointwise conv with the ELU / batch-norm epilogue.  The last layer's global
branch and pointwise conv write their slices of the 480-wide row in place, so nothing is concatenated, and no (B,P,K,.) tensor
is built.  Training mode (train.py's step: per-point logits, batch-statistics batch norm, dropout, the L2 regularisation) is
get_model_training over PointCNNTrainer below.
"""
from __future__ import annotations

import ctypes as C
import math

import torch

from . import _lib, ops
from ._lib import PsaActIn, PsaGradIn, check
from ._lib import ptr as _p
from ._lib import stream as _stream
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
        raise NotImplementedError("pointcnn_cls.get_model runs inference only: train through get_model_training")
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



# ---------------------------------------------------------------------------------------------------------------------
# training mode
# ---------------------------------------------------------------------------------------------------------------------
BN_DECAY = 0.99                  # tf.layers.batch_normalization(momentum=0.99) (pointfly.py:298-302)
DROPOUT_KEEP = 0.2               # fc1's dropout rate 0.8 (modelnet_x3_l4.py:63-66); fc0's rate 0.0 is the identity
WEIGHT_DECAY = 1e-5              # train.py:164, over l2_regularizer(1.0) terms
UNREGULARISED = ("logits/bias",)


class PointCNNTrainer:
    """pointcnn_cls in training mode at one (B, N): forward(points, mask) -> per-point logits (B*128, num_class) with every batch norm
    on the statistics of its batch (moving averages updated with decay 0.99), backward(dlogits) -> every variable's gradient in the
    store's flat gradient bucket.  Per X-Conv layer it keeps the kNN indices, the saved activations a = elu(z) of each batch-normed
    layer (psa_xconv_saved, the pointwise conv's and the global branch's), the core's depthwise output and the layer output; the
    backward's per-layer scratch is one arena.  Buffers are allocated once."""

    def __init__(self, params: VariableStore, b: int, n: int, device):
        from .training import FlatParams
        self.lib = _lib.load()
        self.fp = params._flat if getattr(params, "_flat", None) is not None else FlatParams(params)
        params._flat = self.fp
        fp, self.b, self.n = self.fp, b, n
        f32 = dict(dtype=torch.float32, device=device)
        self.ones, self.zeros = torch.ones(512, **f32), torch.zeros(512, **f32)
        ws_bwd, arena, n_prev = 0, 0, n
        self.layers = []
        for l, (tag, k, d, p, c, c_pts, c_prev, dm, glob) in enumerate(layer_table(), start=1):
            p = n if p == -1 else p
            R, kk, cin = b * p, k * k, c_pts + c_prev
            L = dict(l=l, tag=tag, K=k, D=d, P=p, C=c, Cf=c_pts, Cp=c_prev, dm=dm, glob=glob, cin=cin, R=R, n_prev=n_prev,
                     idx=torch.empty((b, p, k), dtype=torch.int32, device=device),
                     saved={"local": torch.empty((R * k, 3), **f32), "a_p0": torch.empty((R * k, c_pts), **f32),
                            "a_p1": torch.empty((R * k, c_pts), **f32), "a_x0": torch.empty((R, kk), **f32),
                            "a_x1": torch.empty((R, kk), **f32), "a_x2": torch.empty((R, kk), **f32)},
                     dw=torch.empty((R, cin * dm), **f32), out=torch.empty((R, glob + c), **f32), d_out=torch.empty((R, glob + c), **f32))
            sv = L["saved"]
            bns = [("pts0", "nn_fts_from_pts_0", "kernel", sv["a_p0"]), ("pts1", "nn_fts_from_pts", "kernel", sv["a_p1"]),
                   ("x0", "X_0", "kernel", sv["a_x0"]), ("x1", "X_1", "depthwise_weights", sv["a_x1"]), ("x2", "X_2", "depthwise_weights", sv["a_x2"]),
                   ("pw", "fts_conv", "pointwise_kernel", torch.empty((R, c), **f32))]
            if glob:
                bns += [("g0", "fts_global_0", "kernel", torch.empty((R, glob), **f32)), ("g", "fts_global", "kernel", torch.empty((R, glob), **f32))]
                L["h_g0"] = torch.empty((R, glob), **f32)
            L["bn"] = {short: self._bn(params, f"{tag}{layer}", f"{tag}{layer}/{var}", a) for short, layer, var, a in bns}
            L["W_dw"], L["dW_dw"] = fp.views[f"{tag}fts_conv/depthwise_kernel"], fp.gviews[f"{tag}fts_conv/depthwise_kernel"]
            # backward scratch: two (R*K, C_pts), two (R, K*K), d_dw, the pointwise conv's dz, dF_prev, and the global branch's dz / dh
            sizes = [("pA", R * k * c_pts), ("pB", R * k * c_pts), ("xA", R * kk), ("xB", R * kk), ("d_dw", R * cin * dm), ("dz", R * c),
                     ("dF_prev", R * k * c_prev), ("gA", R * glob), ("gB", R * glob)]
            L["scratch"], off = {}, 0
            for name, cnt in sizes:
                L["scratch"][name] = (off, cnt)
                off += (cnt + 63) // 64 * 64
            arena = max(arena, off)
            ws_bwd = max(ws_bwd, int(self.lib.psa_xconv_train_bwd_workspace_bytes(b, p, k, c_pts, c_prev, dm)),
                         int(self.lib.psa_scatter_workspace_bytes(b, n_prev, p * k)))
            for bn in L["bn"].values():
                ws_bwd = max(ws_bwd, int(self.lib.psa_bn_bwd_workspace_bytes(bn["C"])))
                if bn["K"]:
                    ws_bwd = max(ws_bwd, int(self.lib.psa_train_dense_workspace_bytes(bn["rows"], bn["K"], bn["C"])))
            self.layers.append(L)
            n_prev = p
        R = self.layers[-1]["R"]
        self.rows = R
        cin, self.head = self.layers[-1]["glob"] + self.layers[-1]["C"], []
        for i, c in enumerate(FC):
            bn = self._bn(params, f"fc{i}", f"fc{i}/kernel", torch.empty((R, c), **f32))
            bn["h"] = torch.empty((R, c), **f32) if i < len(FC) - 1 else None
            bn["dh"] = torch.empty((R, c), **f32)
            bn["dz"] = torch.empty((R, c), **f32)
            ws_bwd = max(ws_bwd, int(self.lib.psa_bn_bwd_workspace_bytes(c)), int(self.lib.psa_train_dense_workspace_bytes(R, cin, c)))
            self.head.append(bn)
            cin = c
        self.W_l, self.b_l = fp.views["logits/kernel"], fp.views["logits/bias"]
        self.dW_l, self.db_l = fp.gviews["logits/kernel"], fp.gviews["logits/bias"]
        self.num_class = self.b_l.numel()
        self.mask = torch.empty((R, FC[-1]), **f32)
        self.logits = torch.empty((R, self.num_class), **f32)
        ws_bwd = max(ws_bwd, int(self.lib.psa_train_dense_workspace_bytes(R, FC[-1], self.num_class)))
        self.arena = torch.empty(arena, **f32)
        self.ws_bwd_bytes = ws_bwd
        self.ws_bwd = torch.empty(ws_bwd // 4 + 64, **f32)
        self.ws_fwd_bytes, self.ws_fwd = 0, None

    def _bn(self, params, layer, wname, a):
        """one layer BN(elu(x . W)) (X_2: BN(x . W)): its kernel, saved activations a (rows, C), batch norm variables and per-step
        (scale, shift, mean_inv) and backward coefficients"""
        fp, rows, c = self.fp, a.shape[0], a.shape[1]
        w = fp.views[wname]
        dev = a.device
        e = lambda: torch.empty(c, dtype=torch.float32, device=dev)   # noqa: E731
        return dict(layer=layer, a=a, rows=rows, C=c, K=w.numel() // c if not wname.endswith("/depthwise_weights") else 0,
                    W=w, dW=fp.gviews[wname], gamma=fp.views[f"{layer}_bn/gamma"], beta=fp.views[f"{layer}_bn/beta"],
                    dgamma=fp.gviews[f"{layer}_bn/gamma"], dbeta=fp.gviews[f"{layer}_bn/beta"], mov_mean=params[f"{layer}_bn/moving_mean"],
                    mov_var=params[f"{layer}_bn/moving_variance"], s=e(), t=e(), mean_inv=torch.empty((2, c), dtype=torch.float32, device=dev),
                    ca=e(), cb=e(), cc=e())

    # ---- forward ----
    def _fwd_ws(self, rows, k, n):
        """psa_dense_elu_affine's workspace depends on the arithmetic mode of the call: grown on demand"""
        need = int(self.lib.psa_dense_elu_affine_workspace_bytes(rows, k, n))
        if need > self.ws_fwd_bytes:
            self.ws_fwd = torch.empty(need // 4 + 64, dtype=torch.float32, device=self.ones.device)
            self.ws_fwd_bytes = need
        return _p(self.ws_fwd), C.c_size_t(self.ws_fwd_bytes)

    def _finalize(self, bn):
        check(self.lib.psa_bn_finalize_rows(bn["rows"], bn["C"], _p(bn["a"]), _p(bn["gamma"]), _p(bn["beta"]), C.c_float(BN_DECAY),
                                            _p(bn["mov_mean"]), _p(bn["mov_var"]), _p(bn["s"]), _p(bn["t"]), _p(bn["mean_inv"]), _stream()),
              "bn_finalize_rows")

    def _dense(self, bn, x, ldx, out=None, ldo=0):
        """a = elu(x . W) (psa_dense_elu_affine with scale 1, shift 0), its batch statistics, then BN(a) into out when given"""
        rows, k, c = bn["rows"], bn["K"], bn["C"]
        ws, wsn = self._fwd_ws(rows, k, c)
        check(self.lib.psa_dense_elu_affine(rows, k, c, x, ldx, _p(bn["W"]), None, _p(self.ones), _p(self.zeros), _p(bn["a"]), c, ws, wsn, _stream()),
              "dense_elu_affine")
        self._finalize(bn)
        if out is not None:
            check(self.lib.psa_bn_affine_rows(rows, c, _p(bn["a"]), _p(bn["s"]), _p(bn["t"]), out, ldo, _stream()), "bn_affine_rows")

    def _xconv(self, L):
        """the psa_xconv of layer L with each batch norm's batch (s, t)"""
        bn = L["bn"]
        w = {"w_dw": L["W_dw"]}
        for short in ("pts0", "pts1", "x0", "x1", "x2"):
            w[f"w_{short}"], w[f"s_{short}"], w[f"t_{short}"] = bn[short]["W"], bn[short]["s"], bn[short]["t"]
        return _lib.PsaXconv(L["K"], L["Cf"], L["Cp"], L["dm"], *[w[name].data_ptr() for name in ops.XCONV_WEIGHTS])

    def layer_forward(self, L, pts, fts):
        """X-Conv layer L on pts (B, n_prev, 3) and the previous layer's output fts (B*n_prev, C_prev) or None -> L["out"] (B*P, glob + C)"""
        lib, b, k, p, R = self.lib, self.b, L["K"], L["P"], L["R"]
        qrs = pts if p == pts.shape[1] else pts[:, :p].contiguous()          # random sampling: the first P points (pointcnn.py:101)
        L["pts"], L["qrs"], L["fts"] = pts, qrs, fts
        check(lib.psa_knn_dilated(b, pts.shape[1], p, k, L["D"], _p(pts), _p(qrs), _p(L["idx"]), _stream()), "knn_dilated")
        xc = self._xconv(L)
        sv = _lib.PsaXconvSaved(*[L["saved"][f].data_ptr() for f in ("local", "a_p0", "a_p1", "a_x0", "a_x1", "a_x2")])
        bn = L["bn"]
        for stage, done in ((0, ("pts0", "x0")), (1, ("pts1", "x1")), (2, ("x2",))):
            check(lib.psa_xconv_train_stage(stage, b, pts.shape[1], p, _p(pts), _p(qrs), _p(L["idx"]), C.byref(xc), C.byref(sv), _stream()),
                  "xconv_train_stage")
            for short in done:
                self._finalize(bn[short])
        width = L["glob"] + L["C"]
        if L["glob"]:
            self._dense(bn["g0"], qrs.data_ptr(), 3, L["h_g0"].data_ptr(), L["glob"])
            self._dense(bn["g"], L["h_g0"].data_ptr(), L["glob"], L["out"].data_ptr(), width)
        check(lib.psa_xconv_core(b, pts.shape[1], p, _p(pts), _p(qrs), _p(L["idx"]), _p(fts), C.byref(xc), _p(L["dw"]), _stream()), "xconv_core")
        self._dense(bn["pw"], L["dw"].data_ptr(), L["cin"] * L["dm"], L["out"].data_ptr() + 4 * L["glob"], width)
        return L["out"]

    def forward(self, pts, mask):
        """pts (B, N, 3) float32, mask (B*128, 192) fc1's dropout mask or None -> logits (B*128, num_class)"""
        fts = None
        for L in self.layers:
            fts = self.layer_forward(L, pts, fts)
            pts = L["qrs"]
        x, ldx = fts.data_ptr(), fts.shape[1]
        for bn in self.head:
            self._dense(bn, x, ldx, None if bn["h"] is None else bn["h"].data_ptr(), bn["C"])
            if bn["h"] is not None:
                x, ldx = bn["h"].data_ptr(), bn["C"]
        fc1 = self.head[-1]
        self.mask_used = mask
        a = PsaActIn(x=_p(fc1["a"]), ld=fc1["C"], scale=_p(fc1["s"]), shift=_p(fc1["t"]), mask=_p(mask), relu=0)
        ws, wsn = _p(self.ws_bwd), C.c_size_t(self.ws_bwd_bytes)
        check(self.lib.psa_train_dense_fwd(self.rows, fc1["C"], self.num_class, C.byref(a), _p(self.W_l), _p(self.b_l), _p(self.logits), None,
                                           ws, wsn, _stream()), "train_dense_fwd")
        return self.logits

    # ---- backward ----
    def _coeffs(self, bn, dh, ld_dh, mask=None):
        """the batch-norm backward of layer bn from dh, the gradient of its output: dgamma, dbeta and the coefficients -> the
        psa_grad_in that evaluates the gradient of its input a"""
        g = PsaGradIn(y=_p(bn["a"]), ld=bn["C"], dh=dh, ld_dh=ld_dh, mask=_p(mask), pool_k=1, C=bn["C"])
        check(self.lib.psa_bn_bwd_coeffs(bn["rows"], bn["C"], C.byref(g), _p(bn["gamma"]), _p(bn["mean_inv"]), _p(bn["dgamma"]), _p(bn["dbeta"]),
                                         _p(bn["ca"]), _p(bn["cb"]), _p(bn["cc"]), _p(self.ws_bwd), C.c_size_t(self.ws_bwd_bytes), _stream()),
              "bn_bwd_coeffs")
        g.ca, g.cb, g.cc = _p(bn["ca"]), _p(bn["cb"]), _p(bn["cc"])
        return g

    def _dense_bwd(self, bn, dh, ld_dh, x, ldx, act_s=None, act_t=None, dz=None, dx=None, mask=None):
        """backward of a = elu(x . W) -> BN: dz (rows, C) materialised, dW = BN_prev(x)^T . dz, dx = dz . W^T when dx is given"""
        lib, rows, k, c = self.lib, bn["rows"], bn["K"], bn["C"]
        ws, wsn = _p(self.ws_bwd), C.c_size_t(self.ws_bwd_bytes)
        g = self._coeffs(bn, dh, ld_dh, mask)
        check(lib.psa_elu_bn_dy(rows, c, C.byref(g), dz, _stream()), "elu_bn_dy")
        plain = PsaGradIn(dh=dz, ld_dh=c, pool_k=1, C=c)
        a = PsaActIn(x=x, ld=ldx, scale=_p(act_s), shift=_p(act_t), relu=0)
        check(lib.psa_train_dense_bwd_weight(rows, k, c, C.byref(a), C.byref(plain), _p(bn["dW"]), ws, wsn, _stream()), "train_dense_bwd_weight")
        if dx is not None:
            check(lib.psa_train_dense_bwd_input(rows, k, c, C.byref(plain), _p(bn["W"]), dx, k, 0, ws, wsn, _stream()), "train_dense_bwd_input")

    def layer_backward(self, L, d_out, d_fts):
        """d_out (B*P, glob + C) the gradient of L["out"] -> the layer's variable gradients, and d_fts (B*n_prev, C_prev) the gradient of
        its input features when it has any"""
        lib, b, k, R, Cf, kk = self.lib, self.b, L["K"], L["R"], L["Cf"], L["K"] ** 2
        bn, sv, width, glob = L["bn"], L["saved"], L["glob"] + L["C"], L["glob"]
        ar = lambda name: self.arena.data_ptr() + 4 * L["scratch"][name][0]   # noqa: E731
        ws, wsn = _p(self.ws_bwd), C.c_size_t(self.ws_bwd_bytes)
        self._dense_bwd(bn["pw"], d_out.data_ptr() + 4 * glob, width, L["dw"].data_ptr(), L["cin"] * L["dm"], dz=ar("dz"), dx=ar("d_dw"))
        if glob:
            self._dense_bwd(bn["g"], d_out.data_ptr(), width, L["h_g0"].data_ptr(), glob, dz=ar("gA"), dx=ar("gB"))
            self._dense_bwd(bn["g0"], ar("gB"), glob, L["qrs"].data_ptr(), 3, dz=ar("gA"))
        xc = self._xconv(L)
        svs = _lib.PsaXconvSaved(*[sv[f].data_ptr() for f in ("local", "a_p0", "a_p1", "a_x0", "a_x1", "a_x2")])
        check(lib.psa_xconv_train_bwd_top(b, L["pts"].shape[1], L["P"], _p(L["idx"]), _p(L["fts"]), C.byref(xc), C.byref(svs), ar("d_dw"), ar("xA"),
                                          ar("pA"), ar("dF_prev") if L["Cp"] else None, _p(L["dW_dw"]), ws, wsn, _stream()), "xconv_train_bwd_top")
        # X_2 (no ELU), X_1: depthwise backward from dX2n (xA) -> dX1n (xB) -> dX0n (xA)
        for short, prev, elu, src, dst in (("x2", "x1", 0, "xA", "xB"), ("x1", "x0", 1, "xB", "xA")):
            g = self._coeffs(bn[short], ar(src), kk)
            check(lib.psa_xconv_depthwise_bwd(R, k, _p(bn[prev]["a"]), _p(bn[prev]["s"]), _p(bn[prev]["t"]), C.byref(g), elu, _p(bn[short]["W"]),
                                              _p(bn[short]["dW"]), ar(dst), ws, wsn, _stream()), "xconv_depthwise_bwd")
        self._dense_bwd(bn["x0"], ar("xA"), kk, sv["local"].data_ptr(), 3 * k, dz=ar("xB"))
        # the lifting layers from dF_lift (pA): dz_p1 (pB), dh0 (pA), dz_p0 (pB)
        self._dense_bwd(bn["pts1"], ar("pA"), Cf, sv["a_p0"].data_ptr(), Cf, bn["pts0"]["s"], bn["pts0"]["t"], dz=ar("pB"), dx=ar("pA"))
        self._dense_bwd(bn["pts0"], ar("pA"), Cf, sv["local"].data_ptr(), 3, dz=ar("pB"))
        if L["Cp"]:
            check(lib.psa_group_point_grad(b, L["n_prev"], L["Cp"], L["P"], k, ar("dF_prev"), _p(L["idx"]), _p(d_fts), ws, wsn, _stream()),
                  "group_point_grad")

    def backward(self, dlogits):
        """dlogits (B*128, num_class) -> every variable's gradient in the flat bucket"""
        lib, R, nc = self.lib, self.rows, self.num_class
        ws, wsn = _p(self.ws_bwd), C.c_size_t(self.ws_bwd_bytes)
        fc0, fc1 = self.head
        plain = PsaGradIn(dh=_p(dlogits), ld_dh=nc, pool_k=1, C=nc)
        a = PsaActIn(x=_p(fc1["a"]), ld=fc1["C"], scale=_p(fc1["s"]), shift=_p(fc1["t"]), mask=_p(self.mask_used), relu=0)
        check(lib.psa_train_dense_bwd_weight(R, fc1["C"], nc, C.byref(a), C.byref(plain), _p(self.dW_l), ws, wsn, _stream()), "train_dense_bwd_weight")
        check(lib.psa_train_bias_grad(R, nc, C.byref(plain), _p(self.db_l), _stream()), "train_bias_grad")
        check(lib.psa_train_dense_bwd_input(R, fc1["C"], nc, C.byref(plain), _p(self.W_l), _p(fc1["dh"]), fc1["C"], 0, ws, wsn, _stream()),
              "train_dense_bwd_input")
        self._dense_bwd(fc1, fc1["dh"].data_ptr(), fc1["C"], fc0["h"].data_ptr(), fc0["C"], dz=fc1["dz"].data_ptr(), dx=fc0["dh"].data_ptr(),
                        mask=self.mask_used)
        L4 = self.layers[-1]
        self._dense_bwd(fc0, fc0["dh"].data_ptr(), fc0["C"], L4["out"].data_ptr(), L4["out"].shape[1], dz=fc0["dz"].data_ptr(),
                        dx=L4["d_out"].data_ptr())
        for i in range(len(self.layers) - 1, -1, -1):
            L = self.layers[i]
            self.layer_backward(L, L["d_out"], self.layers[i - 1]["d_out"] if i else None)


class _PcnnFn(torch.autograd.Function):
    """PointCNNTrainer as one autograd node over the store's flat parameter vector"""

    @staticmethod
    def forward(ctx, flat, pts, trainer, mask):
        ctx.trainer = trainer
        return trainer.forward(pts, mask).clone()

    @staticmethod
    def backward(ctx, dlogits):
        tr = ctx.trainer
        tr.fp.grad.zero_()
        tr.backward(dlogits.contiguous())
        return tr.fp.grad.clone(), None, None, None


def get_model_training(points, num_class=NUM_CLASSES, *, params: VariableStore, dropout: bool = True, return_end_points: bool = False):
    """Net(points, features=None, is_training=True, setting).logits: points (B,N,3), N >= 384 -> per-point logits (B, 128, num_class)
    (pointcnn_cls.py:13-16 keeps fc1's per-point output in training), differentiable in the store's variables (autograd over its flat
    parameter vector, training.FlatParams).  Every batch norm uses the statistics of its batch (biased variance, eps 1e-3) and
    updates its moving averages as 0.99 moving + 0.01 batch; fc1 is followed by dropout keeping 0.2 (survivors times 5), drawn with
    torch's generator (dropout=False: the identity).  With return_end_points also a dict of the trainer's buffers, overwritten by the
    next call: per layer l = 1..4 ``idx<l>`` (B,P,K), ``local<l>`` (B*P*K, 3), ``dw<l>`` (B*P, C_in*dm) and ``fts<l>`` (B*P, glob + C);
    per batch-normed layer (``<tag>nn_fts_from_pts_0``, ..., ``fc0``, ``fc1``) ``<layer>/a`` = elu(z) (z for X_2), ``<layer>/scale`` and
    ``<layer>/shift``; ``fc1/mask`` (B*128, 192) or None.  Gradients with respect to the points are not implemented."""
    from .training import _cached
    if isinstance(points, torch.Tensor) and points.requires_grad:
        raise NotImplementedError("pointcnn_cls: gradients with respect to the input points are not implemented")
    if params["logits/bias"].numel() != num_class:
        raise ValueError(f"num_class={num_class} but the store's logits layer has {params['logits/bias'].numel()} outputs")
    if not isinstance(points, torch.Tensor) or points.dim() != 3 or points.shape[-1] != 3:
        raise ValueError("pointcnn_cls: points must be a (B, N, 3) tensor")
    b, n, _ = points.shape
    if n < MIN_POINTS:
        raise ValueError(f"pointcnn_cls: N={n} points, fewer than the {MIN_POINTS} queries of layer 2 (tf.slice fails)")
    pts = ops._dev(points, torch.float32, "points", 3)
    tr = _cached(params, ("pointcnn_cls", b, n), lambda: PointCNNTrainer(params, b, n, pts.device))
    mask = tr.mask.bernoulli_(DROPOUT_KEEP).mul_(1.0 / DROPOUT_KEEP) if dropout else None
    logits = _PcnnFn.apply(tr.fp.flat.requires_grad_(True), pts, tr, mask).view(b, -1, num_class)
    if not return_end_points:
        return logits
    ep = {"fc1/mask": mask}
    for L in tr.layers:
        l = L["l"]
        ep.update({f"idx{l}": L["idx"], f"local{l}": L["saved"]["local"], f"dw{l}": L["dw"], f"fts{l}": L["out"]})
    for bn in [bn for L in tr.layers for bn in L["bn"].values()] + tr.head:
        ep.update({f"{bn['layer']}/a": bn["a"], f"{bn['layer']}/scale": bn["s"], f"{bn['layer']}/shift": bn["t"]})
    return logits, ep


def get_loss(logits, label):
    """train.py:138-140: sparse softmax cross-entropy of the per-point logits (B, P, num_class) against the label tiled to every
    point, averaged over B*P"""
    b, p, c = logits.shape
    return torch.nn.functional.cross_entropy(logits.reshape(b * p, c), label.long().reshape(b, 1).expand(b, p).reshape(-1))


def get_regularization_loss(params: VariableStore):
    """WEIGHT_DECAY * sum 0.5 |v|^2 over the regularised variables (train.py:164, pointfly.py:300-345): every kernel and batch-norm
    gamma / beta, not logits/bias or the moving averages.  Built from FlatParams.live views, so its gradient lands in the same flat
    bucket as the model's."""
    from .training import FlatParams
    fp = params._flat if getattr(params, "_flat", None) is not None else FlatParams(params)
    params._flat = fp
    fp.flat.requires_grad_(True)
    total = sum(fp.live(name).square().sum() for name in fp.names if name not in UNREGULARISED)
    return WEIGHT_DECAY * 0.5 * total
