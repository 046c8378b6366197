"""3DmFV-Net/models/3dmfv_net_cls.py on the libpsa kernels, inference mode (the reference's module name starts with a digit).

The reference (3dmfv_net_cls.py:29-102): the modified Fisher vector of the cloud on a grid GMM of r^3 Gaussians (tf_util.get_3dmfv,
(B,20,G)) reshaped to a (B,r,r,r,20) grid -> inception modules of 64, 128 and 256 filters on the r^3 grid -> a SAME 2^3 max pool
(stride 2) -> inception 256 and 512 -> another max pool -> flatten -> fc1 1024, fc2 256, fc3 128 (batch norm, ReLU; dropout is
the identity at inference) -> fc4.  An inception module with n filters is concat[conv1 1^3 (in -> n), conv2 3^3 on conv1 (n ->
n/2), conv3 5^3 on conv1 (n -> n/2), conv4 1^3 on a SAME 3^3 average pool of the input (in -> n)], each conv3d with bias, batch
norm and ReLU.

Here the grid activations are voxel-major rows (B*r^3, C), row = voxel * B + cloud, so that a 128-row tile of the conv kernel
covers few voxels and skips the kernel taps that fall outside the grid for all of them.  Each branch writes its channel slice of
the module's output in place (no concatenation), and conv2 / conv3 read conv1's slice in place.  The Fisher vector is one kernel
that never builds the reference's (B,N,G,3) tiles.  The layout is converted only where the reference's tensors are visible:
the returned ``fv`` and the flatten before fc1 are the reference's.

Training (get_model_training, 3DmFV-Net/train.py:163-173): w, mu and sigma are fed placeholders, so nothing upstream of the Fisher
vector trains and the backward stops at the grid.  Each conv3d writes its pre-batch-norm y = x * W + bias (psa_conv3d_infer in the
current arithmetic mode), batch statistics over all rows give scale / shift, and relu(y * scale + shift) fills the branch's slice of
the module output.  The backward (MfvTrainer.backward, fp32 FMA kernels of csrc/mfv_train.cu) runs the modules in reverse: per conv
the batch-norm coefficients and dy, dW = A^T . dy and dx = dy . W^T with the gathered conv input A never formed, the out-of-grid
taps skipped; conv1's slice adds the data gradients of conv2 and conv3, the module input gets the average-pool backward of conv4's
plus conv1's.  fc1-fc4 train with batch statistics (training.mlp_training).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib, ops
from ._lib import PsaGradIn, check
from ._lib import ptr as _p
from ._lib import stream as _stream
from .tf_util import VariableStore

NUM_CLASSES = 15
INCEPTION = (64, 128, 256, 256, 512)      # filters of inception1..5; a max pool follows inception3 and inception5
KERNEL_SIZES = (3, 5)


def get_3d_grid_gmm(subdivisions=(5, 5, 5), variance=0.04):
    """utils.get_3d_grid_gmm (3DmFV-Net/utils/utils.py:69-92) without sklearn: -> (w (G), mu (G,3), sigma (G,3)) as float32
    numpy arrays, sigma = sqrt(variance) as train.py:280-282 feeds it.  Gaussian g sits at grid cell (g // r^2, g // r % r,
    g % r), the x index first."""
    axes = []
    for s in subdivisions:
        lo, hi = 1.0 / s - 1.0, 1.0 - 1.0 / s
        axes.append(np.arange(s) * ((hi - lo) / (s - 1)) + lo)             # s centres from lo to hi, rounded as np.mgrid rounds
    mu = np.stack(np.meshgrid(*axes, indexing="ij")).reshape(3, -1).T        # (G,3), the last axis fastest
    g = mu.shape[0]
    w = np.full(g, 1.0 / g)
    sigma = np.sqrt(np.full_like(mu, variance))
    return w.astype(np.float32), mu.astype(np.float32), sigma.astype(np.float32)


def _module_widths():
    """[(scope, k, cin, cout)] of every conv3d in the order the reference creates them"""
    out, cin = [], 20
    for l, n in enumerate(INCEPTION, start=1):
        s = f"inception{l}"
        out += [(f"{s}_conv1", 1, cin, n), (f"{s}_conv2", KERNEL_SIZES[0], n, n // 2), (f"{s}_conv3", KERNEL_SIZES[1], n, n // 2),
                (f"{s}_conv4", 1, cin, n)]
        cin = 3 * n
    return out


def init_params(num_classes=NUM_CLASSES, seed=0, device="cuda", randomize_bn=False) -> VariableStore:
    """The reference's variables: inception{1..5}_conv{1..4}/weights (k,k,k,cin,cout), biases and bn/*, then fc1..fc3 (batch norm)
    and fc4.  The flatten before fc1 has 2^3 * 1536 = 12288 entries for the 5^3 grid."""
    p = VariableStore(device=device, seed=seed)
    for scope, k, cin, cout in _module_widths():
        p.add_conv3d(scope, k, cin, cout, randomize_bn=randomize_bn)
    p.add_fc("fc1", 8 * 3 * INCEPTION[-1], 1024, randomize_bn=randomize_bn)
    p.add_fc("fc2", 1024, 256, randomize_bn=randomize_bn)
    p.add_fc("fc3", 256, 128, randomize_bn=randomize_bn)
    p.add_fc("fc4", 128, num_classes, bn=False)
    return p


def _inception(x, r, n, scope, params):
    """inception_module (3dmfv_net_cls.py:86-102) on voxel-major rows x (B*r^3, cin) -> (B*r^3, 3n)"""
    out = torch.empty((x.shape[0], 3 * n), dtype=torch.float32, device=x.device)
    w, sc, sh, _ = params.folded(f"{scope}_conv1")
    ops.conv3d(x, r, w, sc, sh, out=out, offset=0)
    one = out[:, :n]
    w, sc, sh, _ = params.folded(f"{scope}_conv2")
    ops.conv3d(one, r, w, sc, sh, out=out, offset=n)
    w, sc, sh, _ = params.folded(f"{scope}_conv3")
    ops.conv3d(one, r, w, sc, sh, out=out, offset=n + n // 2)
    w, sc, sh, _ = params.folded(f"{scope}_conv4")
    ops.conv3d(ops.pool3d(x, r, "avg"), r, w, sc, sh, out=out, offset=2 * n)
    return out


def get_model(points, w, mu, sigma, is_training, bn_decay=None, weigth_decay=0.005, add_noise=False, num_classes=NUM_CLASSES, *,
              params: VariableStore):
    """3dmfv_net_cls.get_model: points (B,N,3), the grid GMM (w (G), mu (G,3), sigma (G,3)) with G = r^3 -> (logits
    (B,num_classes), fv (B,20,G)).  bn_decay and weigth_decay only matter in training."""
    if is_training:
        raise NotImplementedError("mfv_net_cls.get_model runs inference only: train through get_model_training")
    if isinstance(points, torch.Tensor) and points.requires_grad and torch.is_grad_enabled():
        raise NotImplementedError("mfv_net_cls: gradients with respect to the input points are not implemented")
    if add_noise:
        raise NotImplementedError("mfv_net_cls: the add_noise augmentation is not implemented")
    if params["fc4/biases"].numel() != num_classes:
        raise ValueError(f"num_classes={num_classes} but the store's fc4 has {params['fc4/biases'].numel()} outputs")
    w, mu, sigma = (torch.as_tensor(t, dtype=torch.float32, device=points.device) for t in (w, mu, sigma))
    g = w.shape[0]
    r = int(round(g ** (1.0 / 3.0)))
    if r ** 3 != g:
        raise ValueError(f"mfv_net_cls: G = {g} Gaussians is not a cube r^3 (the model needs a grid GMM)")
    b = points.shape[0]
    fv = ops.fisher_vector(points, w, mu, sigma)                              # (B,G,20)
    net = fv.transpose(0, 1).reshape(g * b, 20)                                # voxel-major rows
    for l in (1, 2, 3):
        net = _inception(net, r, INCEPTION[l - 1], f"inception{l}", params)
    net = ops.pool3d(net, r, "max")
    r = (r + 1) // 2
    for l in (4, 5):
        net = _inception(net, r, INCEPTION[l - 1], f"inception{l}", params)
    net = ops.pool3d(net, r, "max")
    r = (r + 1) // 2
    net = net.reshape(r ** 3, b, -1).transpose(0, 1).reshape(b, -1)           # tf.reshape of (B, d, h, w, C)
    logits = ops.shared_mlp(net, params.mlp(["fc1", "fc2", "fc3", "fc4"], [True, True, True, False]))
    return logits, fv.transpose(1, 2).contiguous()


class MfvTrainer:
    """The five inception modules and two max pools of one (B, r) shape in training mode: forward(fv rows (r^3*B, 20)) -> the
    pooled (ceil(ceil(r/2)/2)^3 * B, 1536) rows, backward(dpooled) -> every conv3d variable's slice of the store's flat gradient.
    Buffers are allocated once."""

    def __init__(self, params: VariableStore, b: int, r: int, device):
        from .training import FlatParams
        self.lib = _lib.load()
        self.fp = params._flat if getattr(params, "_flat", None) is not None else FlatParams(params)
        params._flat = self.fp
        fp, self.b, self.r = self.fp, b, r
        f32 = dict(dtype=torch.float32, device=device)
        self.modules, cin, rr, ws_bwd = [], 20, r, 0
        for l, n in enumerate(INCEPTION, start=1):
            rows = b * rr ** 3
            m = dict(r=rr, rows=rows, cin=cin, n=n, H=torch.empty((rows, 3 * n), **f32), dH=torch.empty((rows, 3 * n), **f32),
                     P=torch.empty((rows, cin), **f32), convs=[])
            for j, (k, c, cout, off) in enumerate([(1, cin, n, 0), (KERNEL_SIZES[0], n, n // 2, n), (KERNEL_SIZES[1], n, n // 2, n + n // 2),
                                                   (1, cin, n, 2 * n)], start=1):
                sc = f"inception{l}_conv{j}"
                w = fp.views[f"{sc}/weights"]
                if tuple(w.shape) != (k, k, k, c, cout):
                    raise ValueError(f"{sc}/weights: shape {tuple(w.shape)}, want {(k, k, k, c, cout)}")
                m["convs"].append(dict(
                    scope=sc, k=k, c=c, cout=cout, off=off, W=w, bias=fp.views[f"{sc}/biases"], gamma=fp.views[f"{sc}/bn/gamma"],
                    beta=fp.views[f"{sc}/bn/beta"], mov_mean=params[f"{sc}/bn/moving_mean"], mov_var=params[f"{sc}/bn/moving_variance"],
                    dW=fp.gviews[f"{sc}/weights"], db=fp.gviews[f"{sc}/biases"], dgamma=fp.gviews[f"{sc}/bn/gamma"],
                    dbeta=fp.gviews[f"{sc}/bn/beta"], y=torch.empty((rows, cout), **f32), scale=torch.empty(cout, **f32),
                    shift=torch.empty(cout, **f32), mean_inv=torch.empty((2, cout), **f32), ca=torch.empty(cout, **f32),
                    cb=torch.empty(cout, **f32), cc=torch.empty(cout, **f32)))
                ws_bwd = max(ws_bwd, self.lib.psa_conv3d_bwd_workspace_bytes(b, rr, k, c, cout), self.lib.psa_bn_bwd_workspace_bytes(cout))
            m["dx4"] = torch.empty((rows, cin), **f32)                   # conv4's data gradient before the average pool's backward
            self.modules.append(m)
            cin = 3 * n
            if l in (3, 5):                                              # the max pools after inception3 and inception5
                ro = (rr + 1) // 2
                m["pooled"] = torch.empty((b * ro ** 3, cin), **f32)
                m["winner"] = torch.empty((b * ro ** 3, cin), dtype=torch.uint8, device=device)
                m["dpooled"] = torch.empty((b * ro ** 3, cin), **f32)
                rr = ro
        self.dy = torch.empty(b * r ** 3 * max(INCEPTION), **f32)
        self.ws_bwd_bytes = ws_bwd
        self.ws_bwd = torch.empty(ws_bwd // 4 + 64, **f32)
        self.ws_fwd_bytes, self.ws_fwd = 0, None
        self.names = [nm for nm in fp.names if nm.startswith("inception")]

    def _fwd_ws(self, need: int):
        """psa_conv3d_infer's workspace depends on the arithmetic mode of the call: grown on demand"""
        if need > self.ws_fwd_bytes:
            self.ws_fwd = torch.empty(need // 4 + 64, dtype=torch.float32, device=self.dy.device)
            self.ws_fwd_bytes = need
        return _p(self.ws_fwd), C.c_size_t(self.ws_fwd_bytes)

    def forward(self, fv_rows: torch.Tensor, decay: float) -> torch.Tensor:
        b, lib = self.b, self.lib
        x = fv_rows
        for m in self.modules:
            r, n = m["r"], m["n"]
            m["X"] = x
            check(lib.psa_pool3d(b, r, m["cin"], 0, _p(x), _p(m["P"]), _stream()), "pool3d")
            for j, cv in enumerate(m["convs"]):
                src, ld = (x, m["cin"]) if j == 0 else (m["H"], 3 * n) if j < 3 else (m["P"], m["cin"])
                self._conv_fwd(m, cv, src, ld, decay)
            x = m["H"]
            if "pooled" in m:
                check(lib.psa_pool3d_max_train(b, r, 3 * n, _p(x), _p(m["pooled"]), _p(m["winner"]), _stream()), "pool3d_max_train")
                x = m["pooled"]
        return x

    def _conv_fwd(self, m, cv, src, ld_src, decay):
        """one conv: y = src . W + bias, batch statistics -> scale / shift (moving averages updated), relu(y * scale + shift) -> its
        slice of the module output"""
        b, r, rows, n, lib = self.b, m["r"], m["rows"], m["n"], self.lib
        k, c, cout = cv["k"], cv["c"], cv["cout"]
        ws, wsn = self._fwd_ws(int(lib.psa_conv3d_workspace_bytes(b, r, k, c, cout)))
        check(lib.psa_conv3d_infer(b, r, k, c, cout, src.data_ptr(), ld_src, _p(cv["W"]), None, _p(cv["bias"]), 0, _p(cv["y"]), cout, ws, wsn,
                                   _stream()), "conv3d")
        check(lib.psa_bn_finalize_rows(rows, cout, _p(cv["y"]), _p(cv["gamma"]), _p(cv["beta"]), C.c_float(decay), _p(cv["mov_mean"]),
                                       _p(cv["mov_var"]), _p(cv["scale"]), _p(cv["shift"]), _p(cv["mean_inv"]), _stream()), "bn_finalize_rows")
        check(lib.psa_mfv_bn_relu(rows, cout, _p(cv["y"]), _p(cv["scale"]), _p(cv["shift"]), m["H"][:, cv["off"]:].data_ptr(), 3 * n, _stream()),
              "mfv_bn_relu")

    def _conv_bwd(self, m, cv, src, ld_src, dx, ld_dx, accumulate):
        """one conv: batch-norm sums and coefficients from its slice of dH, dy, dW, db = 0, and dx (+)= dy . W^T when dx is given"""
        b, r, rows, lib = self.b, m["r"], m["rows"], self.lib
        k, c, cout = cv["k"], cv["c"], cv["cout"]
        wsb, wsn = _p(self.ws_bwd), C.c_size_t(self.ws_bwd_bytes)
        g = PsaGradIn(y=_p(cv["y"]), ld=cout, s=_p(cv["scale"]), t=_p(cv["shift"]), relu=1, ca=_p(cv["ca"]), cb=_p(cv["cb"]), cc=_p(cv["cc"]),
                      dh=m["dH"][:, cv["off"]:].data_ptr(), ld_dh=3 * m["n"], pool_k=1, C=cout)
        check(lib.psa_bn_bwd_coeffs(rows, cout, C.byref(g), _p(cv["gamma"]), _p(cv["mean_inv"]), _p(cv["dgamma"]), _p(cv["dbeta"]), _p(cv["ca"]),
                                    _p(cv["cb"]), _p(cv["cc"]), wsb, wsn, _stream()), "bn_bwd_coeffs")
        cv["db"].zero_()                                                # sum_rows dy = 0 under batch norm
        dy = self.dy[:rows * cout]
        check(lib.psa_mfv_bn_dy(rows, cout, C.byref(g), _p(dy), _stream()), "mfv_bn_dy")
        check(lib.psa_conv3d_bwd_weight(b, r, k, c, cout, src.data_ptr(), ld_src, _p(dy), _p(cv["dW"]), wsb, wsn, _stream()), "conv3d_bwd_weight")
        if dx is not None:
            check(lib.psa_conv3d_bwd_data(b, r, k, c, cout, _p(dy), _p(cv["W"]), dx.data_ptr(), ld_dx, int(accumulate), wsb, wsn, _stream()),
                  "conv3d_bwd_data")

    def backward(self, dpooled: torch.Tensor):
        """dpooled = the gradient of forward()'s return value -> the conv3d variables' gradients in the flat bucket's views"""
        b, lib = self.b, self.lib
        dout = dpooled.contiguous()
        for l in range(len(self.modules) - 1, -1, -1):
            m = self.modules[l]
            r, n, cin = m["r"], m["n"], m["cin"]
            if "pooled" in m:                                          # the max pool after this module: gradient to the winners
                check(lib.psa_pool3d_bwd(b, r, 3 * n, 1, _p(dout), _p(m["winner"]), _p(m["dH"]), _stream()), "pool3d_bwd")
            # the gradient of the module input: the previous module's dH, or the pooled rows' gradient after a max pool; none for inception1
            dX = None if l == 0 else self.modules[l - 1]["dpooled" if "pooled" in self.modules[l - 1] else "dH"]
            c1, c2, c3, c4 = m["convs"]
            H1 = m["H"]
            self._conv_bwd(m, c2, H1, 3 * n, m["dH"], 3 * n, True)    # conv1's slice: dh + dx(conv2) + dx(conv3)
            self._conv_bwd(m, c3, H1, 3 * n, m["dH"], 3 * n, True)
            self._conv_bwd(m, c4, m["P"], cin, None if dX is None else m["dx4"], cin, False)
            if dX is not None:
                check(lib.psa_pool3d_bwd(b, r, cin, 0, _p(m["dx4"]), None, _p(dX), _stream()), "pool3d_bwd")
            self._conv_bwd(m, c1, m["X"], cin, dX, cin, True)          # module input: avg-pool backward of conv4's + conv1's
            dout = dX

    def flat_grad(self) -> torch.Tensor:
        """a gradient bucket holding the conv3d variables' gradients and zeros elsewhere"""
        g = torch.zeros_like(self.fp.grad)
        base = self.fp.grad.data_ptr()
        for nm in self.names:
            v = self.fp.gviews[nm]
            o = (v.data_ptr() - base) // 4
            g[o:o + v.numel()].copy_(v.reshape(-1))
        return g


class _MfvFn(torch.autograd.Function):
    """MfvTrainer as one autograd node over the store's flat parameter vector"""

    @staticmethod
    def forward(ctx, flat, fv_rows, trainer, decay):
        ctx.trainer = trainer
        return trainer.forward(fv_rows, decay).clone()

    @staticmethod
    def backward(ctx, dpooled):
        tr = ctx.trainer
        tr.backward(dpooled)
        return tr.flat_grad(), None, None, None


def get_model_training(points, w, mu, sigma, bn_decay=None, weigth_decay=0.005, num_classes=NUM_CLASSES, *, params: VariableStore,
                       add_noise=False, dropout: bool = True, return_end_points: bool = False):
    """3dmfv_net_cls.get_model with is_training=True: -> (logits (B,num_classes), fv (B,20,G)), the logits differentiable in the
    store's variables (autograd over its flat parameter vector, training.FlatParams).  Every conv3d and fc1-fc3 use batch statistics
    (biased variance, eps 1e-3) and update their moving averages with bn_decay (0.9 for None); dropout keeps 0.7 after fc1, fc2
    and fc3 (dropout=False: the identity).  weigth_decay is accepted and ignored: in the reference it only feeds the `losses`
    collection, which get_loss never reads (and train.py passes 0.0).  With return_end_points a third value, a dict holding each
    conv's pre-batch-norm ``<scope>/y`` (r^3*B, C_out, voxel-major rows), ``<scope>/scale`` and ``<scope>/shift`` and each max pool's
    ``pool1/winner`` / ``pool2/winner`` (uint8, psa_pool3d_max_train); they are the trainer's buffers, overwritten by the next call.
    Gradients with respect to the points and add_noise are not implemented."""
    from .training import DEFAULT_BN_DECAY, _cached, mlp_training
    if isinstance(points, torch.Tensor) and points.requires_grad:
        raise NotImplementedError("mfv_net_cls: gradients with respect to the input points are not implemented")
    if add_noise:
        raise NotImplementedError("mfv_net_cls: the add_noise augmentation is not implemented")
    if params["fc4/biases"].numel() != num_classes:
        raise ValueError(f"num_classes={num_classes} but the store's fc4 has {params['fc4/biases'].numel()} outputs")
    g = len(w)
    r = int(round(g ** (1.0 / 3.0)))
    if r ** 3 != g:
        raise ValueError(f"mfv_net_cls: G = {g} Gaussians is not a cube r^3 (the model needs a grid GMM)")
    points = ops._dev(points, torch.float32, "points", 3)
    w, mu, sigma = (torch.as_tensor(t, dtype=torch.float32, device=points.device) for t in (w, mu, sigma))
    b = points.shape[0]
    fv = ops.fisher_vector(points, w, mu, sigma)                              # (B,G,20)
    rows = fv.transpose(0, 1).reshape(g * b, 20).contiguous()                  # voxel-major rows
    tr = _cached(params, ("mfv_net", b, r), lambda: MfvTrainer(params, b, r, points.device))
    decay = DEFAULT_BN_DECAY if bn_decay is None else float(bn_decay)
    net = _MfvFn.apply(tr.fp.flat.requires_grad_(True), rows, tr, decay)
    net = net.reshape(-1, b, net.shape[-1]).transpose(0, 1).reshape(b, -1)      # tf.reshape of (B, d, h, w, C)
    drop = (lambda v: torch.nn.functional.dropout(v, 0.3, training=True)) if dropout else (lambda v: v)
    for scope in ("fc1", "fc2", "fc3"):
        net = drop(mlp_training(net, [(scope, True)], bn_decay, params))
    logits = mlp_training(net, [("fc4", False)], bn_decay, params)
    fv = fv.transpose(1, 2).contiguous()
    if not return_end_points:
        return logits, fv
    ep = {}
    for m in tr.modules:
        for cv in m["convs"]:
            ep.update({f"{cv['scope']}/y": cv["y"], f"{cv['scope']}/scale": cv["scale"], f"{cv['scope']}/shift": cv["shift"]})
    ep["pool1/winner"], ep["pool2/winner"] = tr.modules[2]["winner"], tr.modules[4]["winner"]
    return logits, fv, ep


def get_loss(pred, label):
    """Mean sparse softmax cross-entropy (3dmfv_net_cls.py:106-115)."""
    return torch.nn.functional.cross_entropy(pred, label.long())
