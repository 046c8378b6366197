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
the returned ``fv`` and the flatten before fc1 are the reference's.  Training mode is not implemented.
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops
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
        raise NotImplementedError("mfv_net_cls: training mode is not implemented (inference only)")
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


def get_loss(pred, label):
    """Mean sparse softmax cross-entropy (3dmfv_net_cls.py:106-115)."""
    return torch.nn.functional.cross_entropy(pred, label.long())
