"""float64 restatement of 3DmFV-Net's classifier (3DmFV-Net/models/3dmfv_net_cls.py:29-102, utils/tf_util.py:254-311, 406-429,
458-495, 578-652) in inference mode.

* fisher_vector: get_3dmfv(flatten=False) (tf_util.py:578-652) with numpy broadcasting over (B,N,G,3) in the reference's order --
  densities w N(x | mu, diag(sigma^2)), their ratio over the Gaussians, the max / min / sum statistics, the power and the L2
  normalisation over the Gaussian axis (tf.nn.l2_normalize, epsilon 1e-12) -- returned as (B,G,20), before the transpose.
* conv3d / pools: torch.nn.functional in float64 on (B,C,D,H,W) grids: conv3d with padding k // 2 (TF's SAME at stride 1),
  avg_pool3d(3, 1, 1, count_include_pad=False) (TF divides by the in-grid count) and max_pool3d(2, 2, ceil_mode=True) (TF's SAME
  pads the far end only).  tests/test_mfv_cpu.py checks both pools against loops with TF's padding.
* batch norm folded from the moving averages with eps 1e-3 (batch_norm_template, tf_util.py:458-495), and the FC head.

forward_from_fv runs the network on a given Fisher vector (the run's own, as the GPU tests do with kNN indices).  The network runs in
float64 on the device of its input: CPU tensors, or CUDA tensors where a test's shapes would take minutes on the CPU."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

BN_EPS = 1e-3
INCEPTION = (64, 128, 256, 256, 512)


def _d(t, device="cpu"):
    return torch.as_tensor(t).to(device=device, dtype=torch.float64)


def fisher_vector(points, w, mu, sigma):
    """tf_util.py:578-652 (flatten=False) -> (B,G,20) float64 numpy, columns [d_pi max, sum | d_mu max, min, sum | d_sigma ...]"""
    x = np.asarray(points, np.float64)[:, :, None, :]                      # (B,N,1,3)
    w = np.asarray(w, np.float64)
    mu = np.asarray(mu, np.float64)[None, None]                            # (1,1,G,3)
    sg = np.asarray(sigma, np.float64)[None, None]
    n = x.shape[1]
    z = (x - mu) / sg                                                      # (B,N,G,3)
    p = np.exp(-0.5 * (z ** 2).sum(-1)) / ((2 * np.pi) ** 1.5 * sg.prod(-1))   # MultivariateNormalDiag.prob
    wp = p * w
    q = wp / wp.sum(-1, keepdims=True)                                     # (B,N,G)
    d_pi_all = ((q - w) / (np.sqrt(w) * n))[..., None]
    d_pi = np.concatenate([d_pi_all.max(1), d_pi_all.sum(1)], axis=2)
    d_mu_all = q[..., None] * z
    d_mu = (1 / (n * np.sqrt(w)))[None, :, None] * np.concatenate([d_mu_all.max(1), d_mu_all.min(1), d_mu_all.sum(1)], axis=2)
    d_sig_all = q[..., None] * (z ** 2 - 1)
    d_sig = (1 / (n * np.sqrt(2 * w)))[None, :, None] * np.concatenate([d_sig_all.max(1), d_sig_all.min(1), d_sig_all.sum(1)], axis=2)
    out = []
    for v in (d_pi, d_mu, d_sig):
        v = np.sign(v) * np.abs(v) ** 0.5
        out.append(v / np.sqrt(np.maximum((v ** 2).sum(1, keepdims=True), 1e-12)))
    return np.concatenate(out, axis=2)


def _folded(p, scope, device):
    """(W, scale, shift) with the bias and batch norm folded: y = (x . W) * scale + shift"""
    v = lambda name: _d(p[f"{scope}/{name}"], device)
    if f"{scope}/bn/gamma" not in p:
        return v("weights"), None, v("biases")
    inv = v("bn/gamma") / torch.sqrt(v("bn/moving_variance") + BN_EPS)
    return v("weights"), inv, (v("biases") - v("bn/moving_mean")) * inv + v("bn/beta")


def conv3d(x, p, scope, relu=True):
    """tf_util.conv3d (SAME, stride 1, bias, inference batch norm, ReLU) on x (B,C,D,H,W)"""
    w, sc, sh = _folded(p, scope, x.device)
    k = w.shape[0]
    y = F.conv3d(x, w.permute(4, 3, 0, 1, 2), padding=k // 2)
    y = y * sc[None, :, None, None, None] + sh[None, :, None, None, None] if sc is not None else y + sh[None, :, None, None, None]
    return torch.relu(y) if relu else y


def avg_pool3(x):
    return F.avg_pool3d(x, 3, stride=1, padding=1, count_include_pad=False)


def max_pool2(x):
    return F.max_pool3d(x, 2, stride=2, ceil_mode=True)


def inception(x, p, scope):
    one = conv3d(x, p, f"{scope}_conv1")
    return torch.cat([one, conv3d(one, p, f"{scope}_conv2"), conv3d(one, p, f"{scope}_conv3"), conv3d(avg_pool3(x), p, f"{scope}_conv4")], 1)


def fc(x, p, scope, relu=True):
    w, sc, sh = _folded(p, scope, x.device)
    y = x @ w
    y = y * sc + sh if sc is not None else y + sh
    return torch.relu(y) if relu else y


def grid_of(fv):
    """(B,G,20) -> the reference's grid_fisher as (B,20,r,r,r): reshape of the (B,20,G) fv, channels first for torch"""
    fv = _d(fv, fv.device if isinstance(fv, torch.Tensor) else "cpu")
    b, g, _ = fv.shape
    r = int(round(g ** (1 / 3)))
    return fv.permute(0, 2, 1).reshape(b, 20, r, r, r)


def forward_from_fv(fv, p):
    """-> (logits (B,num_classes), flattened (B, 8 * 1536) input of fc1), float64"""
    net = grid_of(fv)
    for l in (1, 2, 3):
        net = inception(net, p, f"inception{l}")
    net = max_pool2(net)
    for l in (4, 5):
        net = inception(net, p, f"inception{l}")
    net = max_pool2(net)
    flat = net.permute(0, 2, 3, 4, 1).reshape(net.shape[0], -1)          # tf.reshape of (B,d,h,w,C)
    h = fc(flat, p, "fc1")
    h = fc(h, p, "fc2")
    h = fc(h, p, "fc3")
    return fc(h, p, "fc4", relu=False), flat
