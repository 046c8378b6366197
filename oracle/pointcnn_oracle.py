"""float64 numpy restatement of PointCNN's classifier (PointCNN/pointcnn.py:10-152, pointcnn_cls.py:10-17, pointfly.py:298-347) with
the setting pointcnn_cls/modelnet_x3_l4.py, inference mode, in the reference's own order: the gathered (B,P,K,3) local coordinates,
the lifting dense layers, the (1,K) conv X_0 reshaped to (K,K), the depthwise convs X_1 / X_2 (output channel b*K + m = input
channel b times multiplier m), fts_X = X . F as a batched matmul, the separable conv, the global branch concatenated in front, fc0 /
fc1, the mean over the points and the logits.  Every layer with batch norm is BN(elu(x . W)), BN with the moving statistics and
eps 1e-3.  Everything is materialised.

The kNN indices are an input (the run's own), so the restatement checks the arithmetic; ``knn_dilated`` is the fp32 kNN of
oracle/pointcnn_knn.c:orc_knn_dilated, compiled on first use into a temporary directory.

TEST INFRASTRUCTURE ONLY.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import shutil
import subprocess
import tempfile

import numpy as np

BN_EPS = 1e-3
XCONV = ((8, 1, -1, 48), (12, 2, 384, 96), (16, 2, 128, 192), (16, 3, 128, 384))     # (K, D, P, C), x = 3
FC = (384, 192)


_knn_lib = None


def _knn():
    """oracle/pointcnn_knn.c built with the flags of oracle/Makefile's liboracle.so (-ffp-contract=off: only the written fmaf() fuse)"""
    global _knn_lib
    if _knn_lib is None:
        src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pointcnn_knn.c")
        so = os.path.join(tempfile.mkdtemp(prefix="pointcnn_knn_"), "libpointcnn_knn.so")
        cc = shutil.which("gcc") or shutil.which("cc")
        if cc is None:
            raise RuntimeError("pointcnn_oracle: no C compiler for oracle/pointcnn_knn.c")
        subprocess.run([cc, "-O2", "-std=c11", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fvisibility=hidden", "-o", so, src,
                        "-lm"], check=True)
        _knn_lib = C.CDLL(so)
    return _knn_lib


def knn_dilated(points, queries, k, d):
    """orc_knn_dilated: points (b,n,3), queries (b,m,3) float32 -> (b,m,k) int32"""
    points = np.ascontiguousarray(points, np.float32)
    queries = np.ascontiguousarray(queries, np.float32)
    b, n, _ = points.shape
    m = queries.shape[1]
    idx = np.empty((b, m, k), np.int32)
    _knn().orc_knn_dilated(b, n, m, k, d, points.ctypes.data_as(C.c_void_p), queries.ctypes.data_as(C.c_void_p),
                               idx.ctypes.data_as(C.c_void_p))
    return idx


def _v(p, name):
    t = p[name]
    return np.asarray(t.detach().cpu().numpy() if hasattr(t, "detach") else t, np.float64)


def elu(x):
    """tf.nn.elu: x if x > 0 else expm1(x)"""
    return np.where(x > 0, x, np.expm1(np.minimum(x, 0.0)))


def bn(p, layer, x):
    """tf.layers.batch_normalization(training=False) over the last axis: (x - mean) * gamma / sqrt(var + eps) + beta"""
    g, b = _v(p, f"{layer}_bn/gamma"), _v(p, f"{layer}_bn/beta")
    mu, var = _v(p, f"{layer}_bn/moving_mean"), _v(p, f"{layer}_bn/moving_variance")
    return (x - mu) * (g / np.sqrt(var + BN_EPS)) + b


def dense(p, layer, x, var="kernel"):
    """pf.dense / pf.conv2d (1x1) with with_bn=True: BN(elu(x . W)), no bias (pointfly.py:339-347)"""
    w = _v(p, f"{layer}/{var}")
    return bn(p, layer, elu(x @ w.reshape(-1, w.shape[-1])))


def layer_table():
    """(tag, K, D, P, C, C_pts_fts, C_prev, dm, global width) per layer (pointcnn.py:104-112)"""
    out = []
    for i, (k, d, p, c) in enumerate(XCONV):
        c_prev = 0 if i == 0 else XCONV[i - 1][3]
        c_pts = c // 2 if i == 0 else c_prev // 4
        dm = 4 if i == 0 else math.ceil(c / c_prev)
        out.append((f"xconv_{i + 1}_", k, d, p, c, c_pts, c_prev, dm, c // 4 if i == len(XCONV) - 1 else 0))
    return out


def xconv(p, tag, pts, qrs, idx, fts, K, dm, glob):
    """pointcnn.py:10-52 on pts (B,n,3), qrs (B,P,3), the dilated indices idx (B,P,K) and fts (B,n,C_prev) or None -> dict with the
    depthwise output ``dw`` (B*P, C_in*dm) and the layer output ``out`` (B,P,glob + C)"""
    pts, qrs = np.asarray(pts, np.float64), np.asarray(qrs, np.float64)
    B, P = idx.shape[:2]
    bi = np.arange(B)[:, None, None]
    nn_pts = pts[bi, idx]                                                   # gather_nd (:16)
    local = nn_pts - qrs[:, :, None, :]                                     # (:18)
    lifted = dense(p, f"{tag}nn_fts_from_pts", dense(p, f"{tag}nn_fts_from_pts_0", local))     # (:21-22)
    F = lifted if fts is None else np.concatenate([lifted, np.asarray(fts, np.float64)[bi, idx]], axis=-1)   # (:23-27)
    w0 = _v(p, f"{tag}X_0/kernel")[0]                                       # (K, 3, K*K): the (1,K) VALID conv (:33)
    X0 = bn(p, f"{tag}X_0", elu(np.einsum("bpjd,jdo->bpo", local, w0)))
    X0_KK = X0.reshape(B, P, K, K)                                          # (:34)
    w1 = _v(p, f"{tag}X_1/depthwise_weights")[0]                            # (K, K, K) = (width a, channel b, multiplier m)
    X1 = bn(p, f"{tag}X_1", elu(np.einsum("pqab,abm->pqbm", X0_KK, w1).reshape(B, P, K * K)))     # (:35)
    X1_KK = X1.reshape(B, P, K, K)
    w2 = _v(p, f"{tag}X_2/depthwise_weights")[0]
    X2 = bn(p, f"{tag}X_2", np.einsum("pqab,abm->pqbm", X1_KK, w2).reshape(B, P, K * K))         # activation=None (:37)
    X2_KK = X2.reshape(B, P, K, K)
    fts_X = X2_KK @ F                                                       # tf.matmul (:39)
    wdw = _v(p, f"{tag}fts_conv/depthwise_kernel")[0]                       # (K, C_in, dm)
    dw = np.einsum("pqic,icm->pqcm", fts_X, wdw).reshape(B, P, -1)          # separable conv, depthwise stage (:44)
    conv = dense(p, f"{tag}fts_conv", dw, var="pointwise_kernel")          # pointwise, ELU, BN
    if glob:
        g = dense(p, f"{tag}fts_global", dense(p, f"{tag}fts_global_0", qrs))   # (:47-49)
        conv = np.concatenate([g, conv], axis=-1)                           # (:50)
    return {"dw": dw.reshape(B * P, -1), "out": conv}


def forward(p, points, idx_list):
    """The classifier on points (B,N,3) with the per-layer indices idx_list[l] (B,P_l,K_l) -> dict with ``out<l>``, ``dw<l>``
    (l = 1..4), ``fc0``, ``fc1``, ``fc_mean`` and ``logits`` (B,1,num_class)"""
    pts = np.asarray(points, np.float64)
    n = pts.shape[1]
    fts, res = None, {}
    for l, ((tag, k, _, P, _, _, _, dm, glob), idx) in enumerate(zip(layer_table(), idx_list), start=1):
        P = n if P == -1 else P
        qrs = pts[:, :P]                                                    # tf.slice (:101); the previous points when P repeats
        r = xconv(p, tag, pts, qrs, np.asarray(idx), fts, k, dm, glob)
        res[f"dw{l}"], res[f"out{l}"] = r["dw"], r["out"]
        pts, fts = qrs, r["out"]
    net = fts
    for i in range(len(FC)):
        net = dense(p, f"fc{i}", net)                                       # dropout: identity at inference
        res[f"fc{i}"] = net
    mean = net.mean(axis=1, keepdims=True)                                  # fc_mean (pointcnn_cls.py:13-14)
    res["fc_mean"] = mean[:, 0]
    res["logits"] = mean @ _v(p, "logits/kernel") + _v(p, "logits/bias")    # with_bn=False, activation=None
    return res
