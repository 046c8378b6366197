"""PointCNN training without a GPU: get_model_training's refusals, the new C entries' argument checks, the code shape of the training
kernels (no float atomics, no stack frame or spills), and the GPU tests' float64 restatement against oracle/pointcnn_oracle.py (batch
norm frozen, mean over the points) and against an independent F.batch_norm / F.elu / grouped F.conv2d composition of one layer."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import pointcnn_oracle as po
from scanobjectnn_b200 import pointcnn_cls as M
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import BN_EPS

from .restate import params_as
from .test_pointcnn_train_gpu import pointcnn_training, xconv

KERNELS = ("xconv_stage0_kernel", "xconv_stage1_kernel", "xconv_stage2_kernel", "xconv_bwd_top_kernel", "xconv_dw_bwd_kernel",
           "elu_bn_dy_kernel", "bn_affine_rows_kernel")


def test_get_model_training_refuses_what_it_cannot_run():
    p = M.init_params(device="cpu")
    with pytest.raises(RuntimeError, match="CUDA"):
        M.get_model_training(torch.zeros((1, 512, 3)), params=p)
    with pytest.raises(NotImplementedError):
        M.get_model_training(torch.zeros((1, 512, 3), requires_grad=True), params=p)
    with pytest.raises(ValueError, match="384"):
        M.get_model_training(torch.zeros((1, 300, 3)), params=p)
    with pytest.raises(ValueError, match="num_class"):
        M.get_model_training(torch.zeros((1, 512, 3)), num_class=40, params=p)
    with pytest.raises(NotImplementedError, match="get_model_training"):
        M.get_model(torch.zeros((1, 512, 3)), True, params=p)


def test_training_entries_reject_bad_arguments_without_a_gpu():
    from scanobjectnn_b200 import _lib, ops
    lib = _lib.load()
    null = C.c_void_p(0)
    xc = _lib.PsaXconv(8, 24, 0, 4)
    sv = _lib.PsaXconvSaved()
    assert lib.psa_xconv_train_stage(3, 1, 64, 64, null, null, null, C.byref(xc), C.byref(sv), null) == -1       # stage not 0-2
    assert lib.psa_xconv_train_stage(0, 1, 64, 64, null, null, null, C.byref(xc), C.byref(sv), null) == -1       # null buffers
    assert b"null buffer" in lib.psa_last_error()
    assert lib.psa_xconv_train_stage(0, 0, 64, 64, null, null, null, C.byref(xc), C.byref(sv), null) == 0        # b = 0: a no-op
    bad = _lib.PsaXconv(17, 24, 0, 4)
    assert lib.psa_xconv_train_stage(0, 1, 64, 64, null, null, null, C.byref(bad), C.byref(sv), null) == -1      # K > 16
    assert lib.psa_xconv_train_bwd_top(1, 64, 64, null, null, C.byref(xc), C.byref(sv), null, null, null, null, null, null, 0, null) == -1
    assert lib.psa_xconv_train_bwd_top(1, 64, 64, null, null, C.byref(_lib.PsaXconv(8, 24, 48, 4)), C.byref(sv), null, null, null, null, null,
                                       null, 0, null) == -1                                                       # c_prev > 0 without fts
    assert lib.psa_xconv_train_bwd_workspace_bytes(32, 1024, 8, 24, 0, 4) > 0
    assert lib.psa_xconv_train_bwd_workspace_bytes(32, 1024, 17, 24, 0, 4) == 0
    g = _lib.PsaGradIn(pool_k=1, C=64)
    assert lib.psa_xconv_depthwise_bwd(10, 8, null, null, null, C.byref(g), 1, null, null, null, null, 0, null) == -1
    assert lib.psa_xconv_depthwise_bwd(10, 0, null, null, null, C.byref(g), 1, null, null, null, null, 0, null) == -1
    assert lib.psa_xconv_depthwise_bwd(0, 8, null, null, null, C.byref(g), 1, null, null, null, null, 0, null) == 0
    assert lib.psa_elu_bn_dy(10, 8, C.byref(g), null, null) == -1
    assert lib.psa_elu_bn_dy(0, 8, C.byref(g), null, null) == 0
    assert lib.psa_bn_affine_rows(10, 8, null, null, null, null, 4, null) == -1                  # ldo below the width
    assert lib.psa_bn_affine_rows(10, 8, null, null, null, null, 8, null) == -1
    assert lib.psa_bn_affine_rows(0, 8, null, null, null, null, 8, null) == 0
    z = torch.zeros((4, 64))
    v = torch.zeros(64)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.elu_bn_dy(z, z, v, v, v)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.bn_affine_rows(z, v, v)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.xconv_depthwise_bwd(z, v, v, z, z, v, v, v, torch.zeros((1, 8, 8, 8)), True)


def _sass_functions(lib):
    sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if any(k in m.group(1) for k in KERNELS) else None
            if name:
                funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    return funcs


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_training_kernels_have_no_float_atomics():
    from scanobjectnn_b200.build import build_library
    funcs = _sass_functions(build_library())
    assert all(any(k in f for f in funcs) for k in KERNELS), sorted(funcs)
    for f, lines in funcs.items():
        bad = [ln for ln in lines if re.search(r"\b(RED|ATOM|ATOMG|ATOMS)\b", ln)]
        assert not bad, (f, bad[:3])


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="nvcc not found")
def test_training_kernels_do_not_spill():
    from scanobjectnn_b200.build import CSRC, NVCC_FLAGS, _nvcc
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([_nvcc(), *NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(CSRC, "pointcnn_train.cu"), "-o", os.path.join(d, "p.o")],
                           capture_output=True, text=True, check=True)
    seen, name = set(), None
    for line in r.stderr.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            name = m.group(1) if any(k in m.group(1) for k in KERNELS) else None
            continue
        if name is not None and "stack frame" in line:
            seen.add(name)
            assert re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", line), (name, line)
            name = None
    assert all(any(k in f for f in seen) for k in KERNELS), sorted(seen)


def test_restatement_with_frozen_batch_norm_matches_the_oracle():
    """the GPU tests' float64 restatement, batch norm on the moving averages and the mean over the points, against
    oracle/pointcnn_oracle.py at B=2, N=512"""
    p = M.init_params(seed=3, device="cpu", randomize_bn=True)
    pts = make_clouds("ball", 2, 512, seed=33)
    idx, q = [], pts
    for _, k, d, P, *_ in M.layer_table():
        P = pts.shape[1] if P == -1 else P
        idx.append(po.knn_dilated(q, q[:, :P], k, d))
        q = q[:, :P]
    want = po.forward(p, pts, idx)["logits"]
    got = pointcnn_training(torch.from_numpy(pts).double(), params_as(p, torch.float64), [torch.from_numpy(i) for i in idx], frozen=True,
                            mean=True)
    assert float(np.abs(got.numpy() - want).max()) < 1e-10 * max(1.0, float(np.abs(want).max()))


def _composition(P, tag, pts, qrs, idx, fts, K, dm):
    """one X-Conv layer (no global branch) from F.conv2d / F.batch_norm(training=True) / F.elu in NCHW: X_0 as the (1, K) VALID
    conv, X_1 / X_2 as depthwise convs (groups = K), the separable conv's depthwise stage with groups = C_in"""
    B, Pq = idx.shape[:2]
    bi = torch.arange(B)[:, None, None]
    nchw = lambda x: x.permute(0, 3, 1, 2)                                    # (B, P, K, C) -> (B, C, P, K)  # noqa: E731
    bnl = lambda x, layer: F.batch_norm(x, None, None, P[f"{layer}_bn/gamma"], P[f"{layer}_bn/beta"], training=True, momentum=0.01,  # noqa: E731
                                        eps=BN_EPS)
    conv1 = lambda x, w: F.conv2d(x, w.reshape(-1, w.shape[-1]).t()[:, :, None, None])   # noqa: E731
    local = nchw(pts[bi, idx] - qrs[:, :, None, :])
    h = bnl(F.elu(conv1(local, P[f"{tag}nn_fts_from_pts_0/kernel"])), f"{tag}nn_fts_from_pts_0")
    h = bnl(F.elu(conv1(h, P[f"{tag}nn_fts_from_pts/kernel"])), f"{tag}nn_fts_from_pts")
    Fm = h if fts is None else torch.cat([h, nchw(fts[bi, idx])], dim=1)                 # (B, C_in, P, K)
    w0 = P[f"{tag}X_0/kernel"]                                                           # (1, K, 3, K*K) HWIO
    X = bnl(F.elu(F.conv2d(local, w0.permute(3, 2, 0, 1))), f"{tag}X_0")                 # (B, K*K, P, 1)
    X = X.reshape(B, K, K, Pq).permute(0, 3, 1, 2)                                       # (B, P, K, K)
    for name, act in (("X_1", True), ("X_2", False)):
        w = P[f"{tag}{name}/depthwise_weights"]                                          # (1, K, K, K) = (1, width, channel, mult)
        y = F.conv2d(X.permute(0, 3, 1, 2), w.permute(2, 3, 0, 1).reshape(K * K, 1, 1, K), groups=K)     # (B, K*K, P, 1)
        y = bnl(F.elu(y) if act else y, f"{tag}{name}")
        X = y.reshape(B, K, K, Pq).permute(0, 3, 1, 2)
    fts_X = X @ Fm.permute(0, 2, 3, 1)                                                   # (B, P, K, C_in)
    wdw = P[f"{tag}fts_conv/depthwise_kernel"]                                           # (1, K, C_in, dm)
    cin = wdw.shape[2]
    dw = F.conv2d(nchw(fts_X), wdw.permute(2, 3, 0, 1).reshape(cin * dm, 1, 1, K), groups=cin)          # (B, C_in*dm, P, 1)
    out = bnl(F.elu(conv1(dw, P[f"{tag}fts_conv/pointwise_kernel"])), f"{tag}fts_conv")
    return out[..., 0].permute(0, 2, 1)


def test_restatement_matches_a_batch_norm_composition():
    """batch statistics forward and autograd of one X-Conv layer (layer 2's shape, B=2, N=512) against F.batch_norm(training=True),
    F.elu and grouped F.conv2d, to 1e-10"""
    p = M.init_params(seed=4, device="cpu", randomize_bn=True)
    tag, k, d, P, c, c_pts, c_prev, dm, _ = M.layer_table()[1]
    rng = np.random.default_rng(5)
    pts = torch.from_numpy(make_clouds("ball", 2, 512, seed=44)).double()
    qrs = pts[:, :P]
    idx = torch.from_numpy(po.knn_dilated(pts.numpy().astype(np.float32), qrs.numpy().astype(np.float32), k, d)).long()
    fts = torch.from_numpy(rng.standard_normal((2, 512, c_prev))).requires_grad_(True)
    res = []
    for f in (lambda Q: xconv(Q, tag, pts, qrs, idx, fts, k, 0, False), lambda Q: _composition(Q, tag, pts, qrs, idx, fts, k, dm)):
        Q = params_as(p, torch.float64, grad=True)
        names = [n for n in Q if n.startswith(tag) and not n.endswith(("moving_mean", "moving_variance"))]
        out = f(Q)
        R = torch.from_numpy(np.random.default_rng(6).standard_normal(out.shape))
        res.append((out.detach(), torch.autograd.grad((out * R).sum(), [Q[n] for n in names] + [fts])))
    (o1, g1), (o2, g2) = res
    assert float((o1 - o2).abs().max()) < 1e-10 * max(1.0, float(o2.abs().max()))
    for a, b in zip(g1, g2):
        assert float((a - b).abs().max()) < 1e-10 * max(1.0, float(b.abs().max()))
