"""PointCNN without a GPU: the reference's variable names and TF shapes and a TF checkpoint round trip, the float64 restatement
(oracle/pointcnn_oracle.py) against an independent float64 torch composition (F.conv2d with groups, F.elu, F.batch_norm), the C kNN
oracle against DGCNN's, the refusals that need no device, the C ABI's argument checks, and the new kernels' spills and atomics (the
dense kernel's code shape: test_sass_ring.py)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import oracle as orc
from oracle import pointcnn_oracle as po
from scanobjectnn_b200 import checkpoint as ck
from scanobjectnn_b200 import ops
from scanobjectnn_b200 import pointcnn_cls as M
from scanobjectnn_b200.synthetic import make_clouds

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "scanobjectnn_b200", "libpsa.so")


def _reference_shapes(num_class=15):
    """written out from pointcnn.py / modelnet_x3_l4.py: (K, C_pts_fts, C_in, dm, C) per layer"""
    want = {}
    layers = {1: (8, 24, 24, 4, 48), 2: (12, 12, 60, 2, 96), 3: (16, 24, 120, 2, 192), 4: (16, 48, 240, 2, 384)}

    def bn(layer, c):
        for v in ("gamma", "beta", "moving_mean", "moving_variance"):
            want[f"{layer}_bn/{v}"] = (c,)

    for l, (k, cp, cin, dm, c) in layers.items():
        t = f"xconv_{l}_"
        want[f"{t}nn_fts_from_pts_0/kernel"] = (3, cp); bn(f"{t}nn_fts_from_pts_0", cp)
        want[f"{t}nn_fts_from_pts/kernel"] = (cp, cp); bn(f"{t}nn_fts_from_pts", cp)
        want[f"{t}X_0/kernel"] = (1, k, 3, k * k); bn(f"{t}X_0", k * k)
        want[f"{t}X_1/depthwise_weights"] = (1, k, k, k); bn(f"{t}X_1", k * k)
        want[f"{t}X_2/depthwise_weights"] = (1, k, k, k); bn(f"{t}X_2", k * k)
        want[f"{t}fts_conv/depthwise_kernel"] = (1, k, cin, dm)
        want[f"{t}fts_conv/pointwise_kernel"] = (1, 1, cin * dm, c); bn(f"{t}fts_conv", c)
    want["xconv_4_fts_global_0/kernel"] = (3, 96); bn("xconv_4_fts_global_0", 96)
    want["xconv_4_fts_global/kernel"] = (96, 96); bn("xconv_4_fts_global", 96)
    want["fc0/kernel"] = (480, 384); bn("fc0", 384)
    want["fc1/kernel"] = (384, 192); bn("fc1", 192)
    want["logits/kernel"] = (192, num_class)
    want["logits/bias"] = (num_class,)
    return want


def test_init_params_has_the_reference_variables():
    p = M.init_params(device="cpu")
    assert {k: tuple(v.shape) for k, v in p.items()} == _reference_shapes()
    # Glorot normal truncated at two standard deviations, TF's fans: X_0 (1,16,3,256) of layer 4 has fans 48 and 4096
    std = np.sqrt(2.0 / (48 + 4096)) / 0.87962566103423978
    w = p["xconv_4_X_0/kernel"]
    assert float(w.abs().max()) <= 2 * std + 1e-7 and 0.8 * std < float(w.std()) < std
    assert float(p["logits/bias"].abs().max()) == 0.0


def test_store_survives_a_tf_checkpoint_round_trip(tmp_path):
    p = M.init_params(seed=2, device="cpu", randomize_bn=True)
    src = {k: v.numpy().copy() for k, v in p.items()}
    prefix = str(tmp_path / "model.ckpt")
    ck.write_tf_checkpoint(prefix, src)
    q = M.init_params(seed=7, device="cpu")
    assert ck.restore(q, prefix) == []
    for k, v in src.items():
        assert np.array_equal(q[k].numpy(), v), k


# ---- an independent float64 torch composition of one X-Conv layer, in NCHW with the neighbour axis as the width ----
def _bn_torch(p, layer, x):
    """F.batch_norm over channel axis 1"""
    g = lambda v: p[f"{layer}_bn/{v}"].double()
    return F.batch_norm(x, g("moving_mean"), g("moving_variance"), g("gamma"), g("beta"), False, 0.0, po.BN_EPS)


def _xconv_torch(p, tag, pts, qrs, idx, fts, K, dm, glob):
    B, P = idx.shape[:2]
    w = lambda name: p[f"{tag}{name}"].double()
    nn_pts = torch.stack([pts[b][idx[b]] for b in range(B)])                  # (B,P,K,3)
    local = (nn_pts - qrs[:, :, None, :]).permute(0, 3, 1, 2)                 # NCHW (B,3,P,K)

    def pw(x, kernel, layer, act=True):                                       # 1x1 conv, ELU, BN
        y = F.conv2d(x, kernel.reshape(-1, kernel.shape[-1]).t()[:, :, None, None])
        return _bn_torch(p, layer, F.elu(y) if act else y)

    lifted = pw(pw(local, w("nn_fts_from_pts_0/kernel"), f"{tag}nn_fts_from_pts_0"), w("nn_fts_from_pts/kernel"), f"{tag}nn_fts_from_pts")
    Fin = lifted if fts is None else torch.cat([lifted, torch.stack([fts[b][idx[b]] for b in range(B)]).permute(0, 3, 1, 2)], 1)
    # X_0: a (1,K) VALID conv; TF kernel (1,K,3,K*K) [h][w][in][out] -> torch (out, in, h, w)
    X0 = _bn_torch(p, f"{tag}X_0", F.elu(F.conv2d(local, w("X_0/kernel").permute(3, 2, 0, 1))))      # (B,K*K,P,1)
    X0_KK = X0[..., 0].permute(0, 2, 1).reshape(B, P, K, K)                                           # [a][b]

    def depthwise(x_kk, kernel, layer, act):
        x = x_kk.permute(0, 3, 1, 2)                                          # NCHW: channel b, width a -> (B,K,P,K)
        wt = kernel.permute(2, 3, 0, 1).reshape(K * K, 1, 1, K)              # (in*mult, 1, h, w), out channel b*K + m
        y = F.conv2d(x, wt, groups=K)[..., 0].permute(0, 2, 1)               # (B,P,K*K)
        y = y.permute(0, 2, 1)[..., None]
        return _bn_torch(p, layer, F.elu(y) if act else y)[..., 0].permute(0, 2, 1).reshape(B, P, K, K)

    X1_KK = depthwise(X0_KK, w("X_1/depthwise_weights"), f"{tag}X_1", True)
    X2_KK = depthwise(X1_KK, w("X_2/depthwise_weights"), f"{tag}X_2", False)
    fts_X = torch.einsum("bpij,bcpj->bcpi", X2_KK, Fin)                       # (B,C_in,P,K)
    cin = fts_X.shape[1]
    wdw = w("fts_conv/depthwise_kernel").permute(2, 3, 0, 1).reshape(cin * dm, 1, 1, K)
    dw = F.conv2d(fts_X, wdw, groups=cin)                                     # (B,C_in*dm,P,1)
    conv = pw(dw, w("fts_conv/pointwise_kernel"), f"{tag}fts_conv")
    out = conv[..., 0].permute(0, 2, 1)
    if glob:
        q = qrs.permute(0, 2, 1)[..., None]
        g = pw(pw(q, w("fts_global_0/kernel"), f"{tag}fts_global_0"), w("fts_global/kernel"), f"{tag}fts_global")
        out = torch.cat([g[..., 0].permute(0, 2, 1), out], -1)
    return dw[..., 0].permute(0, 2, 1).reshape(B * P, -1), out


def test_oracle_matches_a_torch_composition():
    b, n = 2, 400
    p = M.init_params(seed=3, device="cpu", randomize_bn=True)
    x = make_clouds("dup", b, n, 5)
    pts, fts, idx_list = x, None, []
    for tag, k, d, P, _, _, _, dm, glob in M.layer_table():
        P = n if P == -1 else P
        qrs = x[:, :P]
        idx = po.knn_dilated(pts, qrs, k, d).astype(np.int64)
        idx_list.append(idx)
        dw_t, out_t = _xconv_torch(p, tag, torch.from_numpy(pts).double(), torch.from_numpy(qrs).double(), torch.from_numpy(idx),
                                   None if fts is None else torch.from_numpy(fts), k, dm, glob)
        r = po.xconv(p, tag, pts, qrs, idx, fts, k, dm, glob)
        for name, got, want in (("dw", r["dw"], dw_t), ("out", r["out"], out_t)):
            scale = max(1.0, float(want.abs().max()))
            assert np.abs(got - want.numpy()).max() < 1e-12 * scale, (tag, name)
        pts, fts = qrs, r["out"]
    res = po.forward(p, x, idx_list)
    assert res["logits"].shape == (b, 1, 15)
    net = torch.from_numpy(res["out4"])
    for i in range(2):
        net = _bn_torch(p, f"fc{i}", F.elu(net @ p[f"fc{i}/kernel"].double()).permute(0, 2, 1)).permute(0, 2, 1)
    logits = net.mean(1, keepdim=True) @ p["logits/kernel"].double() + p["logits/bias"].double()
    assert np.abs(res["logits"] - logits.numpy()).max() < 1e-12


@pytest.mark.parametrize("kind", ["ball", "dup"])
def test_knn_oracle_with_d1_is_dgcnn_knn(kind):
    x = make_clouds(kind, 3, 300, 1)
    assert np.array_equal(po.knn_dilated(x, x, 16, 1), orc.dgcnn_knn(x, 16))


def test_knn_oracle_dilation_keeps_every_dth():
    x = make_clouds("shell", 2, 200, 4)
    full = po.knn_dilated(x, x[:, :50], 48, 1)
    assert np.array_equal(po.knn_dilated(x, x[:, :50], 16, 3), full[:, :, ::3])


def test_invalid_calls_raise_without_a_gpu():
    p = M.init_params(device="cpu")
    x = torch.zeros((2, 1024, 3))
    with pytest.raises(NotImplementedError):
        M.get_model(x, True, params=p)
    with pytest.raises(ValueError):
        M.get_model(torch.zeros((2, 383, 3)), False, params=p)
    with pytest.raises(ValueError):
        M.get_model(x, False, num_class=40, params=p)
    with pytest.raises(NotImplementedError):
        M.get_model(torch.zeros((2, 1024, 3), requires_grad=True), False, params=p)
    with pytest.raises(ValueError):
        ops.knn_dilated(x, x, 16, 5)                  # k*d = 80 > 64
    with pytest.raises(RuntimeError):
        ops.knn_dilated(x, x, 16, 3)                  # a CPU tensor


def test_c_abi_rejects_bad_arguments_without_a_gpu():
    from scanobjectnn_b200 import _lib
    lib = _lib.load()
    null = C.c_void_p(0)
    assert lib.psa_knn_dilated(1, 128, 128, 16, 5, null, null, null, null) == -1
    assert b"k*d" in lib.psa_last_error()
    assert lib.psa_knn_dilated(1, 40, 40, 16, 3, null, null, null, null) == -1
    layer = _lib.PsaXconv(17, 24, 0, 4)
    assert lib.psa_xconv_core(1, 64, 64, null, null, null, null, C.byref(layer), null, null) == -1
    layer = _lib.PsaXconv(8, 24, 48, 4)                # c_prev > 0 without fts
    assert lib.psa_xconv_core(1, 64, 64, null, null, null, null, C.byref(layer), null, null) == -1
    assert lib.psa_dense_elu_affine(128, 96, 48, null, 90, null, null, null, null, null, 48, null, 0, null) == -1     # ldx < K
    assert lib.psa_dense_elu_affine(0, 96, 48, null, 96, null, null, null, null, null, 48, null, 0, null) == 0
    ops.set_mlp_mode(1)
    try:
        assert lib.psa_dense_elu_affine_workspace_bytes(4096, 480, 384) == 0
    finally:
        ops.set_mlp_mode(0)
    assert lib.psa_dense_elu_affine_workspace_bytes(4096, 480, 384) > 0
    assert lib.psa_dense_elu_affine_workspace_bytes(4096, 3, 96) == 0         # K % 4 != 0: the FMA kernel


@pytest.mark.skipif(shutil.which("cuobjdump") is None and not os.path.exists("/usr/local/cuda/bin/cuobjdump"), reason="no cuobjdump")
def test_new_kernels_do_not_spill_and_use_no_float_atomics(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    src = os.path.join(ROOT, "scanobjectnn_b200", "csrc", "pointcnn.cu")
    obj = str(tmp_path / "pointcnn.o")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c", src, "-o", obj],
                       capture_output=True, text=True, check=True)
    log = r.stdout + r.stderr
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(frames) >= 7 and all(f == ("0", "0", "0") for f in frames), log
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    assert not re.search(r"\b(RED|ATOM|ATOMG)\.[A-Z.]*F32", sass)
