"""The row-grouped first layer (psa_shared_mlp_grouped, psa_train_dense_fwd_grouped, psa_train_bias_grad_grouped) against float64
restatements that build the concatenation [x, tile(g)] the way PointNet's segmentation head does (pointnet/models/pointnet_seg.py:81-88)."""
import ctypes as C

import numpy as np
import pytest
import torch

from scanobjectnn_b200 import _lib, ops
from scanobjectnn_b200._lib import PsaActIn, PsaGradIn, check, ptr

from . import gpu_util as G

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["tensor", "fma", "tensor_bf16x3"])
def mlp_mode(request):
    """0 = tensor-core kernels where the shapes allow (fp16x2 operands + range guard), 1 = fp32 FMA kernels only, 2 = tensor-core
    kernels with bf16x3 operands"""
    ops.set_mlp_mode({"tensor": 0, "fma": 1, "tensor_bf16x3": 2}[request.param])
    yield request.param
    ops.set_mlp_mode(0)


def _head(rng, cx, cg, chans):
    """Layers of a 1x1-conv chain whose first layer reads [x (cx), g (cg)]: (W, scale, shift) per layer, W scaled to O(1) outputs."""
    layers, cin = [], cx + cg
    for cout in chans:
        w = (rng.standard_normal((cin, cout)) / np.sqrt(cin)).astype(np.float32)
        layers.append((w, rng.uniform(0.5, 1.5, cout).astype(np.float32), (0.1 * rng.standard_normal(cout)).astype(np.float32)))
        cin = cout
    return layers


def _chain64(h, layers):
    for w, s, t in layers:
        h = np.maximum((h @ w.astype(np.float64)) * s + t, 0.0)
    return h


@pytest.mark.parametrize("b,n,cg,chans", [
    (8, 1024, 1024, [512, 256, 128, 128]),     # the segmentation head, train_seg.py's N
    (4, 2048, 1024, [512, 256, 128, 128]),     # the head at N = 2048
    (3, 1000, 1024, [512, 256]),               # groups straddle the 128-row tiles
    (256, 1, 64, [128, 64]),                   # group_rows = 1
    (1, 1024, 64, [256]),                      # a single group
])
def test_shared_mlp_grouped_matches_the_concatenated_chain(b, n, cg, chans, mlp_mode):
    rng = np.random.default_rng(b * 7919 + n)
    cx = 64
    x = rng.standard_normal((b, n, cx)).astype(np.float32)
    g = np.abs(rng.standard_normal((b, cg))).astype(np.float32)
    layers = _head(rng, cx, cg, chans)
    w0, s0, t0 = layers[0]
    # g . W_g: an ordinary shared_mlp call over the b groups
    ga = ops.shared_mlp(G.cu(g), ops.MlpParams([(G.cu(w0[cx:]), None, G.cu(np.zeros(chans[0], np.float32)), False)]))
    mlp = ops.MlpParams([(G.cu(w0[:cx]), G.cu(s0), G.cu(t0), True)] + [(G.cu(w), G.cu(s), G.cu(t), True) for w, s, t in layers[1:]])
    got = G.npy(ops.shared_mlp_grouped(G.cu(x), mlp, ga))
    concat = np.concatenate([x, np.repeat(g[:, None, :], n, axis=1)], axis=2).astype(np.float64)
    want = _chain64(concat.reshape(b * n, cx + cg), layers).reshape(b, n, -1)
    G.contract_close(got, want, f"shared_mlp_grouped b={b} n={n} {chans} [{mlp_mode}]")


def test_shared_mlp_grouped_rejects_bad_groups():
    rng = np.random.default_rng(0)
    w, s, t = _head(rng, 64, 0, [128])[0]
    mlp = ops.MlpParams([(G.cu(w), G.cu(s), G.cu(t), True)])
    with pytest.raises(ValueError):
        ops.shared_mlp_grouped(G.cu(rng.standard_normal((10, 64)).astype(np.float32)), mlp, torch.zeros((3, 128), device="cuda"))


def _fwd_grouped(x, s_in, t_in, w, bias, ga, group_rows):
    lib = _lib.load()
    rows, k = x.shape
    n = w.shape[1]
    y = torch.empty((rows, n), device="cuda")
    stats = torch.empty((2, n), device="cuda")
    need = lib.psa_train_dense_workspace_bytes(rows, k, n)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    ain = PsaActIn(x=x.data_ptr(), ld=k, scale=s_in.data_ptr(), shift=t_in.data_ptr(), mask=None, relu=1)
    check(lib.psa_train_dense_fwd_grouped(rows, group_rows, k, n, C.byref(ain), ptr(w), ptr(bias), ptr(ga), ptr(y), ptr(stats), ptr(ws),
                                          C.c_size_t(need), None), "train_dense_fwd_grouped")
    return y, stats


@pytest.mark.parametrize("b,n", [(4, 1024), (3, 1000), (2, 2048)])
def test_train_dense_fwd_grouped_matches_fp64_and_repeats(b, n):
    rng = np.random.default_rng(b + n)
    rows, k, c1 = b * n, 64, 512
    x = rng.standard_normal((rows, k)).astype(np.float32)
    s_in = rng.uniform(0.5, 1.5, k).astype(np.float32)
    t_in = (0.1 * rng.standard_normal(k)).astype(np.float32)
    w = (rng.standard_normal((k, c1)) / 8).astype(np.float32)
    bias = (0.1 * rng.standard_normal(c1)).astype(np.float32)
    ga = rng.standard_normal((b, c1)).astype(np.float32)
    args = [G.cu(a) for a in (x, s_in, t_in, w, bias, ga)]
    y, stats = _fwd_grouped(*args, n)
    y2, stats2 = _fwd_grouped(*args, n)
    assert torch.equal(y, y2) and torch.equal(stats, stats2)
    h = np.maximum(x.astype(np.float64) * s_in + t_in, 0.0)
    want = h @ w.astype(np.float64) + np.repeat(ga.astype(np.float64), n, axis=0) + bias
    G.contract_close(G.npy(y), want, "train_dense_fwd_grouped y")
    for i, ref in enumerate((want.sum(0), (want * want).sum(0))):
        err = np.abs(G.npy(stats[i]) - ref).max()
        bound = 1e-5 * np.abs(ref).max()
        print(f"stats[{i}] max|err| = {err:.3e} (bound {bound:.3e})")
        assert err < bound


def _group_sums(rows, group_rows, c, gin):
    lib = _lib.load()
    out = torch.empty((rows // group_rows, c), device="cuda")
    check(lib.psa_train_bias_grad_grouped(rows, group_rows, c, C.byref(gin), ptr(out), None), "train_bias_grad_grouped")
    return out


@pytest.mark.parametrize("b,n", [(4, 1024), (3, 1000), (256, 1)])
def test_group_gradient_sums_match_fp64_and_repeat(b, n):
    rng = np.random.default_rng(b * n + 1)
    rows, c = b * n, 512
    y = rng.standard_normal((rows, c)).astype(np.float32)
    dh = rng.standard_normal((rows, c)).astype(np.float32)
    s, t = rng.uniform(0.5, 1.5, c).astype(np.float32), (0.1 * rng.standard_normal(c)).astype(np.float32)
    ca, cb, cc = (rng.standard_normal(c).astype(np.float32) for _ in range(3))
    ty, tdh, ts, tt, tca, tcb, tcc = (G.cu(a) for a in (y, dh, s, t, ca, cb, cc))
    gin = PsaGradIn(y=ty.data_ptr(), ld=c, s=ts.data_ptr(), t=tt.data_ptr(), relu=1, ca=tca.data_ptr(), cb=tcb.data_ptr(),
                    cc=tcc.data_ptr(), dh=tdh.data_ptr(), ld_dh=c, mask=None, dp=None, pv=None, argk=None, pool_k=1, C=c, mode=0)
    got = _group_sums(rows, n, c, gin)
    assert torch.equal(got, _group_sums(rows, n, c, gin))
    y64 = y.astype(np.float64)
    dz = np.where(y64 * s + t > 0, dh.astype(np.float64), 0.0)
    dy = (ca * dz + cb * y64 + cc).reshape(b, n, c)
    want = dy.sum(1)
    # fp32 evaluates dy with an error relative to its terms, which can cancel (a group of one row is dy itself)
    bound = 1e-5 * (np.abs(ca * dz) + np.abs(cb * y64) + np.abs(cc)).reshape(b, n, c).sum(1)
    err = np.abs(G.npy(got) - want)
    print(f"group sums: max|err| = {err.max():.3e}, max ratio to the bound {(err / bound).max():.3f}")
    assert (err < bound).all()
    # the whole batch as one group is the bias gradient, bit for bit
    db = torch.empty(c, device="cuda")
    check(_lib.load().psa_train_bias_grad(rows, c, C.byref(gin), ptr(db), None), "train_bias_grad")
    assert torch.equal(_group_sums(rows, rows, c, gin)[0], db)
