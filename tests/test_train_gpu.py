"""GPU parity of the training path (forward with batch statistics, backward, Adam) against the float64 restatements
oracle/train_oracle.py / oracle/train_model_oracle.py.  Bound: 1e-4 relative to the largest entry of each gradient tensor
-- the reference's own gradient tests use 1e-4 (pointnet2/tf_ops/grouping/tf_grouping_op_test.py:25,
3d_interpolation/tf_interpolate_op_test.py:21)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import train_model_oracle as M
from oracle import train_oracle as T
from scanobjectnn_b200 import _lib, pointnet2_cls_ssg
from scanobjectnn_b200._lib import PsaActIn, PsaGradIn, ptr, stream
from scanobjectnn_b200.pointnet_util import add_sa_module_params
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import VariableStore
from scanobjectnn_b200.training import LevelSpec, PointNet2ClsTrainer, _plain_grad, _raw_in

from . import gpu_util as G
from .restate import flat_grad, layer, rel

pytestmark = pytest.mark.gpu
GTOL = 1e-4


@pytest.mark.parametrize("rows,K,N", [(1000, 64, 64), (4096, 64, 128), (777, 259, 256), (32, 256, 15), (640, 128, 1024)])
def test_dense_forward_backward_products(rows, K, N):
    """the three products of a layer on the fused GEMM: y = relu(bn(x)).W + b (+ column statistics), dx = dy.W^T, dW = h^T.dy"""
    lib = _lib.load()
    rng = np.random.default_rng(rows + K)
    x = rng.standard_normal((rows, K)).astype(np.float32)
    s = rng.uniform(0.5, 1.5, K).astype(np.float32)
    t = rng.standard_normal(K).astype(np.float32) * 0.3
    W = (rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32) * 0.1
    xd, sd, td, Wd, bd = map(G.cu, (x, s, t, W, b))
    y = torch.empty((rows, N), device="cuda")
    stats = torch.empty((2, N), device="cuda")
    need = lib.psa_train_dense_workspace_bytes(rows, K, N)
    ws = torch.empty(need // 4 + 16, device="cuda")
    a = PsaActIn()
    a.x = xd.data_ptr(); a.ld = K; a.mask = None; a.relu = 1
    if K % 4 == 0:
        a.scale = sd.data_ptr(); a.shift = td.data_ptr()
        h = np.maximum(x.astype(np.float64) * s + t, 0)
    else:
        a.scale = None; a.shift = None; a.relu = 0
        h = x.astype(np.float64)
    assert lib.psa_train_dense_fwd(rows, K, N, C.byref(a), ptr(Wd), ptr(bd), ptr(y), ptr(stats), ptr(ws), C.c_size_t(need), stream()) == 0
    want = h @ W.astype(np.float64) + b
    assert rel(G.npy(y), want) < 1e-5        # wide layers run on the tensor cores (bf16x3 operands): the 1e-5 contract
    np.testing.assert_allclose(G.npy(stats)[0], want.sum(0), rtol=1e-5, atol=1e-3 * np.sqrt(rows))
    np.testing.assert_allclose(G.npy(stats)[1], (want ** 2).sum(0), rtol=1e-5, atol=1e-3)
    # backward products with a plain incoming gradient
    dy = rng.standard_normal((rows, N)).astype(np.float32)
    dyd = G.cu(dy)
    g = _plain_grad(dyd)
    dx = torch.empty((rows, K), device="cuda")
    assert lib.psa_train_dense_bwd_input(rows, K, N, C.byref(g), ptr(Wd), ptr(dx), K, 0, ptr(ws), C.c_size_t(need), stream()) == 0
    assert rel(G.npy(dx), dy.astype(np.float64) @ W.astype(np.float64).T) < 2e-6
    if K > 3:
        dxs = torch.empty((rows, K - 3), device="cuda")
        assert lib.psa_train_dense_bwd_input(rows, K, N, C.byref(g), ptr(Wd), ptr(dxs), K - 3, 3, ptr(ws), C.c_size_t(need), stream()) == 0
        assert rel(G.npy(dxs), (dy.astype(np.float64) @ W.astype(np.float64).T)[:, 3:]) < 2e-6
    dW = torch.empty((K, N), device="cuda")
    assert lib.psa_train_dense_bwd_weight(rows, K, N, C.byref(a), C.byref(g), ptr(dW), ptr(ws), C.c_size_t(need), stream()) == 0
    assert rel(G.npy(dW), h.T @ dy.astype(np.float64)) < 5e-6
    dW2 = torch.empty((K, N), device="cuda")
    assert lib.psa_train_dense_bwd_weight(rows, K, N, C.byref(a), C.byref(g), ptr(dW2), ptr(ws), C.c_size_t(need), stream()) == 0
    assert torch.equal(dW, dW2), "weight gradient is not bit-reproducible"


@pytest.mark.parametrize("groups,pool_k,Cc", [(96, 32, 128), (40, 20, 64)])
def test_bn_relu_pool_layer_backward(groups, pool_k, Cc):
    """batch-norm finalize, max-pool with arg routing, BN backward sums / coefficients and the on-the-fly dy (both dz sources)"""
    lib = _lib.load()
    rng = np.random.default_rng(groups)
    rows = groups * pool_k
    y = rng.standard_normal((rows, Cc)).astype(np.float32) * 1.3 + 0.2
    gamma = rng.uniform(0.5, 1.5, Cc).astype(np.float32)
    beta = rng.standard_normal(Cc).astype(np.float32) * 0.2
    yd, gd, bd = map(G.cu, (y, gamma, beta))
    stats = G.cu(np.stack([y.astype(np.float64).sum(0), (y.astype(np.float64) ** 2).sum(0)]).astype(np.float32))
    f = lambda *s: torch.empty(s, device="cuda")  # noqa: E731
    scale, shift, mean_inv, mm, mv = f(Cc), f(Cc), f(2, Cc), torch.zeros(Cc, device="cuda"), torch.ones(Cc, device="cuda")
    assert lib.psa_bn_finalize(Cc, rows, ptr(stats), ptr(gd), ptr(bd), C.c_float(0.9), ptr(mm), ptr(mv), ptr(scale), ptr(shift), ptr(mean_inv), stream()) == 0
    z64, c_bn, mean, var = T.bn_train_fwd(y.astype(np.float64), gamma.astype(np.float64), beta.astype(np.float64))
    np.testing.assert_allclose(G.npy(mean_inv)[0], mean, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(G.npy(mean_inv)[1], 1 / np.sqrt(var + 1e-3), rtol=1e-5)
    np.testing.assert_allclose(G.npy(mm), 0.1 * mean, rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(G.npy(mv), 0.9 + 0.1 * var, rtol=1e-5)
    pooled, argk = f(groups, Cc), torch.empty((groups, Cc), dtype=torch.int32, device="cuda")
    assert lib.psa_train_pool_fwd(groups, pool_k, Cc, ptr(yd), ptr(scale), ptr(shift), ptr(pooled), ptr(argk), stream()) == 0
    h64, rmask = T.relu_fwd(z64)
    p64, c_pool = T.maxpool_fwd(h64.reshape(groups, pool_k, Cc), axis=1)
    assert np.abs(G.npy(pooled) - p64).max() < 1e-5
    assert (G.npy(argk) == c_pool[0]).mean() > 0.999            # near-ties may pick the other row in fp32
    # ---- backward through pool + relu + BN ----
    dp = rng.standard_normal((groups, Cc)).astype(np.float32)
    dpd = G.cu(dp)
    g = PsaGradIn()
    g.y = yd.data_ptr(); g.ld = Cc; g.s = scale.data_ptr(); g.t = shift.data_ptr(); g.relu = 1
    g.ca = None; g.cb = None; g.cc = None; g.dh = None; g.ld_dh = 0; g.mask = None
    g.dp = dpd.data_ptr(); g.pv = pooled.data_ptr(); g.argk = argk.data_ptr(); g.pool_k = pool_k; g.C = Cc; g.mode = 1
    dgamma, dbeta, ca, cb, cc = f(Cc), f(Cc), f(Cc), f(Cc), f(Cc)
    need = lib.psa_bn_bwd_workspace_bytes(Cc)
    ws = torch.empty(need // 4 + 16, device="cuda")
    assert lib.psa_bn_bwd_coeffs(rows, Cc, C.byref(g), ptr(gd), ptr(mean_inv), ptr(dgamma), ptr(dbeta), ptr(ca), ptr(cb), ptr(cc), ptr(ws),
                                 C.c_size_t(need), stream()) == 0
    # oracle with the GPU's own argmax (so near-tie flips do not enter the comparison)
    dh64 = np.zeros((groups, pool_k, Cc))
    np.put_along_axis(dh64, G.npy(argk)[:, None, :].astype(np.int64), dp[:, None, :].astype(np.float64), axis=1)
    dz64 = dh64.reshape(rows, Cc) * rmask
    dy64, dg64, db64 = T.bn_train_bwd(dz64, c_bn)
    assert rel(G.npy(dgamma), dg64) < GTOL and rel(G.npy(dbeta), db64) < GTOL
    g.ca = ca.data_ptr(); g.cb = cb.data_ptr(); g.cc = cc.data_ptr()
    # dy through an identity-weight input-gradient product
    eye = torch.eye(Cc, device="cuda")
    dy = f(rows, Cc)
    assert lib.psa_train_dense_bwd_input(rows, Cc, Cc, C.byref(g), ptr(eye), ptr(dy), Cc, 0, None, C.c_size_t(0), stream()) == 0
    assert rel(G.npy(dy), dy64) < GTOL
    # dense dz source: same layer fed with the materialised dh
    dhd = G.cu(dh64.reshape(rows, Cc).astype(np.float32))
    g.mode = 0; g.dh = dhd.data_ptr(); g.ld_dh = Cc; g.ca = None; g.cb = None; g.cc = None
    dgamma2, dbeta2 = f(Cc), f(Cc)
    assert lib.psa_bn_bwd_coeffs(rows, Cc, C.byref(g), ptr(gd), ptr(mean_inv), ptr(dgamma2), ptr(dbeta2), ptr(ca), ptr(cb), ptr(cc), ptr(ws),
                                 C.c_size_t(need), stream()) == 0
    assert rel(G.npy(dgamma2), dg64) < GTOL and rel(G.npy(dbeta2), db64) < GTOL


def test_first_layer_backward_ordered_group_point_grad():
    """psa_sa_conv1_bwd: dW_xyz and the ordered-gather GroupPointGrad against np.add.at (tf_grouping_g.cu:61-78)"""
    lib = _lib.load()
    b, n, m, k, c1 = 3, 300, 40, 24, 128
    rng = np.random.default_rng(1)
    xyz = make_clouds("dup", b, n, seed=5)
    new_xyz = orc.gather_point(xyz, orc.fps(xyz, m))
    idx, _ = orc.query_ball_point(0.35, k, xyz, new_xyz, contract=True)
    dy0 = rng.standard_normal((b, m, k, c1)).astype(np.float32)
    dyd = G.cu(dy0.reshape(-1, c1))
    g = _plain_grad(dyd)
    dW = torch.empty((3, c1), device="cuda")
    dU = torch.empty((b * n, c1), device="cuda")
    need = lib.psa_sa_conv1_bwd_workspace_bytes(b, n, m, k, c1, 1)
    ws = torch.empty(need // 4 + 16, device="cuda")
    xyz_d, new_d, idx_d = G.cu(xyz), G.cu(new_xyz), G.cu(idx)       # named: the pointers must outlive the launches
    args = (b, n, m, k, c1, ptr(xyz_d), ptr(new_d), ptr(idx_d), C.byref(g))
    assert lib.psa_sa_conv1_bwd(*args, ptr(dW), ptr(dU), ptr(ws), C.c_size_t(need), stream()) == 0
    d = (orc.group_point(xyz, idx) - new_xyz[:, :, None, :]).astype(np.float64)
    want_dW = np.einsum("bmka,bmkc->ac", d, dy0.astype(np.float64))
    assert rel(G.npy(dW), want_dW) < 1e-5
    want_dU = T.group_bwd(dy0.astype(np.float64), idx.astype(np.int64), n).reshape(b * n, c1)
    assert rel(G.npy(dU), want_dU) < 1e-5
    dU2 = torch.empty_like(dU)
    assert lib.psa_sa_conv1_bwd(*args, ptr(dW), ptr(dU2), ptr(ws), C.c_size_t(need), stream()) == 0
    assert torch.equal(dU, dU2), "ordered GroupPointGrad must be bit-reproducible"


SMALL_LEVELS = [LevelSpec("layer1", 64, 0.3, 16, [64, 64, 128]), LevelSpec("layer2", 16, 0.6, 16, [128, 128, 256]),
                LevelSpec("layer3", None, None, None, [256, 512, 1024], group_all=True)]


def _small_model(seed=0):
    return pointnet2_cls_ssg.init_params(seed=seed, randomize_bn=True)


def _np_params(p):
    return {k: v.detach().cpu().numpy().astype(np.float64) for k, v in p.items()}


def test_training_step_gradients_match_float64_restatement():
    """whole classifier: forward (batch-stat BN everywhere), loss, every parameter gradient, moving averages, one Adam step"""
    B, N = 8, 256
    p = _small_model(seed=3)
    tr = PointNet2ClsTrainer(p, B, N, 15, levels=SMALL_LEVELS)
    xyz = make_clouds("ball", B, N, seed=11)
    labels = np.random.default_rng(0).integers(0, 15, B).astype(np.int32)
    before = _np_params(p)
    tr.draw_dropout()
    masks = {ly.scope: ly.mask.cpu().numpy().astype(np.float64) for ly in tr.head if ly.mask is not None}
    logits = tr.forward(G.cu(xyz), bn_decay=0.7)
    loss, dl = tr.loss_and_grad(logits, G.cu(labels))
    tr.backward(dl)
    torch.cuda.synchronize()
    levels = [(s.scope, s.npoint, s.radius, s.nsample, s.mlp, s.group_all) for s in SMALL_LEVELS]
    head = [("fc1", 512, True, 0.5), ("fc2", 256, True, 0.5), ("fc3", None, False, None)]
    want = M.cls_train_step(xyz, labels, before, levels, head, masks, 15)
    for lv, oidx in zip(tr.levels[:2], want["idx"][:2]):
        assert np.array_equal(G.npy(lv.idx), oidx)
    assert np.abs(G.npy(logits) - want["logits"]).max() < 1e-4 * max(1.0, np.abs(want["logits"]).max())
    assert abs(float(loss.item()) - want["loss"]) < 1e-5 * max(1.0, abs(want["loss"]))
    worst = {}
    for name, gw in want["grads"].items():
        got = G.npy(tr.fp.grad_of(name)).reshape(gw.shape).astype(np.float64)
        if name.endswith("/biases") and f"{name[:-7]}/bn/gamma" in before:
            assert np.abs(got).max() == 0.0 and np.abs(gw).max() < 1e-9       # exact zero here, rounding noise there
            continue
        if np.abs(gw).max() < 1e-9:
            # analytically zero (e.g. the beta of the last BN in front of the max-pool + fc1 + batch norm: a constant shift of
            # the global feature is removed by fc1's batch statistics): only rounding noise on either side
            assert np.abs(got).max() < 1e-5, (name, np.abs(got).max())
            continue
        worst[name] = rel(got, gw)
    bad = {k: v for k, v in worst.items() if v > GTOL}
    print("max relative gradient error:", max(worst.values()), "over", len(worst), "tensors")
    assert not bad, bad
    # moving averages: decay * old + (1 - decay) * batch statistic (tf_util.py:526-531)
    for scope, (mean, var) in want["batch_stats"].items():
        np.testing.assert_allclose(G.npy(p[f"{scope}/bn/moving_mean"]), 0.7 * before[f"{scope}/bn/moving_mean"] + 0.3 * mean, rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(G.npy(p[f"{scope}/bn/moving_variance"]), 0.7 * before[f"{scope}/bn/moving_variance"] + 0.3 * var, rtol=2e-4, atol=1e-6)
    # Adam
    g_before = {k: G.npy(tr.fp.grad_of(k)).astype(np.float64) for k in want["grads"]}
    tr.adam(1e-3)
    for name in ("layer1/conv1/weights", "layer3/conv2/bn/gamma", "fc3/weights", "fc3/biases"):
        pw, _, _ = M.adam_update(before[name], g_before[name].reshape(before[name].shape), 0.0, 0.0, 1, 1e-3)
        np.testing.assert_allclose(G.npy(p[name]).astype(np.float64), pw, rtol=1e-6, atol=1e-7)


def test_training_step_is_bit_reproducible_and_learns():
    B, N = 8, 256
    xyz = G.cu(make_clouds("shell", B, N, seed=2))
    labels = G.cu(np.arange(B, dtype=np.int32) % 15)
    grads = []
    for _ in range(2):
        p = _small_model(seed=5)
        tr = PointNet2ClsTrainer(p, B, N, 15, levels=SMALL_LEVELS)
        tr._gen.manual_seed(7)
        tr.draw_dropout()
        tr.backward(tr.loss_and_grad(tr.forward(xyz, 0.5), labels)[1])
        grads.append(tr.fp.grad.clone())
    assert torch.equal(grads[0], grads[1]), "two runs of the same step must give bit-identical gradients (no atomics)"
    losses = [float(tr.train_step(xyz, labels, lr=2e-3, bn_decay=0.5).item()) for _ in range(30)]
    print("loss", losses[0], "->", losses[-1])
    assert losses[-1] < 0.5 * losses[0]


def test_get_model_is_training_autograd_path():
    """pointnet2_cls_ssg.get_model(is_training=True) no longer raises: logits carry a grad_fn whose backward fills the flat bucket"""
    B, N = 4, 2048
    p = pointnet2_cls_ssg.init_params(seed=1)
    xyz = G.cu(make_clouds("ball", B, N, seed=4))
    labels = G.cu(np.array([1, 3, 5, 7], dtype=np.int32))
    logits, end_points = pointnet2_cls_ssg.get_model(xyz, True, bn_decay=0.5, params=p)
    assert logits.shape == (B, 15) and logits.requires_grad
    loss = pointnet2_cls_ssg.get_loss(logits, labels)
    loss.backward()
    flat = p._flat
    assert flat.flat.grad is not None and torch.isfinite(flat.flat.grad).all() and float(flat.flat.grad.abs().max()) > 0
    assert end_points["l1_indices"].shape == (B, 512, 32)


@pytest.mark.parametrize("c,group_all", [(16, False), (0, False), (24, True)])
def test_pointnet_sa_module_is_training_level_autograd(c, group_all):
    """pointnet_sa_module(is_training=True) on its own: batch-statistics forward, autograd into the input features and the level's
    variables, against the float64 level restatement (oracle/train_oracle.py) on the SAME sampling / grouping indices; two levels
    chained through autograd share one variable store without double-counting each other's gradients."""
    from scanobjectnn_b200.pointnet_util import pointnet_sa_module
    B, N, m, k, r = 3, 256, 64, 16, 0.35
    mlp = [64, 32, 64]                                      # the fused level front takes a first width of 64 or 128
    p = VariableStore(device="cuda", seed=5)
    add_sa_module_params(p, "lv", 3 + c, mlp)
    add_sa_module_params(p, "other", 3 + 8, [16])          # a second level in the same store: its gradients must stay zero here
    rng = np.random.default_rng(c + 1)
    xyz = make_clouds("ball", B, N, seed=31)
    pts = rng.standard_normal((B, N, c)).astype(np.float32) if c else None
    xt = G.cu(xyz)
    pt = G.cu(pts).requires_grad_(True) if c else None
    new_xyz, out, idx = pointnet_sa_module(xt, pt, None if group_all else m, None if group_all else r, None if group_all else k, mlp, None,
                                            group_all, True, 0.5, "lv", params=p)
    mm = 1 if group_all else m
    assert out.shape == (B, mm, mlp[-1]) and out.requires_grad
    R = rng.standard_normal(out.shape).astype(np.float32)
    (out * G.cu(R)).sum().backward()
    # oracle on the same indices
    fps_idx = np.zeros((B, 1), np.int64) if group_all else orc.fps(xyz, m).astype(np.int64)
    idx_np = G.npy(idx).astype(np.int64)
    layers = []
    for i in range(len(mlp)):
        w = G.npy(p[f"lv/conv{i}/weights"]).astype(np.float64)
        layers.append((w.reshape(-1, w.shape[-1]), G.npy(p[f"lv/conv{i}/biases"]).astype(np.float64), G.npy(p[f"lv/conv{i}/bn/gamma"]).astype(np.float64),
                       G.npy(p[f"lv/conv{i}/bn/beta"]).astype(np.float64)))
    x64 = xyz.astype(np.float64)
    if group_all:
        # sample_and_group_all: new_xyz = 0, grouped_xyz = xyz (no centring): same as a centre at the origin
        x_aug = np.concatenate([x64, np.zeros((B, 1, 3))], axis=1)
        fps_idx = np.full((B, 1), N, np.int64)
        pooled, cache, _ = T.sa_level_train_fwd(x_aug, None if pts is None else np.concatenate([pts.astype(np.float64), np.zeros((B, 1, c))], axis=1),
                                                fps_idx, idx_np, layers)
    else:
        pooled, cache, _ = T.sa_level_train_fwd(x64, None if pts is None else pts.astype(np.float64), fps_idx, idx_np, layers)
    assert rel(G.npy(out), pooled) < 1e-5
    _, dpts, grads = T.sa_level_train_bwd(R.astype(np.float64), cache)
    fp = p._flat
    for i, (dw, db, dgamma, dbeta) in enumerate(grads):
        assert rel(G.npy(fp.grad_of(f"lv/conv{i}/weights")).reshape(dw.shape), dw) < GTOL, f"dW{i}"
        assert rel(G.npy(fp.grad_of(f"lv/conv{i}/bn/gamma")), dgamma) < GTOL and rel(G.npy(fp.grad_of(f"lv/conv{i}/bn/beta")), dbeta) < GTOL
        assert float(np.abs(G.npy(fp.grad_of(f"lv/conv{i}/biases"))).max()) < 1e-5       # a bias under batch norm has no gradient
    if c:
        want = dpts[:, :N] if group_all else dpts
        assert rel(G.npy(pt.grad), want) < GTOL
    # autograd on the flat bucket: this level's entries, zeros elsewhere
    g = fp.flat.grad
    assert g is not None and float(g.abs().max()) > 0
    assert float(flat_grad(p, "other/conv0/weights", g).abs().max()) == 0.0


def test_mlp_training_autograd_matches_float64_torch():
    """training.mlp_training (conv / fc chains with batch-statistics batch norm): outputs, input gradient and variable gradients
    against the same chain written in float64 torch ops with torch's autograd."""
    from scanobjectnn_b200.training import mlp_training
    p = VariableStore(device="cuda", seed=9)
    p.add_conv2d("s/c0", 96, 128, bn=True)
    p.add_conv2d("s/c1", 128, 64, bn=True)
    p.add_conv2d("s/c2", 64, 10, bn=False)
    rng = np.random.default_rng(2)
    x = torch.tensor(rng.standard_normal((2, 300, 96)).astype(np.float32), device="cuda", requires_grad=True)
    hid = mlp_training(x, [("s/c0", True), ("s/c1", True)], 0.5, p)                 # activated output (B, N, 64)
    out = mlp_training(hid, [("s/c2", False)], 0.5, p)                               # logits layer, a second autograd node
    R = torch.tensor(rng.standard_normal(tuple(out.shape)).astype(np.float32), device="cuda")
    R2 = torch.tensor(rng.standard_normal(tuple(hid.shape)).astype(np.float32), device="cuda")
    ((out * R).sum() + (hid * R2).sum()).backward()
    fp = p._flat
    # float64 reference
    ws = {k: p[k].detach().double().clone().requires_grad_(True) for k in p.keys() if k.startswith("s/") and "moving" not in k}
    x64 = x.detach().double().reshape(-1, 96).requires_grad_(True)
    h = layer(layer(x64, ws, "s/c0", False), ws, "s/c1", False)
    o = layer(h, ws, "s/c2", False, bn=False)
    ((o * R.double().reshape(-1, 10)).sum() + (h * R2.double().reshape(-1, 64)).sum()).backward()
    assert rel(G.npy(hid).reshape(-1, 64), h.detach().cpu().numpy()) < 1e-5 and rel(G.npy(out).reshape(-1, 10), o.detach().cpu().numpy()) < 1e-5
    assert rel(G.npy(x.grad).reshape(-1, 96), x64.grad.cpu().numpy()) < GTOL
    for k, w in ws.items():
        want = w.grad.cpu().numpy()
        got = G.npy(fp.grad_of(k)).reshape(want.shape)
        if np.abs(want).max() < 1e-9:
            assert np.abs(got).max() < 1e-5, k          # conv bias under batch norm
        else:
            assert rel(got, want) < GTOL, k
    # the bucket autograd accumulated on the flat parameter vector is the sum of the two nodes' buckets = the per-name views
    assert torch.equal(fp.flat.grad, fp.grad) or rel(G.npy(fp.flat.grad), G.npy(fp.grad)) < 1e-6


def test_pointnet2_cls_bga_is_training_backward_runs_and_matches_finite_difference():
    """pointnet2_cls_bga.get_model(is_training=True): both heads carry a grad_fn; a directional finite difference of the joint loss along
    a random direction in parameter space agrees with the autograd gradient (dropout off for the check)."""
    from scanobjectnn_b200 import pointnet2_cls_bga as bga
    B, N = 4, 1024
    p = bga.init_params(seed=3)
    xyz = G.cu(make_clouds("ball", B, N, seed=8))
    labels = G.cu(np.array([1, 4, 7, 11], dtype=np.int64))
    mask = G.cu((np.random.default_rng(0).random((B, N)) > 0.5).astype(np.int64))
    cp, sp = bga.get_model(xyz, True, bn_decay=0.5, params=p)
    assert cp.shape == (B, 15) and sp.shape == (B, N, 2) and cp.requires_grad and sp.requires_grad
    loss, _, _ = bga.get_loss(cp, sp, labels, mask)
    loss.backward()
    g = p._flat.flat.grad.clone()
    assert torch.isfinite(g).all() and float(g.abs().max()) > 0

    def loss_at(flat_values):
        with torch.no_grad():
            p._flat.flat.copy_(flat_values)
        p.invalidate()
        c2, s2 = bga._get_model_training(xyz, 0.5, 15, p, False, dropout=False)
        return float(bga.get_loss(c2, s2, labels, mask)[0].item())

    base = p._flat.flat.detach().clone()
    c2, s2 = bga._get_model_training(xyz, 0.5, 15, p, False, dropout=False)
    p._flat.flat.grad = None
    bga.get_loss(c2, s2, labels, mask)[0].backward()
    g = p._flat.flat.grad.clone()
    d = g / g.norm()                                 # steepest direction: the directional derivative is |g|
    eps = 3e-3 / float(g.norm())                     # a +-3e-3 change of the loss: well above float32 resolution, well inside the linear range
    fd = (loss_at(base + eps * d) - loss_at(base - eps * d)) / (2 * eps)
    an = float((g * d).sum().item())
    loss_at(base)
    assert abs(fd - an) <= 0.05 * max(abs(an), abs(fd)) + 1e-4, (fd, an)


def test_dgcnn_is_training_backward_matches_finite_difference():
    """dgcnn.get_model(is_training=True): EdgeConv layers with batch-statistics batch norm over all edges, the T-net (its 3x3 output is a
    plain torch op on a live view of the flat parameter vector), autograd over group_point / mlp_training; a directional finite difference
    of the loss along the gradient agrees with the autograd gradient (dropout off, neighbour graphs held fixed)."""
    from scanobjectnn_b200 import dgcnn
    B, N = 8, 160                                       # 8 rows in the head's batch norm: two would make it a sign function
    p = dgcnn.init_params(seed=5)
    with torch.no_grad():
        p["transform_net1/transform_XYZ/weights"].normal_(0, 0.01)          # the reference initialises it to zero: give it a gradient path
    xyz = G.cu(make_clouds("ball", B, N, seed=6))
    labels = G.cu(np.array([2, 9, 0, 14, 5, 5, 7, 1], dtype=np.int64))
    logits, end_points = dgcnn.get_model(xyz, True, bn_decay=0.5, params=p)
    assert logits.shape == (B, 15) and logits.requires_grad and end_points["nn_idx4"].shape == (B, N, 20)
    fp = p._flat

    graphs = [end_points[f"nn_idx{i}"] for i in range(5)]     # the graphs depend on the parameters piecewise-constantly: hold them

    def run():
        lg, _ = dgcnn._get_model_training(xyz, 0.5, 15, p, dropout=False, graphs=graphs)
        return torch.nn.functional.cross_entropy(lg, labels)

    fp.flat.grad = None
    run().backward()
    g = fp.flat.grad.clone()
    assert torch.isfinite(g).all() and float(g.abs().max()) > 0
    for name in ("transform_net1/tconv1/weights", "transform_net1/transform_XYZ/weights", "dgcnn1/weights", "dgcnn4/bn/gamma", "agg/weights", "fc3/biases"):
        assert float(flat_grad(p, name, g).abs().max()) > 0, f"no gradient reached {name}"
    base = fp.flat.detach().clone()
    d = g / g.norm()
    eps = 3e-3 / float(g.norm())

    def loss_at(values):
        with torch.no_grad():
            fp.flat.copy_(values)
        p.invalidate()
        with torch.no_grad():
            return float(run().item())

    fd = (loss_at(base + eps * d) - loss_at(base - eps * d)) / (2 * eps)
    an = float((g * d).sum().item())
    loss_at(base)
    assert abs(fd - an) <= 0.05 * max(abs(an), abs(fd)) + 1e-4, (fd, an)


def _directional_check(fp, p, run, tol=0.05):
    fp.flat.grad = None
    run().backward()
    g = fp.flat.grad.clone()
    assert torch.isfinite(g).all() and float(g.abs().max()) > 0
    base = fp.flat.detach().clone()
    d = g / g.norm()
    eps = 3e-3 / float(g.norm())

    def loss_at(values):
        with torch.no_grad():
            fp.flat.copy_(values)
            p.invalidate()
            return float(run().item())

    fd = (loss_at(base + eps * d) - loss_at(base - eps * d)) / (2 * eps)
    an = float((g * d).sum().item())
    loss_at(base)
    assert abs(fd - an) <= tol * max(abs(an), abs(fd)) + 1e-4, (fd, an)
    return g


def test_pointnet_cls_and_dgcnn_bga_is_training():
    """the remaining in-scope model families in training mode: vanilla PointNet (two T-nets, regularised loss) and dgcnn_bga (joint heads)"""
    from scanobjectnn_b200 import dgcnn, pointnet_cls
    B, N = 8, 256
    xyz = G.cu(make_clouds("ball", B, N, seed=12))
    labels = G.cu(np.array([2, 9, 0, 14, 5, 5, 7, 1], dtype=np.int64))
    p = pointnet_cls.init_params(seed=2)
    with torch.no_grad():
        p["transform_net1/transform_XYZ/weights"].normal_(0, 0.01)
        p["transform_net2/transform_feat/weights"].normal_(0, 0.003)
    logits, ep = pointnet_cls.get_model(xyz, True, bn_decay=0.5, params=p)
    assert logits.shape == (B, 15) and logits.requires_grad and ep["transform"].shape == (B, 64, 64)

    def run_pn():
        lg, e2 = pointnet_cls._get_model_training(xyz, 0.5, 15, p, dropout=False)
        return pointnet_cls.get_loss(lg, labels, e2)

    g = _directional_check(p._flat, p, run_pn)
    assert float(flat_grad(p, "transform_net2/transform_feat/weights", g).abs().max()) > 0

    q = dgcnn.init_params(seed=4, bga=True)
    mask = G.cu((np.random.default_rng(1).random((B, N)) > 0.4).astype(np.int64))
    cp, sp = dgcnn.get_model_bga(xyz, True, bn_decay=0.5, params=q)
    assert cp.shape == (B, 15) and sp.shape == (B, N, 2) and cp.requires_grad and sp.requires_grad
    _, _, ep = dgcnn._get_model_training(xyz, 0.5, 15, q, dropout=False, bga=True)
    graphs = [ep[f"nn_idx{i}"] for i in range(5)]

    def run_dg():
        c2, s2, _ = dgcnn._get_model_training(xyz, 0.5, 15, q, dropout=False, graphs=graphs, bga=True)
        f = torch.nn.functional
        return 0.5 * f.cross_entropy(c2, labels) + 0.5 * f.cross_entropy(s2.reshape(-1, 2), mask.reshape(-1))

    _directional_check(q._flat, q, run_dg)
