"""Gradients with respect to the input cloud of DGCNN and vanilla PointNet in inference mode (batch norm frozen on the moving averages:
the training kernels with psa_edgeconv_frozen_bwd / psa_edgeconv2_frozen_bwd and frozen mlp_training nodes) against float64
restatements evaluated on the GPU path's own neighbour graphs.  Bounds as in test_input_grad_gpu.py: outputs
1e-5 of max(1, |largest|), gradients 1e-4 relative to the largest entry.  Ambiguous maxima and near-zero relu inputs are left out
on both sides by the exclusion rule of tests/restate.py."""
import ctypes as C

import numpy as np
import pytest
import torch

from scanobjectnn_b200 import _lib, dgcnn, pointnet_cls, training
from scanobjectnn_b200.synthetic import make_clouds

from . import gpu_util as G
from . import restate
from .restate import Masks, ambiguous, edgeconv_store, edges, grid_x, layer, moving, out_err, params_as, perturb_tnets, rel

OTOL, GTOL = 1e-5, 1e-4
S1, S2 = restate.EC2


def _bit_equal(a: dict, b: dict):
    return a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)


def _randomize_moving(p, scopes, seed):
    rng = np.random.default_rng(seed)
    for s in scopes:
        c = p[f"{s}/bn/moving_mean"].numel()
        p[f"{s}/bn/moving_mean"] = torch.tensor(rng.uniform(-0.5, 0.5, c), dtype=torch.float32, device="cuda")
        p[f"{s}/bn/moving_variance"] = torch.tensor(rng.uniform(0.5, 2.0, c), dtype=torch.float32, device="cuda")


def _dgcnn_setup(b, n, seed, bga=False, tnet_weights=True):
    p = dgcnn.init_params(seed=seed, randomize_bn=True, bga=bga)
    if tnet_weights:
        perturb_tnets(p, seed)
    x = G.cu(make_clouds("ball", b, n, seed=seed + 100))
    return p, x


def _dgcnn_against_float64(b, n, seed, monkeypatch, with_detached=False, frozen=True):
    """(x.grad, float64 x.grad, float64 x.grad with the transform detached (with_detached) or None, logits, float64 logits, masked
    count, count of the elements checked for masking).  frozen=False: training mode (batch statistics, dropout off) on the graphs of
    a first run."""
    p, x0 = _dgcnn_setup(b, n, seed)
    R = G.cu(np.random.default_rng(seed).standard_normal((b, dgcnn.NUM_CLASSES)).astype(np.float32))

    def run(x, graphs=None):
        if frozen:
            return dgcnn.get_model(x, False, params=p)
        return dgcnn._get_model_training(x, 0.5, dgcnn.NUM_CLASSES, p, dropout=False, graphs=graphs)

    _, ep = run(x0.clone().requires_grad_(True))
    graphs = [ep[f"nn_idx{i}"] for i in range(5)]
    P = params_as(p, torch.float64)                  # training mode updates only the moving averages, which batch statistics do not read
    want = []
    for detach in (False, True) if with_detached else (False,):
        masks = Masks()
        x64 = x0.double().requires_grad_(True)
        l64 = restate.dgcnn(x64, P, graphs, frozen, masks, detach_transform=detach)
        (l64 * R.double()).sum().backward()
        want.append((l64.detach(), x64.grad, masks))
    masks = want[0][2]
    with monkeypatch.context() as m:
        masks.patch(m)
        x = x0.clone().requires_grad_(True)
        logits, ep2 = run(x, graphs)
        (logits * R).sum().backward()
    for i in range(5):
        assert torch.equal(ep2[f"nn_idx{i}"], graphs[i])
    masked, total = masks.count()
    return x.grad, want[0][1], want[-1][1] if with_detached else None, logits.detach(), want[0][0], masked, total


# ---------------------------------------------------------------------------------------------------------------------
# 1. argument checks of the C ABI
# ---------------------------------------------------------------------------------------------------------------------
def test_frozen_edgeconv_entry_points_reject_bad_arguments_without_a_gpu():
    lib = _lib.load()
    fake = C.c_void_p(1 << 20)                  # never dereferenced: every check below fails before any launch
    null = C.c_void_p(0)
    big = C.c_size_t(1 << 40)

    def fwd(b, n, c, k, cout, x=fake):          # stats = NULL: the frozen forward
        return lib.psa_edgeconv_train_fwd(b, n, c, k, cout, x, fake, fake, null, fake, null, fake, big, null)

    def bwd1(b, n, c, k, cout, ws=fake, ws_bytes=big, x=fake, dx=fake):
        return lib.psa_edgeconv_frozen_bwd(b, n, c, k, cout, x, *([fake] * 8), dx, ws, ws_bytes, null)

    def bwd2(b, n, c, k, c1=64, c2=128, ws=fake, ws_bytes=big, x=fake, dx=fake, bias2=fake):
        return lib.psa_edgeconv2_frozen_bwd(b, n, c, k, c1, c2, x, *([fake] * 6), bias2, *([fake] * 5), dx, ws, ws_bytes, null)

    for bwd in (bwd1, lambda b, n, c, k, cout=64, **kw: bwd2(b, n, c, k, **kw)):
        assert bwd(0, 16, 3, 20, 64) == -1 and bwd(2, 0, 3, 20, 64) == -1 and bwd(2, 16, 0, 20, 64) == -1 and bwd(2, 16, 3, 0, 64) == -1
        assert b"bad dims" in lib.psa_last_error()
        assert bwd(2, 16, 3, 20, 64, x=null) == -1 and b"null" in lib.psa_last_error()
        assert bwd(2, 16, 3, 20, 64, dx=null) == -1 and b"null" in lib.psa_last_error()
        assert bwd(2, 16, 3, 20, 64, ws=null) == -1
        assert bwd(2, 16, 3, 20, 64, ws=C.c_void_p((1 << 20) + 16)) == -1 and b"aligned" in lib.psa_last_error()
        assert bwd(1, 51201, 3, 20, 64) == -2                                         # beyond the reverse neighbour lists
    need1 = lib.psa_edgeconv_train_workspace_bytes(2, 16, 3, 20, 64)
    assert need1 > 0
    assert bwd1(2, 16, 3, 20, 64, ws_bytes=C.c_size_t(need1 - 1)) == -1 and b"workspace" in lib.psa_last_error()
    assert bwd1(2, 16, 3, 20, 48) == -2 and bwd1(2, 16, 3, 20, 288) == -2            # C_out: a multiple of 32, at most 256
    need2 = lib.psa_edgeconv2_train_workspace_bytes(2, 16, 3, 20, 64, 128)
    assert need2 > 0
    assert bwd2(2, 16, 3, 20, ws_bytes=C.c_size_t(need2 - 1)) == -1 and b"workspace" in lib.psa_last_error()
    for c1, c2 in ((32, 128), (64, 64), (128, 128), (64, 256)):
        assert bwd2(2, 16, 3, 20, c1, c2) == -2
    assert bwd2(2, 16, 3, 33) == -2 and b"mask" in lib.psa_last_error()              # k > 32
    # bias2 may be NULL: the call gets past the buffer checks to the workspace check
    assert bwd2(2, 16, 3, 20, ws_bytes=C.c_size_t(need2 - 1), bias2=null) == -1 and b"workspace" in lib.psa_last_error()
    # the forward without statistics still checks its other buffers and its workspace
    assert fwd(2, 16, 3, 20, 64, x=null) == -1 and b"null" in lib.psa_last_error()
    assert lib.psa_edgeconv_train_fwd(2, 16, 3, 20, 64, fake, fake, fake, null, null, null, fake, big, null) == -1    # PQ
    assert lib.psa_edgeconv_train_fwd(2, 16, 3, 20, 64, fake, fake, fake, null, fake, null, null, big, null) == -1    # workspace
    assert fwd(2, 16, 3, 20, 48) == -2


# ---------------------------------------------------------------------------------------------------------------------
# 2-3. the frozen EdgeConv ops against float64
# ---------------------------------------------------------------------------------------------------------------------
def _flat_state(p):
    fp = p._flat
    return fp.flat.detach().clone(), fp.grad.clone()


def _check_variables_untouched(p, moving0, flat0, grad0):
    fp = p._flat
    assert _bit_equal(moving(p), moving0), "inference mode must not update the moving averages"
    assert torch.equal(fp.flat.detach(), flat0) and torch.equal(fp.grad, grad0), "inference mode must leave the flat buckets alone"
    assert fp.flat.grad is None


@pytest.mark.gpu
@pytest.mark.parametrize("c,cout,k", [(3, 64, 20), (64, 64, 20), (64, 128, 20), (64, 64, 1), (64, 32, 40)])
def test_frozen_edgeconv_matches_float64(c, cout, k):
    """eval-mode batch norm on randomised moving averages; dyadic-grid inputs (every edge value exact in fp32), self-loops and a
    cloud of duplicated points, so tied maxima and their even split occur"""
    b, n, s = 3, 300, "e"
    p = edgeconv_store(c, cout, seed=c + cout + k)
    _randomize_moving(p, [s], seed=k)
    x_np = grid_x(b, n, c, seed=k)
    x_np[1, n // 2:] = x_np[1, :n // 2]
    rng = np.random.default_rng(7)
    idx_np = rng.integers(0, n, (b, n, k)).astype(np.int32)
    idx_np[:, :, 0] = np.arange(n)
    idx_np[1, :, 1 % k] = (np.arange(n) + n // 2) % n
    x = torch.tensor(x_np, device="cuda", requires_grad=True)
    idx = torch.tensor(idx_np, device="cuda")
    R = torch.tensor(np.random.default_rng(11).standard_normal((b, n, cout)).astype(np.float32), device="cuda")
    P = params_as(p, torch.float64)
    moving0 = moving(p)

    out = training.edgeconv_training(x, idx, s, None, p, frozen=True)
    flat0, grad0 = _flat_state(p)
    assert out.shape == (b, n, cout) and out.grad_fn is not None
    (gx,) = torch.autograd.grad(out, [x], R)
    x64 = x.detach().double().requires_grad_(True)
    o64 = layer(edges(x64, idx), P, s, True).amax(dim=2)
    (want,) = torch.autograd.grad(o64, [x64], R.double())
    assert out_err(out.detach().cpu(), o64.detach().cpu()) < OTOL
    assert rel(gx.cpu(), want.cpu()) < GTOL
    _check_variables_untouched(p, moving0, flat0, grad0)
    ties = p._trainers[("edgeconv_frozen", s, b, n, c, k)].ties
    assert k == 1 or int(ties.max()) > 1                                           # the even split was exercised
    assert ("edgeconv", s, b, n, c, k) not in p._trainers


def _store2(c, seed):
    p = restate.edgeconv2_store(c, seed)
    _randomize_moving(p, (S1, S2), seed + 1)
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("k", [20, 1, 32])
def test_frozen_edgeconv2_matches_float64(k):
    b, n, c = 3, 300, 3
    p = _store2(c, seed=k)
    rng = np.random.default_rng(k)
    x_np = rng.standard_normal((b, n, c)).astype(np.float32)
    x_np[1, n // 2:] = x_np[1, :n // 2]
    idx_np = rng.integers(0, n, (b, n, k)).astype(np.int32)
    idx_np[:, :, 0] = np.arange(n)
    idx_np[1, :, 1 % k] = (np.arange(n) + n // 2) % n
    x = torch.tensor(x_np, device="cuda", requires_grad=True)
    idx = torch.tensor(idx_np, device="cuda")
    P = params_as(p, torch.float64)
    moving0 = moving(p)

    x64 = x.detach().double().requires_grad_(True)
    z64 = layer(layer(edges(x64, idx), P, S1, True), P, S2, True)
    o64 = z64.amax(dim=2)
    amb = ambiguous(z64, 2)
    R = torch.tensor(rng.standard_normal((b, n, 128)).astype(np.float32), device="cuda")
    R[amb] = 0.0
    print(f"[frozen edgeconv2 k={k}] ambiguous maxima masked: {int(amb.sum())} of {amb.numel()}")
    assert float(amb.double().mean()) < 0.01

    out = training.edgeconv_training(x, idx, (S1, S2), None, p, frozen=True)
    flat0, grad0 = _flat_state(p)
    assert out.shape == (b, n, 128) and out.grad_fn is not None
    (gx,) = torch.autograd.grad(out, [x], R)
    (want,) = torch.autograd.grad(o64, [x64], R.double())
    assert out_err(out.detach().cpu(), o64.detach().cpu()) < OTOL
    assert rel(gx.cpu(), want.cpu()) < GTOL
    _check_variables_untouched(p, moving0, flat0, grad0)
    mask = p._trainers[("edgeconv2_frozen", (S1, S2), b, n, c, k)].mask
    cnt = np.unpackbits(mask.cpu().numpy().view(np.uint8)).reshape(tuple(mask.shape) + (32,)).sum(-1).astype(np.int64)
    assert cnt.min() >= 1
    assert k == 1 or cnt.max() > 1


# ---------------------------------------------------------------------------------------------------------------------
# DGCNN
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_dgcnn_inference_input_grad_matches_float64(monkeypatch):
    b, n = 8, 256
    gx, want, want_detached, logits, l64, masked, total = _dgcnn_against_float64(b, n, seed=3, monkeypatch=monkeypatch,
                                                                                   with_detached=True)
    print(f"[dgcnn frozen B={b} N={n}] ambiguous maxima masked: {masked} of {total}")
    assert masked <= 0.01 * total
    assert out_err(logits.cpu(), l64.cpu()) < OTOL
    assert rel(gx.cpu(), want.cpu()) < GTOL
    assert rel(want_detached.cpu(), want.cpu()) > 10 * GTOL           # the T-net's share is visible ...
    assert rel(gx.cpu(), want_detached.cpu()) > 10 * GTOL             # ... and the frozen path carries it


@pytest.mark.gpu
def test_dgcnn_inference_routes_by_requires_grad():
    """the frozen path's first graph is the fused path's; its later graphs come from features that differ from the fused kernels' in
    the last bits, which can reorder near-tied neighbours (at this shape graphs 3 and 4 differed at every seed tried), so the logits are
    compared with the frozen path evaluated on the fused path's own graphs"""
    b, n = 4, 2048
    p, x0 = _dgcnn_setup(b, n, seed=4)
    fused, ep_f = dgcnn.get_model(x0, False, params=p)
    assert "_trainers" not in p.__dict__ and getattr(p, "_flat", None) is None
    x = x0.clone().requires_grad_(True)
    with torch.no_grad():
        nograd, _ = dgcnn.get_model(x, False, params=p)
    assert torch.equal(nograd, fused) and "_trainers" not in p.__dict__
    logits, ep = dgcnn.get_model(x, False, params=p)
    assert logits.grad_fn is not None
    assert set(ep) == set(ep_f)
    assert torch.equal(ep["nn_idx0"], ep_f["nn_idx0"])
    assert torch.equal(logits.argmax(-1), fused.argmax(-1))
    on_fused_graphs, _ = dgcnn._get_model_training(x, None, dgcnn.NUM_CLASSES, p, graphs=[ep_f[f"nn_idx{i}"] for i in range(5)], frozen=True)
    assert rel(on_fused_graphs.detach().cpu(), fused.cpu()) < 1e-4
    dgcnn.get_loss(logits, torch.zeros(b, dtype=torch.int64, device="cuda")).backward()
    assert bool(torch.isfinite(x.grad).all()) and float(x.grad.abs().max()) > 0


@pytest.mark.gpu
def test_dgcnn_bga_inference_input_grad_reaches_the_cloud():
    b, n = 4, 512
    p, x0 = _dgcnn_setup(b, n, seed=6, bga=True)
    labels = torch.tensor([1, 4, 0, 9], device="cuda")
    seg_labels = torch.tensor(np.random.default_rng(2).integers(0, 2, (b, n)), device="cuda")
    # one training step first: the flat parameter vector now requires grad, and inference mode must still leave nothing in its .grad
    cp, _ = dgcnn.get_model_bga(x0, True, bn_decay=0.5, params=p)
    torch.nn.functional.cross_entropy(cp, labels).backward()
    assert p._flat.flat.requires_grad and p._flat.flat.grad is not None
    p._flat.flat.grad = None
    moving0 = moving(p)
    grads = []
    for joint in (True, False):
        x = x0.clone().requires_grad_(True)
        cp, sp = dgcnn.get_model_bga(x, False, params=p)
        assert cp.grad_fn is not None and sp.shape == (b, n, 2)
        f = torch.nn.functional
        loss = f.cross_entropy(cp, labels) + (f.cross_entropy(sp.reshape(-1, 2), seg_labels.reshape(-1)) if joint else 0.0)
        loss.backward()
        grads.append(x.grad)
    assert bool(torch.isfinite(grads[0]).all()) and float(grads[0].abs().max()) > 0
    assert rel(grads[0].cpu(), grads[1].cpu()) > 100 * GTOL, "the segmentation head's gradient did not reach the cloud"
    assert _bit_equal(moving(p), moving0)
    assert p._flat.flat.grad is None


@pytest.mark.gpu
def test_dgcnn_training_input_grad(monkeypatch):
    """training mode: logits, the flat gradient bucket and the moving averages are bit-identical whether or not x requires grad, and
    x.grad matches the batch-statistics restatement on the run's graphs"""
    b, n = 32, 256
    runs = []
    for want_grad in (True, False):
        p, x0 = _dgcnn_setup(b, n, seed=7)
        x = x0.clone().requires_grad_(want_grad)
        logits, ep = dgcnn._get_model_training(x, 0.5, dgcnn.NUM_CLASSES, p, dropout=False)
        dgcnn.get_loss(logits, torch.arange(b, device="cuda") % dgcnn.NUM_CLASSES).backward()
        runs.append((logits.detach(), p._flat.flat.grad.clone(), moving(p), x.grad))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1]) and _bit_equal(runs[0][2], runs[1][2])
    assert bool(torch.isfinite(runs[0][3]).all()) and float(runs[0][3].abs().max()) > 0 and runs[1][3] is None
    gx, want, _, _, _, masked, total = _dgcnn_against_float64(b, n, seed=7, monkeypatch=monkeypatch, frozen=False)
    print(f"[dgcnn training B={b} N={n}] masked: {masked} of {total}; x.grad error relative to the largest entry: "
          f"{rel(gx.cpu(), want.cpu()):.2e}")
    assert masked <= 0.01 * total
    assert rel(gx.cpu(), want.cpu()) < GTOL


@pytest.mark.gpu
def test_dgcnn_inference_input_grad_is_bit_reproducible():
    b, n = 8, 1024
    p, x0 = _dgcnn_setup(b, n, seed=9)
    grads = []
    for _ in range(2):
        x = x0.clone().requires_grad_(True)
        logits, _ = dgcnn.get_model(x, False, params=p)
        dgcnn.get_loss(logits, torch.arange(b, device="cuda") % dgcnn.NUM_CLASSES).backward()
        grads.append(x.grad)
    assert torch.equal(grads[0], grads[1])


@pytest.mark.gpu
def test_dgcnn_inference_input_grad_at_the_model_shape(monkeypatch):
    b, n = 32, 2048
    gx, want, _, logits, l64, masked, total = _dgcnn_against_float64(b, n, seed=11, monkeypatch=monkeypatch)
    print(f"[dgcnn frozen B={b} N={n}] ambiguous maxima masked: {masked} of {total}; "
          f"x.grad error relative to the largest entry: {rel(gx.cpu(), want.cpu()):.2e}")
    assert masked <= 0.01 * total
    assert out_err(logits.cpu(), l64.cpu()) < OTOL
    assert rel(gx.cpu(), want.cpu()) < GTOL


# ---------------------------------------------------------------------------------------------------------------------
# 8. vanilla PointNet
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_pointnet_inference_input_grad(monkeypatch):
    b, n = 8, 1024
    p = pointnet_cls.init_params(seed=2, randomize_bn=True)
    perturb_tnets(p, 2)
    x0 = G.cu(make_clouds("ball", b, n, seed=12))
    labels = torch.tensor([3, 1, 4, 1, 5, 9, 2, 6], device="cuda")
    # routing: no gradient asked for -> the fused path, no trainer
    fused, ep_f = pointnet_cls.get_model(x0, False, params=p)
    assert "_trainers" not in p.__dict__ and getattr(p, "_flat", None) is None
    xg = x0.clone().requires_grad_(True)
    with torch.no_grad():
        nograd, _ = pointnet_cls.get_model(xg, False, params=p)
    assert torch.equal(nograd, fused) and "_trainers" not in p.__dict__
    # one training step: the flat parameter vector now requires grad, and inference mode must still leave nothing in its .grad
    lt, ept = pointnet_cls.get_model(x0, True, bn_decay=0.5, params=p)
    pointnet_cls.get_loss(lt, labels, ept).backward()
    assert p._flat.flat.requires_grad and p._flat.flat.grad is not None
    p._flat.flat.grad = None
    p.invalidate()                                           # the step updated the moving averages in place
    with torch.no_grad():
        fused, _ = pointnet_cls.get_model(x0, False, params=p)
    moving0 = moving(p)
    # float64 restatement, then the frozen path with the same maxima masked
    masks = Masks()
    x64 = x0.double().requires_grad_(True)
    l64, t64 = restate.pointnet(x64, params_as(p, torch.float64), masks)
    f = torch.nn.functional
    reg = lambda t: 0.001 * 0.5 * ((torch.bmm(t, t.transpose(1, 2)) - torch.eye(64, dtype=t.dtype, device=t.device)) ** 2).sum()  # noqa: E731
    (f.cross_entropy(l64, labels) + reg(t64)).backward()
    masked, total = masks.count()
    print(f"[pointnet frozen B={b} N={n}] ambiguous maxima masked: {masked} of {total}")
    assert masked <= 0.01 * total
    with monkeypatch.context() as m:
        masks.patch(m)
        x = x0.clone().requires_grad_(True)
        logits, ep = pointnet_cls.get_model(x, False, params=p)
        assert logits.grad_fn is not None and ep["transform"].grad_fn is not None and set(ep) == set(ep_f)
        pointnet_cls.get_loss(logits, labels, ep).backward()
    assert out_err(logits.detach().cpu(), l64.detach().cpu()) < OTOL
    assert rel(logits.detach().cpu(), fused.cpu()) < 1e-4 and torch.equal(logits.argmax(-1), fused.argmax(-1))
    assert rel(x.grad.cpu(), x64.grad.cpu()) < GTOL
    assert _bit_equal(moving(p), moving0)
    assert p._flat.flat.grad is None
