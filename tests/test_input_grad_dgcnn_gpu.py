"""Gradients with respect to the input cloud of DGCNN and vanilla PointNet in inference mode (batch norm frozen on the moving averages:
the training kernels with psa_edgeconv_frozen_bwd / psa_edgeconv2_frozen_bwd and frozen mlp_training nodes) against float64
restatements evaluated on the GPU path's own neighbour graphs.  Bounds as in test_input_grad_gpu.py: outputs
1e-5 of max(1, |largest|), gradients 1e-4 relative to the largest entry.

A max (over k neighbours, or over the N points) whose runner-up lies within 1e-5 of it may be won by another element in fp32 than in
float64, and then routes its gradient elsewhere; likewise a head activation, or a maximum, whose pre-relu value lies within 1e-5 of
zero on either side may fall on the other side of the relu (under batch statistics that changes the gradient of its whole column).
These are properties of the max and the relu, not errors.  The model tests, frozen and training alike, find such elements on the
float64 side and zero the gradient arriving at them on both sides (a hook on the same tensor of each), as test_edgeconv2_train_gpu.py
does for the op's output."""
import ctypes as C

import numpy as np
import pytest
import torch

from scanobjectnn_b200 import _lib, dgcnn, pointnet_cls, training
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import VariableStore

from . import gpu_util as G
from .test_edgeconv_train_gpu import _grid_x
from .test_edgeconv_train_gpu import _store as _store1

OTOL, GTOL = 1e-5, 1e-4
S1, S2 = "t/tconv1", "t/tconv2"


def _rel(got, want):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    return float(np.abs(got - want).max() / max(1e-30, np.abs(want).max()))


def _out_err(got, want):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    return float(np.abs(got - want).max() / max(1.0, np.abs(want).max()))


def _moving(p):
    return {k: v.clone() for k, v in p.items() if k.endswith(("/moving_mean", "/moving_variance"))}


def _bit_equal(a: dict, b: dict):
    return a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)


def _randomize_moving(p, scopes, seed):
    rng = np.random.default_rng(seed)
    for s in scopes:
        c = p[f"{s}/bn/moving_mean"].numel()
        p[f"{s}/bn/moving_mean"] = torch.tensor(rng.uniform(-0.5, 0.5, c), dtype=torch.float32, device="cuda")
        p[f"{s}/bn/moving_variance"] = torch.tensor(rng.uniform(0.5, 2.0, c), dtype=torch.float32, device="cuda")


def _ambiguous(z, dim):
    """True where the max over `dim` has a runner-up of a different value within 1e-5 (of the largest activation) of it, or is a
    positive maximum within that distance of the relu's zero"""
    with torch.no_grad():
        mx = z.amax(dim=dim, keepdim=True)
        below = torch.where(z < mx, z, torch.full_like(z, -1.0)).amax(dim=dim)
        tol = 1e-5 * float(z.abs().max())
        mx = mx.squeeze(dim)
        return ((mx - below) < tol) | ((mx > 0) & (mx < tol))


def _near_zero(z):
    """True where a pre-relu value lies within 1e-5 (of the largest magnitude) of zero"""
    with torch.no_grad():
        return z.abs() < 1e-5 * float(z.abs().max())


def _near_zero_max(pre, dim, scale):
    """True where the max over `dim` of the pre-relu values lies within 1e-5 of `scale` of the relu's zero, on either side: a maximum
    slightly below zero in float64 may lie slightly above it in fp32, and then carries the whole gradient"""
    with torch.no_grad():
        return pre.amax(dim=dim).abs() < 1e-5 * scale


def _inner_flip(pre, inner):
    """True where the edge that wins the max over k (dim 2) of `pre` (b, n, k, c) has a unit of `inner` (b, n, k, c1), the pre-relu
    values of the layer below, within 1e-5 (of the largest magnitude) of zero"""
    with torch.no_grad():
        return _near_zero(inner).any(dim=-1).gather(2, pre.argmax(dim=2))


def _zero_at(t, mask):
    t.register_hook(lambda g: g.masked_fill(mask, 0.0))


# ---------------------------------------------------------------------------------------------------------------------
# float64 restatements
# ---------------------------------------------------------------------------------------------------------------------
def _p64(p):
    return {k: v.detach().double() for k, v in p.items()}


def _layer(h, P, scope, frozen, bn=True, relu=True, stats=None):
    """conv2d / fully_connected (+ batch norm + relu): batch norm on the moving averages (frozen) or on the batch statistics over
    every row (biased variance), eps 1e-3; the batch statistics are recorded in `stats[scope]` when a dict is given"""
    w = P[f"{scope}/weights"]
    y = h @ w.reshape(-1, w.shape[-1]) + P[f"{scope}/biases"]
    if not bn:
        return y
    if frozen:
        mean, var = P[f"{scope}/bn/moving_mean"], P[f"{scope}/bn/moving_variance"]
    else:
        dims = tuple(range(y.dim() - 1))
        mean, var = y.mean(dims), y.var(dims, unbiased=False)
        if stats is not None:
            stats[scope] = (mean.detach(), var.detach())
    z = (y - mean) / torch.sqrt(var + 1e-3) * P[f"{scope}/bn/gamma"] + P[f"{scope}/bn/beta"]
    return torch.relu(z) if relu else z


def _edges(x, idx):
    b, n, c = x.shape
    k = idx.shape[-1]
    neigh = x[torch.arange(b, device=x.device).view(b, 1, 1), idx.long()]
    centre = x.unsqueeze(2).expand(b, n, k, c)
    return torch.cat([centre, neigh - centre], dim=-1)


class _Masks:
    """the ambiguous maxima found by a restatement, in the order the model reaches them: `edge` for the EdgeConv outputs (max over k),
    `pool` for the layers reduced over the N points, keyed by scope; `act` for the head's near-zero relu inputs, keyed by scope"""

    def __init__(self):
        self.edge, self.pool, self.act = [], {}, {}

    def edge_max(self, z, pre=None, inner=None):
        """max over k of the activated edge values z; given their pre-relu values `pre`, a maximum within 1e-5 of the relu's zero on
        either side is ambiguous too, and given a fused first layer's pre-relu values `inner` (b, n, k, c1), so is a maximum whose
        edge has a unit of that layer within 1e-5 of zero (the kernel's relu may fall the other way there)"""
        amb = _ambiguous(z, 2)
        if pre is not None:
            amb |= _near_zero_max(pre, 2, float(z.detach().abs().max()))
        if inner is not None:
            amb |= _inner_flip(pre, inner)
        out = z.amax(dim=2)
        _zero_at(out, amb)
        self.edge.append(amb)
        return out

    def point_max(self, y, scope, pre=None):
        amb = _ambiguous(y, 1)
        if pre is not None:
            amb |= _near_zero_max(pre, 1, float(y.detach().abs().max()))
        _zero_at(y, amb.unsqueeze(1))
        self.pool[scope] = amb
        return y.amax(dim=1)

    def head_layer(self, h, P, scope, frozen, stats=None):
        z = _layer(h, P, scope, frozen, relu=False, stats=stats)
        near = _near_zero(z)
        out = torch.relu(z)
        _zero_at(out, near)
        self.act[scope] = near
        return out

    def count(self):
        ms = self.edge + list(self.pool.values()) + list(self.act.values())
        return sum(int(m.sum()) for m in ms), sum(m.numel() for m in ms)

    def patch(self, monkeypatch):
        """zero the gradient at the same maxima on the GPU path: hooks on the outputs of its EdgeConv and pooled MLP nodes"""
        edge, pool, act = iter(self.edge), self.pool, self.act
        ec, mlp = training.edgeconv_training, training.mlp_training

        def edgeconv_training(*a, **kw):
            out = ec(*a, **kw)
            _zero_at(out, next(edge))
            return out

        def mlp_training(x, layers, *a, **kw):
            out = mlp(x, layers, *a, **kw)
            scope = layers[-1][0]
            if scope in pool:
                _zero_at(out, pool[scope].unsqueeze(1))
            if scope in act:
                _zero_at(out, act[scope])
            return out

        monkeypatch.setattr(training, "edgeconv_training", edgeconv_training)
        monkeypatch.setattr(training, "mlp_training", mlp_training)


def _dgcnn64(x, P, graphs, frozen, masks: _Masks, detach_transform=False, stats=None):
    """dgcnn.get_model (dgcnn.py:24-102, transform_nets.py:10-55) in float64, dropout off, on the given neighbour graphs -> logits;
    stats (a dict): every layer's batch statistics, by scope"""
    b, n, _ = x.shape
    L = lambda h, s, **kw: _layer(h, P, s, frozen, stats=stats, **kw)        # noqa: E731
    sc = "transform_net1"
    y1 = L(_edges(x, graphs[0]), f"{sc}/tconv1", relu=False)
    y = L(torch.relu(y1), f"{sc}/tconv2", relu=False)
    h = masks.edge_max(torch.relu(y), pre=y, inner=y1)
    y = L(h, f"{sc}/tconv3", relu=False)
    h = masks.point_max(torch.relu(y), f"{sc}/tconv3", pre=y)
    h = L(L(h, f"{sc}/tfc1"), f"{sc}/tfc2")
    t = (h @ P[f"{sc}/transform_XYZ/weights"] + P[f"{sc}/transform_XYZ/biases"] + torch.eye(3, dtype=x.dtype, device=x.device).flatten())
    t = t.reshape(b, 3, 3)
    h = torch.bmm(x, t.detach() if detach_transform else t)
    nets = []
    for i, s in enumerate(["dgcnn1", "dgcnn2", "dgcnn3", "dgcnn4"]):
        y = L(_edges(h, graphs[i + 1]), s, relu=False)
        h = masks.edge_max(torch.relu(y), pre=y)
        nets.append(h)
    y = L(torch.cat(nets, dim=-1), "agg", relu=False)
    g = masks.point_max(torch.relu(y), "agg", pre=y)
    for s in ("fc1", "fc2"):
        g = masks.head_layer(g, P, s, frozen, stats)
    return L(g, "fc3", bn=False)


def _dgcnn_setup(b, n, seed, bga=False, tnet_weights=True):
    p = dgcnn.init_params(seed=seed, randomize_bn=True, bga=bga)
    if tnet_weights:             # zero in the reference's initialisation: give the T-net a gradient path
        g = torch.Generator(device="cuda").manual_seed(seed)
        with torch.no_grad():
            p["transform_net1/transform_XYZ/weights"].normal_(0, 0.01, generator=g)
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
    P = _p64(p)                  # training mode updates only the moving averages, which batch statistics do not read
    want = []
    for detach in (False, True) if with_detached else (False,):
        masks = _Masks()
        x64 = x0.double().requires_grad_(True)
        l64 = _dgcnn64(x64, P, graphs, frozen, masks, detach_transform=detach)
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
    assert _bit_equal(_moving(p), moving0), "inference mode must not update the moving averages"
    assert torch.equal(fp.flat.detach(), flat0) and torch.equal(fp.grad, grad0), "inference mode must leave the flat buckets alone"
    assert fp.flat.grad is None


@pytest.mark.gpu
@pytest.mark.parametrize("c,cout,k", [(3, 64, 20), (64, 64, 20), (64, 128, 20), (64, 64, 1), (64, 32, 40)])
def test_frozen_edgeconv_matches_float64(c, cout, k):
    """eval-mode batch norm on randomised moving averages; dyadic-grid inputs (every edge value exact in fp32), self-loops and a
    cloud of duplicated points, so tied maxima and their even split occur"""
    b, n, s = 3, 300, "e"
    p = _store1(c, cout, seed=c + cout + k)
    _randomize_moving(p, [s], seed=k)
    x_np = _grid_x(b, n, c, seed=k)
    x_np[1, n // 2:] = x_np[1, :n // 2]
    rng = np.random.default_rng(7)
    idx_np = rng.integers(0, n, (b, n, k)).astype(np.int32)
    idx_np[:, :, 0] = np.arange(n)
    idx_np[1, :, 1 % k] = (np.arange(n) + n // 2) % n
    x = torch.tensor(x_np, device="cuda", requires_grad=True)
    idx = torch.tensor(idx_np, device="cuda")
    R = torch.tensor(np.random.default_rng(11).standard_normal((b, n, cout)).astype(np.float32), device="cuda")
    P = _p64(p)
    moving0 = _moving(p)

    out = training.edgeconv_training(x, idx, s, None, p, frozen=True)
    flat0, grad0 = _flat_state(p)
    assert out.shape == (b, n, cout) and out.grad_fn is not None
    (gx,) = torch.autograd.grad(out, [x], R)
    x64 = x.detach().double().requires_grad_(True)
    o64 = _layer(_edges(x64, idx), P, s, True).amax(dim=2)
    (want,) = torch.autograd.grad(o64, [x64], R.double())
    assert _out_err(out.detach().cpu(), o64.detach().cpu()) < OTOL
    assert _rel(gx.cpu(), want.cpu()) < GTOL
    _check_variables_untouched(p, moving0, flat0, grad0)
    ties = p._trainers[("edgeconv_frozen", s, b, n, c, k)].ties
    assert k == 1 or int(ties.max()) > 1                                           # the even split was exercised
    assert ("edgeconv", s, b, n, c, k) not in p._trainers


def _store2(c, seed):
    p = VariableStore(device="cuda", seed=seed)
    p.add_conv2d(S1, 2 * c, 64, randomize_bn=True)
    p.add_conv2d(S2, 64, 128, randomize_bn=True)
    rng = np.random.default_rng(seed)
    for s, n in ((S1, 64), (S2, 128)):
        p[f"{s}/biases"] = torch.tensor(rng.standard_normal(n) * 0.1, dtype=torch.float32, device="cuda")
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
    P = _p64(p)
    moving0 = _moving(p)

    x64 = x.detach().double().requires_grad_(True)
    z64 = _layer(_layer(_edges(x64, idx), P, S1, True), P, S2, True)
    o64 = z64.amax(dim=2)
    amb = _ambiguous(z64, 2)
    R = torch.tensor(rng.standard_normal((b, n, 128)).astype(np.float32), device="cuda")
    R[amb] = 0.0
    print(f"[frozen edgeconv2 k={k}] ambiguous maxima masked: {int(amb.sum())} of {amb.numel()}")
    assert float(amb.double().mean()) < 0.01

    out = training.edgeconv_training(x, idx, (S1, S2), None, p, frozen=True)
    flat0, grad0 = _flat_state(p)
    assert out.shape == (b, n, 128) and out.grad_fn is not None
    (gx,) = torch.autograd.grad(out, [x], R)
    (want,) = torch.autograd.grad(o64, [x64], R.double())
    assert _out_err(out.detach().cpu(), o64.detach().cpu()) < OTOL
    assert _rel(gx.cpu(), want.cpu()) < GTOL
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
    assert _out_err(logits.cpu(), l64.cpu()) < OTOL
    assert _rel(gx.cpu(), want.cpu()) < GTOL
    assert _rel(want_detached.cpu(), want.cpu()) > 10 * GTOL           # the T-net's share is visible ...
    assert _rel(gx.cpu(), want_detached.cpu()) > 10 * GTOL             # ... and the frozen path carries it


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
    assert _rel(on_fused_graphs.detach().cpu(), fused.cpu()) < 1e-4
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
    moving0 = _moving(p)
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
    assert _rel(grads[0].cpu(), grads[1].cpu()) > 100 * GTOL, "the segmentation head's gradient did not reach the cloud"
    assert _bit_equal(_moving(p), moving0)
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
        runs.append((logits.detach(), p._flat.flat.grad.clone(), _moving(p), x.grad))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1]) and _bit_equal(runs[0][2], runs[1][2])
    assert bool(torch.isfinite(runs[0][3]).all()) and float(runs[0][3].abs().max()) > 0 and runs[1][3] is None
    gx, want, _, _, _, masked, total = _dgcnn_against_float64(b, n, seed=7, monkeypatch=monkeypatch, frozen=False)
    print(f"[dgcnn training B={b} N={n}] masked: {masked} of {total}; x.grad error relative to the largest entry: "
          f"{_rel(gx.cpu(), want.cpu()):.2e}")
    assert masked <= 0.01 * total
    assert _rel(gx.cpu(), want.cpu()) < GTOL


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
          f"x.grad error relative to the largest entry: {_rel(gx.cpu(), want.cpu()):.2e}")
    assert masked <= 0.01 * total
    assert _out_err(logits.cpu(), l64.cpu()) < OTOL
    assert _rel(gx.cpu(), want.cpu()) < GTOL


# ---------------------------------------------------------------------------------------------------------------------
# 8. vanilla PointNet
# ---------------------------------------------------------------------------------------------------------------------
def _pointnet64(x, P, masks: _Masks):
    """pointnet_cls.get_model (pointnet_cls.py:21-75) in float64 with frozen batch norm -> (logits, feature transform)"""
    b = x.shape[0]
    L = lambda h, s, **kw: _layer(h, P, s, True, **kw)        # noqa: E731

    def tnet(h, scope, K):
        g = masks.point_max(L(L(L(h, f"{scope}/tconv1"), f"{scope}/tconv2"), f"{scope}/tconv3"), f"{scope}/tconv3")
        g = L(L(g, f"{scope}/tfc1"), f"{scope}/tfc2")
        name = "transform_XYZ" if K == 3 else "transform_feat"
        eye = torch.eye(K, dtype=x.dtype, device=x.device).flatten()
        return (g @ P[f"{scope}/{name}/weights"] + P[f"{scope}/{name}/biases"] + eye).reshape(b, K, K)

    h = torch.bmm(x, tnet(x, "transform_net1", 3))
    h = L(L(h, "conv1"), "conv2")
    t2 = tnet(h, "transform_net2", 64)
    h = torch.bmm(h, t2)
    g = masks.point_max(L(L(L(h, "conv3"), "conv4"), "conv5"), "conv5")
    for s in ("fc1", "fc2"):
        g = masks.head_layer(g, P, s, True)
    return L(g, "fc3", bn=False), t2


@pytest.mark.gpu
def test_pointnet_inference_input_grad(monkeypatch):
    b, n = 8, 1024
    p = pointnet_cls.init_params(seed=2, randomize_bn=True)
    with torch.no_grad():
        for s, name in (("transform_net1", "transform_XYZ"), ("transform_net2", "transform_feat")):
            p[f"{s}/{name}/weights"].normal_(0, 0.01, generator=torch.Generator(device="cuda").manual_seed(2))
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
    moving0 = _moving(p)
    # float64 restatement, then the frozen path with the same maxima masked
    masks = _Masks()
    x64 = x0.double().requires_grad_(True)
    l64, t64 = _pointnet64(x64, _p64(p), masks)
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
    assert _out_err(logits.detach().cpu(), l64.detach().cpu()) < OTOL
    assert _rel(logits.detach().cpu(), fused.cpu()) < 1e-4 and torch.equal(logits.argmax(-1), fused.argmax(-1))
    assert _rel(x.grad.cpu(), x64.grad.cpu()) < GTOL
    assert _bit_equal(_moving(p), moving0)
    assert p._flat.flat.grad is None
