"""SpiderCNN's training backward (csrc/spider.cu, spidercnn_cls_xyz.get_model_training) against float64.

1. Each op on random inputs against its float64 formula, relative to each tensor's largest entry, with a plain float32 evaluation of
   the same formula beside it (torch, TF32 off): an error beyond 1e-4 must stay within 2x the float32 one.  Shapes: the four layers,
   c = 3, row counts that leave a partial tile ((9, 1000), (33, 1000)) and B=32, N=1024.
2. One training step (dropout off, loss (logits * R).sum()) against the float64 restatement spidercnn() below, variable by variable:
   logits and the fc1 / fc2 moving averages within 1e-5, every flat-gradient slice within 1e-4 (or 2x float32's own error), fc1 / fc2
   biases exactly zero.  The restatement takes the run's relu gates; pooled entries whose top-2 is within 1e-5 of a tie or of the relu's zero are
   masked on both sides; at most 1% of either.
3. Two steps from the same state give bit-identical gradients and moving averages.
4. The allocation peak of one forward + backward at B=32, N=1024 stays below the 1.68 GB of fanConv4's conv input alone."""
import ctypes as C

import numpy as np
import pytest
import torch

from scanobjectnn_b200 import _lib, ops
from scanobjectnn_b200 import spidercnn_cls_xyz as M
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.training import _plain_grad

from . import gpu_util as G
from .restate import err, flat_grad, layer, params_as, within, zero_at

OTOL, GTOL = 1e-5, 1e-4
K, T = 20, 5
LAYERS = [(3, 32), (32, 64), (64, 128), (128, 256)]


# ---------------------------------------------------------------------------------------------------------------------
# the float64 restatement of spidercnn_cls_xyz in training mode
# ---------------------------------------------------------------------------------------------------------------------
SPIDER_TAYLOR = ("weight_x", "weight_y", "weight_z", "weight_xyz", "weight_xy", "weight_yz", "weight_xz", "biases", "weight_xx",
                 "weight_yy", "weight_zz", "weight_xxy", "weight_xyy", "weight_xxz", "weight_xzz", "weight_yyz", "weight_yzz",
                 "weight_xxx", "weight_yyy", "weight_zzz")


def spider_monomials(delta):
    """(..., 3) -> (..., 20) in the order of SPIDER_TAYLOR"""
    X, Y, Z = delta[..., 0], delta[..., 1], delta[..., 2]
    one = torch.ones_like(X)
    return torch.stack([X, Y, Z, X * Y * Z, X * Y, Y * Z, X * Z, one, X * X, Y * Y, Z * Z, X * X * Y, X * Y * Y, X * X * Z, X * Z * Z,
                        Y * Y * Z, Y * Z * Z, X * X * X, Y * Y * Y, Z * Z * Z], dim=-1)


def spider_gather(feat, idx):
    """feat (B,N,C), idx (B,N,k) -> (B,N,k,C)"""
    return feat[torch.arange(feat.shape[0], device=feat.device)[:, None, None], idx.long()]


def spider_group_norm(y, gamma, beta, G, eps=1e-6):
    """group_norm_for_conv on (B,N,C): moments over (C/G channels, N points) per cloud and group"""
    b, n, c = y.shape
    yt = y.reshape(b, n, G, c // G)
    mean = yt.mean(dim=(1, 3), keepdim=True)
    var = ((yt - mean) ** 2).mean(dim=(1, 3), keepdim=True)
    return ((yt - mean) / torch.sqrt(var + eps)).reshape(b, n, c) * gamma + beta


def spidercnn(xyz, idx, P, gates=None, pool_mask=None, stats=None, info=None):
    """spidercnn_cls_xyz in training mode in P's dtype, dropout off: four spiderConv layers (group norm, relu), top-2 pooling, fc1 / fc2
    with batch statistics (biased variance, recorded in `stats`), fc3.  gates (l -> bool (B,N,C)): the run's relu gates, used in place
    of float64's own, whose disagreements `info` counts ("flips" of "units"); pool_mask (B,960): pooled entries whose gradient is
    zeroed."""
    dt = P["fc1/weights"].dtype
    xyz = xyz.to(dt)
    delta = spider_gather(xyz, idx) - xyz[:, :, None, :]
    mono = spider_monomials(delta)
    feat, hs = xyz, []
    for l in range(1, 5):
        sc = f"fanConv{l}/taylor"
        taylor = torch.cat([P[f"{sc}/{m}"].reshape(1, -1) for m in SPIDER_TAYLOR])              # (20,T)
        g = mono @ taylor                                                                        # (B,N,k,T)
        w = P[f"{sc}/conv/weights"]
        k, ct, cout = w.shape[1:]
        c = feat.shape[-1]
        y = torch.einsum("bnjc,bnjt,jcto->bno", spider_gather(feat, idx), g, w.reshape(k, c, ct // c, cout)) + P[f"{sc}/conv/biases"]
        z = spider_group_norm(y, P[f"{sc}/conv/gn/gamma"], P[f"{sc}/conv/gn/beta"], min(16, cout))
        if gates is not None:
            info["flips"] += int((gates[l] != (z > 0)).sum())
            info["units"] += z.numel()
            h = z * gates[l]
        else:
            h = torch.relu(z)
        hs.append(h)
        feat = h
    pooled = torch.topk(torch.cat(hs, dim=2).permute(0, 2, 1), 2, dim=-1, sorted=True).values.reshape(xyz.shape[0], -1)
    if pool_mask is not None:
        zero_at(pooled, pool_mask)
    net = layer(pooled, P, "fc1", False, stats=stats)
    net = layer(net, P, "fc2", False, stats=stats)
    return layer(net, P, "fc3", False, bn=False)


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


def _inputs(b, n, c, cout, seed):
    gen = torch.Generator(device="cpu").manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=gen)                        # noqa: E731
    d = dict(idx=torch.randint(0, n, (b, n, K), generator=gen, dtype=torch.int32), delta=0.3 * r(b, n, K, 3), taylor=r(20, T) / 3,
             feat=r(b, n, c), W=r(K, c * T, cout) / np.sqrt(K * c * T), dy=r(b, n, cout))
    if c != 3:
        d.update(fs=0.5 + torch.rand(b, c, generator=gen), fu=0.3 * r(b, c))
    return {k: v.cuda() for k, v in d.items()}


def _formulas(x, dt):
    """the backward's float64 (or float32) formulas on the op inputs x; g is the run's own (an input of the products)"""
    c = x["feat"].shape[-1]
    cout = x["dy"].shape[-1]
    h = x["feat"].to(dt)
    if "fs" in x:
        h = torch.relu(h * x["fs"].to(dt)[:, None] + x["fu"].to(dt)[:, None])
    hn = spider_gather(h, x["idx"])                                         # (B,N,k,c)
    g, dy, W = x["g"].to(dt), x["dy"].to(dt), x["W"].to(dt).reshape(K, c, T, cout)
    out = {"g": spider_monomials(x["delta"].to(dt)) @ x["taylor"].to(dt)}
    out["dW"] = torch.einsum("bnjc,bnjt,bno->jcto", hn, g, dy).reshape(K, c * T, cout)
    out["db"] = dy.sum(dim=(0, 1))
    Q = torch.einsum("bno,jcto->bnjct", dy, W)
    out["D"] = torch.einsum("bnjct,bnjt->bnjc", Q, g)
    out["dg"] = torch.einsum("bnjct,bnjc->bnjt", Q, hn)
    del Q
    b, n = dy.shape[:2]
    flat = (x["idx"].long() + torch.arange(b, device=dy.device)[:, None, None] * n).reshape(-1)
    dh = torch.zeros((b * n, c), dtype=dt, device=dy.device)
    out["dh"] = dh.index_add_(0, flat, out["D"].reshape(-1, c)).reshape(b, n, c)
    out["dtaylor"] = torch.einsum("bnjt,bnjm->mt", out["dg"], spider_monomials(x["delta"].to(dt)))
    return out


OP_SHAPES = [(2, 256, c, cout) for c, cout in LAYERS] + [(9, 1000, 32, 64), (33, 1000, 128, 256), (9, 1000, 3, 32), (32, 1024, 128, 256)]


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,c,cout", OP_SHAPES)
def test_spider_conv_backward_ops_match_float64(b, n, c, cout):
    x = _inputs(b, n, c, cout, seed=b * 7 + c)
    fs, fu = x.get("fs"), x.get("fu")
    g = ops.spider_taylor_filter(x["delta"], x["taylor"])
    x["g"] = g
    got = {"g": g, "dW": ops.spider_conv_bwd_weight(x["idx"], x["feat"], g, x["dy"], fs, fu)}
    D, dg = ops.spider_conv_bwd_data(x["idx"], x["feat"], g, x["W"], x["dy"], fs, fu, want_D=c != 3)
    got["dg"] = dg
    got["dtaylor"] = ops.spider_taylor_grad(x["delta"], dg)
    db = torch.empty(cout, device="cuda")
    gi = _plain_grad(x["dy"].view(b * n, cout))
    _lib.check(_lib.load().psa_train_bias_grad(b * n, cout, C.byref(gi), _lib.ptr(db), _lib.stream()), "train_bias_grad")
    got["db"] = db
    if c != 3:
        got["D"] = D
        got["dh"] = _gpg(D, x["idx"], n)
    else:
        assert D is None
    # the float64 formula of dtaylor takes the run's own dg, so that it checks d taylor alone
    w64, w32 = _formulas(x, torch.float64), _formulas(x, torch.float32)
    mono = spider_monomials(x["delta"].double())
    w64["dtaylor"] = torch.einsum("bnjt,bnjm->mt", dg.double(), mono)
    w32["dtaylor"] = torch.einsum("bnjt,bnjm->mt", dg, mono.float())
    for name, v in got.items():
        e, e32 = err(v, w64[name]), err(w32[name], w64[name])
        print(f"{name}: {e:.2e} (float32 {e32:.2e})")
        assert within(e, e32, GTOL, 2), (name, e, e32)


def _gpg(D, idx, n):
    """psa_group_point_grad through group_point's autograd: the gradient of group_point(points, idx) for grad_out = D"""
    pts = torch.zeros((D.shape[0], n, D.shape[-1]), device="cuda", requires_grad=True)
    ops.group_point(pts, idx).backward(D)
    return pts.grad


GN_SHAPES = [(2, 256, 32), (2, 256, 64), (2, 256, 128), (2, 256, 256), (9, 1000, 64), (33, 1000, 256), (32, 1024, 256)]


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,c", GN_SHAPES)
def test_spider_gn_topk_backward_matches_float64(b, n, c):
    gen = torch.Generator(device="cpu").manual_seed(b + c)
    y = (torch.randn(b, n, c, generator=gen) * 2 + 0.5).cuda()
    gamma = (0.8 + 0.4 * torch.rand(c, generator=gen)).cuda()
    beta = (0.2 * torch.randn(c, generator=gen)).cuda()
    P = 480
    off = 7
    dpool = torch.randn(b, P, 2, generator=gen).cuda()
    dh_next = torch.randn(b, n, c, generator=gen).cuda()
    G_ = min(16, c)
    scale, shift = ops.group_norm_affine(y, gamma, beta, G_)
    dy, dgamma, dbeta = ops.spider_gn_bwd(y, scale, shift, gamma, G_, dpool, off, dh_next)
    gate = (y.double() * scale.double()[:, None] + shift.double()[:, None]) > 0          # the run's relu gate

    def formula(dt):
        yy = y.to(dt).requires_grad_(True)
        gm, bt = gamma.to(dt).requires_grad_(True), beta.to(dt).requires_grad_(True)
        yt = yy.reshape(b, n, G_, c // G_)
        mean = yt.mean(dim=(1, 3), keepdim=True)
        var = ((yt - mean) ** 2).mean(dim=(1, 3), keepdim=True)
        z = ((yt - mean) / torch.sqrt(var + 1e-6)).reshape(b, n, c) * gm + bt
        h = z * gate
        top = torch.topk(h.permute(0, 2, 1), 2, dim=-1).values
        ((top * dpool[:, off:off + c].to(dt)).sum() + (h * dh_next.to(dt)).sum()).backward()
        return yy.grad, gm.grad, bt.grad

    w64, w32 = formula(torch.float64), formula(torch.float32)
    for name, v, a, a32 in zip(("dy", "dgamma", "dbeta"), (dy, dgamma, dbeta), w64, w32):
        e, e32 = err(v, a), err(a32, a)
        print(f"{name}: {e:.2e} (float32 {e32:.2e})")
        assert within(e, e32, GTOL, 2), (name, e, e32)


# ---------------------------------------------------------------------------------------------------------------------
# the model-level step
# ---------------------------------------------------------------------------------------------------------------------
def _pool_mask(ep, b):
    """(B,960) pooled entries whose top-2 lies within 1e-5 (of the largest activation) of a tie with the next point or of the relu's
    zero, from the run's own activations"""
    hs = [torch.relu(ep[f"y{l}"].double() * ep[f"scale{l}"].double()[:, None] + ep[f"shift{l}"].double()[:, None]) for l in range(1, 5)]
    h = torch.cat(hs, dim=2).permute(0, 2, 1)
    v = torch.topk(h, 3, dim=-1).values
    tol = 1e-5 * float(h.abs().max())
    amb = ((v[..., 0] - v[..., 1]) < tol) | ((v[..., 1] - v[..., 2]) < tol) | (v[..., 1] < tol)
    return amb[..., None].expand(b, 480, 2).reshape(b, 960)


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,seed", [(4, 256, 1), (16, 1024, 2), (32, 1024, 3)])
def test_spidercnn_training_step_matches_float64(b, n, seed, monkeypatch):
    p = M.init_params(seed=seed, randomize_bn=True)
    xyz = G.cu(make_clouds("ball", b, n, seed=seed + 100))
    R = torch.tensor(np.random.default_rng(seed).standard_normal((b, M.NUM_CLASSES)).astype(np.float32), device="cuda")
    with torch.no_grad():
        _, ep = M.get_model_training(xyz, None, params=p, dropout=False, return_end_points=True)
    idx = ep["idx"].clone()
    gates = {l: (ep[f"y{l}"].double() * ep[f"scale{l}"].double()[:, None] + ep[f"shift{l}"].double()[:, None]) > 0 for l in range(1, 5)}
    mask = _pool_mask(ep, b)
    P0 = params_as(p, torch.float64)

    orig = M._SpiderFn.apply

    def masked_apply(*a):
        out = orig(*a)
        out.register_hook(lambda g: g.masked_fill(mask, 0.0))
        return out

    p._flat.flat.grad = None
    with monkeypatch.context() as m:
        m.setattr(M._SpiderFn, "apply", masked_apply)
        logits = M.get_model_training(xyz, None, params=p, dropout=False)
        (logits * R).sum().backward()

    res = {}
    for dt in (torch.float64, torch.float32):
        P = params_as(P0, dt, grad=True)
        stats, info = {}, {"flips": 0, "units": 0}
        out = spidercnn(xyz, idx, P, gates={l: gates[l] for l in gates}, pool_mask=mask, stats=stats, info=info)
        (out * R.to(dt)).sum().backward()
        res[dt] = (out.detach(), P, stats, info)
    l64, P64, st64, info64 = res[torch.float64]
    l32, P32, st32, _ = res[torch.float32]
    masked, flips = float(mask.double().mean()), info64["flips"] / info64["units"]
    print(f"B={b} N={n}: pooled masked {masked:.2%}, relu gates differing from float64's {flips:.4%}")
    assert masked <= 0.01 and flips <= 0.01

    errs = {"logits": (err(logits, l64), err(l32, l64))}
    for scope in ("fc1", "fc2"):
        for i, suffix in enumerate(("moving_mean", "moving_variance")):
            name = f"{scope}/bn/{suffix}"
            want = 0.1 * st64[scope][i] + 0.9 * P0[name]
            errs[name] = (err(p[name], want), err(0.1 * st32[scope][i].double() + 0.9 * P0[name], want))
    for name in p._flat.names:
        got = flat_grad(p, name)
        if name in ("fc1/biases", "fc2/biases"):
            assert not bool(got.any()), f"{name}: a bias followed by batch norm must get a gradient of exactly zero"
            continue
        want = P64[name].grad
        errs[name] = (err(got, want), err(P32[name].grad, want))
    assert sum(1 for k in errs if "/taylor/weight_" in k or k.endswith("/taylor/biases")) == 80
    bad = []
    for key, (e, e32) in sorted(errs.items()):
        tol = OTOL if key == "logits" or "moving" in key else GTOL
        print(f"  {key}: {e:.2e} (float32 {e32:.2e})")
        if not within(e, e32, tol, 2):
            bad.append((key, e, e32))
    assert not bad, bad


@pytest.mark.gpu
def test_spidercnn_training_step_is_bit_reproducible():
    b, n = 8, 512
    p = M.init_params(seed=4, randomize_bn=True)
    xyz = G.cu(make_clouds("ball", b, n, seed=104))
    R = torch.randn(b, M.NUM_CLASSES, device="cuda")
    moving = [k for k in p if k.endswith(("moving_mean", "moving_variance"))]
    start = {k: p[k].clone() for k in moving}
    runs = []
    for _ in range(2):
        for k in moving:
            p[k].copy_(start[k])
        if getattr(p, "_flat", None) is not None:
            p._flat.flat.grad = None
        logits = M.get_model_training(xyz, None, params=p, dropout=False)
        (logits * R).sum().backward()
        runs.append((p._flat.flat.grad.clone(), [p[k].clone() for k in moving]))
    assert torch.equal(runs[0][0], runs[1][0])
    assert all(torch.equal(a, c) for a, c in zip(runs[0][1], runs[1][1]))


@pytest.mark.gpu
def test_spidercnn_training_allocation_peak():
    b, n = 32, 1024
    p = M.init_params(seed=5)
    xyz = G.cu(make_clouds("ball", b, n, seed=105))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    logits = M.get_model_training(xyz, None, params=p)
    logits.sum().backward()
    torch.cuda.synchronize()
    rise = torch.cuda.max_memory_allocated() - base
    print(f"allocation peak of one forward + backward at B={b}, N={n}: {rise / 1e6:.0f} MB")
    assert rise < 1.68e9
