"""PointCNN's training path (csrc/pointcnn_train.cu, pointcnn_cls.get_model_training) against float64.

1. Each X-Conv layer's forward on the run's own inputs, at B=32, N=1024 and at B=3, N=1000 (partial tiles): the saved activations
   within 1e-5 * max(1, |max|) of float64, the batch statistics and the 0.99 moving-average update within 1e-6 of each vector's
   largest entry (one fp32 rounding of a value near zero is larger than 1e-6 of itself), and the core's
   depthwise output bit-identical to psa_xconv_core called with the batch (s, t).
2. Each layer's backward for a random upstream gradient: every weight and batch-norm gradient and the previous layer's feature
   gradient within 1e-4 of the tensor's largest entry against float64 autograd, or within 2x a float32 evaluation's own error.
3. Whole steps against the float64 restatement pointcnn_training() below, replayed on the run's kNN indices and dropout mask, with the
   tiled cross-entropy and with (logits * R).sum(): logits and every moving average within 1e-5 * max(1, |max|), every flat-gradient
   slice within 1e-4 (or 2x float32's own error), in arithmetic modes 0, 1 and 2, dropout off and on.
4. Two steps from the same state give bit-identical logits, gradients and moving averages.
5. The regularisation loss's gradient is 1e-5 * v on the regularised variables and 0 on logits/bias.
6. Adam (eps 1e-2) on one fixed batch lowers the loss; get_model after a step and params.invalidate() matches the oracle.
7. The allocation peak of one forward + backward at B=32, N=1024 stays under 512 MiB.

ELU's derivative is continuous, so unlike the ReLU models no gate or winner needs to be replayed: only the kNN indices (index ops
carry no gradient) and the dropout mask."""
import numpy as np
import pytest
import torch

from oracle import pointcnn_oracle as po
from scanobjectnn_b200 import ops
from scanobjectnn_b200 import pointcnn_cls as M
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import BN_EPS

from .restate import err, flat_grad, params_as, within

OTOL, GTOL = 1e-5, 1e-4


# ---------------------------------------------------------------------------------------------------------------------
# the float64 restatement of pointcnn_cls in training mode
# ---------------------------------------------------------------------------------------------------------------------
def elu(x):
    """tf.nn.elu"""
    return torch.where(x > 0, x, torch.expm1(torch.clamp(x, max=0.0)))


def bn(x, P, layer, frozen, stats=None):
    """tf.layers.batch_normalization over the last axis: the moving averages when frozen, else the batch's mean and biased variance
    over every other axis (recorded in stats[layer])"""
    c = x.shape[-1]
    if frozen:
        mu, var = P[f"{layer}_bn/moving_mean"].to(x.dtype), P[f"{layer}_bn/moving_variance"].to(x.dtype)
    else:
        flat = x.reshape(-1, c)
        mu, var = flat.mean(0), flat.var(0, unbiased=False)
        if stats is not None:
            stats[layer] = (mu.detach(), var.detach())
    return (x - mu) / torch.sqrt(var + BN_EPS) * P[f"{layer}_bn/gamma"].to(x.dtype) + P[f"{layer}_bn/beta"].to(x.dtype)


def dense(x, P, layer, frozen, stats=None, var="kernel"):
    """pf.dense / pf.conv2d (1x1) with_bn: BN(elu(x . W)), no bias"""
    w = P[f"{layer}/{var}"].to(x.dtype)
    return bn(elu(x @ w.reshape(-1, w.shape[-1])), P, layer, frozen, stats)


def xconv(P, tag, pts, qrs, idx, fts, K, glob, frozen, stats=None, acts=None):
    """pointcnn.py:10-52 -> (B, P, glob + C); acts collects the pre-batch-norm activations a = elu(z) (z for X_2) and dw"""
    B, Pq = idx.shape[:2]
    bi = torch.arange(B, device=idx.device)[:, None, None]
    local = pts[bi, idx] - qrs[:, :, None, :]
    a = {} if acts is None else acts
    h0 = dense(local, P, f"{tag}nn_fts_from_pts_0", frozen, stats)
    lifted = dense(h0, P, f"{tag}nn_fts_from_pts", frozen, stats)
    Fm = lifted if fts is None else torch.cat([lifted, fts[bi, idx]], dim=-1)
    dt = pts.dtype
    w0 = P[f"{tag}X_0/kernel"].to(dt)[0]
    a["x0"] = elu(torch.einsum("bpjd,jdo->bpo", local, w0))
    X0 = bn(a["x0"], P, f"{tag}X_0", frozen, stats).reshape(B, Pq, K, K)
    a["x1"] = elu(torch.einsum("pqab,abm->pqbm", X0, P[f"{tag}X_1/depthwise_weights"].to(dt)[0]).reshape(B, Pq, K * K))
    X1 = bn(a["x1"], P, f"{tag}X_1", frozen, stats).reshape(B, Pq, K, K)
    a["x2"] = torch.einsum("pqab,abm->pqbm", X1, P[f"{tag}X_2/depthwise_weights"].to(dt)[0]).reshape(B, Pq, K * K)
    X2 = bn(a["x2"], P, f"{tag}X_2", frozen, stats).reshape(B, Pq, K, K)
    fts_X = X2 @ Fm
    a["dw"] = torch.einsum("pqic,icm->pqcm", fts_X, P[f"{tag}fts_conv/depthwise_kernel"].to(dt)[0]).reshape(B, Pq, -1)
    out = dense(a["dw"], P, f"{tag}fts_conv", frozen, stats, var="pointwise_kernel")
    if glob:
        out = torch.cat([dense(dense(qrs, P, f"{tag}fts_global_0", frozen, stats), P, f"{tag}fts_global", frozen, stats), out], dim=-1)
    return out


def pointcnn_training(points, P, idx_list, frozen=False, mask=None, stats=None, mean=False):
    """pointcnn_cls on points (B,N,3) in their dtype with the run's kNN indices: batch statistics (recorded in stats) or, frozen, the
    moving averages; fc1 times the dropout mask (B*128, 192) when given; per-point logits (B, 128, num_class), or with mean the
    inference head's mean over the points first (B, 1, num_class)"""
    n = points.shape[1]
    pts, fts = points, None
    for (tag, k, _, p, _, _, _, _, glob), idx in zip(M.layer_table(), idx_list):
        p = n if p == -1 else p
        qrs = pts[:, :p]
        fts = xconv(P, tag, pts, qrs, idx.long(), fts, k, glob, frozen, stats)
        pts = qrs
    net = fts
    for i in range(len(M.FC)):
        net = dense(net, P, f"fc{i}", frozen, stats)
    if mask is not None:
        net = net * mask.reshape(net.shape).to(net.dtype)
    if mean:
        net = net.mean(dim=1, keepdim=True)
    return net @ P["logits/kernel"].to(net.dtype) + P["logits/bias"].to(net.dtype)


def moving_update(P, stats, decay=M.BN_DECAY):
    """the moving averages after one step: decay * moving + (1 - decay) * batch"""
    out = {}
    for layer, (mu, var) in stats.items():
        for v, s in (("moving_mean", mu), ("moving_variance", var)):
            out[f"{layer}_bn/{v}"] = decay * P[f"{layer}_bn/{v}"].double() + (1 - decay) * s
    return out


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def oerr(got, want):
    """max |got - want| relative to max(1, the largest entry of want)"""
    return err(got, want, max(1.0, float(want.detach().abs().max())))


def _setup(b, n, seed):
    p = M.init_params(seed=seed, randomize_bn=True)
    x = torch.from_numpy(make_clouds("ball", b, n, seed=seed + 1)).cuda()
    return p, x


def _idx_list(ep):
    return [ep[f"idx{l}"].clone() for l in range(1, 5)]


# ---------------------------------------------------------------------------------------------------------------------
# 1. / 2. each layer on its own
# ---------------------------------------------------------------------------------------------------------------------
def _layer_inputs(tr, L, x):
    """the layer's points and input features as the run gave them"""
    i = L["l"] - 1
    pts = x if i == 0 else tr.layers[i - 1]["qrs"]
    fts = None if i == 0 else tr.layers[i - 1]["out"]
    return pts, fts


@pytest.mark.gpu
@pytest.mark.parametrize("b,n", [(32, 1024), (3, 1000)])
def test_layer_forward_matches_float64(b, n):
    p, x = _setup(b, n, 11)
    before = {k: v.clone() for k, v in p.items() if k.endswith(("moving_mean", "moving_variance"))}
    M.get_model_training(x, params=p, dropout=False)
    tr = p._trainers[("pointcnn_cls", b, n)]
    P = params_as(p, torch.float64)
    for k, v in before.items():
        P[k] = v.double()
    for L in tr.layers:
        pts, fts = _layer_inputs(tr, L, x)
        stats, acts = {}, {}
        qrs = pts[:, :L["P"]]
        want = xconv(P, L["tag"], pts.double(), qrs.double(), L["idx"].long(), None if fts is None else fts.double().view(b, -1, fts.shape[1]),
                     L["K"], L["glob"], False, stats, acts)
        got = {"x0": L["saved"]["a_x0"], "x1": L["saved"]["a_x1"], "x2": L["saved"]["a_x2"], "dw": L["dw"]}
        for name, g in got.items():
            w = acts[name].reshape(g.shape)
            assert oerr(g, w) < OTOL, (L["tag"], name, oerr(g, w))
        assert oerr(L["out"], want.reshape(L["out"].shape)) < OTOL, L["tag"]
        for short, bnl in L["bn"].items():
            mu, var = stats[bnl["layer"]]
            mi = bnl["mean_inv"].double()
            assert float((mi[0] - mu).abs().max()) < 1e-6 * max(1.0, float(mu.abs().max())), (bnl["layer"], "mean")
            assert float(((mi[1] - 1 / torch.sqrt(var + BN_EPS)) / mi[1]).abs().max()) < 1e-6, (bnl["layer"], "var")
            for v, s in (("moving_mean", mu), ("moving_variance", var)):
                exp = M.BN_DECAY * P[f"{bnl['layer']}_bn/{v}"] + (1 - M.BN_DECAY) * s
                assert err(p[f"{bnl['layer']}_bn/{v}"], exp) < 1e-6, (bnl["layer"], v)
        # the core run with the batch (s, t) gives the stored depthwise output bit for bit
        w = {"w_dw": L["W_dw"]}
        for short in ("pts0", "pts1", "x0", "x1", "x2"):
            w[f"w_{short}"], w[f"s_{short}"], w[f"t_{short}"] = L["bn"][short]["W"], L["bn"][short]["s"], L["bn"][short]["t"]
        dw = ops.xconv_core(pts, qrs.contiguous(), L["idx"], None if fts is None else fts.view(b, -1, fts.shape[1]), w, L["dm"])
        assert torch.equal(dw, L["dw"]), L["tag"]


def _layer_grads(P, L, pts, qrs, idx, fts, dout):
    """float64 / float32 autograd of one layer: the variables' and the input features' gradients for the upstream gradient dout"""
    out = xconv(P, L["tag"], pts, qrs, idx, fts, L["K"], L["glob"], False)
    names = [k for k in P if k.startswith(L["tag"]) and not k.endswith(("moving_mean", "moving_variance"))]
    inputs = [P[k] for k in names] + ([fts] if fts is not None else [])
    g = torch.autograd.grad((out.reshape(dout.shape) * dout.to(out.dtype)).sum(), inputs)
    return dict(zip(names + ["fts"], g))


@pytest.mark.gpu
@pytest.mark.parametrize("b,n", [(32, 1024), (3, 1000)])
def test_layer_backward_matches_float64(b, n):
    p, x = _setup(b, n, 12)
    M.get_model_training(x, params=p, dropout=False)
    tr = p._trainers[("pointcnn_cls", b, n)]
    gen = torch.Generator(device="cuda").manual_seed(b + n)
    for L in tr.layers:
        pts, fts = _layer_inputs(tr, L, x)
        tr.layer_forward(L, pts, fts)
        dout = torch.randn(L["out"].shape, generator=gen, device="cuda")
        d_fts = None if fts is None else torch.empty_like(fts)
        tr.fp.grad.zero_()
        tr.layer_backward(L, dout, d_fts)
        torch.cuda.synchronize()
        qrs = pts[:, :L["P"]]
        res = {}
        for dt in (torch.float64, torch.float32):
            P = params_as(p, dt, grad=True)
            f = None if fts is None else fts.to(dt).view(b, -1, fts.shape[1]).clone().requires_grad_(True)
            res[dt] = _layer_grads(P, L, pts.to(dt), qrs.to(dt), L["idx"].long(), f, dout)
        g64 = res[torch.float64]
        for name, w64 in g64.items():
            g = (d_fts.view(w64.shape) if name == "fts" else flat_grad(p, name, tr.fp.grad))
            scale = max(float(w64.abs().max()), float(g64[name.replace("/beta", "/gamma")].abs().max()) if name.endswith("_bn/beta") else 0.0)
            e, e32 = err(g, w64, scale), err(res[torch.float32][name], w64, scale)
            assert within(e, e32, GTOL, 2.0), (L["tag"], name, e, e32)


# ---------------------------------------------------------------------------------------------------------------------
# 3. whole steps
# ---------------------------------------------------------------------------------------------------------------------
def _step(p, x, label, dropout, loss_kind, R=None):
    logits, ep = M.get_model_training(x, params=p, dropout=dropout, return_end_points=True)
    loss = M.get_loss(logits, label) if loss_kind == "xent" else (logits * R).sum()
    loss.backward()
    return logits.detach().clone(), ep


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("b,n", [(3, 1000), (8, 1024), (32, 1024), (32, 2048)])
@pytest.mark.parametrize("dropout", [False, True])
def test_step_matches_float64(b, n, mode, dropout):
    old = ops.get_mlp_mode()
    ops.set_mlp_mode(mode)
    try:
        p, x = _setup(b, n, 21 + b)
        M.get_model_training(x, params=p, dropout=False)              # creates the flat store
        label = torch.randint(0, M.NUM_CLASSES, (b,), generator=torch.Generator().manual_seed(b)).cuda()
        R = torch.randn((b, 128, M.NUM_CLASSES), generator=torch.Generator(device="cuda").manual_seed(n), device="cuda")
        for loss_kind in ("xent", "dot"):
            before = {k: v.clone() for k, v in p.items()}
            p._flat.flat.grad = None
            logits, ep = _step(p, x, label, dropout, loss_kind, R)
            idx = _idx_list(ep)
            mask = None if ep["fc1/mask"] is None else ep["fc1/mask"].clone()
            grads = {}
            for dt in (torch.float64, torch.float32):
                P = params_as(before, dt, grad=True)
                stats = {}
                out = pointcnn_training(x.to(dt), P, idx, mask=mask, stats=stats)
                loss = M.get_loss(out, label) if loss_kind == "xent" else (out * R.to(dt)).sum()
                names = [k for k in P if not k.endswith(("moving_mean", "moving_variance"))]
                grads[dt] = dict(zip(names, torch.autograd.grad(loss, [P[k] for k in names])))
                if dt == torch.float64:
                    want_logits, mov = out.detach(), moving_update(before, stats)
            assert oerr(logits, want_logits) < OTOL
            for k, v in mov.items():
                assert oerr(p[k], v) < OTOL, k
            g64 = grads[torch.float64]
            for k, w64 in g64.items():
                # X_1's beta has an exactly zero gradient (X_2 is linear in BN_1's output, and the batch-norm backward of X_2 sums to
                # zero over the rows): there both sides hold rounding noise, measured against the same batch norm's gamma gradient
                scale = max(float(w64.abs().max()), float(g64[k.replace("/beta", "/gamma")].abs().max()) if k.endswith("_bn/beta") else 0.0)
                e, e32 = err(flat_grad(p, k), w64, scale), err(grads[torch.float32][k], w64, scale)
                assert within(e, e32, GTOL, 2.0), (k, e, e32)
            for k in before:                                              # restore the moving averages for the second loss
                if k.endswith(("moving_mean", "moving_variance")):
                    p[k].copy_(before[k])
    finally:
        ops.set_mlp_mode(old)


# ---------------------------------------------------------------------------------------------------------------------
# 4. - 7.
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_step_is_bit_reproducible():
    p, x = _setup(8, 1024, 31)
    label = torch.arange(8, device="cuda") % M.NUM_CLASSES
    M.get_model_training(x, params=p, dropout=False)
    state = {k: v.clone() for k, v in p.items()}
    runs = []
    for _ in range(2):
        with torch.no_grad():
            for k, v in state.items():
                p[k].copy_(v)
        p._flat.flat.grad = None
        torch.manual_seed(5)
        logits = M.get_model_training(x, params=p, dropout=True)
        M.get_loss(logits, label).backward()
        runs.append((logits.detach().clone(), p._flat.flat.grad.clone(), {k: v.clone() for k, v in p.items() if "moving" in k}))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    assert all(torch.equal(runs[0][2][k], runs[1][2][k]) for k in runs[0][2])


@pytest.mark.gpu
def test_regularization_loss_gradient():
    p, x = _setup(3, 1000, 41)
    M.get_model_training(x, params=p, dropout=False)
    fp = p._flat
    fp.flat.grad = None
    M.get_regularization_loss(p).backward()
    for name in fp.names:
        g = flat_grad(p, name)
        want = torch.zeros_like(g) if name == "logits/bias" else fp.views[name].detach() * 1e-5
        assert torch.allclose(g, want, rtol=1e-6, atol=0), name
    assert "logits/bias" in fp.names


@pytest.mark.gpu
def test_adam_lowers_the_loss_and_inference_follows():
    p, x = _setup(8, 1024, 51)
    label = torch.arange(8, device="cuda") % M.NUM_CLASSES
    M.get_model_training(x, params=p, dropout=False)
    opt = torch.optim.Adam([p._flat.flat], lr=1e-3, eps=1e-2)
    losses = []
    for _ in range(8):
        opt.zero_grad()
        logits = M.get_model_training(x, params=p, dropout=False)
        loss = M.get_loss(logits, label) + M.get_regularization_loss(p)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert losses[-1] < losses[0], losses
    p.invalidate()
    got, ep = M.get_model(x, False, params=p, return_end_points=True)
    want = po.forward(p, x.cpu().numpy(), [ep[f"idx{l}"].cpu().numpy() for l in range(1, 5)])["logits"]
    assert float(np.abs(got.cpu().numpy() - want).max()) < OTOL * max(1.0, float(np.abs(want).max()))


@pytest.mark.gpu
def test_allocation_peak_at_the_reference_batch():
    """the trainer's buffers (allocated by the first call) included"""
    p, x = _setup(32, 1024, 61)
    label = torch.arange(32, device="cuda") % M.NUM_CLASSES
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    M.get_loss(M.get_model_training(x, params=p), label).backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < 512 * 2 ** 20, peak / 2 ** 20
