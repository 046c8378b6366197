"""3DmFV-Net's training path (csrc/mfv_train.cu, mfv_net_cls.get_model_training) against float64.

1. Each conv3d product on its own, for every conv shape of the model at B=64 and at B=3 (partial tiles, contraction blocks and
   tiles straddling voxels): the weight and data gradients against the float64 autograd of F.conv3d, relative to each tensor's
   largest entry, with a plain float32 evaluation (TF32 off) beside it: an error beyond 1e-4 must stay within 2x the float32 one.
   The accumulating data gradient is bit-identical to base + its plain result, and reruns are bit-identical.  The pools: max-pool
   winners follow the (dz, dy, dx) first-maximum rule on constructed ties and the far-end padding, the max-pool backward is exact,
   the average-pool backward within 1e-6.
2. One training step (dropout off, loss (logits * R).sum()) against the float64 restatement mfv_training() below on the run's own
   Fisher vector, relu gates and max-pool winners: logits and every moving average within 1e-5 * max(1, |max|), every flat-gradient
   slice within 1e-4 (or 2x float32's own error), the conv3d and fc1-fc3 biases exactly zero.  Pooled entries whose window has a
   runner-up within 1e-5 of its maximum, or a maximum within 1e-5 of the relu's zero, are masked on both sides; at most 1% of them.
3. Two steps from the same state give bit-identical gradients and moving averages; bn_decay=None decays at 0.9.
4. Adam on one fixed batch lowers the loss."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import mfv_oracle as mo
from scanobjectnn_b200 import mfv_net_cls as M
from scanobjectnn_b200 import ops
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import BN_EPS

from .restate import RunDecisions, err, flat_grad, layer, params_as, within, zero_at

OTOL, GTOL = 1e-5, 1e-4


# ---------------------------------------------------------------------------------------------------------------------
# the float64 restatement of 3dmfv_net_cls in training mode
# ---------------------------------------------------------------------------------------------------------------------
def grid(rows, b, r):
    """voxel-major rows (b*r^3, C) -> (b, C, r, r, r)"""
    return rows.reshape(r ** 3, b, -1).permute(1, 2, 0).reshape(b, -1, r, r, r)


def max_pool_at(x, win):
    """the SAME 2^3 stride-2 max taken at the given winners (b, C, ro, ro, ro) (window position dz * 4 + dy * 2 + dx), so that the
    gradient goes where the run sends it; the far-end padding cells are never a winner"""
    b, c, r = x.shape[:3]
    ro = (r + 1) // 2
    xp = F.pad(x, (0, 2 * ro - r) * 3)
    w = xp.reshape(b, c, ro, 2, ro, 2, ro, 2).permute(0, 1, 2, 4, 6, 3, 5, 7).reshape(b, c, ro, ro, ro, 8)
    return w.gather(-1, win.long().unsqueeze(-1)).squeeze(-1)


def conv_bn(x, P, scope, frozen, gates=None, stats=None, info=None):
    """tf_util.conv3d (SAME, stride 1, bias) + batch norm (moving averages when frozen, else the batch's, biased) + relu; gates
    (b, C, r, r, r): the run's relu decisions in place of x's dtype's own"""
    dt = x.dtype
    w = P[f"{scope}/weights"].to(dt)
    y = F.conv3d(x, w.permute(4, 3, 0, 1, 2), padding=w.shape[0] // 2) + P[f"{scope}/biases"].to(dt)[None, :, None, None, None]
    if frozen:
        mean, var = P[f"{scope}/bn/moving_mean"].to(dt), P[f"{scope}/bn/moving_variance"].to(dt)
    else:
        mean, var = y.mean(dim=(0, 2, 3, 4)), y.var(dim=(0, 2, 3, 4), unbiased=False)
        if stats is not None:
            stats[scope] = (mean.detach(), var.detach())
    v = lambda t: t[None, :, None, None, None]                              # noqa: E731
    z = (y - v(mean)) / torch.sqrt(v(var) + BN_EPS) * v(P[f"{scope}/bn/gamma"].to(dt)) + v(P[f"{scope}/bn/beta"].to(dt))
    if gates is None:
        return torch.relu(z)
    g = gates[scope]
    info["flips"] += int((g != (z > 0)).sum())
    info["near"] += int((z.detach().abs() < 1e-5 * float(z.detach().abs().max())).sum())
    info["units"] += g.numel()
    return z * g


def mfv_training(fv, P, frozen=False, gates=None, winners=None, pool_mask=None, stats=None, run=None, info=None):
    """3dmfv_net_cls.get_model on the Fisher vector fv (B,G,20) in its dtype, dropout off: batch statistics (recorded in `stats`) or,
    frozen, the moving averages.  gates / winners: the run's relu decisions and max-pool winners (grids); pool_mask: the entries of the
    last max pool whose gradient is zeroed; run (restate.RunDecisions): the FC head's relu gates"""
    b, g, _ = fv.shape
    r = int(round(g ** (1 / 3)))
    net = fv.permute(0, 2, 1).reshape(b, 20, r, r, r)
    for l in range(1, 6):
        s = f"inception{l}"
        cb = lambda x, j: conv_bn(x, P, f"{s}_conv{j}", frozen, gates, stats, info)   # noqa: E731
        one = cb(net, 1)
        net = torch.cat([one, cb(one, 2), cb(one, 3), cb(mo.avg_pool3(net), 4)], 1)
        if l in (3, 5):
            net = mo.max_pool2(net) if winners is None else max_pool_at(net, winners[l])
    if pool_mask is not None:
        zero_at(net, pool_mask)
    h = net.permute(0, 2, 3, 4, 1).reshape(b, -1)
    for scope in ("fc1", "fc2", "fc3"):
        h = layer(h, P, scope, frozen, stats=stats, run=run, info=info)
    return layer(h, P, "fc4", frozen, bn=False)


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


# ---------------------------------------------------------------------------------------------------------------------
# each product on its own
# ---------------------------------------------------------------------------------------------------------------------
CONVS = sorted({(3 if s.startswith(("inception4", "inception5")) else 5, k, cin, cout) for s, k, cin, cout in M._module_widths()})


@pytest.mark.gpu
@pytest.mark.parametrize("b", [64, 3])
@pytest.mark.parametrize("r,k,cin,cout", CONVS)
def test_conv3d_products_match_float64(b, r, k, cin, cout):
    gen = torch.Generator(device="cuda").manual_seed(b * 7 + r * 100 + k * 10 + cin)
    rows = b * r ** 3
    buf = torch.zeros((rows, cin + 8), device="cuda")                        # x read as a column slice of a wider buffer
    buf[:, 4:4 + cin] = torch.relu(torch.randn((rows, cin), generator=gen, device="cuda"))
    x = buf[:, 4:4 + cin]
    W = torch.randn((k, k, k, cin, cout), generator=gen, device="cuda") / np.sqrt(k ** 3 * cin)
    dy = torch.randn((rows, cout), generator=gen, device="cuda")
    got = {"dW": ops.conv3d_bwd_weight(x, r, dy, k), "dx": ops.conv3d_bwd_data(dy, r, W)}

    def formula(dt):
        xg = grid(x.to(dt), b, r).requires_grad_(True)
        wg = W.to(dt).requires_grad_(True)
        y = F.conv3d(xg, wg.permute(4, 3, 0, 1, 2), padding=k // 2)
        (y * grid(dy.to(dt), b, r)).sum().backward()
        return {"dW": wg.grad, "dx": xg.grad.reshape(b, cin, r ** 3).permute(2, 0, 1).reshape(rows, cin)}

    w64, w32 = formula(torch.float64), formula(torch.float32)
    for name, v in got.items():
        e, e32 = err(v, w64[name]), err(w32[name], w64[name])
        print(f"b={b} r={r} k={k} {cin}->{cout} {name}: {e:.2e} (float32 {e32:.2e})")
        assert within(e, e32, GTOL, 2), (name, e, e32)
    # reruns are bit-identical; accumulate adds the same product to what the buffer holds
    assert torch.equal(got["dW"], ops.conv3d_bwd_weight(x, r, dy, k))
    assert torch.equal(got["dx"], ops.conv3d_bwd_data(dy, r, W))
    out = torch.randn((rows, cin + 16), generator=gen, device="cuda")
    base = out.clone()
    ops.conv3d_bwd_data(dy, r, W, out=out[:, 8:], accumulate=True)
    assert torch.equal(out[:, 8:8 + cin], base[:, 8:8 + cin] + got["dx"])
    assert torch.equal(out[:, :8], base[:, :8]) and torch.equal(out[:, 8 + cin:], base[:, 8 + cin:])
    issued_w, issued_d, in_grid = ops.conv3d_bwd_macs(b, r, k, cin, cout)
    assert in_grid <= issued_w and in_grid <= issued_d <= rows * k ** 3 * cin * cout


def _winners_ref(x, b, r):
    """first maximum in (dz, dy, dx) order of each 2^3 window, the far-end padding at -inf"""
    ro = (r + 1) // 2
    xg = F.pad(grid(x, b, r), (0, 2 * ro - r) * 3, value=-float("inf"))
    c = xg.shape[1]
    w = xg.reshape(b, c, ro, 2, ro, 2, ro, 2).permute(0, 1, 2, 4, 6, 3, 5, 7).reshape(b, c, ro, ro, ro, 8)
    return w.argmax(-1)                                                      # torch.argmax: the first maximal value


@pytest.mark.gpu
@pytest.mark.parametrize("r", [5, 3, 8])
def test_pools_winners_and_backward(r):
    b, c = 3, 40
    gen = torch.Generator(device="cuda").manual_seed(r)
    x = torch.randn((b * r ** 3, c), generator=gen, device="cuda")
    x[:, :8] = torch.randint(0, 3, (b * r ** 3, 8), generator=gen, device="cuda").float()   # many ties within a window
    x[:, 8] = 1.0                                                            # a whole channel tied: the first in-grid cell wins
    out, win = ops.pool3d_max_train(x, r)
    ro = (r + 1) // 2
    assert torch.equal(out, ops.pool3d(x, r, "max"))
    want = _winners_ref(x, b, r)
    assert torch.equal(grid(win, b, ro).long(), want)
    assert not bool((grid(win, b, ro)[:, 8] != 0).any())
    # max backward: a copy to the winners
    dout = torch.randn((b * ro ** 3, c), generator=gen, device="cuda")
    dx = ops.pool3d_bwd(dout, r, "max", win)
    xg = grid(x, b, r).double().requires_grad_(True)
    max_pool_at(xg, grid(win, b, ro)).backward(grid(dout, b, ro).double())
    assert torch.equal(grid(dx, b, r).double(), xg.grad)
    # average backward: a gather of dout / count
    dout = torch.randn((b * r ** 3, c), generator=gen, device="cuda")
    dx = ops.pool3d_bwd(dout, r, "avg")
    xg = grid(x, b, r).double().requires_grad_(True)
    mo.avg_pool3(xg).backward(grid(dout, b, r).double())
    assert err(grid(dx, b, r), xg.grad) < 1e-6
    assert torch.equal(dx, ops.pool3d_bwd(dout, r, "avg"))


# ---------------------------------------------------------------------------------------------------------------------
# the model-level step
# ---------------------------------------------------------------------------------------------------------------------
def _gmm(r):
    return [torch.from_numpy(t).cuda() for t in M.get_3d_grid_gmm((r, r, r))]


def _run_decisions(ep, b, r):
    """the run's relu gates per conv (grids), max-pool winners by module, and the mask of ambiguous last-pool entries"""
    gates, hs, rr = {}, {}, r
    for l in range(1, 6):
        for j in range(1, 5):
            s = f"inception{l}_conv{j}"
            z = ep[f"{s}/y"].double() * ep[f"{s}/scale"].double() + ep[f"{s}/shift"].double()
            gates[s] = grid(z > 0, b, rr)
            hs[s] = grid(torch.relu(z), b, rr)
        if l in (3, 5):
            rr = (rr + 1) // 2
    ro4, ro = (r + 1) // 2, ((r + 1) // 2 + 1) // 2
    winners = {3: grid(ep["pool1/winner"], b, ro4), 5: grid(ep["pool2/winner"], b, ro)}
    h5 = torch.cat([hs[f"inception5_conv{j}"] for j in range(1, 5)], 1)
    r5 = h5.shape[-1]
    hp = F.pad(h5, (0, 2 * ro - r5) * 3, value=-1.0)
    c = h5.shape[1]
    w = hp.reshape(b, c, ro, 2, ro, 2, ro, 2).permute(0, 1, 2, 4, 6, 3, 5, 7).reshape(b, c, ro, ro, ro, 8)
    top = torch.topk(w, 2, dim=-1).values
    tol = 1e-5 * float(h5.abs().max())
    mask = ((top[..., 0] - top[..., 1]) < tol) & (top[..., 0] > 0) | ((top[..., 0] > 0) & (top[..., 0] < tol))
    return gates, winners, mask


def _step(p, pts, gmm, R, mask_rows=None, monkeypatch=None):
    """one forward + backward of get_model_training, dropout off; mask_rows zeroes the gradient at the conv stack's output rows"""
    p_flat = getattr(p, "_flat", None)
    if p_flat is not None:
        p_flat.flat.grad = None
    if mask_rows is None:
        logits, fv = M.get_model_training(pts, *gmm, None, params=p, dropout=False)
    else:
        orig = M._MfvFn.apply

        def masked_apply(*a):
            out = orig(*a)
            out.register_hook(lambda g: g.masked_fill(mask_rows, 0.0))
            return out

        with monkeypatch.context() as m:
            m.setattr(M._MfvFn, "apply", masked_apply)
            logits, fv = M.get_model_training(pts, *gmm, None, params=p, dropout=False)
    (logits * R).sum().backward()
    return logits.detach(), fv


STEP = [(64, 1024, 5, 0), (64, 1024, 5, 1), (64, 1024, 5, 2), (16, 1024, 5, 0), (3, 1000, 5, 0), (8, 1024, 8, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,r,mode", STEP)
def test_training_step_matches_float64(b, n, r, mode, monkeypatch):
    seed = b + r + mode
    p = M.init_params(seed=seed, randomize_bn=True)
    pts = torch.from_numpy(make_clouds("ball", b, n, seed=seed + 100)).cuda()
    gmm = _gmm(r)
    R = torch.tensor(np.random.default_rng(seed).standard_normal((b, M.NUM_CLASSES)).astype(np.float32), device="cuda")
    ops.set_mlp_mode(mode)
    try:
        with torch.no_grad():
            _, fv, ep = M.get_model_training(pts, *gmm, None, params=p, dropout=False, return_end_points=True)
        gates, winners, mask = _run_decisions(ep, b, r)
        ro = mask.shape[-1]
        mask_rows = mask.permute(2, 3, 4, 0, 1).reshape(ro ** 3 * b, -1)    # the conv stack's output rows (voxel-major)
        P0 = params_as(p, torch.float64)
        logits, fv = _step(p, pts, gmm, R, mask_rows, monkeypatch)
    finally:
        ops.set_mlp_mode(0)
    run = RunDecisions(p, frozen=False, stats=False)
    res = {}
    for dt in (torch.float64, torch.float32):
        P = params_as(P0, dt, grad=True)
        stats, info = {}, {"flips": 0, "near": 0, "units": 0}
        out = mfv_training(fv.transpose(1, 2).to(dt), P, gates=gates, winners=winners, pool_mask=mask, stats=stats, run=run, info=info)
        (out * R.to(dt)).sum().backward()
        res[dt] = (out.detach(), P, stats, info)
    l64, P64, st64, info64 = res[torch.float64]
    l32, P32, st32, _ = res[torch.float32]
    masked, flips, near = float(mask.double().mean()), info64["flips"] / info64["units"], info64["near"] / info64["units"]
    print(f"B={b} N={n} r={r} mode={mode}: last pool masked {masked:.3%}, conv pre-activations within 1e-5 of zero {near:.4%}, "
          f"relu gates differing from float64's {flips:.4%}")
    assert masked <= 0.01 and near <= 0.01 and flips <= 0.01

    errs = {"logits": (err(logits, l64, max(1.0, float(l64.abs().max()))), err(l32, l64, max(1.0, float(l64.abs().max()))))}
    for name, (m64, v64) in st64.items():
        m32, v32 = st32[name]
        for i, (suffix, w64, w32) in enumerate((("moving_mean", m64, m32), ("moving_variance", v64, v32))):
            key = f"{name}/bn/{suffix}"
            want = 0.1 * w64 + 0.9 * P0[key]
            sc = max(1.0, float(want.abs().max()))
            errs[key] = (err(p[key], want, sc), err(0.1 * w32.double() + 0.9 * P0[key], want, sc))
    assert sum(1 for k in errs if "moving" in k) == 2 * 23
    for name in p._flat.names:
        got = flat_grad(p, name)
        if name.endswith("/biases") and name != "fc4/biases":
            assert not bool(got.any()), f"{name}: a bias followed by batch norm must get a gradient of exactly zero"
            continue
        errs[name] = (err(got, P64[name].grad), err(P32[name].grad, P64[name].grad))
    bad = []
    for key, (e, e32) in sorted(errs.items()):
        tol = OTOL if key == "logits" or "moving" in key else GTOL
        print(f"  {key}: {e:.2e} (float32 {e32:.2e})")
        if not within(e, e32, tol, 2):
            bad.append((key, e, e32))
    assert not bad, bad


@pytest.mark.gpu
def test_training_step_is_bit_reproducible_and_decays_at_0_9():
    b, n, r = 8, 512, 5
    p = M.init_params(seed=4, randomize_bn=True)
    pts = torch.from_numpy(make_clouds("ball", b, n, seed=104)).cuda()
    gmm = _gmm(r)
    R = torch.randn(b, M.NUM_CLASSES, device="cuda")
    moving = [k for k in p if k.endswith(("moving_mean", "moving_variance"))]
    start = {k: p[k].clone() for k in moving}
    runs = []
    for _ in range(2):
        for k in moving:
            p[k].copy_(start[k])
        _step(p, pts, gmm, R)
        runs.append((p._flat.flat.grad.clone(), [p[k].clone() for k in moving]))
    assert torch.equal(runs[0][0], runs[1][0])
    assert all(torch.equal(a, c) for a, c in zip(runs[0][1], runs[1][1]))
    # bn_decay=None: moving = 0.9 moving + 0.1 batch, here for a conv3d batch norm (its y is the batch)
    for k in moving:
        p[k].copy_(start[k])
    with torch.no_grad():
        _, _, ep = M.get_model_training(pts, *gmm, None, params=p, dropout=False, return_end_points=True)
    y = ep["inception3_conv3/y"].double()
    want = 0.9 * start["inception3_conv3/bn/moving_mean"].double() + 0.1 * y.mean(0)
    assert err(p["inception3_conv3/bn/moving_mean"], want) < 1e-6
    want = 0.9 * start["inception3_conv3/bn/moving_variance"].double() + 0.1 * y.var(0, unbiased=False)
    assert err(p["inception3_conv3/bn/moving_variance"], want) < 1e-6


@pytest.mark.gpu
def test_adam_on_one_batch_lowers_the_loss():
    b, n, r = 16, 1024, 5
    torch.manual_seed(0)
    p = M.init_params(seed=6)
    pts = torch.from_numpy(make_clouds("ball", b, n, seed=106)).cuda()
    labels = torch.arange(b, device="cuda") % M.NUM_CLASSES
    gmm = _gmm(r)
    M.get_model_training(pts, *gmm, None, params=p)                          # the flat parameter vector exists from here on
    opt = torch.optim.Adam([p._flat.flat], lr=1e-3)
    losses = []
    for _ in range(30):
        opt.zero_grad()
        logits, _ = M.get_model_training(pts, *gmm, None, params=p)
        loss = M.get_loss(logits, labels)
        loss.backward()
        opt.step()
        p.invalidate()
        losses.append(float(loss.detach()))
    print("losses:", " ".join(f"{v:.3f}" for v in losses))
    assert np.mean(losses[-5:]) < np.mean(losses[:5])
