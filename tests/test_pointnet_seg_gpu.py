"""pointnet_seg and pointnet_partseg against float64 restatements that build tile + concat as the reference does
(pointnet/models/pointnet_seg.py:24-134, pointnet_partseg.py:23-124): inference outputs, one training step (outputs, moving
averages, the flat gradient) and the inference-mode gradient with respect to the cloud.

Where fp32 and float64 can legitimately disagree, the comparison of gradients does what tests/test_input_grad_dgcnn_gpu.py does:
the gradient arriving at a max over the points whose runner-up is within 1e-5 of it, or at an FC-head activation within 1e-5 of the
relu's zero, is zeroed on both sides.  The segmentation head gives every point a gradient path of its own through conv1-conv9, so a
relu that fp32 and float64 decide differently there moves that point's gradient visibly; those layers run inside one autograd node
each, so instead of zeroing, the restatement takes the relu decisions the run took (fmaf(y, scale, shift) > 0 of the run's own
pre-batch-norm activations, evaluated exactly).  Both counts are printed.  In training mode the restatement also takes the values
of the run's batch statistics (its derivative stays float64's): fp32 sums of y and y^2 give the variance with an error relative to
E[y^2], not to the variance, and that error is bounded on its own (1e-4 of E[y^2]) instead of through every later layer."""
import pytest
import torch

from scanobjectnn_b200 import ops, pointnet_partseg, pointnet_seg
from scanobjectnn_b200.synthetic import make_clouds

from . import gpu_util as G
from .test_input_grad_dgcnn_gpu import _Masks, _near_zero, _out_err, _rel, _zero_at

pytestmark = pytest.mark.gpu
OTOL, GTOL = 1e-5, 1e-4
F = torch.nn.functional
MODELS = {"seg": pointnet_seg, "partseg": pointnet_partseg}


def _layer(h, P, scope, frozen, info, run, bn=True, relu=True):
    """conv2d / fully_connected (+ batch norm + relu) in float64; batch statistics (biased variance) are recorded in info["stats"].
    With a `run` (_Run), its batch statistics are used (see below) and its relu decisions: the relu is z * gate, and the decisions
    that differ from float64's are counted."""
    w = P[f"{scope}/weights"]
    y = h @ w.reshape(-1, w.shape[-1]) + P[f"{scope}/biases"]
    if not bn:
        return y
    if frozen:
        mean, var = P[f"{scope}/bn/moving_mean"], P[f"{scope}/bn/moving_variance"]
    else:
        dims = tuple(range(y.dim() - 1))
        mean, var = y.mean(dims), y.var(dims, unbiased=False)
        if run is not None and scope in run.stats:
            # the run's batch statistics as values, float64's for the derivative: fp32 sums of y and y^2 give the variance with an
            # error relative to E[y^2], which the comparison of the run's statistics below bounds on its own
            rmean, rinv = run.stats[scope][0].to(y.dtype), run.stats[scope][1].to(y.dtype)
            rvar = 1.0 / (rinv * rinv) - 1e-3
            ms = float((y.detach() ** 2).mean(dims).max())
            info["stat_err"] = max(info["stat_err"], float((rmean - mean.detach()).abs().max()) / ms ** 0.5,
                                   float((rvar - var.detach()).abs().max()) / ms)
            mean, var = mean + (rmean - mean).detach(), var + (rvar - var).detach()
        info["stats"][scope] = (mean.detach(), var.detach())
    z = (y - mean) / torch.sqrt(var + 1e-3) * P[f"{scope}/bn/gamma"] + P[f"{scope}/bn/beta"]
    if not relu:
        return z
    if run is not None and scope in run.gates:
        gate = run.gates[scope].view(z.shape)
        info["flips"] += int((gate != (z > 0)).sum())
        info["units"] += gate.numel()
        return z * gate
    return torch.relu(z)


class _Run:
    """per scope, from the last run of every cached MLP trainer: the relu decisions fmaf(y, scale, shift) > 0 (exact in float64) and,
    in training mode, the batch statistics (mean, 1 / sqrt(var + eps)) batch norm used"""

    def __init__(self, p, frozen):
        self.gates, self.stats = {}, {}
        for key, tr in p.__dict__.get("_trainers", {}).items():
            if key[0] != ("mlp_frozen" if frozen else "mlp"):
                continue
            for ly in tr.layers:
                if ly.bn:
                    self.gates[ly.scope] = (ly.y.double() * ly.scale.double() + ly.shift.double()) > 0
                    if not frozen:
                        self.stats[ly.scope] = ly.mean_inv


class _SameMasks(_Masks):
    """the masks of an earlier pass, applied again: the second pass takes the run's batch statistics, which moves values by far less
    than the 1e-5 that makes a maximum ambiguous, but enough to move a few of them across that threshold"""

    def __init__(self, first: _Masks):
        super().__init__()
        self.first = first

    def point_max(self, y, scope):
        self.pool[scope] = amb = self.first.pool[scope]
        _zero_at(y, amb.unsqueeze(1))
        return y.amax(dim=1)


def _model64(x, P, frozen, masks: _Masks, classify: bool, run: _Run | None = None):
    """the model in float64, dropout off -> ([class_pred,] seg_pred, feature transform, {"stats", "flips", "units", "stat_err"})"""
    b, n, _ = x.shape
    info = {"stats": {}, "flips": 0, "units": 0, "stat_err": 0.0}
    L = lambda h, s, **kw: _layer(h, P, s, frozen, info, run, **kw)        # noqa: E731

    def tnet(h, scope, K):
        g = masks.point_max(L(L(L(h, f"{scope}/tconv1"), f"{scope}/tconv2"), f"{scope}/tconv3"), f"{scope}/tconv3")
        g = L(L(g, f"{scope}/tfc1"), f"{scope}/tfc2")
        name = "transform_XYZ" if K == 3 else "transform_feat"
        eye = torch.eye(K, dtype=x.dtype, device=x.device).flatten()
        return (g @ P[f"{scope}/{name}/weights"] + P[f"{scope}/{name}/biases"] + eye).reshape(b, K, K)

    h = L(L(torch.bmm(x, tnet(x, "transform_net1", 3)), "conv1"), "conv2")
    t2 = tnet(h, "transform_net2", 64)
    point_feat = torch.bmm(h, t2)
    g = masks.point_max(L(L(L(point_feat, "conv3"), "conv4"), "conv5"), "conv5")
    out = []
    if classify:
        c = g
        for s in ("fc1", "fc2"):
            z = L(c, s, relu=False)
            near = masks.first.act[s] if isinstance(masks, _SameMasks) else _near_zero(z)
            c = torch.relu(z)
            _zero_at(c, near)
            masks.act[s] = near
        out.append(L(c, "fc3", bn=False))
    h = torch.cat([point_feat, g.unsqueeze(1).expand(b, n, g.shape[-1])], dim=2)          # tile + concat
    for s in pointnet_seg.HEAD:
        h = L(h, s)
    out.append(L(h, "conv10", bn=False))
    return out, t2, info


def _loss64(kind, outs, t2, labels, parts):
    reg = 0.001 * 0.5 * ((torch.bmm(t2, t2.transpose(1, 2)) - torch.eye(64, dtype=t2.dtype, device=t2.device)) ** 2).sum()
    seg = F.cross_entropy(outs[-1].transpose(1, 2), parts, reduction="none").mean(1).mean()
    if kind == "seg":
        return 0.5 * F.cross_entropy(outs[0], labels) + 0.5 * seg + reg
    return seg + reg


def _loss(kind, outs, ep, labels, parts):
    if kind == "seg":
        return pointnet_seg.get_loss(outs[0], outs[1], labels, parts, ep)[0]
    return pointnet_partseg.get_loss(outs[0], parts, ep)


def _setup(kind, b, n, seed):
    mod = MODELS[kind]
    p = mod.init_params(seed=seed, randomize_bn=True)
    with torch.no_grad():                          # zero in the reference's initialisation: give the T-nets a gradient path
        for s, name in (("transform_net1", "transform_XYZ"), ("transform_net2", "transform_feat")):
            p[f"{s}/{name}/weights"].normal_(0, 0.01, generator=torch.Generator(device="cuda").manual_seed(seed))
    x = G.cu(make_clouds("ball", b, n, seed=seed + 100))
    gen = torch.Generator(device="cuda").manual_seed(seed)
    labels = torch.randint(0, 15, (b,), device="cuda", generator=gen)
    nseg = p["conv10/weights"].shape[-1]
    parts = torch.randint(0, nseg, (b, n), device="cuda", generator=gen)
    return mod, p, x, labels, parts


def _outs(kind, res):
    return list(res[:2]) if kind == "seg" else [res[0]]


def _p64(p, grad=False):
    return {k: v.detach().double().requires_grad_(grad) for k, v in p.items()}


@pytest.mark.parametrize("kind", ["seg", "partseg"])
@pytest.mark.parametrize("n", [1024, 2048])
def test_inference_outputs_match_float64(kind, n):
    mod, p, x, _, _ = _setup(kind, 4, n, seed=n + len(kind))
    with torch.no_grad():
        res = mod.get_model(x, False, params=p)
    want, _, _ = _model64(x.double().requires_grad_(True), _p64(p), True, _Masks(), kind == "seg")   # (the masks hook gradients)
    got = _outs(kind, res)
    assert got[-1].shape == (4, n, 2 if kind == "seg" else 6)
    for g, w in zip(got, want):
        err = _out_err(g.cpu(), w.detach().cpu())
        print(f"[{kind} inference N={n}] output error {err:.2e}")
        assert err < OTOL
    assert res[-1]["transform"].shape == (4, 64, 64) and res[-1]["global"].shape == (4, 1024)


def _grad_errors(p, P, P32):
    """per variable: (max|run - float64|, max|float32 restatement - float64|), and the largest float64 entry"""
    fp = p._flat
    errs, scale = {}, 0.0
    for name in fp.names:
        v = fp.views[name]
        off = (v.data_ptr() - fp.flat.data_ptr()) // 4
        want = P[name].grad if P[name].grad is not None else torch.zeros_like(P[name])
        g32 = P32[name].grad if P32[name].grad is not None else torch.zeros_like(P32[name])
        got = fp.flat.grad[off:off + v.numel()].double().view(v.shape)
        errs[name] = (float((got - want).abs().max()), float((g32.double() - want).abs().max()))
        scale = max(scale, float(want.abs().max()))
    return errs, scale


def _against_float64(kind, b, n, seed, frozen, monkeypatch):
    """one GPU pass (training step or frozen inference with x.grad) and its float64 restatement on the same relu decisions
    -> (p, P, x, x64, outputs, float64 outputs, info)"""
    mod, p, x0, labels, parts = _setup(kind, b, n, seed)
    with torch.no_grad():
        fused = _outs(kind, mod.get_model(x0, False, params=p)) if frozen else None
    P0 = _p64(p)
    moving0 = {k: v.clone() for k, v in p.items() if k.endswith(("/moving_mean", "/moving_variance"))}
    masks = _Masks()                                   # pass 1: the ambiguous maxima and near-zero FC activations
    _model64(x0.double().requires_grad_(True), P0, frozen, masks, kind == "seg")
    masked, total = masks.count()
    with monkeypatch.context() as m:
        masks.patch(m)
        x = x0.clone().requires_grad_(frozen)
        if frozen:
            res = mod.get_model(x, False, params=p)
        elif kind == "seg":
            res = pointnet_seg._get_model_training(x, 0.5, p, dropout=False)
        else:
            res = pointnet_partseg.get_model(x, True, bn_decay=0.5, params=p)
        assert res[0].grad_fn is not None
        _loss(kind, _outs(kind, res), res[-1], labels, parts).backward()
    P = {k: v.clone().requires_grad_(not frozen) for k, v in P0.items()}
    masks2 = _SameMasks(masks)                         # pass 2, with the run's relu decisions (and batch statistics)
    x64 = x0.double().requires_grad_(True)
    want, t64, info = _model64(x64, P, frozen, masks2, kind == "seg", _Run(p, frozen))
    _loss64(kind, want, t64, labels, parts).backward()
    assert masks2.count() == (masked, total)
    print(f"[{kind} {'frozen' if frozen else 'training'} B={b} N={n}] masked: {masked} of {total}; relu decisions that differ "
          f"from float64's: {info['flips']} of {info['units']}; batch statistics' error relative to E[y^2]: {info['stat_err']:.2e}")
    assert masked <= 0.01 * total and info["flips"] <= 1e-4 * info["units"] and info["stat_err"] < GTOL
    if frozen:                                         # the frozen path agrees with the fused one and touches no variable
        for g, f in zip(_outs(kind, res), fused):
            assert _rel(g.detach().cpu(), f.cpu()) < 1e-4
        assert all(torch.equal(p[k], v) for k, v in moving0.items()) and p._flat.flat.grad is None
        return p, P, x, x64, _outs(kind, res), want, info
    # the same restatement in float32 (same relu decisions, statistics and masks): how far plain fp32 lands from float64
    P32 = {k: v.detach().float().requires_grad_(True) for k, v in P0.items()}
    want32, t32, _ = _model64(x0.clone(), P32, frozen, _SameMasks(masks), kind == "seg", _Run(p, frozen))
    _loss64(kind, want32, t32, labels, parts).backward()
    return p, (P, P32), x, x64, _outs(kind, res), (want, want32), info


@pytest.mark.parametrize("kind", ["seg", "partseg"])
def test_one_training_step_matches_float64(kind, monkeypatch):
    """Outputs and gradients within 1e-4 of the largest entry, or, where fp32 itself does not resolve 1e-4, within 3x of a float32
    evaluation of the same restatement (printed).  That is the case for the gradients of the trunk's early layers (the input T-net,
    conv1, conv2): sums over all B*N points of terms that largely cancel, since every point has a gradient of its own through the
    segmentation head."""
    p, (P, P32), _, _, got, (want, want32), info = _against_float64(kind, 32, 1024, 5, False, monkeypatch)
    for g, w, w32 in zip(got, want, want32):
        err, err32 = _out_err(g.detach().cpu(), w.detach().cpu()), _out_err(w32.detach().cpu(), w.detach().cpu())
        print(f"[{kind} training] output error {err:.2e} (float32 restatement: {err32:.2e})")
        assert err < GTOL or err <= 3 * err32
    # moving averages: decay 0.5 from the store's initial values towards the batch statistics
    for scope, (mean, var) in info["stats"].items():
        for suffix, batch in (("moving_mean", mean), ("moving_variance", var)):
            w = 0.5 * P[f"{scope}/bn/{suffix}"].detach() + 0.5 * batch
            assert _rel(p[f"{scope}/bn/{suffix}"].cpu(), w.cpu()) < OTOL, (scope, suffix)
    errs, scale = _grad_errors(p, P, P32)
    over = {k: (e / scale, e32 / scale) for k, (e, e32) in errs.items() if e > GTOL * scale}
    worst = max(errs, key=lambda k: errs[k][0])
    print(f"[{kind} training] gradient error relative to the largest entry: {errs[worst][0] / scale:.2e} ({worst}); beyond 1e-4 "
          f"(run, float32 restatement): {over}")
    assert all(e <= 3 * e32 for e, e32 in over.values()), over


@pytest.mark.parametrize("kind", ["seg", "partseg"])
def test_inference_input_grad_matches_float64(kind, monkeypatch):
    _, _, x, x64, got, want, _ = _against_float64(kind, 8, 1024, 9, True, monkeypatch)
    for g, w in zip(got, want):
        assert _out_err(g.detach().cpu(), w.detach().cpu()) < OTOL
    err = _rel(x.grad.cpu(), x64.grad.cpu())
    print(f"[{kind} frozen] x.grad error relative to its largest entry: {err:.2e}")
    assert err < GTOL


def test_training_step_is_bit_reproducible():
    runs = []
    for _ in range(2):
        _, p, x, labels, parts = _setup("seg", 4, 1024, seed=3)
        cls, seg, ep = pointnet_seg._get_model_training(x, 0.5, p, dropout=False)
        pointnet_seg.get_loss(cls, seg, labels, parts, ep)[0].backward()
        runs.append((cls.detach(), seg.detach(), p._flat.flat.grad.clone()))
    assert all(torch.equal(a, b) for a, b in zip(*runs))


def _peak_mib(fn):
    fn()                                           # folded weights and weight images are cached on the store by the first call
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2**20


def test_inference_memory_stays_below_the_concatenation():
    """At B=32, N=2048 the (B*N, 1088) concatenation alone would take 272 MiB."""
    b, n = 32, 2048
    p = pointnet_seg.init_params(seed=1, randomize_bn=True)
    x = G.cu(make_clouds("ball", b, n, seed=1))

    def composition():
        from scanobjectnn_b200 import pointnet_cls
        point_feat, g, _ = pointnet_cls.trunk(x, p)
        h = ops.shared_mlp(torch.cat([point_feat, g[:, None, :].expand(b, n, 1024)], dim=2), p.mlp(pointnet_seg.HEAD))
        return ops.shared_mlp(h, p.mlp(["conv10"], [False]))

    with torch.no_grad():
        grouped = _peak_mib(lambda: pointnet_seg.get_model(x, False, params=p))
        concat = _peak_mib(composition)
        diff = float((pointnet_seg.get_model(x, False, params=p)[1] - composition()).abs().max())
    print(f"[memory B={b} N={n}] inference allocation peak: grouped head {grouped:.1f} MiB, tile + concat {concat:.1f} MiB; "
          f"max|seg_pred difference| {diff:.2e}")
    assert grouped < 272
