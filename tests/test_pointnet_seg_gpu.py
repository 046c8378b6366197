"""pointnet_seg and pointnet_partseg against float64 restatements that build tile + concat as the reference does
(pointnet/models/pointnet_seg.py:24-134, pointnet_partseg.py:23-124): inference outputs, one training step (outputs, moving
averages, the flat gradient) and the inference-mode gradient with respect to the cloud.

Where fp32 and float64 can legitimately disagree, the comparison of gradients applies the exclusion rule of tests/restate.py:
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
from . import restate
from .restate import Masks, RunDecisions, grad_errors, moving, out_err, params_as, perturb_tnets, rel, within

pytestmark = pytest.mark.gpu
OTOL, GTOL = 1e-5, 1e-4
F = torch.nn.functional
MODELS = {"seg": pointnet_seg, "partseg": pointnet_partseg}


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
    perturb_tnets(p, seed)
    x = G.cu(make_clouds("ball", b, n, seed=seed + 100))
    gen = torch.Generator(device="cuda").manual_seed(seed)
    labels = torch.randint(0, 15, (b,), device="cuda", generator=gen)
    nseg = p["conv10/weights"].shape[-1]
    parts = torch.randint(0, nseg, (b, n), device="cuda", generator=gen)
    return mod, p, x, labels, parts


def _outs(kind, res):
    return list(res[:2]) if kind == "seg" else [res[0]]


@pytest.mark.parametrize("kind", ["seg", "partseg"])
@pytest.mark.parametrize("n", [1024, 2048])
def test_inference_outputs_match_float64(kind, n):
    mod, p, x, _, _ = _setup(kind, 4, n, seed=n + len(kind))
    with torch.no_grad():
        res = mod.get_model(x, False, params=p)
    want, _, _ = restate.pointnet_seg(x.double().requires_grad_(True), params_as(p, torch.float64), True, Masks(), kind == "seg")
    got = _outs(kind, res)
    assert got[-1].shape == (4, n, 2 if kind == "seg" else 6)
    for g, w in zip(got, want):
        err = out_err(g.cpu(), w.detach().cpu())
        print(f"[{kind} inference N={n}] output error {err:.2e}")
        assert err < OTOL
    assert res[-1]["transform"].shape == (4, 64, 64) and res[-1]["global"].shape == (4, 1024)


def _against_float64(kind, b, n, seed, frozen, monkeypatch):
    """one GPU pass (training step or frozen inference with x.grad) and its float64 restatement on the same relu decisions
    -> (p, P, x, x64, outputs, float64 outputs, info)"""
    mod, p, x0, labels, parts = _setup(kind, b, n, seed)
    with torch.no_grad():
        fused = _outs(kind, mod.get_model(x0, False, params=p)) if frozen else None
    P0 = params_as(p, torch.float64)
    moving0 = moving(p)
    masks = Masks()                                    # pass 1: the ambiguous maxima and near-zero FC activations
    restate.pointnet_seg(x0.double().requires_grad_(True), P0, frozen, masks, kind == "seg")
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
    P = params_as(P0, torch.float64, grad=not frozen)
    masks2 = masks.replay()                            # pass 2, with the run's relu decisions (and batch statistics)
    x64 = x0.double().requires_grad_(True)
    want, t64, info = restate.pointnet_seg(x64, P, frozen, masks2, kind == "seg", RunDecisions(p, frozen))
    _loss64(kind, want, t64, labels, parts).backward()
    assert masks2.count() == (masked, total)
    print(f"[{kind} {'frozen' if frozen else 'training'} B={b} N={n}] masked: {masked} of {total}; relu decisions that differ "
          f"from float64's: {info['flips']} of {info['units']}; batch statistics' error relative to E[y^2]: {info['stat_err']:.2e}")
    assert masked <= 0.01 * total and info["flips"] <= 1e-4 * info["units"] and info["stat_err"] < GTOL
    if frozen:                                         # the frozen path agrees with the fused one and touches no variable
        for g, f in zip(_outs(kind, res), fused):
            assert rel(g.detach().cpu(), f.cpu()) < 1e-4
        assert all(torch.equal(p[k], v) for k, v in moving0.items()) and p._flat.flat.grad is None
        return p, P, x, x64, _outs(kind, res), want, info
    # the same restatement in float32 (same relu decisions, statistics and masks): how far plain fp32 lands from float64
    P32 = params_as(P0, torch.float32, grad=True)
    want32, t32, _ = restate.pointnet_seg(x0.clone(), P32, frozen, masks.replay(), kind == "seg", RunDecisions(p, frozen))
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
        err, err32 = out_err(g.detach().cpu(), w.detach().cpu()), out_err(w32.detach().cpu(), w.detach().cpu())
        print(f"[{kind} training] output error {err:.2e} (float32 restatement: {err32:.2e})")
        assert within(err, err32, GTOL, 3)
    # moving averages: decay 0.5 from the store's initial values towards the batch statistics
    for scope, (mean, var) in info["stats"].items():
        for suffix, batch in (("moving_mean", mean), ("moving_variance", var)):
            w = 0.5 * P[f"{scope}/bn/{suffix}"].detach() + 0.5 * batch
            assert rel(p[f"{scope}/bn/{suffix}"].cpu(), w.cpu()) < OTOL, (scope, suffix)
    errs, scale = grad_errors(p, P, P32)
    over = {k: (e / scale, e32 / scale) for k, (e, e32) in errs.items() if e > GTOL * scale}
    worst = max(errs, key=lambda k: errs[k][0])
    print(f"[{kind} training] gradient error relative to the largest entry: {errs[worst][0] / scale:.2e} ({worst}); beyond 1e-4 "
          f"(run, float32 restatement): {over}")
    assert all(within(e, e32, GTOL, 3) for e, e32 in over.values()), over


@pytest.mark.parametrize("kind", ["seg", "partseg"])
def test_inference_input_grad_matches_float64(kind, monkeypatch):
    _, _, x, x64, got, want, _ = _against_float64(kind, 8, 1024, 9, True, monkeypatch)
    for g, w in zip(got, want):
        assert out_err(g.detach().cpu(), w.detach().cpu()) < OTOL
    err = rel(x.grad.cpu(), x64.grad.cpu())
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
