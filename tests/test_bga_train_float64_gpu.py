"""The two background-aware classifiers, pointnet2_cls_bga and dgcnn_bga, against float64 restatements (tests/restate.py): one
training step with dropout on and the joint loss, variable by variable, and the inference-mode gradient with respect to the cloud.

Dropout is on.  torch.nn.functional.dropout is replaced by a recorder that draws each mask from a seeded generator, records (mask, p)
and applies t * mask / (1 - p); the restatement applies the same masks in the same order.  The calls must be the reference's: dp1,
dp2, then the segmentation head's.  The class vector that feeds the segmentation branch is fc2's output before dp2
(pointnet2_cls_bga.py:45-48, dgcnn_bga.py:107-114); with dropout on, taking it after dp2 would change every segmentation gradient.

A first training-mode forward gives the run's FPS and ball-query indices (or neighbour graphs) and the dropout masks; the step
under test starts from the moving averages it left.  A float64 pass finds the elements the exclusion rule of tests/restate.py leaves
out; the GPU step runs with those masked; the float64 restatement then takes the run's relu decisions inside multi-layer MLP nodes
(RunDecisions), and a float32 evaluation of it is the yardstick of what fp32 resolves.  Each error is relative to its own float64
tensor: class_pred and seg_pred 1e-5 of max(1, largest); every batch norm's moving mean and variance 1e-5, against decay * old +
(1 - decay) * float64's batch statistic, with decay 0.5 except 0.9 for dgcnn_bga's seg/conv1 and seg/conv2; every variable's gradient
1e-4.  A bias followed by batch norm gets a gradient of exactly zero.  Where the float32 restatement itself misses a bound, the run
must stay within 2x of it."""
import time

import numpy as np
import pytest
import torch

from scanobjectnn_b200 import dgcnn, pointnet2_cls_bga
from scanobjectnn_b200.synthetic import make_clouds

from . import gpu_util as G
from . import restate
from .restate import Masks, RunDecisions, err, flat_grad, params_as, perturb_tnets, rel, within

pytestmark = pytest.mark.gpu
OTOL, GTOL = 1e-5, 1e-4
DECAY = 0.5
SEG_WEIGHT = 0.5
NUM_CLASS = 15
DROPS = {"pointnet2_cls_bga": [0.5, 0.5, 0.5], "dgcnn_bga": [0.5, 0.5, 0.3]}     # dp1, dp2, the segmentation head's
# Batch norms built without bn_decay: the reference's default 0.9 whatever the model's decay (dgcnn_bga.py:125-128).
FIXED_DECAY = {"dgcnn_bga": ("seg/conv1", "seg/conv2")}
# The beta of a layer max-pooled over the points whose pooled output reaches only batch norms over whole columns: a shift of beta shifts
# every pooled value alike (where the maxima are positive), which those batch norms remove, so its exact gradient is zero and its error
# is taken relative to the layer's dgamma.  pointnet2_cls_bga's layer3 feeds fc1 (over the B clouds); DGCNN's T-net tconv3 feeds tfc1;
# dgcnn_bga's agg feeds fc1 and, tiled over the N points, the agg columns of seg/conv1, batch-normed over all B*N rows: a constant
# shift there too.
POOLED_BETAS = {"pointnet2_cls_bga": ("layer3/conv2/bn/beta",), "dgcnn_bga": ("transform_net1/tconv3/bn/beta", "agg/bn/beta")}


class DropoutRecorder:
    """torch.nn.functional.dropout drawing its masks from a seeded generator and recording (mask, p); with `replay`, the recorded
    masks are applied again in order instead"""

    def __init__(self, seed, replay=None):
        self.gen = torch.Generator(device="cuda").manual_seed(seed)
        self.calls, self.replay = [], replay

    def __call__(self, t, p=0.5, training=True, inplace=False):
        assert training and not inplace
        if self.replay is not None:
            mask, q = self.replay[len(self.calls)]
            assert q == p and mask.shape == t.shape
        else:
            mask = (torch.rand(t.shape, generator=self.gen, device=t.device) >= p).to(t.dtype)
        self.calls.append((mask, p))
        return t * mask / (1 - p)


def _setup(model, b, n, seed):
    if model == "pointnet2_cls_bga":
        p = pointnet2_cls_bga.init_params(seed=seed, randomize_bn=True)
    else:
        p = dgcnn.init_params(seed=seed, randomize_bn=True, bga=True)
        perturb_tnets(p, seed)
    x = G.cu(make_clouds("ball", b, n, seed=seed + 100))
    rng = np.random.default_rng(seed)
    labels = torch.tensor(rng.integers(0, NUM_CLASS, b), device="cuda")
    mask = torch.tensor(rng.integers(0, 2, (b, n)), device="cuda")
    return p, x, labels, mask


def _loss(model, cp, sp, labels, mask):
    """the model's joint loss -> (total, classify, seg)"""
    f = pointnet2_cls_bga.get_loss if model == "pointnet2_cls_bga" else dgcnn.get_loss_bga
    return f(cp, sp, labels, mask, seg_weight=SEG_WEIGHT)


def _gpu(model, p, x, frozen, discrete=None):
    """one GPU pass -> (class_pred, seg_pred, the run's discrete choices: level indices or neighbour graphs)"""
    if model == "pointnet2_cls_bga":
        cp, sp = (pointnet2_cls_bga.get_model(x, False, params=p) if frozen else
                  pointnet2_cls_bga._get_model_training(x, DECAY, NUM_CLASS, p, False))
        return cp, sp, restate.pn2_indices(p, "level_frozen" if frozen else "level")
    cp, sp, ep = dgcnn._get_model_training(x, DECAY, NUM_CLASS, p, graphs=discrete, bga=True, frozen=frozen)
    return cp, sp, [ep[f"nn_idx{i}"] for i in range(5)]


def _restate(model, x, P, frozen, masks, discrete, run=None, drops=None):
    """the float restatement in x's dtype -> (class_pred, seg_pred, info)"""
    if model == "pointnet2_cls_bga":
        return restate.pointnet2_bga(x, P, frozen, masks, discrete, run=RunDecisions(run, frozen) if run is not None else None, drops=drops)
    info = {"stats": {}, "flips": 0, "units": 0, "stat_err": 0.0}
    dec = RunDecisions(run, frozen, stats=False) if run is not None else None
    cp, sp = restate.dgcnn(x, P, discrete, frozen, masks, stats=info["stats"], bga=True, run=dec, info=info, drops=drops)
    return cp, sp, info


def _passes(model, b, n, seed, frozen, monkeypatch):
    """a first pass, the exclusion masks, the GPU pass under test and its float64 and float32 restatements -> dict of what the checks
    compare"""
    p, x0, labels, segmask = _setup(model, b, n, seed)
    rec = DropoutRecorder(seed)
    with monkeypatch.context() as m:
        m.setattr(torch.nn.functional, "dropout", rec)
        _, _, discrete = _gpu(model, p, x0.clone().requires_grad_(frozen), frozen)
    drops = None if frozen else list(rec.calls)
    assert [q for _, q in rec.calls] == ([] if frozen else DROPS[model]), "dropout calls differ from the reference's"
    discrete = [d.clone() for d in discrete] if model == "dgcnn_bga" else discrete
    P0 = params_as(p, torch.float64)                  # the moving averages the step starts from
    before = {k: v.clone() for k, v in p.items()}
    masks = Masks()                                   # pass 1: the ambiguous maxima and near-zero head activations
    _restate(model, x0.double().requires_grad_(True), P0, frozen, masks, discrete, drops=drops)
    masked, total = masks.count()
    torch.cuda.empty_cache()

    if getattr(p, "_flat", None) is not None:
        p._flat.flat.grad = None
    replay = DropoutRecorder(seed, replay=drops)
    with monkeypatch.context() as m:
        masks.patch(m)
        m.setattr(torch.nn.functional, "dropout", replay)
        x = x0.clone().requires_grad_(frozen)
        cp, sp, run_discrete = _gpu(model, p, x, frozen, None if model == "pointnet2_cls_bga" else discrete)
        _loss(model, cp, sp, labels, segmask)[0].backward()
    assert len(replay.calls) == len(rec.calls)
    got, want = _flatten(run_discrete), _flatten(discrete)
    assert len(got) == len(want) and all(torch.equal(a, c) for a, c in zip(got, want)), "the run sampled other indices or graphs"

    res = dict(p=p, x=x, cp=cp.detach(), sp=sp.detach(), P0=P0, before=before, masked=masked, total=total)
    for dtype, tag in ((torch.float64, "64"), (torch.float32, "32")):
        if frozen and tag == "32":
            break
        P = params_as(P0, dtype, grad=not frozen)
        xd = x0.to(dtype, copy=True).requires_grad_(True)
        again = masks.replay()
        c, s, info = _restate(model, xd, P, frozen, again, discrete, run=p, drops=drops)
        total_loss, classify, _ = _loss(model, c, s, labels, segmask)
        if not frozen and tag == "64":            # fc2's gradient from the classification loss alone
            res["fc2_cls"] = torch.autograd.grad((1 - SEG_WEIGHT) * classify, P["fc2/weights"], retain_graph=True)[0]
        total_loss.backward()
        res.update({f"cp{tag}": c.detach(), f"sp{tag}": s.detach(), f"P{tag}": P, f"x{tag}": xd.grad, f"info{tag}": info})
        assert again.count() == (masked, total)
    return res


def _flatten(t):
    return [t] if isinstance(t, torch.Tensor) else [u for v in t for u in _flatten(v)]


@pytest.mark.parametrize("model,b,n,seed", [("pointnet2_cls_bga", 16, 1024, 1), ("pointnet2_cls_bga", 32, 2048, 2),
                                            ("dgcnn_bga", 16, 1024, 3), ("dgcnn_bga", 8, 256, 7), ("dgcnn_bga", 8, 256, 8)])
def test_training_step_with_dropout_matches_float64(model, b, n, seed, monkeypatch):
    """B=8 N=256 seeds 7 and 8: where DGCNN's EdgeConv backward differed from float64 before maxima just below the relu's zero were
    masked (DESIGN.md, "EdgeConv in training mode")"""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    r = _passes(model, b, n, seed, False, monkeypatch)
    p, P, P32, info, info32 = r["p"], r["P64"], r["P32"], r["info64"], r["info32"]
    scale = lambda t: max(1.0, float(t.abs().max()))          # noqa: E731
    errs = {"class_pred": (err(r["cp"], r["cp64"], scale(r["cp64"])), err(r["cp32"], r["cp64"], scale(r["cp64"])), OTOL),
            "seg_pred": (err(r["sp"], r["sp64"], scale(r["sp64"])), err(r["sp32"], r["sp64"], scale(r["sp64"])), OTOL)}
    # moving averages: float64's own batch statistics (where the restatement took the run's, "own" holds float64's)
    stats, stats32 = {**info["stats"], **info.get("own", {})}, {**info32["stats"], **info32.get("own", {})}
    fixed = FIXED_DECAY.get(model, ())
    assert set(fixed) <= set(stats)
    for scope in stats:
        decay = 0.9 if scope in fixed else DECAY
        for i, suffix in enumerate(("moving_mean", "moving_variance")):
            name = f"{scope}/bn/{suffix}"
            want = decay * r["P0"][name] + (1 - decay) * stats[scope][i]
            yard = decay * r["P0"][name] + (1 - decay) * stats32[scope][i].double()
            errs[name] = (err(p[name], want), err(yard, want), OTOL)
    bn_biases = {f"{s}/biases" for s in stats}
    for name in p._flat.names:
        got = flat_grad(p, name)
        if name in bn_biases:
            assert not bool(got.any()), f"{name}: a bias followed by batch norm must get a gradient of exactly zero"
            continue
        want = P[name].grad
        s = float(want.abs().max())
        if name in POOLED_BETAS[model]:
            s = max(s, float(P[name.replace("/beta", "/gamma")].grad.abs().max()))
        errs[name] = (err(got, want, s), err(P32[name].grad, want, s), GTOL)
    # the segmentation loss reaches fc2 through the class vector
    fc2_seg = rel(P["fc2/weights"].grad.cpu(), r["fc2_cls"].cpu())
    assert fc2_seg > 100 * GTOL, f"fc2's gradient hardly changes with the segmentation loss: {fc2_seg:.1e}"
    # every moving average and every variable gradient is checked
    assert {k for k in errs if "/moving_" in k} == {k for k in p if k.endswith(restate.MOVING)}
    assert {k for k in errs if "/moving_" not in k and k not in ("class_pred", "seg_pred")} | bn_biases == set(p._flat.names)

    grads = [k for k in errs if "/moving_" not in k and k not in ("class_pred", "seg_pred")]
    movs = [k for k in errs if "/moving_" in k]
    wg, wm = max(grads, key=lambda k: errs[k][0]), max(movs, key=lambda k: errs[k][0])
    print(f"[{model} step B={b} N={n} seed={seed}] masked {r['masked']} of {r['total']}; gates flipped {info['flips']} of "
          f"{info['units']}; error (float32 restatement's): class_pred {errs['class_pred'][0]:.2e} ({errs['class_pred'][1]:.2e}), "
          f"seg_pred {errs['seg_pred'][0]:.2e} ({errs['seg_pred'][1]:.2e}), worst variable gradient {errs[wg][0]:.2e} "
          f"({errs[wg][1]:.2e}, {wg}), worst moving average {errs[wm][0]:.2e} ({errs[wm][1]:.2e}, {wm}); fc2 with / without the "
          f"segmentation loss {fc2_seg:.1e}; {time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
    assert r["masked"] <= 0.01 * r["total"]
    assert info["flips"] <= 1e-4 * max(1, info["units"]) and info["stat_err"] < GTOL
    over = {k: f"{e:.2e} ({e32:.2e}) > {tol:.0e}" for k, (e, e32, tol) in errs.items() if not within(e, e32, tol, 2)}
    assert not over, over


@pytest.mark.parametrize("model", ["pointnet2_cls_bga", "dgcnn_bga"])
def test_inference_input_grad_of_the_joint_loss_matches_float64(model, monkeypatch):
    """inference mode with a cloud that requires a gradient: class_pred and seg_pred within 1e-5, x.grad of the joint loss within 1e-4
    of its largest entry; no dropout, and no variable and no moving average moves"""
    b, n = 16, 1024
    r = _passes(model, b, n, 5, True, monkeypatch)
    p = r["p"]
    scale = lambda t: max(1.0, float(t.abs().max()))          # noqa: E731
    e_cp, e_sp = err(r["cp"], r["cp64"], scale(r["cp64"])), err(r["sp"], r["sp64"], scale(r["sp64"]))
    e_x = err(r["x"].grad, r["x64"])
    info = r["info64"]
    print(f"[{model} frozen B={b} N={n}] masked {r['masked']} of {r['total']}; gates flipped {info['flips']} of {info['units']}; "
          f"class_pred {e_cp:.2e}, seg_pred {e_sp:.2e}, x.grad {e_x:.2e}")
    assert all(torch.equal(v, r["before"][k]) for k, v in p.items()), "inference mode moved a variable or a moving average"
    assert p._flat.flat.grad is None
    assert r["masked"] <= 0.01 * r["total"] and info["flips"] <= 1e-4 * max(1, info["units"])
    assert e_cp < OTOL and e_sp < OTOL and e_x < GTOL
