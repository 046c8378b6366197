"""DGCNN's training step (dgcnn._get_model_training: batch statistics everywhere, dropout off) against a float64 restatement,
variable by variable, and each of its fused EdgeConv ops in isolation on the model's own activations.

1. The model: one step on the graphs of a first run, against restate.dgcnn on the same graphs.  Each tensor is
   compared relative to its own largest entry: the logits and every batch-norm layer's moving averages within 1e-5, every variable's
   slice of the flat gradient (the T-net's included) and x.grad within 1e-4.  A bias followed by batch norm has a gradient of exactly
   zero.  Near-tied maxima, maxima near the relu's zero and near-zero head activations are masked on both sides by the exclusion
   rule of tests/restate.py.  Next to each error stands that of the restatement evaluated in float32 with the same masks; where
   float32 itself misses the bound, the step must stay within 2x of it.
2. The ops: the input, graph and arriving gradient of every EdgeConv of a GPU step (dgcnn1..4 and the T-net's tconv1 + tconv2) are
   captured, and the op is run again on exactly those inputs against the float64 formula (output, batch statistics, dW, dgamma, dbeta,
   dx).  Next to each error stands that of a plain float32 evaluation of the same formula (torch autograd over the materialised
   edges): the yardstick of what fp32 resolves on that input.  An error beyond the bound must stay within 2x the yardstick's.
3. The head's batch statistics: psa_bn_finalize_rows against float64 on the pre-BN output of tfc1 and fc1, whose columns have a
   mean up to ~60 times their spread."""
import ctypes as C

import numpy as np
import pytest
import torch

from scanobjectnn_b200 import _lib, dgcnn, training
from scanobjectnn_b200._lib import ptr, stream
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import VariableStore

from . import gpu_util as G
from . import restate
from .restate import Masks, edges, err, flat_grad, layer, params_as, perturb_tnets, rel, within

OTOL, GTOL = 1e-5, 1e-4
DECAY = 0.5                      # the model's bn_decay
OP_DECAY = 0.9                   # the ops re-run on their own: decay and 1 - decay differ, so a swap of the two would show
TNET = ("transform_net1/tconv1", "transform_net1/tconv2")
BN_SUFFIXES = ("weights", "biases", "bn/gamma", "bn/beta", "bn/moving_mean", "bn/moving_variance")
# The beta of a layer pooled over the N points that feeds a layer batch-normed over the B clouds: a shift of beta shifts every cloud's
# pooled value alike, which the next batch norm removes, so its exact gradient is zero wherever all B maxima are positive and unmasked.
# Relative to its own largest entry the error would compare rounding with rounding; it is taken relative to the layer's dgamma.
POOLED_BETAS = ("transform_net1/tconv3/bn/beta", "agg/bn/beta")


def _loss_weights(b, seed):
    return torch.tensor(np.random.default_rng(seed).standard_normal((b, dgcnn.NUM_CLASSES)).astype(np.float32), device="cuda")


def _first_run(b, n, seed):
    """the store, the cloud and the five neighbour graphs of a first training-mode forward (which also moves the moving averages)"""
    p = dgcnn.init_params(seed=seed, randomize_bn=True)
    perturb_tnets(p, seed)
    x0 = G.cu(make_clouds("ball", b, n, seed=seed + 100))
    _, ep = dgcnn._get_model_training(x0, DECAY, dgcnn.NUM_CLASSES, p, dropout=False)
    return p, x0, [ep[f"nn_idx{i}"] for i in range(5)]


# ---------------------------------------------------------------------------------------------------------------------
# 1. the model-level step
# ---------------------------------------------------------------------------------------------------------------------
def _restatement(x0, P0, graphs, R, masks, dtype):
    """restate.dgcnn in `dtype` with the loss (logits * R).sum() differentiated -> (logits, x.grad, variables, batch statistics)"""
    P = params_as(P0, dtype, grad=True)
    x = x0.to(dtype, copy=True).requires_grad_(True)
    stats = {}
    logits = restate.dgcnn(x, P, graphs, False, masks, stats=stats)
    (logits * R.to(dtype)).sum().backward()
    return logits.detach(), x.grad, P, stats


def _step_against_float64(b, n, seed, monkeypatch):
    """one GPU training step and its float64 restatement -> ({quantity: (error of the step, error of the float32 restatement)}, each
    relative to the float64 tensor's largest entry, for "logits", "x.grad", ("grad", variable), ("moving", variable); masked and checked
    counts)"""
    p, x0, graphs = _first_run(b, n, seed)
    R = _loss_weights(b, seed)
    P0 = params_as(p, torch.float64)                 # the moving averages the step starts from
    trainable = set(p._flat.names)
    masks = Masks()
    l64, gx64, P, stats = _restatement(x0, P0, graphs, R, masks, torch.float64)
    l32, gx32, P32, stats32 = _restatement(x0, P0, graphs, R, masks.replay(), torch.float32)

    p._flat.flat.grad = None
    with monkeypatch.context() as m:
        masks.patch(m)
        x = x0.clone().requires_grad_(True)
        logits, ep = dgcnn._get_model_training(x, DECAY, dgcnn.NUM_CLASSES, p, dropout=False, graphs=graphs)
        (logits * R).sum().backward()
    assert all(torch.equal(ep[f"nn_idx{i}"], graphs[i]) for i in range(5))

    errs = {"logits": (err(logits, l64), err(l32, l64)), "x.grad": (err(x.grad, gx64), err(gx32, gx64))}
    bn_biases = {f"{s}/biases" for s in stats}
    for name in sorted(trainable):
        got = flat_grad(p, name)
        if name in bn_biases:
            assert not bool(got.any()), f"{name}: a bias followed by batch norm must get a gradient of exactly zero"
            continue
        want = P[name].grad
        scale = float(want.abs().max())
        if name in POOLED_BETAS:
            scale = max(scale, float(P[name.replace("/beta", "/gamma")].grad.abs().max()))
        errs[("grad", name)] = (err(got, want, scale), err(P32[name].grad, want, scale))
    for scope, (mean, var) in stats.items():
        for i, suffix in enumerate(("moving_mean", "moving_variance")):
            name = f"{scope}/bn/{suffix}"
            want = (1 - DECAY) * (mean, var)[i] + DECAY * P0[name]
            errs[("moving", name)] = (err(p[name], want), err((1 - DECAY) * stats32[scope][i].double() + DECAY * P0[name], want))
    assert {f"{s}/biases" for s in ("dgcnn1", "dgcnn4", "agg", "fc2", TNET[0], "transform_net1/tfc2")} <= bn_biases
    assert ("grad", "transform_net1/transform_XYZ/weights") in errs and ("grad", "fc3/biases") in errs
    return errs, masks.count()


def _within(key, e, e32):
    """the bound of an output or a gradient, or where float32 itself does not reach it, 2x the float32 restatement's error"""
    output = key in ("logits", "out") or (isinstance(key, tuple) and (key[0] == "moving" or key[1] in ("moving_mean", "moving_variance")))
    return within(e, e32, OTOL if output else GTOL, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,seed", [(8, 256, 7), (8, 256, 8), (8, 256, 0), (32, 256, 7), (32, 1024, 2)])
def test_dgcnn_training_step_matches_float64(b, n, seed, monkeypatch):
    """B=8 seeds 7 and 8 are the two of seeds 0-9 whose x.grad differed from float64 by 4.8e-3 and 2.0e-3 before the restatement
    masked maxima just below the relu's zero (DESIGN.md, "EdgeConv in training mode")"""
    errs, (masked, total) = _step_against_float64(b, n, seed, monkeypatch)
    fmt = lambda k: "/".join(k) if isinstance(k, tuple) else k          # noqa: E731
    grads = {k: v for k, v in errs.items() if isinstance(k, tuple) and k[0] == "grad"}
    moving = {k: v for k, v in errs.items() if isinstance(k, tuple) and k[0] == "moving"}
    worst_g, worst_m = max(grads, key=lambda k: grads[k][0]), max(moving, key=lambda k: moving[k][0])
    print(f"[dgcnn step B={b} N={n} seed={seed}] masked {masked} of {total}; error (float32 restatement's): "
          f"logits {errs['logits'][0]:.2e} ({errs['logits'][1]:.2e}), x.grad {errs['x.grad'][0]:.2e} ({errs['x.grad'][1]:.2e}), "
          f"worst variable gradient {grads[worst_g][0]:.2e} ({grads[worst_g][1]:.2e}, {worst_g[1]}), "
          f"worst moving average {moving[worst_m][0]:.2e} ({moving[worst_m][1]:.2e}, {worst_m[1]})")
    assert masked <= 0.01 * total
    over = {fmt(k): f"{e:.2e} ({e32:.2e})" for k, (e, e32) in errs.items() if not _within(k, e, e32)}
    assert not over, over


# ---------------------------------------------------------------------------------------------------------------------
# 2. each fused EdgeConv on the model's own activations
# ---------------------------------------------------------------------------------------------------------------------
def _capture(b, n, seed, monkeypatch):
    """the store and, for every EdgeConv of one training step in the order the model runs them, its scopes, input, graph and the
    gradient arriving at its output"""
    p, x0, graphs = _first_run(b, n, seed)
    R = _loss_weights(b, seed)
    seen, ec = [], training.edgeconv_training

    def spy(x, nn_idx, scope, *a, **kw):
        out = ec(x, nn_idx, scope, *a, **kw)
        rec = {"scopes": (scope,) if isinstance(scope, str) else tuple(scope), "x": x.detach().clone(), "idx": nn_idx.clone()}
        out.register_hook(lambda g: rec.__setitem__("dout", g.detach().clone()))
        seen.append(rec)
        return out

    with monkeypatch.context() as m:
        m.setattr(training, "edgeconv_training", spy)
        x = x0.clone().requires_grad_(True)
        logits, _ = dgcnn._get_model_training(x, DECAY, dgcnn.NUM_CLASSES, p, dropout=False, graphs=graphs)
        (logits * R).sum().backward()
    assert [r["scopes"] for r in seen] == [TNET, ("dgcnn1",), ("dgcnn2",), ("dgcnn3",), ("dgcnn4",)]
    return p, seen


def _formula(p, scopes, x, idx, dout, dtype, amb=None):
    """[x_i, x_j - x_i] -> (conv + batch norm + relu) per scope -> max over k in `dtype`, differentiated by torch autograd against
    dout (zeroed at `amb`, by default the maxima Masks.edge_max finds ambiguous) -> (amb, output, batch statistics by scope,
    {quantity: tensor})"""
    P = {f"{s}/{v}": p[f"{s}/{v}"].detach().to(dtype, copy=True).requires_grad_(True) for s in scopes for v in BN_SUFFIXES[:4]}
    xd = x.detach().to(dtype, copy=True).requires_grad_(True)
    stats, pre, h = {}, [], edges(xd, idx)
    for s in scopes:
        pre.append(layer(h, P, s, False, relu=False, stats=stats))
        h = torch.relu(pre[-1])
    if amb is None:
        masks = Masks()
        masks.edge_max(h, pre=pre[-1], inner=pre[0] if len(scopes) == 2 else None)
        amb = masks.edge[0]
    out = h.amax(dim=2)
    (out * dout.to(dtype).masked_fill(amb, 0.0)).sum().backward()
    res = {"dx": xd.grad}
    for s in scopes:
        res.update({(s, "dW"): P[f"{s}/weights"].grad.reshape(-1, P[f"{s}/weights"].shape[-1]), (s, "dgamma"): P[f"{s}/bn/gamma"].grad,
                    (s, "dbeta"): P[f"{s}/bn/beta"].grad})
    return amb, out.detach(), stats, res


def _op_against_float64(p, rec):
    """-> ({quantity: (error of the op, error of the float32 formula)}, masked count, checked count)"""
    scopes, x, idx, dout = rec["scopes"], rec["x"], rec["idx"], rec["dout"]
    amb, o64, st64, g64 = _formula(p, scopes, x, idx, dout, torch.float64)
    _, o32, st32, g32 = _formula(p, scopes, x, idx, dout, torch.float32, amb)
    q = VariableStore(device="cuda")                 # the op alone, on a store of its own variables
    for s in scopes:
        for v in BN_SUFFIXES:
            q[f"{s}/{v}"] = p[f"{s}/{v}"].detach().clone()
    moving0 = {k: v.double() for k, v in q.items() if k.endswith(("/moving_mean", "/moving_variance"))}
    xin = x.clone().requires_grad_(True)
    out = training.edgeconv_training(xin, idx, scopes[0] if len(scopes) == 1 else scopes, OP_DECAY, q)
    (out * dout.masked_fill(amb, 0.0)).sum().backward()
    got = {"dx": xin.grad}
    for s in scopes:
        got.update({(s, "dW"): flat_grad(q, f"{s}/weights").reshape(-1, q[f"{s}/weights"].shape[-1]),
                    (s, "dgamma"): flat_grad(q, f"{s}/bn/gamma"), (s, "dbeta"): flat_grad(q, f"{s}/bn/beta")})
        assert not bool(flat_grad(q, f"{s}/biases").any())
    errs = {"out": (rel(out.detach().cpu(), o64.cpu()), rel(o32.cpu(), o64.cpu()))}
    for s in scopes:
        for i, suffix in enumerate(("moving_mean", "moving_variance")):
            name = f"{s}/bn/{suffix}"
            want = (1 - OP_DECAY) * st64[s][i] + OP_DECAY * moving0[name]
            yard = (1 - OP_DECAY) * st32[s][i].double() + OP_DECAY * moving0[name]
            errs[(s, suffix)] = (rel(q[name].cpu(), want.cpu()), rel(yard.cpu(), want.cpu()))
    for key, want in g64.items():
        errs[key] = (rel(got[key].cpu(), want.cpu()), rel(g32[key].cpu(), want.cpu()))
    return errs, int(amb.sum()), amb.numel()


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,seed", [(8, 256, 7), (8, 256, 8), (32, 2048, 11)])
def test_dgcnn_edgeconv_ops_match_float64_on_the_models_activations(b, n, seed, monkeypatch):
    p, seen = _capture(b, n, seed, monkeypatch)
    failures = []
    for rec in seen:
        errs, masked, total = _op_against_float64(p, rec)
        name = "+".join(s.rsplit("/", 1)[-1] for s in rec["scopes"])
        print(f"[dgcnn op {name} B={b} N={n} seed={seed}] masked {masked} of {total}; error of the op (of fp32 torch):",
              {"/".join(k) if isinstance(k, tuple) else k: f"{e:.2e} ({e32:.2e})" for k, (e, e32) in errs.items()})
        assert masked <= 0.01 * total
        failures += [(name, key, e, e32) for key, (e, e32) in errs.items() if not _within(key, e, e32)]
        torch.cuda.empty_cache()
    assert not failures, failures


# ---------------------------------------------------------------------------------------------------------------------
# 3. the head's batch statistics on the model's own activations
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("b,n,seed", [(8, 256, 7), (32, 1024, 2)])
def test_head_batch_statistics_match_float64(b, n, seed):
    """The FC layers after a max over the points (T-net tfc1, fc1) have columns whose mean is up to ~60 times their spread.  Their
    batch norm (psa_bn_finalize_rows: two fp64 passes over y) agrees with float64 on their own pre-BN output; E[y^2] - mean^2 from
    correctly rounded fp32 sums (psa_bn_finalize's input) is printed beside it."""
    p, _, _ = _first_run(b, n, seed)
    lib = _lib.load()
    st = stream()
    ratio = 0.0
    for scope in ("transform_net1/tfc1", "fc1"):
        ly = next(ly for tr in p._trainers.values() for ly in tr.layers if ly.scope == scope)
        y = ly.y.clone()
        y64 = y.double()
        mean, var = y64.mean(0), y64.var(0, unbiased=False)
        ratio = max(ratio, float((mean * mean / var).max()))
        want = torch.stack([mean, 1 / torch.sqrt(var + 1e-3)])
        errs = {}
        for path in ("rows", "fp32 sums"):
            f = lambda: torch.empty(ly.N, device="cuda")          # noqa: E731
            scale, shift, mean_inv, mm, mv = f(), f(), torch.empty((2, ly.N), device="cuda"), torch.zeros(ly.N, device="cuda"), f()
            mv.fill_(1.0)
            args = (ptr(ly.gamma), ptr(ly.beta), C.c_float(OP_DECAY), ptr(mm), ptr(mv), ptr(scale), ptr(shift), ptr(mean_inv), st)
            if path == "rows":
                assert lib.psa_bn_finalize_rows(b, ly.N, ptr(y), *args) == 0
            else:
                stats = torch.stack([y64.sum(0), (y64 * y64).sum(0)]).float()
                assert lib.psa_bn_finalize(ly.N, b, ptr(stats), *args) == 0
            errs[path] = (rel(mean_inv[0].cpu(), want[0].cpu()), float(((mean_inv[1].double() - want[1]) / want[1]).abs().max()))
            if path == "rows":
                assert rel(mm.cpu(), ((1 - OP_DECAY) * mean).cpu()) < 1e-6
                assert rel(mv.cpu(), (OP_DECAY + (1 - OP_DECAY) * var).cpu()) < 1e-6
                g64, b64 = ly.gamma.detach().double(), ly.beta.detach().double()
                assert rel(scale.cpu(), (g64 * want[1]).cpu()) < 1e-6 and rel(shift.cpu(), (b64 - mean * g64 * want[1]).cpu()) < 1e-6
        print(f"[dgcnn head B={b} N={n} seed={seed}] {scope}: (mean, 1/sigma) errors by path {errs}")
        assert errs["rows"][0] < 1e-6 and errs["rows"][1] < 1e-6
    print(f"[dgcnn head B={b} N={n} seed={seed}] largest mean^2 / var: {ratio:.0f}")
    assert ratio > 100                                             # the regime that needs the centred variance

