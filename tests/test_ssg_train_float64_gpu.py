"""The benchmarked PointNet++ training step (PointNet2ClsTrainer at B=32, N=2048 with SSG_LEVELS and the FC head) against a float64
restatement, variable by variable, over several consecutive steps; and the loss and optimizer kernels on their own.

1. The step.  train_step's order -- draw_dropout, forward (batch statistics), loss_and_grad, backward with the coordinate gradient,
   adam -- four times in a row, so every step after the first starts from moved weights, moving averages and non-zero Adam moments.
   After each backward, restate.ssg restates the model in float64 on the trainer's own FPS and ball-query indices
   (which must equal the CPU oracle's), and takes the run's discrete decisions: each batch-normed layer's relu gate
   fmaf(y, scale, shift) > 0, each level's max-pool winner argk (its first winning row: a tie, or a ball-query padding row that
   duplicates a real row, gives the same gradients whichever copy it routes to) and the head's dropout masks.  Batch statistics are
   float64's own.  Each error is relative to the float64 tensor's largest entry:
     logits 1e-5; every batch-norm layer's moving mean and variance, against decay * (the GPU's previous value) + (1 - decay) *
     (float64's batch statistic), 1e-5; every variable's gradient and the input cloud's gradient 1e-4.
   tr.loss and tr.dlogits are checked against float64 on the run's own logits: 1e-6 * max(1, loss) and 1e-6 / B.  A bias followed by
   batch norm gets a gradient of exactly zero.  Beside each error stands that of the same restatement evaluated in float32; where
   float32 itself misses the bound, the step must stay within 2x of it.  Flipped gates stay within 1e-4 of the units, and float64's
   value at every winner within 1e-5 (of the largest activation) of float64's own maximum.
   Adam is checked against float64 Adam applied to the GPU's own previous parameters, moments and gradient: the moments to a few
   units of fp32 rounding of their terms, the parameter's increment within 1e-5 of lr_t beyond the rounding of the stored parameter.
   The same restatement with frozen=True checks inference-mode logits and the input cloud's gradient at the same shape.
2. psa_softmax_xent and psa_adam_step called directly against float64, at the shapes and values where they could go wrong."""
import ctypes as C
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import oracle as orc
from scanobjectnn_b200 import _lib, pointnet2_cls_ssg
from scanobjectnn_b200._lib import ptr, stream
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.training import PointNet2ClsTrainer

from . import restate
from .restate import err, params_as, within

pytestmark = pytest.mark.gpu

OTOL, GTOL = 1e-5, 1e-4
LR, DECAY, NUM_CLASS = 1e-3, 0.5, 15
B1, B2, EPS = float(np.float32(0.9)), float(np.float32(0.999)), float(np.float32(1e-8))      # as the kernel receives them
U32 = 2.0 ** -24                    # fp32's unit roundoff
SUB32 = 2.0 ** -149                 # the spacing of fp32's subnormals
# The beta of the group-all level's last layer: a shift of it shifts every cloud's pooled feature alike, which fc1's batch norm
# removes, so its exact gradient is zero wherever the maxima are positive.  Its error is taken relative to the layer's dgamma.
POOLED_BETAS = ("layer3/conv2/bn/beta",)


def _lr_t(lr, step):
    return lr * np.sqrt(1.0 - B2 ** step) / (1.0 - B1 ** step)


def _adam_errors(p0, m0, v0, g, p1, m1, v1, lr, step, gscale):
    """the kernel's step (p1, m1, v1) from (p0, m0, v0) and gradient g, against float64 Adam on the same inputs -> (m error, v error,
    increment error), each relative to its allowance (<= 1 passes): the moments a few units of fp32 rounding of their terms (plus
    the subnormal spacing, where g^2 underflows), the increment 1e-5 of lr_t beyond half a unit in the last place of the stored p"""
    p0, m0, v0, g, p1, m1, v1 = (t.double() for t in (p0, m0, v0, g, p1, m1, v1))
    gi = g * gscale
    bm, tm = B1 * m0, (1 - B1) * gi
    bv, tv = B2 * v0, (1 - B2) * gi * gi
    m64, v64 = bm + tm, bv + tv
    lr_t = _lr_t(lr, step)
    inc64 = -lr_t * m64 / (torch.sqrt(v64) + EPS)
    half_ulp = 0.5 * (torch.nextafter(p1.float().abs(), torch.tensor(float("inf"), device=p1.device)).double() - p1.abs())
    em = ((m1 - m64).abs() / (4 * U32 * (bm.abs() + tm.abs()) + 4 * SUB32)).max()
    ev = ((v1 - v64).abs() / (4 * U32 * (bv + tv) + 4 * SUB32)).max()
    ei = (((p1 - p0) - inc64).abs() / (1e-5 * lr_t + half_ulp)).max()
    return float(em), float(ev), float(ei)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the trainer against float64
# ---------------------------------------------------------------------------------------------------------------------
def _check_indices(tr):
    """the trainer's FPS and ball-query indices of every sampled level equal the CPU oracle's on the same input coordinates"""
    for lv, (cur_xyz, _) in zip(tr.levels, tr.in_xyz):
        if lv.spec.group_all:
            continue
        cur = cur_xyz.detach().cpu().numpy()
        fps = orc.fps(cur, lv.m)
        assert np.array_equal(lv.fps_idx.cpu().numpy(), fps), f"{lv.spec.scope}: FPS differs from the oracle"
        idx, _ = orc.query_ball_point(lv.spec.radius, lv.k, cur, orc.gather_point(cur, fps), contract=True)
        assert np.array_equal(lv.idx.cpu().numpy(), idx), f"{lv.spec.scope}: ball query differs from the oracle"


def _restate(tr, p, xyz, labels, dtype):
    """restate.ssg on the run's decisions in `dtype`, mean cross-entropy differentiated -> (logits, x.grad, {variable: grad}, info)"""
    P = params_as(p, dtype, grad=not tr.frozen)
    x = xyz.detach().to(dtype, copy=True).requires_grad_(True)
    masks = {ly.scope: ly.mask for ly in tr.head if ly.mask is not None}
    info = {"flips": 0, "units": 0, "pool_gap": 0.0}
    logits = restate.ssg(x, P, tr.levels, tr.frozen, masks, run=tr, info=info)
    F.cross_entropy(logits, labels.long()).backward()
    grads = {} if tr.frozen else {k: P[k].grad for k in tr.fp.names}
    return logits.detach(), x.grad, grads, info


def _step_errors(tr, p, xyz, labels, logits, moving_before):
    """-> ({quantity: (error of the run, error of the float32 restatement, bound)}, the float64 restatement's info) for one step whose
    backward has run (with the coordinate gradient)"""
    l64, gx64, g64, info = _restate(tr, p, xyz, labels, torch.float64)
    l32, gx32, g32, info32 = _restate(tr, p, xyz, labels, torch.float32)
    errs = {"logits": (err(logits, l64), err(l32, l64), OTOL), "x.grad": (err(tr.input_xyz_grad(), gx64), err(gx32, gx64), GTOL)}
    # the loss kernel on the run's own logits
    gl = logits.detach().double()
    loss64 = float(F.cross_entropy(gl, labels.long()))
    dl64 = (torch.softmax(gl, 1) - F.one_hot(labels.long(), NUM_CLASS).double()) / tr.B
    errs["loss"] = (abs(float(tr.loss) - loss64) / max(1.0, loss64), 0.0, 1e-6)
    errs["dlogits"] = (err(tr.dlogits, dl64, 1.0 / tr.B), 0.0, 1e-6)
    if tr.frozen:
        return errs, info
    stats, stats32 = info["stats"], info32["stats"]
    assert len(stats) == 11                          # 3 x 3 level layers + fc1 + fc2
    for name in sorted(g64):
        got = tr.fp.grad_of(name)
        if name.endswith("/biases") and name[:-len("/biases")] in stats:
            assert not bool(got.any()), f"{name}: a bias followed by batch norm must get a gradient of exactly zero"
            continue
        scale = float(g64[name].abs().max())
        if name in POOLED_BETAS:
            scale = max(scale, float(g64[name.replace("/beta", "/gamma")].abs().max()))
        errs[name] = (err(got, g64[name], scale), err(g32[name], g64[name], scale), GTOL)
    for scope in stats:
        for i, suffix in enumerate(("moving_mean", "moving_variance")):
            name = f"{scope}/bn/{suffix}"
            want = DECAY * moving_before[name] + (1 - DECAY) * stats[scope][i]
            yard = DECAY * moving_before[name] + (1 - DECAY) * stats32[scope][i].double()
            errs[name] = (err(p[name], want), err(yard, want), OTOL)
    return errs, info


def _report(tag, errs, info, seconds):
    worst = max(errs, key=lambda k: errs[k][0] / errs[k][2])
    grads = [k for k in errs if k.endswith(("/weights", "/biases", "/gamma", "/beta"))]
    wg = max(grads, key=lambda k: errs[k][0]) if grads else None
    moving = [k for k in errs if "/moving_" in k]
    wm = max(moving, key=lambda k: errs[k][0]) if moving else None
    line = (f"[{tag}] flips {info['flips']} of {info['units']}, pool gap {info['pool_gap']:.1e}; error (float32 restatement's): "
            f"logits {errs['logits'][0]:.2e} ({errs['logits'][1]:.2e}), x.grad {errs['x.grad'][0]:.2e} ({errs['x.grad'][1]:.2e}), "
            f"loss {errs['loss'][0]:.1e}, dlogits {errs['dlogits'][0]:.1e}")
    if wg is not None:
        line += (f", worst variable gradient {errs[wg][0]:.2e} ({errs[wg][1]:.2e}, {wg}), "
                 f"worst moving average {errs[wm][0]:.2e} ({errs[wm][1]:.2e}, {wm})")
    line += (f"; worst against its bound: {worst}; {seconds:.1f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
    print(line)


def _check_step(tag, errs, info):
    assert info["flips"] <= 1e-4 * info["units"], (tag, info["flips"], info["units"])
    assert info["pool_gap"] <= 1e-5, (tag, info["pool_gap"])
    over = {k: f"{e:.2e} ({e32:.2e}) > {tol:.0e}" for k, (e, e32, tol) in errs.items() if not within(e, e32, tol, 2)}
    assert not over, (tag, over)


def _train_steps(p, cloud, b, n, steps, seed0):
    """steps consecutive training steps of the benchmark's trainer, each checked against float64 together with its Adam update"""
    tr = PointNet2ClsTrainer(p, b, n, NUM_CLASS)
    labels = torch.from_numpy(np.random.default_rng(0).integers(0, NUM_CLASS, b).astype(np.int32)).cuda()
    moving_names = [k for k in p.keys() if k.endswith(("/moving_mean", "/moving_variance"))]
    fp = tr.fp
    for i in range(steps):
        tag = f"ssg step {i + 1} {cloud} B={b} N={n}"
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        xyz = torch.from_numpy(make_clouds(cloud, b, n, seed=seed0 + i)).cuda()
        moving_before = {k: p[k].double().clone() for k in moving_names}
        tr.draw_dropout()
        logits = tr.forward(xyz, DECAY)
        _, dl = tr.loss_and_grad(logits, labels)
        tr.backward(dl, xyz_grad=True)
        _check_indices(tr)
        errs, info = _step_errors(tr, p, xyz, labels, logits, moving_before)
        state = [t.clone() for t in (fp.flat, fp.adam_m, fp.adam_v, fp.grad)]
        tr.adam(LR)
        torch.cuda.synchronize()
        em, ev, ei = _adam_errors(*state, fp.flat, fp.adam_m, fp.adam_v, LR, fp.step_count, 1.0)
        _report(tag, errs, info, time.perf_counter() - t0)
        print(f"[{tag}] adam (error / allowance): m {em:.2f}, v {ev:.2f}, increment {ei:.2f}")
        _check_step(tag, errs, info)
        assert em <= 1 and ev <= 1 and ei <= 1, (tag, em, ev, ei)
        del errs, info, state
        torch.cuda.empty_cache()


def test_benchmarked_training_steps_match_float64():
    """bench.py's training workload: init_params(seed=1), make_clouds("ball", 32, 2048, seed=2001 + i) for step i, lr 1e-3, decay 0.5,
    dropout on; four consecutive steps"""
    _train_steps(pointnet2_cls_ssg.init_params(seed=1), "ball", 32, 2048, 4, 2001)


def test_training_step_on_duplicated_points_matches_float64():
    """a quarter of every cloud duplicates its first point: exact ties in FPS, in the ball query and in the max-pool"""
    _train_steps(pointnet2_cls_ssg.init_params(seed=3, randomize_bn=True), "dup", 32, 1024, 1, 2001)


def test_inference_mode_logits_and_xyz_grad_match_float64():
    """the frozen trainer (batch norm on the moving averages) at the benchmarked shape: logits 1e-5, the input cloud's gradient 1e-4"""
    b, n = 32, 2048
    p = pointnet2_cls_ssg.init_params(seed=1, randomize_bn=True)
    tr = PointNet2ClsTrainer(p, b, n, NUM_CLASS, frozen=True)
    labels = torch.from_numpy(np.random.default_rng(0).integers(0, NUM_CLASS, b).astype(np.int32)).cuda()
    xyz = torch.from_numpy(make_clouds("ball", b, n, seed=2001)).cuda()
    moving = restate.moving(p)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    logits = tr.forward(xyz)
    _, dl = tr.loss_and_grad(logits, labels)
    tr.backward(dl, xyz_grad=True)
    _check_indices(tr)
    errs, info = _step_errors(tr, p, xyz, labels, logits, None)
    tag = f"ssg frozen B={b} N={n}"
    _report(tag, errs, info, time.perf_counter() - t0)
    assert all(torch.equal(moving[k], p[k]) for k in moving), "inference mode must not move the moving averages"
    _check_step(tag, errs, info)


# ---------------------------------------------------------------------------------------------------------------------
# 2. the loss and optimizer kernels on their own
# ---------------------------------------------------------------------------------------------------------------------
def _softmax_xent(logits, labels):
    b, c = logits.shape
    loss = torch.full((1,), float("nan"), device="cuda")
    dl = torch.full((b, c), float("nan"), device="cuda")
    _lib.check(_lib.load().psa_softmax_xent(b, c, ptr(logits), ptr(labels), ptr(loss), ptr(dl), stream()), "softmax_xent")
    torch.cuda.synchronize()
    return loss, dl


@pytest.mark.parametrize("offset", [0.0, 30.0, 1e3, 1e4])
@pytest.mark.parametrize("c", [1, 2, 15, 40])
@pytest.mark.parametrize("b", [1, 31, 32, 33, 1024])
def test_softmax_xent_matches_float64(b, c, offset):
    """mean cross-entropy and its gradient against float64 on the same fp32 logits: N(0, 3) plus a common offset, which leaves the
    loss unchanged and must not cost it digits; labels at 0 and c-1; a row of equal logits and a row whose label logit is 80 below
    the row's max.  loss within 1e-6 * max(1, loss), dlogits within 1e-6 / b."""
    rng = np.random.default_rng(b * 100 + c)
    x = rng.normal(0.0, 3.0, (b, c))
    lab = rng.integers(0, c, b)
    lab[0], lab[-1] = 0, c - 1
    if b >= 3:
        x[1] = 0.25                                                  # equal logits
    if b >= 4 and c >= 2:
        lab[2] = 0
        x[2, 0] = x[2, 1:].max() - 80.0                              # the label's probability is ~e^-80
    logits = torch.from_numpy((x + offset).astype(np.float32)).cuda()
    labels = torch.from_numpy(lab.astype(np.int32)).cuda()
    loss, dl = _softmax_xent(logits, labels)
    l64 = logits.double()
    want = F.cross_entropy(l64, labels.long())
    want_dl = (torch.softmax(l64, 1) - F.one_hot(labels.long(), c).double()) / b
    e_loss = abs(float(loss) - float(want)) / max(1.0, float(want))
    e_dl = float((dl.double() - want_dl).abs().max()) * b
    assert e_loss <= 1e-6, f"loss {float(loss)!r} vs {float(want)!r}: error {e_loss:.2e} of max(1, loss)"
    assert e_dl <= 1e-6, f"dlogits error {e_dl:.2e} of 1/b"


def test_softmax_xent_refuses_more_than_1024_rows():
    """one block holds the batch: b = 1025 is refused"""
    b, c = 1025, 15
    logits = torch.zeros((b, c), device="cuda")
    labels = torch.zeros(b, dtype=torch.int32, device="cuda")
    with pytest.raises(_lib.PsaError, match="1024"):
        _softmax_xent(logits, labels)


@pytest.mark.parametrize("gscale", [1.0, 0.5])
@pytest.mark.parametrize("step", [1, 2, 10, 10000])
@pytest.mark.parametrize("count", [0, 1, 255, 257, 270_337, 1_500_000])
def test_adam_step_matches_float64(count, step, gscale):
    """psa_adam_step against float64 Adam on the same inputs: gradients of magnitudes 1e-3 .. 1e3, exact zeros (with zero moments, so
    the parameter must not move), values whose square underflows fp32; half the parameters zero, so their increment is seen
    unrounded.  count past 8 * 132 * 256 = 270,336 runs the kernel's grid-stride loop; nothing past count is written; two calls on
    the same inputs agree bit for bit."""
    pad = 64
    gen = torch.Generator(device="cuda")
    gen.manual_seed(count * 31 + step)
    n = count + pad
    mag = 10.0 ** (torch.rand(n, generator=gen, device="cuda") * 6 - 3)
    g = torch.randn(n, generator=gen, device="cuda") * mag
    sel = torch.randint(0, 8, (n,), generator=gen, device="cuda")
    g = torch.where(sel == 0, torch.zeros_like(g), g)                # exact zeros
    g = torch.where(sel == 1, torch.randn(n, generator=gen, device="cuda") * 1e-25, g)      # g^2 underflows
    # moments as a run leaves them: |m| / sqrt(v) <= 0.3
    r = torch.randn(n, generator=gen, device="cuda")
    m = 0.3 * mag * r
    v = mag * mag * (r * r + torch.randn(n, generator=gen, device="cuda") ** 2)
    m = torch.where(sel == 0, torch.zeros_like(m), m)
    v = torch.where(sel == 0, torch.zeros_like(v), v)
    p = torch.randn(n, generator=gen, device="cuda") * (torch.arange(n, device="cuda") % 2)
    lib = _lib.load()
    outs = []
    for _ in range(2):
        p1, m1, v1 = p.clone(), m.clone(), v.clone()
        _lib.check(lib.psa_adam_step(count, ptr(p1), ptr(g), ptr(m1), ptr(v1), C.c_float(LR), C.c_float(B1), C.c_float(B2), C.c_float(EPS),
                                     step, C.c_float(gscale), stream()), "adam_step")
        outs.append((p1, m1, v1))
    torch.cuda.synchronize()
    (p1, m1, v1), (p2, m2, v2) = outs
    assert torch.equal(p1, p2) and torch.equal(m1, m2) and torch.equal(v1, v2), "two calls on the same inputs must agree bit for bit"
    for got, before in ((p1, p), (m1, m), (v1, v)):
        assert torch.equal(got[count:], before[count:]), "psa_adam_step wrote past count"
    if count == 0:
        return
    k = slice(0, count)
    still = sel[k] == 0
    assert torch.equal(p1[k][still], p[k][still]), "a zero gradient with zero moments must leave the parameter where it is"
    em, ev, ei = _adam_errors(p[k], m[k], v[k], g[k], p1[k], m1[k], v1[k], LR, step, gscale)
    assert em <= 1 and ev <= 1 and ei <= 1, f"error / allowance: m {em:.2f}, v {ev:.2f}, increment {ei:.2f}"
