"""pointnet2_cls_partseg against a float64 restatement that builds fa_layer1's input as the reference does
(pointnet2/models/pointnet2_cls_partseg.py:20-87, pointnet_util.py:199-229): three_nn with the missing neighbours at infinity, the
inverse-distance weights, the interpolation (a tile of l3_points) and the concatenation with l2_points, on the run's own FPS and
ball-query indices.  Inference outputs, one training step (outputs, moving averages, the flat gradient) and the inference-mode
gradient with respect to the cloud; then the grouped fa_layer1 against pointnet_fp_module on the materialised input, and the
generalised grouped helpers in their default (point rows first) order.

Where fp32 and float64 can legitimately disagree, the comparisons apply the exclusion rule of tests/restate.py: a max over a
neighbourhood whose runner-up is within 1e-5 of it has its gradient zeroed on both sides, and the restatement takes the run's relu
decisions and, in training mode, the values of its batch statistics.  Both counts are printed."""
import pytest
import torch

from scanobjectnn_b200 import ops, pointnet2_cls_partseg, pointnet_seg, training
from scanobjectnn_b200.pointnet_util import pointnet_fp_module, pointnet_fp_module_broadcast
from scanobjectnn_b200.synthetic import make_clouds

from . import gpu_util as G
from . import restate
from .restate import Masks, RunDecisions, flat_grad, grad_errors, moving, out_err, params_as, rel, within

pytestmark = pytest.mark.gpu
OTOL, GTOL = 1e-5, 1e-4
F = torch.nn.functional
M = pointnet2_cls_partseg
LEVELS = [("layer1", 512, 0.2, 64), ("layer2", 128, 0.4, 64)]          # (scope, npoint, radius, nsample); layer3 groups all
FA1 = ["fa_layer1/conv_0", "fa_layer1/conv_1"]


def _indices(p, x, mode):
    """per level (fps_idx, ball-query idx) as int64: those the run's level trainers used (mode "level" / "level_frozen"), or for the
    fused inference path the same kernels' results on the run's coordinates"""
    if mode is not None:
        lv = {key[1]: tr.levels[0] for key, tr in p.__dict__["_trainers"].items() if key[0] == mode}
        return [(lv[s].fps_idx.long(), lv[s].idx.long()) for s, _, _, _ in LEVELS]
    out, cur = [], x.detach()
    for _, m, r, k in LEVELS:
        f = ops.farthest_point_sample(m, cur)
        new = ops.gather_point(cur, f)
        out.append((f.long(), ops.query_ball_point(r, k, cur, new)[0].long()))
        cur = new
    return out


def _setup(b, n, seed):
    p = M.init_params(seed=seed, randomize_bn=True)
    x = G.cu(make_clouds("ball", b, n, seed=seed + 100))
    parts = torch.randint(0, M.NUM_CLASSES, (b, n), device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed))
    return p, x, parts


@pytest.mark.parametrize("b,n", [(4, 1024), (32, 2048)])
def test_inference_outputs_match_float64(b, n):
    p, x, parts = _setup(b, n, seed=n + b)
    with torch.no_grad():
        seg = M.get_model(x, False, params=p)
        seg2, ep = M.get_model(x, False, params=p, return_end_points=True)
    assert seg.shape == (b, n, 6) and torch.equal(seg, seg2)
    assert ep["l3_points"].shape == (b, 1, 1024) and ep["l2_points"].shape == (b, 128, 256) and ep["feats"].shape == (b, n, 128)
    want, _ = restate.pointnet2_partseg(x.double().requires_grad_(True), params_as(p, torch.float64), True, Masks(), _indices(p, x, None))
    want = want.detach()
    err = out_err(seg.cpu(), want.cpu())
    print(f"[partseg inference B={b} N={n}] output error {err:.2e}")
    assert err < OTOL
    assert abs(float(M.get_loss(seg, parts)) - float(F.cross_entropy(want.transpose(1, 2), parts, reduction="none").mean(1).mean())) < 1e-5
    with pytest.raises(ValueError, match="num_class=4"):
        M.get_model(x, False, num_class=4, params=p)


def _against_float64(b, n, seed, frozen, monkeypatch):
    """one GPU pass (training step without dropout, or frozen inference with x.grad) and its float64 restatement on the same
    indices, relu decisions and masks -> (p, P, x, x64, seg_pred, float64 seg_pred, info)"""
    p, x0, parts = _setup(b, n, seed)
    with torch.no_grad():
        fused = M.get_model(x0, False, params=p) if frozen else None
    P0 = params_as(p, torch.float64)
    moving0 = moving(p)
    idx = _indices(p, x0, None)                        # sampling and grouping depend on the coordinates only
    masks = Masks()                                    # pass 1: the ambiguous maxima
    restate.pointnet2_partseg(x0.double().requires_grad_(True), P0, frozen, masks, idx)
    masked, total = masks.count()
    x = x0.clone().requires_grad_(frozen)
    with monkeypatch.context() as m:
        masks.patch(m)
        seg = M.get_model(x, False, params=p) if frozen else M._get_model_training(x, 0.5, p, dropout=False)
        assert seg.grad_fn is not None
        M.get_loss(seg, parts).backward()
    run_idx = _indices(p, x0, "level_frozen" if frozen else "level")
    assert all(torch.equal(a, c) and torch.equal(a2, c2) for (a, a2), (c, c2) in zip(run_idx, idx)), "the run sampled other indices"
    P = params_as(P0, torch.float64, grad=not frozen)
    masks2 = masks.replay()                            # pass 2, with the run's relu decisions (and batch statistics)
    x64 = x0.double().requires_grad_(True)
    want, info = restate.pointnet2_partseg(x64, P, frozen, masks2, run_idx, RunDecisions(p, frozen))
    F.cross_entropy(want.transpose(1, 2), parts, reduction="none").mean(1).mean().backward()
    assert masks2.count() == (masked, total)
    print(f"[partseg {'frozen' if frozen else 'training'} B={b} N={n}] masked: {masked} of {total}; relu decisions that differ "
          f"from float64's: {info['flips']} of {info['units']}; batch statistics' error relative to E[y^2]: {info['stat_err']:.2e}")
    assert masked <= 0.01 * total and info["flips"] <= 1e-4 * info["units"] and info["stat_err"] < GTOL
    if frozen:                                         # the frozen path agrees with the fused one and touches no variable
        assert rel(seg.detach().cpu(), fused.cpu()) < 1e-4
        assert all(torch.equal(p[k], v) for k, v in moving0.items()) and p._flat.flat.grad is None
        return p, P, x, x64, seg, want, info
    P32 = params_as(P0, torch.float32, grad=True)
    want32, _ = restate.pointnet2_partseg(x0.clone(), P32, frozen, masks.replay(), run_idx, RunDecisions(p, frozen))
    F.cross_entropy(want32.transpose(1, 2), parts, reduction="none").mean(1).mean().backward()
    return p, (P, P32), x, x64, seg, (want, want32), info


@pytest.mark.parametrize("b,n", [(4, 1024), (32, 2048)])
def test_one_training_step_matches_float64(b, n, monkeypatch):
    """Outputs within 1e-5, moving averages, and the flat gradient within 1e-4 of its largest entry, or, where fp32 itself does not
    resolve 1e-4, within 3x of a float32 evaluation of the same restatement (printed)"""
    p, (P, P32), _, _, got, (want, want32), info = _against_float64(b, n, 5, False, monkeypatch)
    err, err32 = out_err(got.detach().cpu(), want.detach().cpu()), out_err(want32.detach().cpu(), want.detach().cpu())
    print(f"[partseg training B={b} N={n}] output error {err:.2e} (float32 restatement: {err32:.2e})")
    assert within(err, err32, OTOL, 3)
    for scope, (mean, var) in info["stats"].items():
        for suffix, batch in (("moving_mean", mean), ("moving_variance", var)):
            w = 0.5 * P[f"{scope}/bn/{suffix}"].detach() + 0.5 * batch
            assert rel(p[f"{scope}/bn/{suffix}"].cpu(), w.cpu()) < OTOL, (scope, suffix)
    assert {s.rsplit("/", 1)[0] for s in info["stats"]} >= {"layer3", "fa_layer1", "seg_fc1"}
    errs, scale = grad_errors(p, P, P32)
    over = {k: (e / scale, e32 / scale) for k, (e, e32) in errs.items() if e > GTOL * scale}
    worst = max(errs, key=lambda k: errs[k][0])
    print(f"[partseg training B={b} N={n}] gradient error relative to the largest entry: {errs[worst][0] / scale:.2e} ({worst}); "
          f"beyond 1e-4 (run, float32 restatement): {over}")
    assert all(within(e, e32, GTOL, 3) for e, e32 in over.values()), over
    # fa_layer1/conv_0's two row blocks (l3_points' 1024 rows first, then l2_points' 256) and the group-all level's variables
    w0 = flat_grad(p, "fa_layer1/conv_0/weights").view(1280, 256).double()
    want0 = P["fa_layer1/conv_0/weights"].grad.view(1280, 256)
    for name, rows in (("l3_points rows", slice(0, 1024)), ("l2_points rows", slice(1024, 1280))):
        e = float((w0[rows].cpu() - want0[rows].cpu()).abs().max()) / scale
        print(f"[partseg training B={b} N={n}] fa_layer1/conv_0 {name}: {e:.2e} of the largest entry")
        assert e < GTOL
        assert float(want0[rows].abs().max()) > 0
    for k in [k for k in errs if k.startswith("layer3/")]:
        assert errs[k][0] < GTOL * scale or errs[k][0] <= 3 * errs[k][1], k


def test_inference_input_grad_matches_float64(monkeypatch):
    _, _, x, x64, got, want, _ = _against_float64(4, 1024, 9, True, monkeypatch)
    assert out_err(got.detach().cpu(), want.detach().cpu()) < OTOL
    err = rel(x.grad.cpu(), x64.grad.cpu())
    print(f"[partseg frozen] x.grad error relative to its largest entry: {err:.2e}")
    assert err < GTOL


def _fa1_inputs(b, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    l2_xyz = torch.rand((b, 128, 3), device="cuda", generator=gen) * 2 - 1
    l3_xyz = torch.zeros((b, 1, 3), device="cuda")                      # the group-all level's centre
    l2_points = torch.relu(torch.randn((b, 128, 256), device="cuda", generator=gen))
    l3_points = torch.relu(torch.randn((b, 1, 1024), device="cuda", generator=gen))
    return l2_xyz, l3_xyz, l2_points, l3_points


@pytest.mark.parametrize("b", [4, 32])
def test_grouped_fa_layer1_matches_the_materialised_fp_module(b):
    """pointnet_fp_module_broadcast against pointnet_fp_module (three_nn + interpolation + concat, K = 1280) on the same inputs: in
    inference, and in training mode (outputs, the gradients of l2_points and l3_points, and fa_layer1's variable gradients)"""
    p = M.init_params(seed=b, randomize_bn=True)
    l2_xyz, l3_xyz, l2_points, l3_points = _fa1_inputs(b, b)
    args = (l2_xyz, l3_xyz)
    with torch.no_grad():
        g = pointnet_fp_module_broadcast(*args, l2_points, l3_points, [256, 256], False, None, "fa_layer1", params=p)
        c = pointnet_fp_module(*args, l2_points, l3_points, [256, 256], False, None, "fa_layer1", params=p)
    diff = rel(g.cpu(), c.cpu())
    print(f"[fa_layer1 inference B={b}] grouped vs materialised: {diff:.2e} of the largest entry")
    assert g.shape == (b, 128, 256) and diff < 5e-6
    R = torch.randn((b, 128, 256), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    names = [f"{s}/{v}" for s in FA1 for v in ("weights", "biases", "bn/gamma", "bn/beta")]
    res = []
    for fn in (pointnet_fp_module_broadcast, pointnet_fp_module):
        x2, x3 = l2_points.clone().requires_grad_(True), l3_points.clone().requires_grad_(True)
        out = fn(*args, x2, x3, [256, 256], True, 0.5, "fa_layer1", params=p)
        (out * R).sum().backward()
        res.append((out.detach(), x2.grad, x3.grad, torch.cat([flat_grad(p, k).reshape(-1) for k in names])))
        p._flat.flat.grad = None
    for name, a, c in zip(("output", "d l2_points", "d l3_points", "variable gradients"), *res):
        d = rel(a.cpu(), c.cpu())
        print(f"[fa_layer1 training B={b}] {name}: grouped vs materialised {d:.2e} of the largest entry")
        assert d < 5e-6, name


def test_fold_needs_a_single_known_point():
    p = M.init_params(seed=0)
    l2_xyz, _, l2_points, l3_points = _fa1_inputs(2, 0)
    with pytest.raises(ValueError, match="one point"):
        pointnet_fp_module_broadcast(l2_xyz, l2_xyz[:, :2], l2_points, l3_points.expand(2, 2, 1024), [256, 256], False, None, "fa_layer1",
                                     params=p)


def test_grouped_helpers_default_to_point_rows_first():
    """VariableStore.grouped_mlp and MlpTrainer without group_first slice the first weight as [points; group], as pointnet_seg's
    head uses them; with group_first as [group; points], and the gradient views are the matching rows of the flat bucket"""
    p = pointnet_seg.init_params(seed=1, randomize_bn=True)
    w = p.folded("conv6")[0]
    for first, (pts, glob) in ((False, (w[:64], w[64:])), (True, (w[1024:], w[:1024]))):
        rows_mlp, global_mlp = p.grouped_mlp(["conv6"], 64, group_first=first)
        assert torch.equal(rows_mlp._weights[0], pts) and torch.equal(global_mlp._weights[0], glob)
    assert p.grouped_mlp(["conv6"], 64) is p.grouped_mlp(["conv6"], 64, group_first=False)
    for first in (False, True):
        tr = training.MlpTrainer(p, 4 * 16, 64, [("conv6", True)], groups=4, group_channels=1024, group_first=first)
        W, dW = tr.layers[0].W, tr.layers[0].dW
        x_rows, g_rows = (slice(1024, None), slice(0, 1024)) if first else (slice(0, 64), slice(64, None))
        for got, want in ((tr.W_x, W[x_rows]), (tr.W_g, W[g_rows]), (tr.dW_x, dW[x_rows]), (tr.dW_g, dW[g_rows])):
            assert got.data_ptr() == want.data_ptr() and got.shape == want.shape
    tr = training.MlpTrainer(p, 64, 64, [("conv6", True)], groups=4, group_channels=1024)
    assert tr.W_x.data_ptr() == tr.layers[0].W.data_ptr() and tr.W_x.shape == (64, 512) and tr.W_g.shape == (1024, 512)
    assert tr.W_g.data_ptr() == tr.layers[0].W[64].data_ptr() and tr.dW_g.data_ptr() == tr.layers[0].dW[64].data_ptr()
