"""Inference layers and models against float64 with batch norm CALIBRATED to the data they see.

The other parity tests draw batch-norm statistics that have nothing to do with the activations (tf_util.VariableStore._bn), so the
folded scale gamma / sqrt(moving_var + 1e-3) stays between 0.65 and 1.7.  A trained checkpoint's moving statistics are those of the
pre-batch-norm activations themselves: the folded scale is gamma / sqrt(var(y) + 1e-3), up to 31.6 gamma, and every MLP kernel
applies it after the product, so an absolute error of the product reaches the output multiplied by it.  Batch norm also makes a
layer's output independent of the scale of its weights (up to eps), so a checkpoint may carry weights of any magnitude.

Here every batch-norm layer's weights are multiplied by s, then its moving mean and (biased) variance are set to the float64
statistics of its own pre-batch-norm output on a calibration batch (another draw of the same generator), and the layer / model is
held to the 1e-5 contract against float64 on a fresh batch, in every arithmetic mode.  Each case asserts that it ran in the regime
(largest folded scale > 10), so a calibration that silently did nothing fails."""
import numpy as np
import pytest
import torch

from oracle import mlp_oracle as mo
from oracle import oracle as orc
from scanobjectnn_b200 import dgcnn, ops, pointnet2_cls_bga, pointnet2_cls_ssg, pointnet_cls, pointnet_seg
from scanobjectnn_b200.engine import pointnet2_cls_ssg_engine
from scanobjectnn_b200.pointnet_util import (add_fp_module_params, add_sa_module_params, pointnet_fp_module,
                                              pointnet_fp_module_broadcast, pointnet_sa_module)
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import BN_EPS, VariableStore

from . import gpu_util as G

pytestmark = pytest.mark.gpu
SCALES = [1.0, 0.1, 0.01, 1e-4]
REGIME = 10.0          # the largest folded scale a case must reach (s <= 0.1, and SA1's conv0 at s = 1)


@pytest.fixture(params=[0, 1, 2], ids=["tensor", "fma", "tensor_bf16x3"])
def mlp_mode(request):
    """0 = tensor cores where the shapes allow (fp16x2 operands + range guard), 1 = fp32 FMA kernels, 2 = tensor cores, bf16x3"""
    ops.set_mlp_mode(request.param)
    try:
        yield request.param
    finally:
        ops.set_mlp_mode(0)


def _bn_scopes(p):
    return [k[: -len("/bn/gamma")] for k in p if k.endswith("/bn/gamma")]


def _scale_weights(p, s):
    """multiply the weights of every batch-norm layer by s (the layer's output after calibration does not depend on it)"""
    for scope in _bn_scopes(p):
        p[f"{scope}/weights"] = p[f"{scope}/weights"] * s


def calibrate(p, monkeypatch, oracle_pass):
    """Run ``oracle_pass()`` (a float64 oracle evaluation on a calibration batch) with mlp_oracle.conv_bn_relu wrapped so that every
    batch-norm layer of ``p`` it reaches first gets moving_mean / moving_variance := the mean / biased variance over all rows of its
    float64 pre-batch-norm output.  Every oracle model runs its layers through mlp_chain -> conv_bn_relu in forward order, so one
    pass calibrates each layer on inputs produced by the already calibrated layers before it.  -> the calibrated scopes."""
    done = []
    orig = mo.conv_bn_relu

    def wrapper(x, params, scope, relu=True, dtype=np.float64):
        if params is p and f"{scope}/bn/gamma" in params and scope not in done:
            w = mo._np(params[f"{scope}/weights"], np.float64)
            y = np.asarray(x, np.float64) @ w.reshape(-1, w.shape[-1]) + mo._np(params[f"{scope}/biases"], np.float64)
            y = y.reshape(-1, y.shape[-1])
            dev = params[f"{scope}/bn/gamma"].device
            params[f"{scope}/bn/moving_mean"] = torch.tensor(y.mean(0), dtype=torch.float32, device=dev)
            params[f"{scope}/bn/moving_variance"] = torch.tensor(y.var(0), dtype=torch.float32, device=dev)
            done.append(scope)
        return orig(x, params, scope, relu, dtype)

    with monkeypatch.context() as m:
        m.setattr(mo, "conv_bn_relu", wrapper)
        oracle_pass()
    p.invalidate()
    return done


def folded_scale(p, scope):
    v = p[f"{scope}/bn/gamma"].double() / torch.sqrt(p[f"{scope}/bn/moving_variance"].double() + BN_EPS)
    return float(v.abs().max())


def check_regime(p, scopes, s, first=None):
    """every batch-norm layer of the case was calibrated; the largest folded scale it runs with (printed) reaches the regime for
    s <= 0.1, and so does ``first`` (SA1's conv0, whose inputs are offsets of at most r = 0.2) at any s"""
    assert scopes and sorted(scopes) == sorted(_bn_scopes(p)), f"calibration missed {set(_bn_scopes(p)) - set(scopes)}"
    big = max(folded_scale(p, x) for x in scopes)
    print(f"[regime] s={s:g}: largest folded scale {big:.2f}" + (f", {first}: {folded_scale(p, first):.2f}" if first else ""))
    if s <= 0.1:
        assert big > REGIME, f"largest folded scale {big:.2f}: batch norm was not calibrated into the regime"
    if first is not None:
        assert folded_scale(p, first) > REGIME, f"{first}: folded scale {folded_scale(p, first):.2f}"
    return big


def _relu_normal(rng, shape):
    return np.maximum(rng.standard_normal(shape), 0.0).astype(np.float32)


def _store(seed):
    return VariableStore(device="cuda", seed=seed)


def _close(got, want, what):
    return G.contract_close(got, want, what)


# ------------------------------------------------------------------------------------------------------------------------------
# layers
# ------------------------------------------------------------------------------------------------------------------------------
def _chain_rows(rng, rows, c0):
    """rows as the SA3 / head layers see them: coordinates in the unit ball first, then post-ReLU features"""
    x = _relu_normal(rng, (rows, c0))
    x[:, :3] = rng.uniform(-1, 1, (rows, 3))
    return x


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("case", ["sa3_pool", "dense", "fc_head"])
def test_shared_mlp_calibrated(case, s, mlp_mode, monkeypatch):
    rows, pool_k, chans, relus = {
        "sa3_pool": (8 * 128, 128, [259, 256, 512, 1024], None),          # the group-all chain, pool_k = n
        "dense": (2048, 1, [128, 256, 128], None),                        # pool_k = 1, eligible for the tensor cores
        "fc_head": (32, 1, [1024, 512, 256, 15], [True, True, False]),    # the FC head at 32 rows, last layer without batch norm
    }[case]
    p = _store(17)
    scopes = [f"m/l{i}" for i in range(len(chans) - 1)]
    for i, sc in enumerate(scopes):
        p.add_conv2d(sc, chans[i], chans[i + 1], bn=relus is None or relus[i], randomize_bn=True)
    relus = relus or [True] * len(scopes)
    _scale_weights(p, s)
    rng = np.random.default_rng(5)
    xc = _chain_rows(rng, rows, chans[0])
    done = calibrate(p, monkeypatch, lambda: mo.mlp_chain(xc, p, scopes, relus))
    check_regime(p, done, s)
    x = _chain_rows(rng, rows, chans[0])
    got = G.npy(ops.shared_mlp(G.cu(x), p.mlp(scopes, relus), pool_k=pool_k))
    want = mo.mlp_chain(x, p, scopes, relus)
    if pool_k > 1:
        want = want.reshape(rows // pool_k, pool_k, -1).max(1)
    _close(got, want, f"shared_mlp {case} s={s:g} mode {mlp_mode}")


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("level", ["sa1", "sa2"])
def test_sa_module_calibrated(level, s, mlp_mode, monkeypatch):
    n, m, r, k, c, mlp = {"sa1": (2048, 512, 0.2, 32, 0, [64, 64, 128]), "sa2": (512, 128, 0.4, 64, 128, [128, 128, 256])}[level]
    b = 8
    p = _store(23)
    add_sa_module_params(p, "sa", 3 + c, mlp, randomize_bn=True)
    _scale_weights(p, s)
    rng = np.random.default_rng(7)

    def batch(seed):
        return make_clouds("ball", b, n, seed=seed), (_relu_normal(rng, (b, n, c)) if c else None)

    xyz_c, pts_c = batch(100)
    done = calibrate(p, monkeypatch, lambda: mo.sa_module(xyz_c, pts_c, m, r, k, mlp, False, "sa", p))
    check_regime(p, done, s, first="sa/conv0" if level == "sa1" else None)
    xyz, pts = batch(200)
    _, got, idx = pointnet_sa_module(G.cu(xyz), G.cu(pts) if c else None, m, r, k, mlp, None, False, False, None, "sa", params=p)
    _, want, oidx = mo.sa_module(xyz, pts, m, r, k, mlp, False, "sa", p)
    assert np.array_equal(G.npy(idx), oidx)
    _close(G.npy(got), want, f"sa_module {level} s={s:g} mode {mlp_mode}")


@pytest.mark.parametrize("s", SCALES)
def test_sa_group_all_calibrated(s, mlp_mode, monkeypatch):
    """sa_group_all_infer: the feature rows of the first layer on the tensor cores, its xyz rows added in the epilogue"""
    b, n, c, mlp = 8, 128, 256, [256, 512, 1024]
    p = _store(29)
    add_sa_module_params(p, "sa", 3 + c, mlp, randomize_bn=True)
    _scale_weights(p, s)
    rng = np.random.default_rng(11)

    def batch(seed):
        return make_clouds("ball", b, n, seed=seed), _relu_normal(rng, (b, n, c))

    xyz_c, pts_c = batch(300)
    done = calibrate(p, monkeypatch, lambda: mo.sa_module(xyz_c, pts_c, None, None, None, mlp, True, "sa", p))
    check_regime(p, done, s)
    xyz, pts = batch(400)
    _, got, _ = pointnet_sa_module(G.cu(xyz), G.cu(pts), None, None, None, mlp, None, True, False, None, "sa", params=p)
    _, want, _ = mo.sa_module(xyz, pts, None, None, None, mlp, True, "sa", p)
    _close(G.npy(got).reshape(want.shape), want, f"sa_group_all s={s:g} mode {mlp_mode}")


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("case", ["single", "tnet"])
def test_edgeconv_calibrated(case, s, mlp_mode, monkeypatch):
    """single: one layer, c = 64 -- the (W_a - W_b) . x_i + W_b . x_j algebra, its GEMM without a scale; tnet: DGCNN's two-layer
    transform-net EdgeConv over 3-D points (the set-abstraction kernel with centre weights)"""
    c, mlp = {"single": (64, [64]), "tnet": (3, [64, 128])}[case]
    b, n, k = 2, 1024, 20
    p = _store(31)
    scopes, cin = [], 2 * c
    for i, co in enumerate(mlp):
        p.add_conv2d(f"e/conv{i}", cin, co, bn=True, randomize_bn=True)
        scopes.append(f"e/conv{i}")
        cin = co
    _scale_weights(p, s)
    rng = np.random.default_rng(13)

    def batch(seed):
        return make_clouds("ball", b, n, seed=seed) if c == 3 else rng.standard_normal((b, n, c)).astype(np.float32)

    xc = batch(500)
    done = calibrate(p, monkeypatch, lambda: mo.edgeconv(xc, orc.dgcnn_knn(xc, k), p, scopes))
    check_regime(p, done, s)
    x = batch(600)
    idx = orc.dgcnn_knn(x, k)
    got = G.npy(ops.edgeconv_infer(G.cu(x), G.cu(idx), p.mlp(scopes)))
    _close(got, mo.edgeconv(x, idx, p, scopes), f"edgeconv {case} s={s:g} mode {mlp_mode}")


@pytest.mark.parametrize("s", SCALES)
def test_shared_mlp_grouped_calibrated(s, mlp_mode, monkeypatch):
    """PointNet's segmentation head: conv6 reads [point features (64), tiled global feature (1024)]; the global rows run once per
    cloud and the point layer adds their product per group of rows before its batch norm"""
    b, n = 8, 1024
    p = _store(37)
    for scope, cin, cout in zip(pointnet_seg.HEAD, [1088, 512, 256, 128], [512, 256, 128, 128]):
        p.add_conv2d(scope, cin, cout, bn=True, randomize_bn=True)
    _scale_weights(p, s)
    rng = np.random.default_rng(19)

    def batch():
        return _relu_normal(rng, (b, n, 64)), _relu_normal(rng, (b, 1024))

    def concat(x, g):
        return np.concatenate([x, np.broadcast_to(g[:, None, :], (b, n, 1024))], axis=2)

    xc, gc = batch()
    done = calibrate(p, monkeypatch, lambda: mo.mlp_chain(concat(xc, gc), p, pointnet_seg.HEAD))
    check_regime(p, done, s)
    x, g = batch()
    rows_mlp, global_mlp = p.grouped_mlp(pointnet_seg.HEAD[:1], 64)
    net = ops.shared_mlp_grouped(G.cu(x), rows_mlp, ops.shared_mlp(G.cu(g), global_mlp))
    got = G.npy(ops.shared_mlp(net, p.mlp(pointnet_seg.HEAD[1:])))
    _close(got, mo.mlp_chain(concat(x, g), p, pointnet_seg.HEAD), f"shared_mlp_grouped s={s:g} mode {mlp_mode}")


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("case", ["fp", "fp_broadcast"])
def test_fp_module_calibrated(case, s, mlp_mode, monkeypatch):
    """pointnet_fp_module (three-NN interpolation + concat + convs) and pointnet_fp_module_broadcast (one known point, its rows
    added per cloud as a group input)"""
    b = 8
    n1, n2, c1, c2, mlp = {"fp": (512, 128, 128, 256, [256, 128]), "fp_broadcast": (128, 1, 256, 1024, [256, 256])}[case]
    p = _store(41)
    add_fp_module_params(p, "fp", c2 + c1, mlp, randomize_bn=True)
    _scale_weights(p, s)
    rng = np.random.default_rng(43)

    def batch(seed):
        xyz2 = make_clouds("ball", b, n2, seed=seed + 1) if n2 > 1 else np.zeros((b, 1, 3), np.float32)
        return make_clouds("ball", b, n1, seed=seed), xyz2, _relu_normal(rng, (b, n1, c1)), _relu_normal(rng, (b, n2, c2))

    cal = batch(700)
    done = calibrate(p, monkeypatch, lambda: mo.fp_module(*cal, mlp, "fp", p))
    check_regime(p, done, s)
    xyz1, xyz2, p1, p2 = batch(800)
    fn = pointnet_fp_module if case == "fp" else pointnet_fp_module_broadcast
    got = G.npy(fn(G.cu(xyz1), G.cu(xyz2), G.cu(p1), G.cu(p2), mlp, False, None, "fp", params=p))
    _close(got, mo.fp_module(xyz1, xyz2, p1, p2, mlp, "fp", p), f"{case} s={s:g} mode {mlp_mode}")


# ------------------------------------------------------------------------------------------------------------------------------
# models: calibrated at s = 1 in every mode, and at s = 0.1 in mode 0.  Stage by stage: each stage's oracle is fed the GPU's inputs
# of that stage.  End to end, calibrated batch norm amplifies the rounding of every stage by its folded scale, and plain fp32 (mode 1)
# itself lands 1.2e-5 (relative) from float64 on the SSG logits and 1.1e-5 on the BGA segmentation logits; the 1e-5 contract is one
# of the layers, and each stage is held to it.
# ------------------------------------------------------------------------------------------------------------------------------
MODEL_CASES = [(0, 1.0), (1, 1.0), (2, 1.0), (0, 0.1)]
MODEL_IDS = ["tensor-s1", "fma-s1", "tensor_bf16x3-s1", "tensor-s0.1"]


@pytest.fixture(params=MODEL_CASES, ids=MODEL_IDS)
def model_case(request):
    mode, s = request.param
    ops.set_mlp_mode(mode)
    try:
        yield mode, s
    finally:
        ops.set_mlp_mode(0)


def _ssg_stages(xyz, logits, ep, p, tag):
    """pointnet2_cls_ssg's levels and head against the oracle, each fed the GPU's inputs of that stage"""
    b = xyz.shape[0]
    _, l1, idx1 = mo.sa_module(xyz, None, 512, 0.2, 32, [64, 64, 128], False, "layer1", p)
    assert np.array_equal(G.npy(ep["l1_indices"]), idx1)
    _close(G.npy(ep["l1_points"]), l1, f"ssg l1_points {tag}")
    _, l2, idx2 = mo.sa_module(G.npy(ep["l1_xyz"]), G.npy(ep["l1_points"]), 128, 0.4, 64, [128, 128, 256], False, "layer2", p)
    assert np.array_equal(G.npy(ep["l2_indices"]), idx2)
    _close(G.npy(ep["l2_points"]), l2, f"ssg l2_points {tag}")
    _, l3, _ = mo.sa_module(G.npy(ep["l2_xyz"]), G.npy(ep["l2_points"]), None, None, None, [256, 512, 1024], True, "layer3", p)
    _close(G.npy(ep["l3_points"]).reshape(l3.shape), l3, f"ssg l3_points {tag}")
    want = mo.mlp_chain(G.npy(ep["l3_points"]).reshape(b, -1), p, ["fc1", "fc2", "fc3"], [True, True, False])
    _close(G.npy(logits), want, f"ssg logits {tag}")


def test_pointnet2_cls_ssg_engine_calibrated(model_case, monkeypatch):
    """The benchmarked workload, B = 32, N = 2048, through the engine bench.py drives: 13 batches on 6 slots, each result read
    before its slot comes round again and bit-equal to the eager forward; the eager forward's levels and logits within the contract
    of float64."""
    mode, s = model_case
    b, n = 32, 2048
    p = pointnet2_cls_ssg.init_params(seed=1, randomize_bn=True)
    _scale_weights(p, s)
    cal = make_clouds("ball", b, n, seed=900)
    done = calibrate(p, monkeypatch, lambda: mo.pointnet2_cls_ssg(cal, p))
    check_regime(p, done, s, first="layer1/conv0")
    slots = 6
    engine = pointnet2_cls_ssg_engine(p, batch=b, npoints=n, num_class=15, slots=slots)
    batches = [make_clouds(("ball", "shell", "dup")[i % 3], b, n, seed=1000 + i) for i in range(13)]
    got, pending = {}, []
    for i, xyz in enumerate(batches):                 # up to `slots` batches in flight; a slot is read before it is reused
        if len(pending) == slots:
            j, slot = pending.pop(0)
            got[j] = engine.result(slot).clone()
        pending.append((i, engine.submit(G.cu(xyz))))
    for j, slot in pending:
        got[j] = engine.result(slot).clone()
    for i, xyz in enumerate(batches):
        logits, ep = pointnet2_cls_ssg.get_model(G.cu(xyz), False, params=p)
        assert torch.equal(got[i], logits), f"batch {i}: engine result differs from the eager forward"
        if i in (0, 12):
            _ssg_stages(xyz, logits, ep, p, f"batch {i} s={s:g} mode {mode}")


def test_pointnet2_cls_bga_calibrated(model_case, monkeypatch):
    """every set-abstraction and feature-propagation level of the forward is recorded with its GPU inputs and held against the
    oracle on those inputs; the heads are fed the GPU's l3_points and fa_layer3 output"""
    mode, s = model_case
    b, n = 8, 2048
    p = pointnet2_cls_bga.init_params(seed=3, randomize_bn=True)
    _scale_weights(p, s)
    cal = make_clouds("ball", b, n, seed=901)
    done = calibrate(p, monkeypatch, lambda: mo.pointnet2_cls_bga(cal, p))
    check_regime(p, done, s, first="layer1/conv0")
    xyz = make_clouds("shell", b, n, seed=902)
    calls = []

    def record(fn):
        def run(*args, **kw):
            out = fn(*args, **kw)
            calls.append((fn, args, kw, out))
            return out
        return run

    with monkeypatch.context() as m:
        m.setattr(pointnet2_cls_bga, "pointnet_sa_module", record(pointnet_sa_module))
        m.setattr(pointnet2_cls_bga, "pointnet_fp_module", record(pointnet_fp_module))
        cls, seg, ep = pointnet2_cls_bga.get_model(G.cu(xyz), False, params=p, return_end_points=True)
    tag = f"s={s:g} mode {mode}"
    assert len(calls) == 6
    for fn, args, kw, out in calls:
        h = [None if a is None else G.npy(a) if isinstance(a, torch.Tensor) else a for a in args]
        if fn is pointnet_sa_module:            # (xyz, points, npoint=, radius=, nsample=, mlp=, group_all=, scope=, ...)
            _, want, _ = mo.sa_module(h[0], h[1], kw["npoint"], kw["radius"], kw["nsample"], kw["mlp"], kw["group_all"], kw["scope"], p)
            _close(G.npy(out[1]).reshape(want.shape), want, f"bga {kw['scope']} {tag}")
        else:                                   # (xyz1, xyz2, points1, points2, mlp, is_training, bn_decay, scope=, ...)
            want = mo.fp_module(h[0], h[1], h[2], h[3], h[4], kw["scope"], p)
            _close(G.npy(out), want, f"bga {kw['scope']} {tag}")
    l3 = G.npy(ep["l3_points"]).reshape(b, -1)
    _close(G.npy(cls), mo.mlp_chain(mo.mlp_chain(l3, p, ["fc1", "fc2"]), p, ["fc3"], [False]), f"bga class_pred {tag}")
    _close(G.npy(ep["feats"]), mo.mlp_chain(G.npy(calls[-1][3]), p, ["seg_fc1"]), f"bga feats {tag}")
    _close(G.npy(seg), mo.mlp_chain(G.npy(ep["feats"]), p, ["seg_fc2"], [False]), f"bga seg_pred {tag}")


def test_pointnet_cls_calibrated(model_case, monkeypatch):
    """the input T-net, conv1-conv2, the feature T-net, conv3-conv5 + max and the FC head, each against the oracle on the GPU's
    inputs of that stage; the stages are the calls the forward makes (its feature transform and global feature, bit for bit)"""
    mode, s = model_case
    b, n = 8, 1024
    p = pointnet_cls.init_params(seed=6, randomize_bn=True)
    for name in ("transform_net1/transform_XYZ/weights", "transform_net2/transform_feat/weights"):
        p[name] = 0.01 * torch.randn(p[name].shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    _scale_weights(p, s)
    cal = make_clouds("shell", b, n, seed=903)
    done = calibrate(p, monkeypatch, lambda: mo.pointnet_cls(cal, p))
    check_regime(p, done, s)
    xyz = make_clouds("ball", b, n, seed=904)
    tag = f"s={s:g} mode {mode}"
    x = G.cu(xyz)
    logits, ep = pointnet_cls.get_model(x, False, params=p)
    t1 = pointnet_cls.transform_net(x, p, "transform_net1", 3)
    _close(G.npy(t1), mo._tnet(xyz, p, "transform_net1", 3, np.float64), f"pointnet input transform {tag}")
    xt = torch.bmm(x, t1).contiguous()
    net = ops.shared_mlp(xt.reshape(b * n, 3), p.mlp(["conv1", "conv2"])).reshape(b, n, 64)
    _close(G.npy(net), mo.mlp_chain(G.npy(xt), p, ["conv1", "conv2"]), f"pointnet conv2 {tag}")
    t2 = pointnet_cls.transform_net(net, p, "transform_net2", 64)
    assert torch.equal(t2, ep["transform"])
    _close(G.npy(t2), mo._tnet(G.npy(net), p, "transform_net2", 64, np.float64), f"pointnet feature transform {tag}")
    pf = torch.bmm(net, t2).contiguous()
    glob = ops.shared_mlp(pf.reshape(b * n, 64), p.mlp(["conv3", "conv4", "conv5"]), pool_k=n)
    assert torch.equal(glob, ep["global"])
    _close(G.npy(glob), mo.mlp_chain(G.npy(pf), p, ["conv3", "conv4", "conv5"]).max(axis=1), f"pointnet global {tag}")
    _close(G.npy(logits), mo.mlp_chain(G.npy(glob), p, ["fc1", "fc2", "fc3"], [True, True, False]), f"pointnet logits {tag}")


def _dgcnn_oracle_logits(xyz, p, k=20):
    """dgcnn.get_model in float64 on the oracle's own graphs (only used to calibrate: every layer in forward order)"""
    t = mo.edgeconv(xyz, orc.dgcnn_knn(xyz, k), p, ["transform_net1/tconv1", "transform_net1/tconv2"])
    t = mo.mlp_chain(t, p, ["transform_net1/tconv3"]).max(axis=1)
    t = mo.mlp_chain(t, p, ["transform_net1/tfc1", "transform_net1/tfc2"])
    tr = (t @ G.npy(p["transform_net1/transform_XYZ/weights"]).astype(np.float64) + np.eye(3).flatten()).reshape(-1, 3, 3)
    feats, cat = (xyz.astype(np.float64) @ tr).astype(np.float32), []
    for scope in ["dgcnn1", "dgcnn2", "dgcnn3", "dgcnn4"]:
        feats = mo.dgcnn_stage(feats, k, p, [scope])[1].astype(np.float32)
        cat.append(feats)
    glob = mo.mlp_chain(np.concatenate(cat, -1), p, ["agg"]).max(axis=1)
    return mo.mlp_chain(glob, p, ["fc1", "fc2", "fc3"], [True, True, False])


def test_dgcnn_stagewise_calibrated(model_case, monkeypatch):
    """stage by stage, each stage's oracle fed the GPU's input features of that stage (as test_models_gpu does), so that a last-bit
    difference cannot change a kNN graph"""
    mode, s = model_case
    b, n = 2, 1024
    p = dgcnn.init_params(seed=5, randomize_bn=True)
    p["transform_net1/transform_XYZ/weights"] = 0.01 * torch.randn((256, 9), device="cuda",
                                                                   generator=torch.Generator(device="cuda").manual_seed(5))
    _scale_weights(p, s)
    cal = make_clouds("ball", b, n, seed=905)
    done = calibrate(p, monkeypatch, lambda: _dgcnn_oracle_logits(cal, p))
    check_regime(p, done, s)
    xyz = make_clouds("ball", b, n, seed=906)
    cls, ep = dgcnn.get_model(G.cu(xyz), False, params=p)
    tag = f"s={s:g} mode {mode}"
    assert np.array_equal(G.npy(ep["nn_idx0"]), orc.dgcnn_knn(xyz, 20))
    t = mo.edgeconv(xyz, G.npy(ep["nn_idx0"]), p, ["transform_net1/tconv1", "transform_net1/tconv2"])
    t = mo.mlp_chain(t, p, ["transform_net1/tconv3"]).max(axis=1)
    t = mo.mlp_chain(t, p, ["transform_net1/tfc1", "transform_net1/tfc2"])
    tr = t @ G.npy(p["transform_net1/transform_XYZ/weights"]).astype(np.float64) + np.eye(3).flatten()
    _close(G.npy(ep["transform"]).reshape(b, 9), tr, f"dgcnn transform {tag}")
    feats = G.npy(ep["point_cloud_transformed"])
    for i, scope in enumerate(["dgcnn1", "dgcnn2", "dgcnn3", "dgcnn4"]):
        idx, y = mo.dgcnn_stage(feats, 20, p, [scope])
        assert np.array_equal(G.npy(ep[f"nn_idx{i + 1}"]), idx), scope
        _close(G.npy(ep[f"net{i + 1}"]), y, f"dgcnn {scope} {tag}")
        feats = G.npy(ep[f"net{i + 1}"])
    cat = np.concatenate([G.npy(ep[f"net{i}"]) for i in (1, 2, 3, 4)], -1)
    glob = mo.mlp_chain(cat, p, ["agg"]).max(axis=1)
    _close(G.npy(ep["global"]), glob, f"dgcnn global {tag}")
    _close(G.npy(cls), mo.mlp_chain(glob, p, ["fc1", "fc2", "fc3"], [True, True, False]), f"dgcnn logits {tag}")


# ------------------------------------------------------------------------------------------------------------------------------
# non-finite weights: the column keeps factor 1 and raises the flag of the weight image
# ------------------------------------------------------------------------------------------------------------------------------
def _nonfinite_case(mode, where):
    ops.set_mlp_mode(mode)
    try:
        rng = np.random.default_rng(3)
        if where == "dense":
            w = (rng.standard_normal((256, 128)) / 16).astype(np.float32)
            w[5, 7], w[9, 70] = np.inf, np.nan
            x = rng.standard_normal((512, 256)).astype(np.float32)
            s, t = rng.uniform(0.5, 1.5, 128).astype(np.float32), rng.uniform(-0.1, 0.1, 128).astype(np.float32)
            got = G.npy(ops.shared_mlp(G.cu(x), ops.MlpParams([(G.cu(w), G.cu(s), G.cu(t), False)])))
            want = (x.astype(np.float64) @ w.astype(np.float64)) * s + t
            return got, want
        p = _store(47)
        add_sa_module_params(p, "sa", 3, [64, 64, 128], randomize_bn=True)
        p["sa/conv1/weights"][0, 0, 4, 9] = np.inf
        p.invalidate()
        xyz = make_clouds("ball", 2, 2048, seed=48)
        _, got, _ = pointnet_sa_module(G.cu(xyz), None, 512, 0.2, 32, [64, 64, 128], None, False, False, None, "sa", params=p)
        return G.npy(got), mo.sa_module(xyz, None, 512, 0.2, 32, [64, 64, 128], False, "sa", p)[1]
    finally:
        ops.set_mlp_mode(0)


@pytest.mark.parametrize("where", ["dense", "sa"])
def test_nonfinite_weight_reruns_on_bf16x3(where):
    """mode 0 with a non-finite weight: the weight image raises its flag and the op is rerun with bf16x3 operands, bit for bit what
    mode 2 computes.  A single dense layer (no ReLU to turn an inf or NaN back into a number): the outputs fp32 (mode 1) leaves
    non-finite are the non-finite ones, and the finite ones meet the contract."""
    got0, want = _nonfinite_case(0, where)
    got2, _ = _nonfinite_case(2, where)
    assert np.array_equal(got0, got2, equal_nan=True)
    if where == "dense":
        fin = np.isfinite(_nonfinite_case(1, where)[0])
        assert not fin.all() and np.array_equal(np.isfinite(got0), fin)
        G.contract_close(got0[fin], want[fin], "non-finite weight (dense), finite outputs")
