"""The float64 torch restatements of the models that the GPU tests compare against, and the pieces they share.

A restatement evaluates a model with torch ops in the dtype of its input (float64; float32 as the yardstick of what fp32 itself
resolves), on the GPU run's own discrete choices: neighbour graphs, FPS and ball-query indices.

Where fp32 and float64 can legitimately disagree, the comparisons leave the element out on both sides instead of widening a bound.
A max (over k neighbours, or over the N points) whose runner-up lies within 1e-5 of it may be won by another element in fp32 than
in float64, and then routes its gradient elsewhere; likewise a head activation, or a maximum, whose pre-relu value lies within 1e-5
of zero on either side may fall on the other side of the relu (under batch statistics that changes the gradient of its whole
column).  These are properties of the max and the relu, not errors.  `Masks` finds such elements on the float64 side and zeroes the
gradient arriving at them on both sides (a hook on the same tensor of each).  Layers that run inside one autograd node on the GPU,
where no hook reaches, take the run's own relu decisions (and max-pool winners) from `RunDecisions` instead.

Nothing here touches a GPU at import time."""
import numpy as np
import torch

from scanobjectnn_b200 import training
from scanobjectnn_b200.pointnet_seg import HEAD as SEG_HEAD
from scanobjectnn_b200.tf_util import BN_EPS, VariableStore

MOVING = ("/moving_mean", "/moving_variance")
SSG_HEAD = [("fc1", True), ("fc2", True), ("fc3", False)]
EC2 = ("t/tconv1", "t/tconv2")                   # the two scopes of the two-layer EdgeConv stores


# ---------------------------------------------------------------------------------------------------------------------
# variables
# ---------------------------------------------------------------------------------------------------------------------
def params_as(p, dtype, grad=False):
    """a detached copy of every variable in `dtype`; leaves of autograd when `grad`"""
    return {k: v.detach().to(dtype, copy=True).requires_grad_(grad) for k, v in p.items()}


def flat_grad(p, name, g=None):
    """variable `name`'s slice of a gradient of the flat parameter vector: by default the one autograd left on it"""
    fp = p._flat
    v = fp.views[name]
    off = (v.data_ptr() - fp.flat.data_ptr()) // 4
    return (fp.flat.grad if g is None else g)[off:off + v.numel()].view(v.shape)


def moving(p):
    """a copy of every batch norm's moving averages"""
    return {k: v.clone() for k, v in p.items() if k.endswith(MOVING)}


def perturb_tnets(p, seed):
    """the reference initialises the T-nets' transform layers to zero, which leaves the T-nets without a gradient: draw them from
    N(0, 0.01) instead"""
    with torch.no_grad():
        for name in ("transform_net1/transform_XYZ/weights", "transform_net2/transform_feat/weights"):
            if name in p:
                p[name].normal_(0, 0.01, generator=torch.Generator(device="cuda").manual_seed(seed))


def grid_x(b, n, c, seed):
    """coordinates on the 1/16 grid: with edgeconv_store's weights every edge value is exact in fp32"""
    return np.random.default_rng(seed).integers(-32, 33, (b, n, c)).astype(np.float32) / 16.0


def edgeconv_store(c, cout, seed, scope="e"):
    """one conv2d(2c -> cout) + batch norm with weights, bias, gamma and beta on dyadic grids"""
    rng = np.random.default_rng(seed)
    p = VariableStore(device="cuda", seed=seed)
    p.add_conv2d(scope, 2 * c, cout)
    p[f"{scope}/weights"] = torch.tensor(rng.integers(-16, 17, (1, 1, 2 * c, cout)) / 64.0, dtype=torch.float32, device="cuda")
    p[f"{scope}/biases"] = torch.tensor(rng.integers(-8, 9, cout) / 64.0, dtype=torch.float32, device="cuda")
    p[f"{scope}/bn/gamma"] = torch.tensor(1.0 + rng.integers(-32, 33, cout) / 64.0, dtype=torch.float32, device="cuda")
    p[f"{scope}/bn/beta"] = torch.tensor(rng.integers(-8, 9, cout) / 64.0, dtype=torch.float32, device="cuda")
    return p


def edgeconv2_store(c, seed):
    """the two layers EC2 of DGCNN's T-net EdgeConv (2c -> 64 -> 128), batch norm randomised, biases N(0, 0.1)"""
    p = VariableStore(device="cuda", seed=seed)
    p.add_conv2d(EC2[0], 2 * c, 64, randomize_bn=True)
    p.add_conv2d(EC2[1], 64, 128, randomize_bn=True)
    rng = np.random.default_rng(seed)
    for s, n in zip(EC2, (64, 128)):
        p[f"{s}/biases"] = torch.tensor(rng.standard_normal(n) * 0.1, dtype=torch.float32, device="cuda")
    return p


# ---------------------------------------------------------------------------------------------------------------------
# one layer, and the run's decisions it can take
# ---------------------------------------------------------------------------------------------------------------------
class RunDecisions:
    """A GPU run's discrete decisions, by scope: every batch-normed layer's relu gate fmaf(y, scale, shift) > 0 (exact in float64)
    in `gates`, in training mode the batch statistics (mean, 1 / sqrt(var + eps)) its batch norm used in `stats`, and every level's
    max-pool winners in `argk`.  Read from a PointNet2ClsTrainer, or from a VariableStore: the last run of each MLP and level
    trainer it caches for that mode.  stats=False leaves the batch statistics out, so a restatement keeps float64's own."""

    def __init__(self, src, frozen, stats=True):
        if isinstance(src, VariableStore):
            trainers = src.__dict__.get("_trainers", {}).items()
            layers = [ly for key, tr in trainers if key[0] == ("mlp_frozen" if frozen else "mlp") for ly in tr.layers]
            levels = [tr.levels[0] for key, tr in trainers if key[0] == ("level_frozen" if frozen else "level")]
        else:
            layers, levels = src.head, src.levels
        self.gates, self.stats = {}, {}
        for ly in layers + [ly for lv in levels for ly in lv.layers]:
            if ly.bn:
                self.gates[ly.scope] = (ly.y.double() * ly.scale.double() + ly.shift.double()) > 0
                if stats and not frozen:
                    self.stats[ly.scope] = ly.mean_inv
        self.argk = {lv.spec.scope: lv.argk for lv in levels}


def layer(h, P, scope, frozen, *, bn=True, relu=True, stats=None, run=None, info=None):
    """conv2d / fully_connected (+ batch norm + relu) in h's dtype.  Batch norm on the moving averages (frozen) or on the batch
    statistics over every row (biased variance), eps BN_EPS; the batch statistics are recorded in `stats[scope]` when a dict is given.

    With a `run` (RunDecisions) the relu is z * the run's gate, and `info` counts the gates that differ from float64's own ("flips"
    of "units").  In training mode the batch statistics then take the run's values, float64's derivative: fp32 sums of y and y^2
    give the variance with an error relative to E[y^2], not to the variance, and that error is bounded on its own
    (info["stat_err"], relative to E[y^2]) instead of through every later layer; info["own"] keeps h's dtype's own batch statistics,
    by scope, for the moving averages."""
    dt = h.dtype
    w = P[f"{scope}/weights"].to(dt)
    y = h @ w.reshape(-1, w.shape[-1]) + P[f"{scope}/biases"].to(dt)
    if not bn:
        return y
    if frozen:
        mean, var = P[f"{scope}/bn/moving_mean"].to(dt), P[f"{scope}/bn/moving_variance"].to(dt)
    else:
        dims = tuple(range(y.dim() - 1))
        mean, var = y.mean(dims), y.var(dims, unbiased=False)
        if run is not None and scope in run.stats:
            info.setdefault("own", {})[scope] = (mean.detach(), var.detach())          # dtype's own batch statistics
            rmean, rinv = run.stats[scope][0].to(dt), run.stats[scope][1].to(dt)
            rvar = 1.0 / (rinv * rinv) - BN_EPS
            ms = float((y.detach() ** 2).mean(dims).max())
            info["stat_err"] = max(info["stat_err"], float((rmean - mean.detach()).abs().max()) / ms ** 0.5,
                                   float((rvar - var.detach()).abs().max()) / ms)
            mean, var = mean + (rmean - mean).detach(), var + (rvar - var).detach()
        if stats is not None:
            stats[scope] = (mean.detach(), var.detach())
    z = (y - mean) / torch.sqrt(var + BN_EPS) * P[f"{scope}/bn/gamma"].to(dt) + P[f"{scope}/bn/beta"].to(dt)
    if not relu:
        return z
    if run is not None and scope in run.gates:
        gate = run.gates[scope].view(z.shape)
        info["flips"] += int((gate != (z > 0)).sum())
        info["units"] += gate.numel()
        return z * gate
    return torch.relu(z)


# ---------------------------------------------------------------------------------------------------------------------
# the exclusion rule
# ---------------------------------------------------------------------------------------------------------------------
def ambiguous(z, dim):
    """True where the max over `dim` has a runner-up of a different value within 1e-5 (of the largest activation) of it, or is a
    positive maximum within that distance of the relu's zero"""
    with torch.no_grad():
        mx = z.amax(dim=dim, keepdim=True)
        below = torch.where(z < mx, z, torch.full_like(z, -1.0)).amax(dim=dim)
        tol = 1e-5 * float(z.abs().max())
        mx = mx.squeeze(dim)
        return ((mx - below) < tol) | ((mx > 0) & (mx < tol))


def near_zero(z):
    """True where a pre-relu value lies within 1e-5 (of the largest magnitude) of zero"""
    with torch.no_grad():
        return z.abs() < 1e-5 * float(z.abs().max())


def near_zero_max(pre, dim, scale):
    """True where the max over `dim` of the pre-relu values lies within 1e-5 of `scale` of the relu's zero, on either side: a maximum
    slightly below zero in float64 may lie slightly above it in fp32, and then carries the whole gradient"""
    with torch.no_grad():
        return pre.amax(dim=dim).abs() < 1e-5 * scale


def inner_flip(pre, inner):
    """True where the edge that wins the max over k (dim 2) of `pre` (b, n, k, c) has a unit of `inner` (b, n, k, c1), the pre-relu
    values of the layer below, within 1e-5 (of the largest magnitude) of zero"""
    with torch.no_grad():
        return near_zero(inner).any(dim=-1).gather(2, pre.argmax(dim=2))


def zero_at(t, mask):
    t.register_hook(lambda g: g.masked_fill(mask, 0.0))


def dropper(drops):
    """dropout that applies the given (mask, p) pairs in call order: t * mask / (1 - p); without `drops` the identity.  The returned
    function's `left()` counts the pairs not yet applied."""
    it = iter(drops or ())

    def drop(t):
        if drops is None:
            return t
        mask, p = next(it)
        assert mask.shape == t.shape, (mask.shape, t.shape)
        return t * mask.to(t.dtype) / (1 - p)

    drop.left = lambda: sum(1 for _ in it)
    return drop


class Masks:
    """The elements a comparison leaves out, in the order the model reaches them: `edge` for the maxima over k neighbours (EdgeConv
    outputs, set-abstraction levels), `pool` for the maxima over the N points, keyed by scope, `act` for the head's near-zero relu
    inputs, keyed by scope.

    Masks(replay=first), or first.replay(), looks for none: it applies the masks `first` recorded, whatever the values and the
    `pre` / `inner` arguments, so that a second pass (in float32, or on the run's batch statistics, which move values by far less
    than 1e-5 but may move a few across it) leaves out the same elements."""

    def __init__(self, replay=None):
        self.edge, self.pool, self.act = [], {}, {}
        self._first = replay

    def replay(self):
        return Masks(replay=self)

    def edge_max(self, z, pre=None, inner=None):
        """max over k of the activated edge values z; given their pre-relu values `pre`, a maximum within 1e-5 of the relu's zero on
        either side is ambiguous too, and given a fused first layer's pre-relu values `inner` (b, n, k, c1), so is a maximum whose
        edge has a unit of that layer within 1e-5 of zero (the kernel's relu may fall the other way there)"""
        if self._first is not None:
            amb = self._first.edge[len(self.edge)]
        else:
            amb = ambiguous(z, 2)
            if pre is not None:
                amb |= near_zero_max(pre, 2, float(z.detach().abs().max()))
            if inner is not None:
                amb |= inner_flip(pre, inner)
        out = z.amax(dim=2)
        zero_at(out, amb)
        self.edge.append(amb)
        return out

    def point_max(self, y, scope, pre=None):
        if self._first is not None:
            amb = self._first.pool[scope]
        else:
            amb = ambiguous(y, 1)
            if pre is not None:
                amb |= near_zero_max(pre, 1, float(y.detach().abs().max()))
        zero_at(y, amb.unsqueeze(1))
        self.pool[scope] = amb
        return y.amax(dim=1)

    def head_layer(self, h, P, scope, frozen, **kw):
        """layer(), its relu's near-zero inputs left out"""
        z = layer(h, P, scope, frozen, relu=False, **kw)
        near = self._first.act[scope] if self._first is not None else near_zero(z)
        out = torch.relu(z)
        zero_at(out, near)
        self.act[scope] = near
        return out

    def count(self):
        ms = self.edge + list(self.pool.values()) + list(self.act.values())
        return sum(int(m.sum()) for m in ms), sum(m.numel() for m in ms)

    def patch(self, monkeypatch):
        """zero the gradient at the same elements on the GPU path: hooks on the outputs of its EdgeConv and set-abstraction nodes
        (`edge`, in the order the model calls them) and of its MLP nodes (`pool` and `act`, by the node's last scope)"""
        edge, pool, act = iter(self.edge), self.pool, self.act
        ec, sa, mlp = training.edgeconv_training, training.sa_module_training, training.mlp_training

        def edgeconv_training(*a, **kw):
            out = ec(*a, **kw)
            zero_at(out, next(edge))
            return out

        def sa_module_training(*a, **kw):
            new_xyz, out, idx = sa(*a, **kw)
            zero_at(out, next(edge))
            return new_xyz, out, idx

        def mlp_training(x, layers, *a, **kw):
            out = mlp(x, layers, *a, **kw)
            scope = layers[-1][0]
            if scope in pool:
                zero_at(out, pool[scope].unsqueeze(1))
            if scope in act:
                zero_at(out, act[scope])
            return out

        monkeypatch.setattr(training, "edgeconv_training", edgeconv_training)
        monkeypatch.setattr(training, "sa_module_training", sa_module_training)
        monkeypatch.setattr(training, "mlp_training", mlp_training)


# ---------------------------------------------------------------------------------------------------------------------
# model pieces
# ---------------------------------------------------------------------------------------------------------------------
def edges(x, idx):
    """the EdgeConv input [x_i, x_j - x_i] (b, n, k, 2c) over the neighbour graph idx (b, n, k)"""
    b, n, c = x.shape
    k = idx.shape[-1]
    neigh = x[torch.arange(b, device=x.device).view(b, 1, 1), idx.long()]
    centre = x.unsqueeze(2).expand(b, n, k, c)
    return torch.cat([centre, neigh - centre], dim=-1)


def tnet(h, P, scope, K, L, masks):
    """PointNet's transform net (pointnet/models/transform_nets.py) on h (b, n, c) -> (b, K, K); L: the caller's layer()"""
    g = masks.point_max(L(L(L(h, f"{scope}/tconv1"), f"{scope}/tconv2"), f"{scope}/tconv3"), f"{scope}/tconv3")
    g = L(L(g, f"{scope}/tfc1"), f"{scope}/tfc2")
    name = "transform_XYZ" if K == 3 else "transform_feat"
    eye = torch.eye(K, dtype=h.dtype, device=h.device).flatten()
    return (g @ P[f"{scope}/{name}/weights"] + P[f"{scope}/{name}/biases"] + eye).reshape(h.shape[0], K, K)


def sa_level(xyz, pts, fps=None, ball=None):
    """a set-abstraction level's grouping on given int64 FPS and ball-query indices -> (new_xyz, rows (b, m, k, 3 + c): the
    coordinates relative to their centre, then the features); without indices group all: one group of every point, centre 0"""
    if fps is None:
        return torch.zeros_like(xyz[:, :1]), (xyz if pts is None else torch.cat([xyz, pts], -1))[:, None]
    ar = torch.arange(xyz.shape[0], device=xyz.device)
    new_xyz = xyz[ar[:, None], fps]
    h = xyz[ar[:, None, None], ball] - new_xyz[:, :, None, :]
    if pts is not None:
        h = torch.cat([h, pts[ar[:, None, None], ball]], -1)
    return new_xyz, h


def interpolate(xyz1, xyz2, points2):
    """three_nn (tf_interpolate.cpp:60-103: squared distances, neighbours not found stay at 1e40 = inf in float, index 0), weights
    (1/max(d,1e-10)) / sum (pointnet_util.py:211-216), no gradient through them, and three_interpolate"""
    b = xyz1.shape[0]
    with torch.no_grad():
        d = ((xyz1.detach()[:, :, None, :] - xyz2.detach()[:, None, :, :]) ** 2).sum(-1)
        if d.shape[-1] < 3:
            d = torch.cat([d, torch.full((*d.shape[:2], 3 - d.shape[-1]), float("inf"), dtype=d.dtype, device=d.device)], dim=-1)
        dist, idx = d.topk(3, dim=-1, largest=False, sorted=True)
        idx[torch.isinf(dist)] = 0
        inv = 1.0 / dist.clamp_min(1e-10)
        w = inv / inv.sum(-1, keepdim=True)
    ar = torch.arange(b, device=xyz1.device)[:, None, None]
    return (points2[ar, idx] * w[..., None]).sum(dim=2)


def pn2_levels(x, L, masks, idx):
    """the three set-abstraction levels of pointnet2_cls_bga / _partseg ([64, 64, 128], [128, 128, 256], group all [256, 512, 1024])
    on the given indices [(fps, ball)] * 2, max-pooled through masks.edge_max -> [(new_xyz, pooled)] * 3; L: the caller's layer()"""
    out, xyz, pts = [], x, None
    for scope, ind in (("layer1", idx[0]), ("layer2", idx[1]), ("layer3", (None, None))):
        xyz, h = sa_level(xyz, pts, *ind)
        for i in range(3):
            h = L(h, f"{scope}/conv{i}")
        pts = masks.edge_max(h)
        out.append((xyz, pts))
    return out


def pn2_fp(xyz1, xyz2, pts1, pts2, L, scope, n):
    """pointnet_fp_module (pointnet_util.py:199-229): interpolate pts2 onto xyz1, concatenate pts1, n layers"""
    h = interpolate(xyz1, xyz2, pts2)
    h = torch.cat([h, pts1], dim=2) if pts1 is not None else h          # a tile + concat for fa_layer1
    for i in range(n):
        h = L(h, f"{scope}/conv_{i}")
    return h


def pn2_indices(p, mode):
    """per sampled level (fps_idx, ball-query idx) as int64, from the last run of the level trainers cached on store `p` for `mode`
    ("level" or "level_frozen")"""
    lv = {key[1]: tr.levels[0] for key, tr in p.__dict__["_trainers"].items() if key[0] == mode}
    return [(lv[s].fps_idx.long(), lv[s].idx.long()) for s in ("layer1", "layer2")]


def _argk_pool(h, argk, info):
    """the max over dim 2 taken at the run's winner argk (its first winning row), so the gradient goes where the kernel sends it;
    info["pool_gap"]: how far below h's own maximum that row lies, relative to h's largest entry"""
    B, m, _, c = h.shape
    out = h.gather(2, argk.long().view(B, m, 1, c)).squeeze(2)
    with torch.no_grad():
        gap = float((h.amax(dim=2) - out).max()) / max(float(h.abs().max()), 1e-30)
        info["pool_gap"] = max(info["pool_gap"], gap)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# the models
# ---------------------------------------------------------------------------------------------------------------------
def ssg(xyz, p, levels, frozen, masks, run=None, info=None):
    """pointnet2_cls_ssg (or bga's classification branch) restated in torch ops of xyz's dtype on the levels' FPS / ball-query
    indices; `masks`: the head's dropout masks, by scope.  run: the PointNet2ClsTrainer whose discrete decisions are taken instead of
    the restatement's own -- every batch-normed layer's relu gate and every level's max-pool winner (batch statistics stay
    float64's); `info` then collects the batch statistics ("stats"), the flipped gates ("flips" of "units") and the largest pool gap
    ("pool_gap")."""
    dec = None if run is None else RunDecisions(run, frozen, stats=False)
    stats = None if info is None else info.setdefault("stats", {})
    L = lambda h, s, **kw: layer(h, p, s, frozen, stats=stats, run=dec, info=info, **kw)        # noqa: E731
    cur_xyz, cur_pts = xyz, None
    for lv in levels:
        sp = lv.spec
        new_xyz, h = sa_level(cur_xyz, cur_pts, *((None, None) if sp.group_all else (lv.fps_idx.long(), lv.idx.long())))
        for i in range(len(sp.mlp)):
            h = L(h, f"{sp.scope}/conv{i}")
        cur_xyz, cur_pts = new_xyz, h.amax(dim=2) if dec is None else _argk_pool(h, dec.argk[sp.scope], info)
    h = cur_pts.reshape(xyz.shape[0], -1)
    for scope, bn in SSG_HEAD:
        h = L(h, scope, bn=bn)
        if scope in masks:
            h = h * masks[scope].to(h.dtype)
    return h


def dgcnn(x, P, graphs, frozen, masks, detach_transform=False, stats=None, bga=False, run=None, info=None, drops=None):
    """dgcnn.get_model (dgcnn.py:24-102, transform_nets.py:10-55) on the given neighbour graphs -> logits; stats (a dict): every
    layer's batch statistics, by scope.  bga: dgcnn_bga.get_model (dgcnn_bga.py:27-134) -> (class_pred, seg_pred), the segmentation
    head on concat[class vector (fc2's output, before dp2), the pooled agg, net1..net4] (1600 channels).  run (RunDecisions) and
    info as for layer(); drops: the dropout masks (dp1, dp2 and, with bga, the segmentation head's), see dropper()."""
    b, n = x.shape[:2]
    L = lambda h, s, **kw: layer(h, P, s, frozen, stats=stats, run=run, info=info, **kw)        # noqa: E731
    drop = dropper(drops)
    sc = "transform_net1"
    y1 = L(edges(x, graphs[0]), f"{sc}/tconv1", relu=False)
    y = L(torch.relu(y1), f"{sc}/tconv2", relu=False)
    h = masks.edge_max(torch.relu(y), pre=y, inner=y1)
    y = L(h, f"{sc}/tconv3", relu=False)
    h = masks.point_max(torch.relu(y), f"{sc}/tconv3", pre=y)
    h = L(L(h, f"{sc}/tfc1"), f"{sc}/tfc2")
    t = (h @ P[f"{sc}/transform_XYZ/weights"] + P[f"{sc}/transform_XYZ/biases"] + torch.eye(3, dtype=x.dtype, device=x.device).flatten())
    t = t.reshape(b, 3, 3)
    h = torch.bmm(x, t.detach() if detach_transform else t)
    nets = []
    for i, s in enumerate(["dgcnn1", "dgcnn2", "dgcnn3", "dgcnn4"]):
        y = L(edges(h, graphs[i + 1]), s, relu=False)
        h = masks.edge_max(torch.relu(y), pre=y)
        nets.append(h)
    y = L(torch.cat(nets, dim=-1), "agg", relu=False)
    g = masks.point_max(torch.relu(y), "agg", pre=y)
    kw = dict(stats=stats, run=run, info=info)
    c = drop(masks.head_layer(g, P, "fc1", frozen, **kw))
    c = masks.head_layer(c, P, "fc2", frozen, **kw)
    class_pred = L(drop(c), "fc3", bn=False)
    if not bga:
        return class_pred
    h = torch.cat([c.unsqueeze(1).expand(b, n, c.shape[-1]), g.unsqueeze(1).expand(b, n, g.shape[-1]), *nets], dim=-1)
    h = L(L(h, "seg/conv1"), "seg/conv2")
    return class_pred, L(drop(h), "seg/conv3", bn=False)


def pointnet(x, P, masks):
    """pointnet_cls.get_model (pointnet_cls.py:21-75) with frozen batch norm -> (logits, feature transform)"""
    L = lambda h, s, **kw: layer(h, P, s, True, **kw)        # noqa: E731
    h = torch.bmm(x, tnet(x, P, "transform_net1", 3, L, masks))
    h = L(L(h, "conv1"), "conv2")
    t2 = tnet(h, P, "transform_net2", 64, L, masks)
    h = torch.bmm(h, t2)
    g = masks.point_max(L(L(L(h, "conv3"), "conv4"), "conv5"), "conv5")
    for s in ("fc1", "fc2"):
        g = masks.head_layer(g, P, s, True)
    return L(g, "fc3", bn=False), t2


def pointnet_seg(x, P, frozen, masks, classify, run=None):
    """pointnet_seg (classify) or pointnet_partseg, dropout off, building tile + concat as the reference does
    (pointnet/models/pointnet_seg.py:24-134, pointnet_partseg.py:23-124) -> ([class_pred,] seg_pred, feature transform,
    {"stats", "flips", "units", "stat_err"}); run: RunDecisions"""
    b, n, _ = x.shape
    info = {"stats": {}, "flips": 0, "units": 0, "stat_err": 0.0}
    kw = dict(stats=info["stats"], run=run, info=info)
    L = lambda h, s, **k: layer(h, P, s, frozen, **kw, **k)        # noqa: E731
    h = L(L(torch.bmm(x, tnet(x, P, "transform_net1", 3, L, masks)), "conv1"), "conv2")
    t2 = tnet(h, P, "transform_net2", 64, L, masks)
    point_feat = torch.bmm(h, t2)
    g = masks.point_max(L(L(L(point_feat, "conv3"), "conv4"), "conv5"), "conv5")
    out = []
    if classify:
        c = g
        for s in ("fc1", "fc2"):
            c = masks.head_layer(c, P, s, frozen, **kw)
        out.append(L(c, "fc3", bn=False))
    h = torch.cat([point_feat, g.unsqueeze(1).expand(b, n, g.shape[-1])], dim=2)          # tile + concat
    for s in SEG_HEAD:
        h = L(h, s)
    out.append(L(h, "conv10", bn=False))
    return out, t2, info


def pointnet2_partseg(x, P, frozen, masks, idx, run=None):
    """pointnet2_cls_partseg, dropout off, on the given level indices [(fps, ball)] * 2, building fa_layer1's input as the reference
    does (pointnet2/models/pointnet2_cls_partseg.py:20-87, pointnet_util.py:199-229) -> (seg_pred, {"stats", "flips", "units",
    "stat_err"}); run: RunDecisions"""
    info = {"stats": {}, "flips": 0, "units": 0, "stat_err": 0.0}
    L = lambda h, s, **kw: layer(h, P, s, frozen, stats=info["stats"], run=run, info=info, **kw)        # noqa: E731
    (l1_xyz, l1), (l2_xyz, l2), (l3_xyz, l3) = pn2_levels(x, L, masks, idx)
    l2 = pn2_fp(l2_xyz, l3_xyz, l2, l3, L, "fa_layer1", 2)
    l1 = pn2_fp(l1_xyz, l2_xyz, l1, l2, L, "fa_layer2", 2)
    l0 = pn2_fp(x, l1_xyz, None, l1, L, "fa_layer3", 3)
    return L(L(l0, "seg_fc1"), "seg_fc2", bn=False), info


def pointnet2_bga(x, P, frozen, masks, idx, run=None, drops=None):
    """pointnet2_cls_bga (pointnet2/models/pointnet2_cls_bga.py:21-75) on the given level indices [(fps, ball)] * 2 -> (class_pred,
    seg_pred, {"stats", "flips", "units", "stat_err"[, "own"]}).  The class vector is fc2's output before dp2; fa_layer1 interpolates
    it from the group-all level's single point (weights (1, 0, 0)) and concatenates l2_points.  run: RunDecisions; drops: the
    dropout masks of dp1, dp2 and seg_dp1, see dropper()."""
    info = {"stats": {}, "flips": 0, "units": 0, "stat_err": 0.0}
    kw = dict(stats=info["stats"], run=run, info=info)
    L = lambda h, s, **k: layer(h, P, s, frozen, **kw, **k)        # noqa: E731
    drop = dropper(drops)
    (l1_xyz, l1), (l2_xyz, l2), (l3_xyz, l3) = pn2_levels(x, L, masks, idx)
    net = drop(masks.head_layer(l3.reshape(x.shape[0], -1), P, "fc1", frozen, **kw))
    net = masks.head_layer(net, P, "fc2", frozen, **kw)
    class_pred = L(drop(net), "fc3", bn=False)
    l2 = pn2_fp(l2_xyz, l3_xyz, l2, net.unsqueeze(1), L, "fa_layer1", 2)
    l1 = pn2_fp(l1_xyz, l2_xyz, l1, l2, L, "fa_layer2", 2)
    l0 = pn2_fp(x, l1_xyz, None, l1, L, "fa_layer3", 3)
    seg_pred = L(drop(L(l0, "seg_fc1")), "seg_fc2", bn=False)
    assert drop.left() == 0, "dropout masks left over"
    return class_pred, seg_pred, info


# ---------------------------------------------------------------------------------------------------------------------
# plans of the shared ring GEMM's three ops (csrc/mfv.cu conv_plan, csrc/pointcnn.cu pd_plan, csrc/spider.cu spider_ws with
# csrc/tc_mlp.cu tc_dense_nt): the tile widths, splits and workspace bytes the launchers pick, so that a test can name the path a
# shape takes.  tests/test_ring_gemm_plan_cpu.py checks the byte counts against the library's workspace queries.
# ---------------------------------------------------------------------------------------------------------------------
PLAN_SMS = 132                    # kNumSMs (csrc/common.cuh): what the plans assume, whatever the device has


def _al256(x):
    return (x + 255) & ~255


def image_bytes(K, N, np_):
    """tc_image_alloc_bytes (csrc/tc_common.cuh): the blocks, np = 2's column factors, the 256-byte trailer"""
    blocks = _al256(K * N * 2 * np_)
    return blocks + (_al256(N * 4) if np_ == 2 else 0) + 256


def wide_tiles(tiles, Np):
    """the 128-wide column tile of tc_dense_nt and conv_plan: when Np allows it and those tiles alone fill more than half the SMs"""
    return Np % 128 == 0 and 2 * tiles * (Np // 128) > PLAN_SMS


def conv_active_taps(b, r, k, tile, rows):
    """conv3d_tapmask_kernel: the taps of a k^3 kernel that reach inside the r^3 grid for some row of 128-row tile `tile`"""
    h, r0, r1 = k // 2, tile * 128, min(rows, tile * 128 + 128) - 1
    vox = [(v // (r * r), v // r % r, v % r) for v in range(r0 // b, r1 // b + 1)]
    offs = [(t // (k * k) - h, t // k % k - h, t % k - h) for t in range(k ** 3)]
    return sum(any(all(0 <= p + o < r for p, o in zip(v, off)) for v in vox) for off in offs)


def conv_plan(b, r, k, c, n, np_):
    """conv_plan (csrc/mfv.cu) -> dict: tiles, Np, Nt, splits, units (all column tiles and splits) and the workspace `total` for
    np_ = 2 (mode 0) or 3 (mode 2)"""
    rows, K, CB = b * r ** 3, k ** 3 * c, c // 64
    tiles, Np = -(-rows // 128), -(-n // 64) * 64
    Nt = 128 if wide_tiles(tiles, Np) else 64
    units = tiles * (Np // Nt)
    reach = min(k, 2 * r - 1)
    maxk = reach ** 3 * CB
    s = min(1 if units >= PLAN_SMS else PLAN_SMS // units, 16)
    s = s if s < maxk // 2 else max(maxk // 2, 1)
    total = 256 + _al256(tiles * 16)
    if Np != n:
        total += _al256(K * Np * 4)
    total += image_bytes(K, Np, 2) if np_ == 2 and image_bytes(K, Np, 2) > image_bytes(K, Np, 3) else image_bytes(K, Np, 3)
    if s > 1:
        total += _al256(s * rows * Np * 4)
    return dict(rows=rows, tiles=tiles, Np=Np, Nt=Nt, splits=s, units=units * s, total=total)


def conv_unit_blocks(b, r, k, c, splits):
    """per 128-row tile, the K blocks of each of its split units (Conv3dOp::unit): the tile's active blocks divided in order"""
    rows = b * r ** 3
    nact = [conv_active_taps(b, r, k, t, rows) * (c // 64) for t in range(-(-rows // 128))]
    return [[a * (sp + 1) // splits - a * sp // splits for sp in range(splits)] for a in nact]


def pd_plan(rows, K, N, np_):
    """pd_plan (csrc/pointcnn.cu): K padded to 64, N to 64-wide blocks taken two at a time when their count is even"""
    Kp, nblk = -(-K // 64) * 64, -(-N // 64)
    Nt, Np = (128 if nblk % 2 == 0 else 64), nblk * 64
    total = 256 + _al256(K * Np * 4) + (image_bytes(Kp, Np, 2) if np_ == 2 else 0) + image_bytes(Kp, Np, 3)
    return dict(Kp=Kp, Np=Np, Nt=Nt, units=-(-rows // 128) * (Np // Nt), total=total)


def spider_tensor_shape(rows, c, k, t, n):
    """spider_tc_eligible (csrc/spider.cu) for aligned pointers"""
    return rows >= 128 and c % 32 == 0 and k * t * c % 64 == 0 and n % 64 == 0 and (n == 64 or n % 128 == 0)


def spider_plan(b, npts, c, k, t, n):
    """spider_ws (csrc/spider.cu) and the tile width of tc_dense_nt; the workspace holds both images in every mode"""
    rows, K = b * npts, k * t * c
    tiles = -(-rows // 128)
    Nt = 128 if wide_tiles(tiles, n) else 64
    total = 256 + _al256(rows * k * t * 4)
    if spider_tensor_shape(rows, c, k, t, n):
        total += _al256(K * n * 4) + image_bytes(K, n, 2) + image_bytes(K, n, 3)
    return dict(rows=rows, Nt=Nt, units=tiles * (n // Nt), total=total)


# ---------------------------------------------------------------------------------------------------------------------
# plans of the inference dense layers (csrc/tc_mlp.cu): the chain of psa_shared_mlp / psa_sa_group_all_infer, the
# set-abstraction level and EdgeConv.  `mode` is psa_set_mlp_mode's.  tests/test_dense_chain_plan_cpu.py checks them against
# the library's workspace queries and psa_mlp_image_plan.
# ---------------------------------------------------------------------------------------------------------------------
FC_KS = 64                        # kFcKs (csrc/mlp.cu): the K slice of one fc_small partial


def dense_image_bytes(K, N):
    """tc_dense_image_bytes: an fp16x2 image and the bf16x3 image of its rerun, K padded to 64"""
    Kp = -(-K // 64) * 64
    return image_bytes(Kp, N, 2) + image_bytes(Kp, N, 3)


def dense_on_tc(rows, K, N, pool_k, mode):
    """dense_on_tc / tc_dense_eligible: the tensor-core path of one dense layer"""
    pool_ok = pool_k in (1, 32, 64) or (pool_k >= 128 and pool_k % 128 == 0)
    return (mode != 1 and rows >= 128 and K >= 32 and N >= 64 and N % 64 == 0 and (N == 64 or N % 128 == 0) and pool_ok
            and (pool_k == 1 or rows % pool_k == 0))


def dense_nt(rows, N, mode):
    """tc_dense_nt: the tile width with the image format flag of the mode"""
    return (128 if wide_tiles(-(-rows // 128), N) else 64) | (0x100 if mode == 2 else 0x200)


def plan_image_bytes(Kp, N, mode):
    """tc_plan_image_bytes: a prebuilt image, fp16x2 blocks followed by their bf16x3 twin in mode 0"""
    return image_bytes(Kp, N, 3) + (image_bytes(Kp, N, 2) if mode == 0 else 0)


def chain_plan(rows, channels, K0):
    """chain_plan: (K, N) per layer and the workspace bytes -- two ping-pong halves of the widest inner activation, an image
    slot per layer, fc_small's partials when rows <= 32, the 256-byte word region"""
    KN = [(K0 if l == 0 else channels[l], channels[l + 1]) for l in range(len(channels) - 1)]
    inner = [K for K, _ in KN[1:]]
    total = 2 * _al256(rows * max(inner) * 4) if inner else 0
    total += sum(dense_image_bytes(K, max(N, 64)) for K, N in KN)
    if rows <= 32:
        total += _al256(max(-(-K // FC_KS) * 32 * N * 4 for K, N in KN))
    return dict(layers=KN, total=total + 256)


def chain_images(rows, pool_k, channels, row0, mode):
    """psa_mlp_image_plan for a chain: (nt, row0, bytes) of each layer on the tensor cores, zeros for the others"""
    out = []
    KN = chain_plan(rows, channels, channels[0] - row0)["layers"]
    for l, (K, N) in enumerate(KN):
        pk = pool_k if l == len(KN) - 1 else 1
        on = dense_on_tc(rows, K, N, pk, mode)
        out.append((dense_nt(rows, N, mode), row0 if l == 0 else 0, plan_image_bytes(-(-K // 64) * 64, N, mode)) if on else (0, 0, 0))
    return out


def sa_tc_layers(channels, c, nsample, mode):
    """tc_sa_eligible for both splits: [(Kd, Ntot)] of the level's tensor layers, or None for the FMA fused kernel"""
    L = len(channels) - 1
    if mode == 1 or not 2 <= L <= 3 or nsample not in (32, 64, 128) or channels[0] != 3 + c or channels[1] not in (64, 128):
        return None
    layers = [(channels[1 + l], channels[2 + l]) for l in range(L - 1)]
    for l, (K, N) in enumerate(layers):
        if K not in (64, 128) or (l < len(layers) - 1 and N not in (64, 128)) or (l == len(layers) - 1 and N != 64 and N % 128):
            return None
    # tc_sa_layout at np = 3, which the fp16x2 layout never exceeds: every layer resident, or the last one streamed through two
    # slots of one 64-channel chunk
    fixed = 7 * channels[1] * 4 + sum(2 * N * 4 for _, N in layers)          # w1x, w1c (3 C1 each), t1; scale, shift per layer
    resident = sum(K * N * 2 * 3 for K, N in layers)
    streamed = resident - layers[-1][0] * layers[-1][1] * 2 * 3 + 2 * (layers[-1][0] // 64) * 64 * 128 * 3
    return layers if min(resident, streamed) + fixed + 1024 <= 220 * 1024 else None


def sa_workspace(b, n, c, channels, layers):
    """tc_sa_workspace_bytes: the word region, both images of every tensor layer, the U rows and the U GEMM's image slot"""
    total = 256 + sum(image_bytes(K, N, 2) + image_bytes(K, N, 3) for K, N in layers)
    return total + (_al256(b * n * channels[1] * 4) + dense_image_bytes(c, channels[1]) if c > 0 else 0)


def sa_images(rows, c, nsample, channels, mode):
    """psa_mlp_image_plan for a set-abstraction level: the U GEMM (row0 = 3) and the level's 64-wide tensor layers"""
    out = [(0, 0, 0)] * 4
    layers = sa_tc_layers(channels, c, nsample, mode)
    if layers is None:
        return out
    if c > 0 and dense_on_tc(rows, c, channels[1], 1, mode):
        out[0] = (dense_nt(rows, channels[1], mode), 3, plan_image_bytes(-(-c // 64) * 64, channels[1], mode))
    for l, (K, N) in enumerate(layers):
        out[1 + l] = (64 | (0x100 if mode == 2 else 0x200), 0, plan_image_bytes(K, N, mode))
    return out


def edgeconv_workspace(b, n, c, k, channels, mode):
    """psa_edgeconv_workspace_bytes: the dual-SA path (c = 3, two layers or more), the algebra path (one layer), else none"""
    rows = b * n
    if mode != 1 and c == 3 and 1 <= k <= 32 and len(channels) >= 3:
        layers = sa_tc_layers([3] + list(channels[1:]), 0, 32, mode)
        if layers is not None:
            return _al256(rows * 32 * 4) + sa_workspace(b, n, 0, channels, layers)
    N = channels[1]
    if mode == 1 or len(channels) != 2 or rows < 128 or k > 32 or N not in (32, 64, 128, 256):
        return 0
    return _al256(c * 2 * N * 4) + _al256(rows * 2 * N * 4) + dense_image_bytes(c, 2 * N) + 256


# ---------------------------------------------------------------------------------------------------------------------
# routing of the training GEMM's launchers (csrc/train.cu): which kernel path, tile and contraction split each product takes,
# and psa_train_dense_workspace_bytes.  tests/test_train_gemm_plan_cpu.py checks the workspace against the library, and that
# the cases of tests/test_train_gemm_gpu.py reach every path.
# ---------------------------------------------------------------------------------------------------------------------
TRAIN_SMALL_M = 1024              # kSmallM: rows up to this split the contraction of the forward / input gradient
TRAIN_BK = 16                     # kGemmBK


def tc_train_fwd_eligible(rows, K, N):
    return rows >= 128 and 128 <= K <= 512 and N >= 128 and N % 128 == 0


def small_m_splits(contraction):
    return max(1, min(16, contraction // 64))


def weight_grad_splits(rows, tiles):
    """(splits, k_per_split) of the weight gradient's contraction over the rows"""
    want = max(1, min((2 * PLAN_SMS + tiles - 1) // tiles, (rows + 255) // 256))
    kps = -(-(-(-rows // want)) // TRAIN_BK) * TRAIN_BK
    return -(-rows // kps), kps


def _split_k(contraction):
    """(nz, k_per_split) of a small-M product: small_m_splits rounded to whole BK blocks"""
    s = small_m_splits(contraction)
    kps = -(-(-(-contraction // s)) // TRAIN_BK) * TRAIN_BK
    return -(-contraction // kps), kps


def train_fwd_plan(rows, K, N, ld=None, mask=False):
    """psa_train_dense_fwd: path "tc" (the tensor-core forward), "split" (small M, contraction split over CTAs, statistics from
    col_stats_kernel) or "fp32" (one pass, statistics from the epilogue); the tile width bn of the fp32 paths"""
    if tc_train_fwd_eligible(rows, K, N) and (ld is None or ld == K) and not mask:
        return dict(path="tc")
    bn = 64 if N <= 64 else 128
    if rows <= TRAIN_SMALL_M and small_m_splits(K) > 1:
        nz, kps = _split_k(K)
        return dict(path="split", bn=bn, splits=nz, kps=kps)
    return dict(path="fp32", bn=bn, splits=1)


def train_bwd_input_plan(rows, K, N, workspace_bytes):
    """psa_train_dense_bwd_input: "split" when small M and the workspace holds the partials, else "fp32" (one split)"""
    bn = 64 if K <= 64 else 128
    if rows <= TRAIN_SMALL_M and small_m_splits(N) > 1 and workspace_bytes >= small_m_splits(N) * rows * K * 4:
        nz, kps = _split_k(N)
        return dict(path="split", bn=bn, splits=nz, kps=kps)
    return dict(path="fp32", bn=bn, splits=1)


def train_bwd_weight_plan(rows, K, N):
    """psa_train_dense_bwd_weight: the (bm, bn) tiling over (K, N) and the split of the rows"""
    bm, bn = (64 if K <= 64 else 128), (64 if N <= 64 else 128)
    splits, kps = weight_grad_splits(rows, -(-K // bm) * -(-N // bn))
    return dict(bm=bm, bn=bn, splits=splits, kps=kps)


def train_dense_workspace(rows, K, N):
    """psa_train_dense_workspace_bytes"""
    fwd = -(-rows // 128) * 2 * N * 4
    w = train_bwd_weight_plan(rows, K, N)
    need = max(fwd, w["splits"] * K * N * 4 if w["splits"] > 1 else 0, 16 * rows * max(K, N) * 4 if rows <= TRAIN_SMALL_M else 0)
    if tc_train_fwd_eligible(rows, K, N):
        need = max(need, _al256(fwd) + dense_image_bytes(K, N))
    return need + 256


# The dense cases of tests/test_train_gemm_gpu.py.  act: "raw" (x as is), "bn" (relu(x * scale + shift)), "bn_mask" (and a dropout
# mask); x layout: "dense" (ld = K), "slice" (a column slice, ld = K + 8), "ld_odd" (ld = K + 3), "offset" (x, mask, scale and
# shift 4 bytes past a 16-byte boundary).  src: the psa_grad_in flags joined by "+": mask, gate (the relu gate from s / t),
# coeffs (ca / cb / cc), pool20 / pool32 (mode 1, the max-pool routing), scalar (dh with an odd ld_dh, y with ld = N + 3).
#            id            rows   K    N    act        x         bias   stats
FWD_CASES = [("fp32_n48", 300, 40, 48, "bn", "dense", True, True),
             ("fp32_n100", 1500, 72, 100, "raw", "dense", False, True),
             ("split_stats", 200, 300, 130, "bn", "dense", True, True),
             ("split_nostats", 33, 256, 40, "raw", "dense", True, False),
             ("tc_gate_in", 128, 128, 128, "bn", "dense", True, True),
             ("rows127", 127, 128, 128, "bn", "dense", True, True),
             ("k127", 128, 127, 128, "bn", "dense", False, True),
             ("tc_k512", 256, 512, 256, "bn", "dense", True, True),
             ("k513", 256, 513, 256, "bn", "dense", True, True),
             ("n192", 256, 200, 192, "bn", "dense", True, True),
             ("tc_kpad", 384, 200, 128, "bn", "dense", True, True),
             ("tc_plain", 1000, 256, 384, "raw", "dense", False, False),
             ("tc_shape_mask", 256, 128, 128, "bn_mask", "dense", True, True),
             ("slice", 1100, 128, 128, "bn", "slice", True, True),
             ("ld_odd", 1100, 64, 72, "bn_mask", "ld_odd", False, True),
             ("offset", 1100, 64, 48, "bn_mask", "offset", True, True)]
#                  id                rows  K    N    src                     col_skip ld_dx
BWD_INPUT_CASES = [("k48", 1100, 48, 72, "plain", 0, None),
                   ("k100", 1100, 100, 40, "mask+gate+coeffs", 0, None),
                   ("mask", 1100, 64, 64, "mask", 0, None),
                   ("gate", 1100, 64, 64, "gate", 0, None),
                   ("coeffs", 1100, 96, 64, "coeffs", 0, None),
                   ("split", 200, 72, 300, "gate", 0, None),
                   ("split_k40", 64, 40, 1024, "mask+coeffs", 0, None),
                   ("skip_odd", 1100, 70, 64, "mask", 3, 69),
                   ("skip_odd_split", 200, 70, 256, "plain", 3, 69),
                   ("pool20", 800, 96, 64, "pool20", 0, None),
                   ("pool32", 1536, 64, 128, "pool32+coeffs", 0, None),
                   ("pool20_split", 600, 48, 256, "pool20+coeffs", 0, None),
                   ("scalar", 1100, 64, 66, "scalar+mask+gate+coeffs", 0, None)]
#                   id                rows   K    N    act        x         src
BWD_WEIGHT_CASES = [("t64x64", 200, 40, 48, "bn", "dense", "plain"),
                    ("t64x128", 3000, 40, 100, "bn_mask", "dense", "mask+gate+coeffs"),
                    ("t128x64_pool", 1000, 100, 60, "bn", "dense", "pool20+coeffs"),
                    ("t128x128", 250, 130, 200, "bn_mask", "dense", "coeffs"),
                    ("t64x128_pool32", 2048, 64, 128, "raw", "dense", "pool32"),
                    ("scalar", 1500, 66, 70, "bn_mask", "ld_odd", "scalar+mask+gate"),
                    ("offset", 700, 64, 64, "bn", "offset", "gate"),
                    ("large", 40009, 72, 136, "bn", "dense", "gate")]


# ---------------------------------------------------------------------------------------------------------------------
# metrics
# ---------------------------------------------------------------------------------------------------------------------
def rel(got, want):
    """max |got - want| relative to the largest entry of want"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    return float(np.abs(got - want).max() / max(1e-30, np.abs(want).max()))


def out_err(got, want):
    """max |got - want| relative to max(1, the largest entry of want)"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    return float(np.abs(got - want).max() / max(1.0, np.abs(want).max()))


def err(got, want, scale=None):
    """max |got - want| of two tensors relative to `scale`, by default the largest entry of want"""
    want = want.detach().double()
    scale = float(want.abs().max()) if scale is None else scale
    return float((got.detach().double() - want).abs().max()) / max(scale, 1e-30)


def within(e, e32, tol, factor):
    """the bound, or where the float32 restatement itself misses it, `factor` times the float32 restatement's error"""
    return e < tol or e <= factor * e32


def grad_errors(p, P, P32):
    """per variable: (max|run - float64|, max|float32 restatement - float64|), and the largest float64 entry"""
    errs, scale = {}, 0.0
    for name in p._flat.names:
        want = P[name].grad if P[name].grad is not None else torch.zeros_like(P[name])
        g32 = P32[name].grad if P32[name].grad is not None else torch.zeros_like(P32[name])
        errs[name] = (float((flat_grad(p, name).double() - want).abs().max()), float((g32.double() - want).abs().max()))
        scale = max(scale, float(want.abs().max()))
    return errs, scale
