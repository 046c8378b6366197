"""The set-abstraction kernel (tc_sa_kernel) against float64 at every instantiation, unit kind and V-layer path a level can take.

A level runs on tc_sa_kernel<NP, C1, NL, N0>: NP = 2 (fp16x2, mode 0) or 3 (bf16x3, mode 2 and mode 0's guarded rerun) pieces
per operand, times six level shapes.  Its launcher picks one of three kinds of units from what fits in shared memory: a
warpgroup on its own, both warpgroups as one joint unit, or a joint unit that streams the last layer 64 columns at a time.
The fit is decided again at NP = 3, whose weight images are larger, so a level may run on another kind of unit in the rerun
than in its fp16x2 pass.  With input features, the level's first layer reads V = s (points . W1[3:] + xyz . W1[:3]) + t,
which the dense layer in front of it computes on the tensor cores or, for narrow features, on the fp32 FMA kernel.

`_route` restates those choices from the C++ (each line names what it restates); `test_case_table_reaches_every_route` checks
without a GPU that the levels below reach all of them.  Each level is then compared with float64 at 1e-5 of
max(1, max |want|) in modes 0 and 2, run twice (units claim chunks in whatever order they reach the counter, and a max does not
depend on it, so the two runs agree bit for bit), on explicit ball-query indices whose neighbourhood sizes cycle through the
16-row slot edges, and with a group count that leaves a partial last chunk for every chunk size."""
from collections import namedtuple

import numpy as np
import pytest
import torch

from scanobjectnn_b200 import ops

from . import restate

# ---------------------------------------------------------------------------------------------------------------------
# the route of a level (csrc/tc_mlp.cu)
# ---------------------------------------------------------------------------------------------------------------------
SMEM_BUDGET = 220 * 1024          # kSmemBudget
POOL_LIMIT = 223 * 1024           # launch_tc_sa_np: `limit`, the layout and the units' pooling buffers
SHAPES = [(64, 1, 0), (128, 1, 0), (64, 2, 64), (64, 2, 128), (128, 2, 64), (128, 2, 128)]   # (C1, NL, N0) of launch_tc_sa_np


def _layout_total(layers, c1, np_, stream_last):
    """tc_sa_layout(a).total"""
    last = len(layers) - 1
    # resident layers: tc_image_bytes(Kd, Ntot, np)
    total = sum(K * N * 2 * np_ for l, (K, N) in enumerate(layers) if not (stream_last and l == last))
    if stream_last:                                       # ring[0], ring[1]: (Kd / 64) * tc_block_bytes(kSaNt, np) each
        total += 2 * (layers[last][0] // 64) * 64 * 128 * np_
    total += 7 * c1 * 4                                   # w1x (3 C1), w1c (3 C1), t1
    return total + sum(2 * N * 4 for _, N in layers)      # scale and shift of every tensor layer


def _pool_bytes(layers, k, joint, stream_last):
    """sa_pool_bytes: per unit, sa_chunk(K, joint) rows of sa_pool_cols words"""
    chunk = (128 if joint else 512) // k                  # sa_chunk
    cols = 64 if stream_last else layers[-1][1]           # sa_pool_cols
    return (1 if joint else 2) * chunk * cols * 4


def _route(widths, c, k, np_):
    """(instantiation (NP, C1, NL, N0), unit kind, stream_last) of a level on tc_sa_kernel, or None when it runs on the FMA
    fused kernel"""
    # tc_sa_eligible(mlp, c, nsample, out): the shape, and a layout that fits at np = 3 (which the guarded default needs too)
    layers = restate.sa_tc_layers(widths, c, k, 0 if np_ == 2 else 2)
    if layers is None:
        return None
    c1 = widths[1]
    # tc_sa_eligible(..., np): `if (tc_sa_layout(a).total + 1024 > kSmemBudget) a.stream_last = 1;`
    stream = _layout_total(layers, c1, np_, False) + 1024 > SMEM_BUDGET
    assert _layout_total(layers, c1, np_, stream) + 1024 <= SMEM_BUDGET
    # launch_tc_sa_np: `a.joint = a.K == 128 || a.stream_last;`, then a joint unit when the warpgroups' buffers do not fit,
    # then a streamed last layer when the joint buffer does not fit next to the resident one
    joint = k == 128 or stream

    def fits():
        return _layout_total(layers, c1, np_, stream) + 1024 + _pool_bytes(layers, k, joint, stream) <= POOL_LIMIT

    if not joint and not fits():
        joint = True
    if not fits():
        stream = True
    assert fits(), "sa_module: internal error (pooling buffer does not fit)"
    # launch_tc_sa_shape<NP, C1, NL, N0>: N0 = Ntot[0] when NL = 2
    inst = (np_, c1, len(layers), layers[0][1] if len(layers) == 2 else 0)
    return inst, "streamed" if stream else "joint" if joint else "warpgroup", stream


# ---------------------------------------------------------------------------------------------------------------------
# the levels
# ---------------------------------------------------------------------------------------------------------------------
# widths: the MLP's channels, C_in = 3 + c (EdgeConv: 2 * 3); k: the neighbourhood size; neg: the last layer without ReLU and
# its shift pushed negative, so that most pooled values are negative; rerun: also checked with inputs scaled by 3e5 in mode 0;
# b, n, m: clouds, points per cloud, centres per cloud (b * m = 111 leaves a partial last chunk for chunks of 16, 8, 4 and 2)
Level = namedtuple("Level", "widths c k neg rerun b n m edge", defaults=(False, False, 3, 256, 37, False))
LEVELS = {
    "64-128": Level([3, 64, 128, 256], 0, 32, neg=True),
    "64-128-feat": Level([3 + 64, 64, 128, 128], 64, 64, rerun=True),
    "fold64-fma-v": Level([3 + 5, 64, 64, 128], 5, 32),
    "fold64-tc-v": Level([3 + 32, 64, 64, 128], 32, 32),
    "last64-nl2": Level([3, 64, 64, 64], 0, 32, neg=True),
    "last64-nl1": Level([3 + 16, 128, 64], 16, 64, neg=True),
    "128-64-joint": Level([3 + 16, 128, 64, 128], 16, 128, neg=True),
    "joint-2layer": Level([3 + 64, 128, 128, 256], 64, 128, neg=True, rerun=True),
    "streamed-nl1": Level([3, 128, 1024], 0, 32),
    "640": Level([3, 64, 640], 0, 32, neg=True, rerun=True),
    "edgeconv": Level([6, 64, 128, 256], 3, 20, n=111, edge=True),     # 333 points
    # 32769 neighbourhoods: 2049 chunks of 16, the last of one, several for each unit of the persistent grid
    "many-chunks": Level([3, 64, 64, 128], 0, 32, m=10923, n=12288),
}
EC_K = 32                          # EdgeConv's neighbours are padded to a 32-row neighbourhood (edge_pad_idx_kernel)


def _level_shape(lv):
    """(widths, c, k) of the level tc_sa_kernel runs: EdgeConv over 3-D points is a level with no features whose centre
    weights are W1[0:3] (edgeconv_dual_ok)"""
    return ([3] + lv.widths[1:], 0, EC_K) if lv.edge else (lv.widths, lv.c, lv.k)


def _v_path(lv):
    """where V runs: dense_on_tc(b * n, c, C1, 1) in tc_sa_run, or nowhere for a level without features"""
    _, c, _ = _level_shape(lv)
    if c == 0:
        return None
    return "tc" if restate.dense_on_tc(lv.b * lv.n, c, lv.widths[1], 1, 0) else "fma"


def test_case_table_reaches_every_route():
    """all 12 instantiations, the three unit kinds at both NP, V on both dense kernels, levels whose NP = 2 and NP = 3 routes
    differ (with a rerun among them), a last layer without ReLU on every shape, a rerun on warpgroup and joint units"""
    routes = {name: {np_: _route(*_level_shape(lv), np_) for np_ in (2, 3)} for name, lv in LEVELS.items()}
    for name, r in routes.items():
        assert r[2] is not None and r[3] is not None, f"{name} does not run on tc_sa_kernel"
    insts = {r[np_][0] for r in routes.values() for np_ in (2, 3)}
    assert insts == {(np_,) + s for np_ in (2, 3) for s in SHAPES}, sorted(insts)
    kinds = {(np_, r[np_][1]) for r in routes.values() for np_ in (2, 3)}
    assert kinds == {(np_, kind) for np_ in (2, 3) for kind in ("warpgroup", "joint", "streamed")}, sorted(kinds)
    assert {_v_path(lv) for lv in LEVELS.values()} == {None, "tc", "fma"}
    differ = {name for name, r in routes.items() if r[2][1:] != r[3][1:]}
    assert differ and any(LEVELS[name].rerun for name in differ), routes
    assert {routes[name][2][0][1:] for name, lv in LEVELS.items() if lv.neg} == set(SHAPES)
    assert {routes[name][2][1] for name, lv in LEVELS.items() if lv.rerun} >= {"warpgroup", "joint"}
    # a partial last chunk for every chunk size in use (16, 8, 4 or 2 neighbourhoods; a joint unit at K = 128 takes one)
    for name, lv in LEVELS.items():
        for np_ in (2, 3):
            _, kind, _ = routes[name][np_]
            chunk = (128 if kind != "warpgroup" else 512) // _level_shape(lv)[2]
            assert chunk == 1 or (lv.b * (lv.n if lv.edge else lv.m)) % chunk, (name, np_, chunk)


# ---------------------------------------------------------------------------------------------------------------------
# inputs and the float64 restatement
# ---------------------------------------------------------------------------------------------------------------------
def _layers(lv, rng):
    """(W, scale, shift, relu) per layer: W ~ N(0, 1 / C_in), BN scale in [0.5, 2], shift N(0, 0.1) (- 4 on a `neg` last layer)"""
    out, L = [], len(lv.widths) - 1
    for l in range(L):
        w = rng.standard_normal((lv.widths[l], lv.widths[l + 1])) / np.sqrt(lv.widths[l])
        s, t = rng.uniform(0.5, 2.0, lv.widths[l + 1]), rng.standard_normal(lv.widths[l + 1]) * 0.1
        relu = not (lv.neg and l == L - 1)
        if not relu:
            t = t - 4.0
        out.append((w.astype(np.float32), s.astype(np.float32), t.astype(np.float32), relu))
    return out


def _sa_inputs(lv, rng, scale):
    """xyz, new_xyz (the first m points), features, and ball-query indices whose counts cycle through 1 (cnt = 0), the 16-row
    slot edges and k - 1, k, padded by repeating the first index as the ball query does (no other entry repeats it).  `scale`
    multiplies the features, or the coordinates of a level without any"""
    xyz = (rng.uniform(-1.0, 1.0, (lv.b, lv.n, 3)) * (1.0 if lv.c else scale)).astype(np.float32)
    pts = (rng.standard_normal((lv.b, lv.n, lv.c)) * scale).astype(np.float32) if lv.c else None
    groups = lv.b * lv.m
    sizes = np.resize([1, 15, 16, 17, lv.k - 1, lv.k], groups)
    idx = rng.integers(0, lv.n, (groups, lv.k))
    idx[:, 1:] = np.where(idx[:, 1:] == idx[:, :1], (idx[:, 1:] + 1) % lv.n, idx[:, 1:])
    idx = np.where(np.arange(lv.k) < sizes[:, None], idx, idx[:, :1]).astype(np.int32)
    return xyz, xyz[:, :lv.m].copy(), pts, idx.reshape(lv.b, lv.m, lv.k)


def _edge_inputs(lv, rng):
    """points and a k-neighbour graph whose first neighbour is the point itself, as a kNN gives it"""
    x = rng.uniform(-1.0, 1.0, (lv.b, lv.n, 3)).astype(np.float32)
    idx = np.empty((lv.b, lv.n, lv.k), np.int32)
    for b in range(lv.b):
        for i in range(lv.n):
            others = rng.choice(lv.n - 1, size=lv.k - 1, replace=False)
            idx[b, i] = np.concatenate([[i], others + (others >= i)])
    return x, idx


def _mlp64(h, layers):
    """h @ W * s + t per layer, ReLU where configured (the last layer's too), in h's dtype and on its device"""
    for w, s, t, relu in layers:
        w, s, t = (torch.from_numpy(a).to(h) for a in (w, s, t))
        h = h @ w * s + t
        if relu:
            h = torch.clamp_min(h, 0.0)
    return h


def _reference(lv, inputs, layers, device="cpu"):
    """the level in float64 -> (its output, max |layer 1|): rows (relative coordinates, then features; EdgeConv:
    [x_i, x_j - x_i]), the MLP, max over k"""
    t64 = lambda a: None if a is None else torch.from_numpy(a).to(device, torch.float64)  # noqa: E731
    if lv.edge:
        x, idx = inputs
        h = restate.edges(t64(x), torch.from_numpy(idx).to(device))
    else:
        xyz, _, pts, idx = inputs                       # the centres are the first m points: sa_level's FPS indices 0..m-1
        fps = torch.arange(lv.m, device=device).expand(lv.b, lv.m)
        h = restate.sa_level(t64(xyz), t64(pts), fps, torch.from_numpy(idx).to(device).long())[1]
    first = _mlp64(h, layers[:1])
    return _mlp64(first, layers[1:]).amax(dim=2).cpu().numpy(), float(first.abs().max())


def _run(lv, inputs, layers, mode):
    """the level on the GPU in `mode`, twice -> the first result; the second must equal it bit for bit"""
    dev = lambda a: None if a is None else torch.from_numpy(a).cuda()  # noqa: E731
    mlp = ops.MlpParams([(dev(w), dev(s), dev(t), relu) for w, s, t, relu in layers])
    ops.set_mlp_mode(mode)
    try:
        if lv.edge:
            x, idx = (dev(a) for a in inputs)
            call = lambda: ops.edgeconv_infer(x, idx, mlp)  # noqa: E731
        else:
            xyz, new_xyz, pts, idx = (dev(a) for a in inputs)
            call = lambda: ops.sa_module_infer(xyz, new_xyz, pts, 0.4, lv.k, mlp, idx=idx)  # noqa: E731
        first, second = call(), call()
        torch.cuda.synchronize()
    finally:
        ops.set_mlp_mode(0)
    assert torch.equal(first, second), "two runs of the level differ"
    return first.cpu().numpy()


def _check(got, want):
    """max |got - want| <= 1e-5 max(1, max |want|), every value finite"""
    assert got.shape == want.shape
    err = float(np.abs(got - want).max())
    assert np.isfinite(got).all() and err <= 1e-5 * max(1.0, float(np.abs(want).max())), \
        f"max |err| {err:.3e}, max |want| {np.abs(want).max():.3e}"


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("name", list(LEVELS))
def test_level_matches_float64(name, mode):
    lv = LEVELS[name]
    rng = np.random.default_rng(sum(lv.widths) + lv.k)
    layers = _layers(lv, rng)
    inputs = _edge_inputs(lv, rng) if lv.edge else _sa_inputs(lv, rng, 1.0)
    want, _ = _reference(lv, inputs, layers, "cuda")
    if lv.neg:
        assert 0.5 < (want < 0).mean() < 1.0, "the last layer's outputs must be mostly, not all, negative"
    _check(_run(lv, inputs, layers, mode), want)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [name for name, lv in LEVELS.items() if lv.rerun])
def test_fp16_overflow_reruns_on_bf16x3(name):
    """inputs scaled by 3e5: layer 1's activations leave the fp16 range, the fp16x2 pass raises its flag and the bf16x3 rerun,
    which may run on another kind of unit, replaces the result; it meets the bound relative to its own magnitude"""
    lv = LEVELS[name]
    rng = np.random.default_rng(sum(lv.widths) + lv.k + 1)
    layers = _layers(lv, rng)
    inputs = _sa_inputs(lv, rng, 3.0e5)
    want, first = _reference(lv, inputs, layers, "cuda")
    assert first > 65504.0, "layer 1 must leave the fp16 range"
    _check(_run(lv, inputs, layers, 0), want)
