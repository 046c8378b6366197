"""SpiderCNN (spidercnn_cls_xyz) on the GPU against the float64 restatement oracle/spidercnn_oracle.py, on the run's own kNN
indices: the kNN order itself, each fused spiderConv shape in the three arithmetic modes up to the benchmarked B=32 (128-wide
column tiles on a persistent grid), spiderConv at other k, T, C and C_out with its dispatch pinned, the misaligned-pointer
fallback, the group-norm affine and top-2 pooling at their edges, the whole model, the fp16 range guard, determinism, CUDA-graph
replay and the allocation peak."""
import contextlib
import ctypes as C
import io

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import spidercnn_oracle as so
from scanobjectnn_b200 import _lib, ops
from scanobjectnn_b200 import spidercnn_cls_xyz as M
from scanobjectnn_b200.engine import InferenceEngine
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import VariableStore

from . import gpu_util as G

pytestmark = pytest.mark.gpu
LAYERS = [(1, 3, 32), (2, 32, 64), (3, 64, 128), (4, 128, 256)]
# (b, n) of the layer checks: the small shapes, then (9, 1000) with 71 row tiles, the benchmarked B=32 and (33, 1000), whose 258th
# row tile holds 104 rows
LAYER_SHAPES = [(2, 1024), (2, 2048), (3, 1000), (1, 1024), (9, 1000), (32, 1024), (32, 2048), (33, 1000)]
PLAN_SMS = 132                                                                # kNumSMs (csrc/common.cuh), what tc_dense_nt plans with


@pytest.fixture(params=[0, 1, 2], ids=["tensor", "fma", "tensor_bf16x3"])
def mode(request):
    ops.set_mlp_mode(request.param)
    yield request.param
    ops.set_mlp_mode(0)


@pytest.fixture(scope="module")
def params():
    return M.init_params(seed=11, randomize_bn=True)


@pytest.fixture(scope="module")
def signed_params():
    """group-norm gammas drawn from [-1.2, 1.2], as a trained net has them: a negative gamma reverses the order topk_pool sees and
    changes what the ReLU in the next layer's operand split keeps"""
    p = M.init_params(seed=11, randomize_bn=True)
    gen = torch.Generator().manual_seed(12)
    for l, cout in enumerate(M.CHANNELS, start=1):
        p[f"fanConv{l}/taylor/conv/gn/gamma"] = (torch.rand(cout, generator=gen) * 2.4 - 1.2).cuda()
        assert float(p[f"fanConv{l}/taylor/conv/gn/gamma"].min()) < 0
    return p


def _cloud(b, n, seed=0, kind="ball", scale=1.0):
    return torch.from_numpy(make_clouds(kind, b, n, seed) * np.float32(scale)).cuda()


def _plan(rows, c_out):
    """(column-tile width, tiles) of tc_dense_nt (csrc/tc_mlp.cu), which psa_spider_conv_infer plans with: 128-wide when c_out
    allows it and the 128-wide tiles alone fill more than half of the 132 SMs.  The grid is min(tiles, the device's SM count)."""
    row_tiles = -(-rows // 128)
    width = 128 if c_out % 128 == 0 and 2 * row_tiles * (c_out // 128) > PLAN_SMS else 64
    return width, row_tiles * (c_out // width)


def _tensor_shape(rows, c, k, t, c_out):
    """spider_tc_eligible (csrc/spider.cu) for aligned pointers"""
    return rows >= 128 and c % 32 == 0 and k * t * c % 64 == 0 and c_out % 64 == 0 and (c_out == 64 or c_out % 128 == 0)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _path(rows, c, k, t, c_out, mode):
    if mode == 1 or not _tensor_shape(rows, c, k, t, c_out):
        return "fma"
    width, tiles = _plan(rows, c_out)
    return f"{width}-wide, {tiles} tiles" + (f", persistent on {_sms()} SMs" if tiles > _sms() else "")


@pytest.mark.parametrize("kind", ["ball", "shell", "dup"])
def test_knn_point_is_selection_sort_order(kind):
    xyz = _cloud(2, 1024, seed=4, kind=kind)
    _, idx = ops.knn_point(20, xyz, xyz)
    d = xyz[:, None, :, :] - xyz[:, :, None, :]                               # (b, query, dataset, 3)
    dist = ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).contiguous()
    oi, _ = ops.select_top_k(20, dist)
    assert torch.equal(idx, oi[..., :20])
    if orc.refgpu_available():
        ri, _ = G.ref_selection_sort(20, dist)
        assert torch.equal(idx, ri[..., :20])


def _layer_inputs(b, n, cin, seed, scale=1.0):
    xyz = _cloud(b, n, seed, scale=scale)
    _, idx = ops.knn_point(20, xyz, xyz)
    delta = (ops.group_point(xyz, idx) - xyz.unsqueeze(2)).contiguous()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    if cin == 3:
        return xyz, idx, delta, xyz, None, None
    feat = torch.randn((b, n, cin), generator=gen, device="cuda")
    s = torch.rand((b, cin), generator=gen, device="cuda") + 0.5
    u = torch.rand((b, cin), generator=gen, device="cuda") - 0.5
    return xyz, idx, delta, feat, s, u


def _layer64(p, scope, idx, delta, feat, s, u):
    """float64 pre-norm y, one cloud at a time: a cloud's (n, k, C*T) product is at most 210 MB (fanConv4 at n = 2048)"""
    out = []
    for i in range(feat.shape[0]):
        h = feat[i:i + 1].double()
        if s is not None:
            h = torch.relu(h * s[i:i + 1].double()[:, None, :] + u[i:i + 1].double()[:, None, :])
        out.append(so.spider_conv_prenorm(h, idx[i:i + 1], delta[i:i + 1].double(), p, scope))
    return torch.cat(out)


def _forward64(xyz, idx, p):
    """so.forward one cloud at a time (group norm and top-2 pooling are per cloud, the FC head per row) -> (logits, pooled)"""
    outs = [so.forward(xyz[i:i + 1], idx[i:i + 1], p)[:2] for i in range(xyz.shape[0])]
    return torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])


def _per_cloud_close(got, want, what):
    """G.contract_close on each cloud on its own, so that the bound follows that cloud's largest value; prints the worst error"""
    worst = 0.0
    with contextlib.redirect_stdout(io.StringIO()):
        for i in range(got.shape[0]):
            worst = max(worst, G.contract_close(G.npy(got[i]), G.npy(want[i]), f"{what} cloud {i}"))
    print(f"[spider] {what}: worst max|err| over {got.shape[0]} clouds = {worst:.2e}")


def test_layer_shapes_reach_wide_and_persistent_tiles():
    """what LAYER_SHAPES run on, by the launcher's plan"""
    sms = _sms()
    plan = {(b, n, l): _plan(b * n, cout) for b, n in LAYER_SHAPES for l, _, cout in LAYERS}
    # (9, 1000): 71 row tiles; fanConv3 128-wide on 71 tiles (one per CTA), fanConv4 128-wide on 142 (some CTAs take a second)
    assert plan[9, 1000, 3] == (128, 71) and plan[9, 1000, 4] == (128, 142)
    assert 71 <= sms < 142, sms
    # B=32: every tensor-core layer on a persistent grid
    assert all(plan[32, n, l][1] > sms for n in (1024, 2048) for l in (2, 3, 4))
    # (33, 1000): 258 row tiles, the last one 104 rows, and tiles that straddle clouds (per-cloud scale / shift change inside one)
    assert plan[33, 1000, 2] == (64, 258) and 33 * 1000 - 257 * 128 == 104 and 1000 % 128
    # (2, 2048), the control: fanConv4 64-wide on 128 tiles
    assert plan[2, 2048, 4] == (64, 128)
    for l in (3, 4):
        assert any(plan[b, n, l][0] == 128 and plan[b, n, l][1] > sms for b, n in LAYER_SHAPES), f"fanConv{l}: no wide persistent case"


@pytest.mark.parametrize("b,n", LAYER_SHAPES)
@pytest.mark.parametrize("l,cin,cout", LAYERS)
def test_spider_conv_matches_float64(mode, params, b, n, l, cin, cout):
    _, idx, delta, feat, s, u = _layer_inputs(b, n, cin, seed=l + n)
    taylor, w, bias, _, _ = params.spider(f"fanConv{l}/taylor")
    y = ops.spider_conv(delta, idx, feat, taylor, w, bias, s, u)
    want = _layer64(params, f"fanConv{l}/taylor", idx, delta, feat, s, u)
    what = f"fanConv{l} b={b} n={n} mode={mode}"
    err = G.contract_close(G.npy(y), G.npy(want), what)
    print(f"[spider] {what} ({_path(b * n, cin, 20, 5, cout, mode)}): max|err| = {err:.2e}, max|y| = {float(want.abs().max()):.3f}")


@pytest.mark.parametrize("c_out", [64, 128, 192, 256])
@pytest.mark.parametrize("c", [64, 96])
@pytest.mark.parametrize("t", [3, 5])
@pytest.mark.parametrize("k", [1, 7, 16, 32])
def test_spider_conv_other_shapes_match_float64(k, t, c, c_out):
    """spider_conv beyond the model's k = 20, T = 5, on random in-range neighbour indices at b = 9, n = 1000 (128-wide tiles for
    c_out = 128 and 256): k = 32 fills the staged neighbour slots, c = 96 has K blocks that cross (j, t) slices, c_out = 192 and
    k*T*c % 64 != 0 are not tensor-core shapes.  All three modes against float64; where the launcher takes the FMA kernel, mode 0
    and mode 2 are bit for bit mode 1."""
    b, n = 9, 1000
    seed = k * 1000 + t * 100 + c + c_out
    xyz = _cloud(b, n, seed)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    idx = torch.randint(0, n, (b, n, k), generator=gen, device="cuda", dtype=torch.int32)
    delta = (ops.group_point(xyz, idx) - xyz.unsqueeze(2)).contiguous()
    feat = torch.randn((b, n, c), generator=gen, device="cuda")
    s = torch.rand((b, c), generator=gen, device="cuda") * 2 - 0.5              # a quarter of the scales negative
    u = torch.rand((b, c), generator=gen, device="cuda") - 0.5
    p = VariableStore(device="cuda", seed=seed)
    p.add_spider_conv("spider", c, c_out, k, t)
    p["spider/biases"] = torch.rand((1, 1, 1, t), generator=gen, device="cuda") - 0.5          # the filters' constant term
    p["spider/conv/biases"] = torch.rand(c_out, generator=gen, device="cuda") - 0.5
    taylor, w, bias, _, _ = p.spider("spider")
    want = G.npy(_layer64(p, "spider", idx, delta, feat, s, u))
    got = {}
    for m in (0, 1, 2):
        ops.set_mlp_mode(m)
        try:
            got[m] = ops.spider_conv(delta, idx, feat, taylor, w, bias, s, u)
        finally:
            ops.set_mlp_mode(0)
        err = G.contract_close(G.npy(got[m]), want, f"k={k} T={t} {c}->{c_out} mode={m}")
        print(f"[spider] k={k} T={t} {c}->{c_out} mode={m} ({_path(b * n, c, k, t, c_out, m)}): max|err| = {err:.2e}")
    if _path(b * n, c, k, t, c_out, 0) == "fma":
        assert torch.equal(got[0], got[1]) and torch.equal(got[2], got[1]), "an FMA-kernel shape did not take the FMA kernel"


def test_misaligned_pointers_take_the_fma_kernel(params):
    """bias, feat_scale / feat_shift or y 4 bytes off an 8-byte boundary, or feat off a 16-byte one, are contiguous but cannot
    feed the tensor path's float2 and 16-byte accesses: at a tensor-core shape (b = 2, n = 1024, 64 -> 128) the call is served by
    the FMA kernel, bit for bit what mode 1 returns on aligned copies, and within the contract of float64"""
    b, n, c, c_out = 2, 1024, 64, 128
    assert _path(b * n, c, 20, 5, c_out, 0) != "fma"
    _, idx, delta, feat, s, u = _layer_inputs(b, n, c, seed=13)
    taylor, w, bias, _, _ = params.spider("fanConv3/taylor")
    ops.set_mlp_mode(1)
    try:
        fma = ops.spider_conv(delta, idx, feat, taylor, w, bias, s, u)
    finally:
        ops.set_mlp_mode(0)
    want = G.npy(_layer64(params, "fanConv3/taylor", idx, delta, feat, s, u))

    def shifted(x):
        """a copy of x one float into a fresh buffer: 4 mod 8 and 4 mod 16 bytes"""
        buf = torch.zeros(x.numel() + 1, device="cuda")
        buf[1:] = x.reshape(-1)
        return buf[1:].view(x.shape)

    mb, ms, mu, mf = shifted(bias), shifted(s), shifted(u), shifted(feat)
    assert mb.data_ptr() % 8 == 4 and ms.data_ptr() % 8 == 4 and mu.data_ptr() % 8 == 4 and mf.data_ptr() % 16 != 0
    cases = {"bias": (feat, mb, s, u), "feat_scale / feat_shift": (feat, bias, ms, mu), "feat": (mf, bias, s, u)}
    for what, (f, bi, sc, sh) in cases.items():
        y = ops.spider_conv(delta, idx, f, taylor, w, bi, sc, sh)
        assert torch.equal(y, fma), f"misaligned {what}: not the FMA kernel's result"
        G.contract_close(G.npy(y), want, f"misaligned {what}")
    # y itself through the C ABI (ops.spider_conv always allocates it aligned); the float before it must stay untouched
    lib = _lib.load()
    out = torch.full((b * n * c_out + 1,), 7.25, device="cuda")
    y = out[1:].view(b, n, c_out)
    need = lib.psa_spider_conv_workspace_bytes(b, n, c, 20, 5, c_out)
    ws = torch.empty((need + 3) // 4, device="cuda")
    assert y.data_ptr() % 8 == 4 and ws.data_ptr() % 256 == 0
    P = _lib.ptr
    assert lib.psa_spider_conv_infer(b, n, c, 20, 5, c_out, P(delta), P(idx), P(feat), P(s), P(u), P(taylor), P(w), P(bias), P(y),
                                     P(ws), C.c_size_t(need), _lib.stream()) == 0
    assert torch.equal(y, fma) and float(out[0]) == 7.25, "misaligned y: not the FMA kernel's result"


def _check_group_norm(y, gamma, beta, groups, s, u):
    """scale and shift against the float64 moments of contiguous channel groups -> the float64 variance (b, groups)"""
    b, n, c = y.shape
    yg = y.double().reshape(b, n, groups, c // groups)
    mean = yg.mean(dim=(1, 3))
    var = ((yg - mean[:, None, :, None]) ** 2).mean(dim=(1, 3))
    s64 = gamma.double() / torch.sqrt(var.repeat_interleave(c // groups, dim=1) + 1e-6)
    ms = mean.repeat_interleave(c // groups, dim=1) * s64
    u64 = beta.double() - ms
    assert float(((s.double() - s64).abs() / s64.abs()).max()) < 1e-6
    assert float(((u.double() - u64).abs() / (beta.double().abs() + ms.abs())).max()) < 1e-6
    return var


def test_group_norm_affine_matches_float64():
    gen = torch.Generator(device="cuda").manual_seed(1)
    b, n, c, groups = 3, 1000, 64, 16
    y = torch.randn((b, n, c), generator=gen, device="cuda") * 3 + 5
    y[1, :, 4:8] = 0.37                                                       # cloud 1, group 1: constant
    gamma = torch.rand(c, generator=gen, device="cuda") + 0.5
    beta = torch.rand(c, generator=gen, device="cuda") - 0.5
    out, s, u = ops.group_norm_affine(y, gamma, beta, groups, 1e-6, apply=True, relu=True)
    var = _check_group_norm(y, gamma, beta, groups, s, u)
    assert float(var[1, 1]) == 0.0
    G.contract_close(G.npy(out), G.npy(torch.relu(so.group_norm(y.double(), gamma, beta, groups))), "group norm + relu")


@pytest.mark.parametrize("n,c,groups,offset", [(1000, 64, 16, 1e4), (1000, 64, 1, 0.0), (1000, 64, 64, 0.0), (4096, 128, 16, 0.0)])
def test_group_norm_affine_edges_match_float64(n, c, groups, offset):
    """a common offset of 1e4 on std-1 data (the variance must not cancel), one group over all channels, one group per channel,
    and n = 4096; gammas of both signs.  At the offset only the affine is checked: its fp32 shift is beta - 1e4 * scale, and
    applying it in fp32 loses about ulp(1e4) to cancellation whatever the kernel does."""
    gen = torch.Generator(device="cuda").manual_seed(n + c + groups)
    b = 3
    y = torch.randn((b, n, c), generator=gen, device="cuda") + offset
    gamma = torch.rand(c, generator=gen, device="cuda") * 2.4 - 1.2
    beta = torch.rand(c, generator=gen, device="cuda") - 0.5
    out, s, u = ops.group_norm_affine(y, gamma, beta, groups, 1e-6, apply=True, relu=True)
    var = _check_group_norm(y, gamma, beta, groups, s, u)
    assert float(var.min()) > 0.5
    if offset == 0.0:
        G.contract_close(G.npy(out), G.npy(torch.relu(so.group_norm(y.double(), gamma, beta, groups))), f"group norm groups={groups} n={n}")


def test_topk_pool_matches_torch_topk():
    gen = torch.Generator(device="cuda").manual_seed(2)
    y = torch.randn((2, 1000, 96), generator=gen, device="cuda")
    y[0, 10:20, 3] = 7.0                                                      # a repeated maximum
    out = ops.topk_pool(y, 2)
    want = torch.topk(y.permute(0, 2, 1), 2, dim=-1).values
    assert torch.equal(out, want)
    assert float(out[0, 3, 0]) == float(out[0, 3, 1]) == 7.0


@pytest.mark.parametrize("c", [33, 480])
@pytest.mark.parametrize("n", [2, 3, 7, 8, 9, 4096])
def test_topk_pool_affine_edges(n, c):
    """top-2 of h = y [* scale + shift] [then ReLU] with scales of both signs, for n around the kernel's 8 point slices, a partial
    32-channel block (c = 33) and the model's 480, with -inf entries and a channel the ReLU cuts to 0 everywhere, written at an
    offset of a wider out whose other channels must not change.  Against torch.topk of h computed in float64 and rounded to fp32:
    within one fp32 ulp, as the kernel's fmaf rounds once."""
    b, off, extra, fill = 3, 5, 7, 7.25
    gen = torch.Generator(device="cuda").manual_seed(n * 1000 + c)
    y = torch.randn((b, n, c), generator=gen, device="cuda") * 3
    y[0, n // 2, 1] = float("-inf")
    y[1, :, 2] = float("-inf")                                                # -inf at every point
    y[:, :, 0] = y[:, :, 0].abs() + 1
    scale = torch.rand((b, c), generator=gen, device="cuda") * 4 - 2
    scale[scale.abs() < 0.01] = 0.5                                           # -inf * 0 would be NaN
    shift = torch.rand((b, c), generator=gen, device="cuda") - 0.5
    scale[:, 0], shift[:, 0] = 1.0, -1e3                                      # channel 0: negative everywhere before the ReLU
    assert (scale < 0).any()
    for affine in (False, True):
        for relu in (False, True):
            s, u = (scale, shift) if affine else (None, None)
            out = torch.full((b, off + c + extra, 2), fill, device="cuda")
            ops.topk_pool(y, 2, s, u, relu=relu, out=out, offset=off)
            what = f"n={n} c={c} affine={affine} relu={relu}"
            assert bool((out[:, :off] == fill).all() and (out[:, off + c:] == fill).all()), f"{what}: wrote outside its channels"
            h = y.double() if s is None else y.double() * s.double()[:, None, :] + u.double()[:, None, :]
            h = h.float()
            if relu:
                h = torch.relu(h)
            want = G.npy(torch.topk(h.permute(0, 2, 1), 2, dim=-1).values).astype(np.float64)
            got = G.npy(out[:, off:off + c]).astype(np.float64)
            fin = np.isfinite(want)
            assert np.array_equal(got[~fin], want[~fin]), f"{what}: infinite maxima differ"
            tol = np.spacing(np.maximum(np.abs(got[fin]), np.abs(want[fin])).astype(np.float32))
            assert (np.abs(got[fin] - want[fin]) <= tol).all(), f"{what}: max|err| = {np.abs(got[fin] - want[fin]).max():.3e}"
            if affine and relu:
                assert not got[:, 0].any(), f"{what}: channel 0 is not cut to 0"
            if not affine and not relu:
                assert (got[1, 2] == -np.inf).all(), f"{what}: an all -inf channel"


MODEL_CASES = [pytest.param(4, 1024, "ball", False, id="4-1024"), pytest.param(2, 1000, "ball", False, id="2-1000"),
               *(pytest.param(32, n, kind, False, id=f"32-{n}-{kind}") for n in (1024, 2048) for kind in ("ball", "shell", "dup")),
               pytest.param(33, 1000, "ball", False, id="33-1000"),
               pytest.param(32, 1024, "ball", True, id="32-1024-signed-gamma")]


@pytest.mark.parametrize("b,n,kind,signed", MODEL_CASES)
def test_model_matches_float64(mode, request, b, n, kind, signed):
    """pooled features and logits of every cloud against float64 on the run's own kNN indices, up to the timed B=32 shapes; `dup`
    clouds have zero deltas and identical neighbour rows"""
    p = request.getfixturevalue("signed_params" if signed else "params")
    xyz = _cloud(b, n, seed=21, kind=kind)
    logits, ep = M.get_model(xyz, False, params=p, return_end_points=True)
    want_logits, want_pooled = _forward64(xyz, ep["idx"], p)
    what = f"b={b} n={n} {kind}{' signed gamma' if signed else ''} mode={mode}"
    _per_cloud_close(ep["pooled"], want_pooled, f"pooled {what}")
    _per_cloud_close(logits, want_logits, f"logits {what}")


def test_range_guard_reruns_on_bf16x3(params):
    """A cloud scaled x100 puts the cubic Taylor terms far past 65504: the fp16x2 pass must raise its flag, and what mode 0
    returns is then bit for bit what mode 2 computes -- at B=2 and at B=32, where fanConv3 / fanConv4 run 128-wide tiles on a
    persistent grid.  The flag is global: a B=32 batch with one cloud scaled is rerun whole, and every cloud stays right."""
    for b in (2, 32):
        for l, cin, cout in LAYERS[1:]:
            _, idx, delta, feat, s, u = _layer_inputs(b, 1024, cin, seed=5, scale=100.0)
            taylor, w, bias, _, _ = params.spider(f"fanConv{l}/taylor")
            got = {}
            for m in (0, 2):
                ops.set_mlp_mode(m)
                try:
                    got[m] = ops.spider_conv(delta, idx, feat, taylor, w, bias, s, u)
                finally:
                    ops.set_mlp_mode(0)
            assert torch.equal(got[0], got[2]), f"fanConv{l} b={b}: mode 0 is not the bf16x3 rerun"
            want = _layer64(params, f"fanConv{l}/taylor", idx, delta, feat, s, u)
            G.contract_close(G.npy(got[0]), G.npy(want), f"fanConv{l} b={b} x100 ({_path(b * 1024, cin, 20, 5, cout, 0)})")
    one = _cloud(32, 1024, seed=6)
    one[7] *= 100.0
    for xyz in (_cloud(2, 1024, seed=6, scale=100.0), one):
        out = {}
        for m in (0, 2):
            ops.set_mlp_mode(m)
            try:
                out[m] = M.get_model(xyz, False, params=params, return_end_points=True)
            finally:
                ops.set_mlp_mode(0)
        assert torch.equal(out[0][0], out[2][0])
        want_logits, _ = _forward64(xyz, out[0][1]["idx"], params)
        _per_cloud_close(out[0][0], want_logits, f"logits x100 b={xyz.shape[0]}")


def test_deterministic_and_graph_replay_is_bit_equal(params):
    """at B=32, where every tensor-core layer runs on a persistent grid"""
    xyz = _cloud(32, 1024, seed=8)
    a = M.get_model(xyz, False, params=params)
    b = M.get_model(xyz, False, params=params)
    assert torch.equal(a, b)
    eng = InferenceEngine(lambda x: M.get_model(x, False, params=params), (32, 1024, 3), (32, M.NUM_CLASSES), slots=1)
    slot = eng.submit(xyz)
    assert torch.equal(eng.result(slot), a)


def test_allocation_peak_rules_out_materialising():
    p = M.init_params(seed=3)
    xyz = _cloud(32, 1024, seed=9)
    M.get_model(xyz, False, params=p)                                         # warm-up: cached weights and taylor matrices
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    M.get_model(xyz, False, params=p)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print(f"[peak] B=32 N=1024 forward: {peak / 2**20:.1f} MiB above the inputs and weights")
    assert peak < 256 * 2**20
