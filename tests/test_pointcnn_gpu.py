"""PointCNN (pointcnn_cls) on the GPU: the dilated kNN bit for bit against oracle/pointcnn_knn.c:orc_knn_dilated, the X-Conv core and
the ELU / batch-norm GEMM stage by stage against float64 on the run's own indices in the three arithmetic modes, the fp16 range guard,
the whole model against oracle/pointcnn_oracle.py with random and with calibrated batch norm, determinism, CUDA-graph replay and the
allocation peak."""
import numpy as np
import pytest
import torch

from oracle import pointcnn_oracle as po
from scanobjectnn_b200 import _lib, ops
from scanobjectnn_b200 import pointcnn_cls as M
from scanobjectnn_b200.engine import pointcnn_cls_engine
from scanobjectnn_b200.synthetic import make_clouds

from . import gpu_util as G

pytestmark = pytest.mark.gpu
MODEL_SHAPES = [(32, 1024), (32, 2048), (3, 1000)]


@pytest.fixture(params=[0, 1, 2], ids=["tensor", "fma", "tensor_bf16x3"])
def mode(request):
    ops.set_mlp_mode(request.param)
    yield request.param
    ops.set_mlp_mode(0)


@pytest.fixture(scope="module")
def params():
    return M.init_params(seed=5, randomize_bn=True)


def _cloud(b, n, kind="ball", seed=0, scale=1.0):
    return torch.from_numpy(make_clouds(kind, b, n, seed) * np.float32(scale)).cuda()


def _knn_cases(n):
    """(points per cloud, queries, k, d) of the four layers on n points: prefix queries, as random sampling takes them"""
    return [(n, n, 8, 1), (n, 384, 12, 2), (384, 128, 16, 2), (128, 128, 16, 3)]


@pytest.mark.parametrize("kind", ["ball", "shell", "dup"])
@pytest.mark.parametrize("b,n", [(32, 1024), (32, 2048), (3, 1000), (3, 384)])
def test_knn_dilated_bit_exact(kind, b, n):
    x = _cloud(b, n, kind, seed=n)
    for npts, m, k, d in _knn_cases(n):
        pts, qrs = x[:, :npts].contiguous(), x[:, :m].contiguous()
        got = G.npy(ops.knn_dilated(pts, qrs, k, d))
        want = po.knn_dilated(G.npy(pts), G.npy(qrs), k, d)
        assert np.array_equal(got, want), f"{kind} b={b} n={npts} m={m} k={k} d={d}: {(got != want).sum()} indices differ"


@pytest.mark.parametrize("kind", ["ball", "dup"])
def test_knn_dilated_takes_every_point(kind):
    """k * d == n: every point is a candidate, and the list keeps every third of the whole ordering"""
    x = _cloud(4, 48, kind, seed=3)
    got = G.npy(ops.knn_dilated(x, x, 16, 3))
    assert np.array_equal(got, po.knn_dilated(G.npy(x), G.npy(x), 16, 3))


def test_xconv_core_matches_float64(params):
    """the core kernel's (B*P, C_in*dm) depthwise output of each layer at B=32, N=1024 on the model's own indices and inputs (fp32 FMA
    in every mode, so one mode covers it)"""
    x = _cloud(32, 1024, "dup", 1)
    _, ep = M.get_model(x, False, params=params, return_end_points=True)
    pts, fts = x, None
    for l, (tag, k, _, p, _, _, _, dm, glob) in enumerate(M.layer_table(), start=1):
        p = x.shape[1] if p == -1 else p
        qrs = x[:, :p].contiguous()
        idx = ep[f"idx{l}"]
        got = ops.xconv_core(pts, qrs, idx, fts, M.xconv_weights(params, tag), dm)
        want = po.xconv(params, tag, G.npy(pts), G.npy(qrs), G.npy(idx).astype(np.int64), None if fts is None else G.npy(fts), k, dm,
                        glob)["dw"]
        G.contract_close(G.npy(got), want, f"core layer {l}")
        pts, fts = qrs, ep[f"fts{l}"]


# (rows, K, N) of every dense layer of the model at B=32 (pointwise convs, global branch, fc0, fc1), then edges: K and N padded
# inside a block, rows below one tile, a 4-wide K, N = 1
DENSE_SHAPES = [(32768, 96, 48), (12288, 120, 96), (4096, 240, 192), (4096, 480, 384), (4096, 3, 96), (4096, 96, 96),
                (4096, 384, 192), (1000, 100, 70), (300, 64, 64), (130, 4, 200), (127, 96, 48), (1500, 68, 1)]


def _dense_case(rows, k, n, seed, big=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((rows, k), generator=g)
    if big is not None:
        x[rows // 2, k // 2] = big
    w = torch.randn((k, n), generator=g) / np.sqrt(k)
    s = torch.rand(n, generator=g) * 2 + 0.5
    t = torch.randn(n, generator=g) * 0.1
    bias = torch.randn(n, generator=g) * 0.1
    return [a.cuda() for a in (x, w, s, t, bias)]


def _dense64(x, w, s, t, bias=None):
    y = G.npy(x).astype(np.float64) @ G.npy(w).astype(np.float64)
    if bias is not None:
        y = y + G.npy(bias)
    return po.elu(y) * G.npy(s) + G.npy(t)


def _tensor_path(rows, k, n, x):
    """the dispatch of psa_dense_elu_affine: the tensor kernel exactly when the workspace query asks for an image and x is aligned"""
    need = _lib.load().psa_dense_elu_affine_workspace_bytes(rows, k, n)
    return need > 0 and x.data_ptr() % 16 == 0 and x.stride(0) % 4 == 0


@pytest.mark.parametrize("rows,k,n", DENSE_SHAPES)
def test_dense_elu_affine_matches_float64(mode, rows, k, n):
    x, w, s, t, bias = _dense_case(rows, k, n, rows + k + n)
    tc = _tensor_path(rows, k, n, x)
    assert tc == (mode != 1 and rows >= 128 and k % 4 == 0), (mode, rows, k, n, tc)
    G.contract_close(G.npy(ops.dense_elu_affine(x, w, s, t)), _dense64(x, w, s, t), f"dense {rows}x{k}x{n} mode {mode} tc={tc}")
    G.contract_close(G.npy(ops.dense_elu_affine(x, w, s, t, bias=bias)), _dense64(x, w, s, t, bias), f"dense+bias {rows}x{k}x{n}")


def test_dense_elu_affine_strided_slices(mode):
    """layer 4's row: the global branch and the pointwise conv each write their slice of a 480-wide buffer; a column slice as input"""
    rows = 4096
    out = torch.full((rows, 480), float("nan"), device="cuda")
    xg, wg, sg, tg, _ = _dense_case(rows, 96, 96, 1)
    xc, wc, sc, tc_, _ = _dense_case(rows, 480, 384, 2)
    ops.dense_elu_affine(xg, wg, sg, tg, out=out, offset=0)
    ops.dense_elu_affine(xc, wc, sc, tc_, out=out, offset=96)
    G.contract_close(G.npy(out[:, :96]), _dense64(xg, wg, sg, tg), "global slice")
    G.contract_close(G.npy(out[:, 96:]), _dense64(xc, wc, sc, tc_), "conv slice")
    wide = torch.randn((rows, 200), device="cuda")
    for off in (4, 1):                                     # 16-byte aligned slice: tensor path; off = 1: the FMA kernel
        xs = wide[:, off:off + 96]
        assert _tensor_path(rows, 96, 96, xs) == (mode != 1 and off % 4 == 0)
        G.contract_close(G.npy(ops.dense_elu_affine(xs, wg, sg, tg)), _dense64(xs, wg, sg, tg), f"slice at {off}")


@pytest.mark.parametrize("rows,k,n", [(4096, 480, 384), (12288, 120, 96), (32768, 96, 48)])
def test_dense_range_guard_reruns_on_bf16x3(rows, k, n):
    """an input beyond the fp16 range raises the flag of the fp16x2 pass; the bf16x3 rerun then writes every output: mode 0 equals
    mode 2 bit for bit and meets the contract"""
    x, w, s, t, _ = _dense_case(rows, k, n, 9, big=1e5)
    try:
        ops.set_mlp_mode(0)
        y0 = ops.dense_elu_affine(x, w, s, t)
        ops.set_mlp_mode(2)
        y2 = ops.dense_elu_affine(x, w, s, t)
    finally:
        ops.set_mlp_mode(0)
    assert torch.equal(y0, y2)
    G.contract_close(G.npy(y0), _dense64(x, w, s, t), "range guard")


def _calibrate(params, x, idx_list):
    """moving statistics of every batch norm := those of its post-ELU input on the batch x, layer after layer in forward order (the
    float64 restatement with its bn() calibrating each layer the first time it runs)"""
    real_bn = po.bn

    def calib_bn(p, layer, z):
        axes = tuple(range(z.ndim - 1))
        p[f"{layer}_bn/moving_mean"] = torch.from_numpy(z.mean(axis=axes).astype(np.float32)).cuda()
        p[f"{layer}_bn/moving_variance"] = torch.from_numpy(z.var(axis=axes).astype(np.float32)).cuda()
        return real_bn(p, layer, z)

    po.bn = calib_bn
    try:
        po.forward(params, G.npy(x), idx_list)
    finally:
        po.bn = real_bn
    folded = max(float((params[k.replace("moving_variance", "gamma")] / torch.sqrt(params[k] + 1e-3)).abs().max())
                 for k in params if k.endswith("moving_variance"))
    assert folded > 10, folded
    return params


@pytest.mark.parametrize("bn", ["random", "calibrated"])
@pytest.mark.parametrize("b,n", MODEL_SHAPES)
def test_model_matches_float64(mode, b, n, bn):
    x = _cloud(b, n, "dup" if b == 32 else "shell", seed=b + n)
    p = M.init_params(seed=7, randomize_bn=True)
    if bn == "calibrated":
        _, ep = M.get_model(x, False, params=p, return_end_points=True)
        _calibrate(p, x, [G.npy(ep[f"idx{l}"]).astype(np.int64) for l in range(1, 5)])
    logits, ep = M.get_model(x, False, params=p, return_end_points=True)
    assert tuple(logits.shape) == (b, 1, 15)
    want = po.forward(p, G.npy(x), [G.npy(ep[f"idx{l}"]).astype(np.int64) for l in range(1, 5)])
    for l in range(1, 5):
        G.contract_close(G.npy(ep[f"fts{l}"]), want[f"out{l}"], f"layer {l} ({b},{n}) mode {mode} {bn}")
    for name in ("fc0", "fc1"):
        G.contract_close(G.npy(ep[name]), want[name].reshape(-1, want[name].shape[-1]), f"{name} mode {mode} {bn}")
    G.contract_close(G.npy(logits), want["logits"], f"logits ({b},{n}) mode {mode} {bn}")


def test_reruns_and_graph_replay_are_bit_identical(params):
    x = _cloud(32, 1024, "ball", 4)
    y1 = M.get_model(x, False, params=params)
    y2 = M.get_model(x, False, params=params)
    assert torch.equal(y1, y2)
    eng = pointcnn_cls_engine(params, batch=32, npoints=1024, slots=2)
    for _ in range(2):
        for j in range(2):
            eng.submit(x)
        for j in range(2):
            assert torch.equal(eng.result(j), y1)


def test_allocation_peak_rules_out_materialising(params):
    """at B=32, N=1024 (mode 0) the forward's peak stays within 1 MiB of what one layer's live buffers need: the previous layer's
    output, the indices, the depthwise output, the layer output and the pointwise GEMM's workspace.  Layer 1's (B,P,K,C_in)
    neighbour tensor alone is larger."""
    b, n = 32, 1024
    x = _cloud(b, n, "ball", 2)
    M.get_model(x, False, params=params)                     # weights' caches built outside the window
    torch.cuda.synchronize()
    ws = _lib.load().psa_dense_elu_affine_workspace_bytes
    bound, prev = 0, 0
    for tag, k, _, p, c, c_pts, c_prev, dm, glob in M.layer_table():
        p = n if p == -1 else p
        rows, cdw = b * p, (c_pts + c_prev) * dm
        bound = max(bound, prev + 4 * rows * (k + cdw + glob + c) + ws(rows, cdw, c))
        prev = 4 * rows * (glob + c)
    bound += 1 << 20
    materialised = 4 * b * n * 8 * 24
    assert bound < materialised
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    M.get_model(x, False, params=params)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print(f"[alloc] peak {peak / 2**20:.2f} MiB, bound {bound / 2**20:.2f} MiB, layer-1 neighbour tensor {materialised / 2**20:.2f} MiB")
    assert peak < bound
