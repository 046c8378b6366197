"""3DmFV-Net (mfv_net_cls) on the GPU against the float64 restatement oracle/mfv_oracle.py: the Fisher vector on three kinds of
cloud, every conv3d shape of the model in the three arithmetic modes (plain and with calibrated batch norm), both pools, the whole
model on the run's own Fisher vector, determinism, CUDA-graph replay, the refusals and the allocation peak."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import mfv_oracle as mo
from scanobjectnn_b200 import mfv_net_cls as M
from scanobjectnn_b200 import ops
from scanobjectnn_b200.engine import InferenceEngine
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import VariableStore

from . import gpu_util as G

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# every (r, k, cin, cout) of the model's 20 conv3d layers at the default configuration
CONVS = sorted({(3 if s.startswith(("inception4", "inception5")) else 5, k, cin, cout) for s, k, cin, cout in M._module_widths()})


@pytest.fixture(params=[0, 1, 2], ids=["tensor", "fma", "tensor_bf16x3"])
def mode(request):
    ops.set_mlp_mode(request.param)
    yield request.param
    ops.set_mlp_mode(0)


def _gmm(r):
    return [torch.from_numpy(t).cuda() for t in M.get_3d_grid_gmm((r, r, r))]


@pytest.mark.parametrize("kind", ["ball", "shell", "dup"])
@pytest.mark.parametrize("b,n,r", [(1, 1024, 5), (3, 1000, 5), (32, 1024, 5), (2, 2048, 8)])
def test_fisher_vector_matches_float64(kind, b, n, r):
    pts = make_clouds(kind, b, n, seed=b + n + r)
    w, mu, s = _gmm(r)
    got = ops.fisher_vector(torch.from_numpy(pts).cuda(), w, mu, s)
    want = mo.fisher_vector(pts, G.npy(w), G.npy(mu), G.npy(s))
    err = float(np.abs(G.npy(got).astype(np.float64) - want).max())
    print(f"[fv] {kind} b={b} n={n} r={r}: max|err| = {err:.2e}")
    assert err < 1e-6
    assert torch.equal(got, ops.fisher_vector(torch.from_numpy(pts).cuda(), w, mu, s))


def _grid(rows, b, r, device="cpu"):
    """voxel-major rows (b*r^3, C) -> (b, C, r, r, r) float64"""
    return rows.detach().to(device=device, dtype=torch.float64).reshape(r ** 3, b, -1).permute(1, 2, 0).reshape(b, -1, r, r, r)


def _conv_case(r, k, cin, cout, b, seed, weight_scale=1.0):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    p = VariableStore(device="cuda", seed=seed)
    p.add_conv3d("c", k, cin, cout, randomize_bn=True)
    p["c/weights"] = p["c/weights"] * weight_scale
    rows = b * r ** 3
    buf = torch.zeros((rows, cin + 32), device="cuda")                       # x is read as a column slice of a wider buffer
    if cin == 20:                                                              # the Fisher vector's range
        buf[:, 16:16 + cin] = torch.rand((rows, cin), generator=gen, device="cuda") * 2 - 1
    else:                                                                      # post-ReLU activations
        buf[:, 16:16 + cin] = torch.relu(torch.randn((rows, cin), generator=gen, device="cuda"))
    return p, buf[:, 16:16 + cin]


def _calibrate(p, x, b, r):
    """batch norm set to the float64 statistics of the layer's own pre-norm output on x"""
    y = torch.nn.functional.conv3d(_grid(x, b, r), mo._d(p["c/weights"]).permute(4, 3, 0, 1, 2), padding=p["c/weights"].shape[0] // 2)
    y = y + mo._d(p["c/biases"])[None, :, None, None, None]
    p["c/bn/moving_mean"] = y.mean(dim=(0, 2, 3, 4)).float().cuda()
    p["c/bn/moving_variance"] = y.var(dim=(0, 2, 3, 4), unbiased=False).float().cuda()


def _check_conv(p, x, b, r, cout, what, device="cpu"):
    W, sc, sh, _ = p.folded("c")
    out = torch.zeros((x.shape[0], cout + 64), device="cuda")
    ops.conv3d(x, r, W, sc, sh, out=out, offset=32)
    assert not out[:, :32].any() and not out[:, 32 + cout:].any(), f"{what}: wrote outside its channel slice"
    want = mo.conv3d(_grid(x, b, r, device), p, "c")
    got = _grid(out[:, 32:32 + cout], b, r)
    G.contract_close(got.numpy(), G.npy(want), what)
    return float(sc.max())


@pytest.mark.parametrize("r,k,cin,cout", CONVS)
def test_conv3d_matches_float64(mode, r, k, cin, cout):
    b = 3                                                                      # 128-row tiles end inside a cloud's voxels
    p, x = _conv_case(r, k, cin, cout, b, seed=r * 1000 + k * 100 + cin)
    _check_conv(p, x, b, r, cout, f"conv r={r} k={k} {cin}->{cout} mode={mode}")
    # calibrated batch norm: the weights scaled down so that the folded scale is large (> 10) and amplifies every rounding
    p, x = _conv_case(r, k, cin, cout, b, seed=r * 1000 + k * 100 + cin + 1, weight_scale=0.05)
    _calibrate(p, x, b, r)
    big = _check_conv(p, x, b, r, cout, f"calibrated conv r={r} k={k} {cin}->{cout} mode={mode}")
    assert big > 10, big


def _tile_width(b, r, cout):
    """the column-tile width conv_plan (csrc/mfv.cu) picks: 128 when the padded width allows it and the 128-wide tiles alone
    fill more than half of the 132 SMs"""
    tiles, np_ = -(-b * r ** 3 // 128), -(-cout // 64) * 64
    return 128 if np_ % 128 == 0 and 2 * tiles * (np_ // 128) > 132 else 64


def test_conv3d_at_the_model_batch_sizes():
    """B=32 and B=64 with the split tap loop on 64-wide column tiles, modes 0 and 2, against float64 (evaluated on the GPU)"""
    for b in (32, 64):
        for r, k, cin, cout in [(5, 5, 256, 128), (3, 5, 512, 256), (5, 3, 64, 32), (3, 1, 768, 512)]:
            assert _tile_width(b, r, cout) == 64
            p, x = _conv_case(r, k, cin, cout, b, seed=b + k + cin)
            for m in (0, 2):
                ops.set_mlp_mode(m)
                try:
                    _check_conv(p, x, b, r, cout, f"conv b={b} r={r} k={k} {cin}->{cout} mode={m}", "cuda")
                finally:
                    ops.set_mlp_mode(0)


# shapes whose plan takes 128-wide column tiles (tc_conv3d_kernel<NP, 2>): inception3_conv1 / conv4 at B=64, and the large 3^3 / 5^3
# layers at B=128 and B=256
WIDE = [(64, 5, 1, 384, 256), (128, 5, 5, 256, 128), (128, 5, 3, 256, 128), (256, 3, 3, 512, 256), (256, 3, 5, 512, 256)]


@pytest.mark.parametrize("m", [0, 2], ids=["tensor", "tensor_bf16x3"])
@pytest.mark.parametrize("b,r,k,cin,cout", WIDE)
def test_conv3d_wide_tiles_match_float64(m, b, r, k, cin, cout):
    assert _tile_width(b, r, cout) == 128
    ops.set_mlp_mode(m)
    try:
        p, x = _conv_case(r, k, cin, cout, b, seed=b + r + k + cin)
        _check_conv(p, x, b, r, cout, f"wide conv b={b} r={r} k={k} {cin}->{cout} mode={m}", "cuda")
        p, x = _conv_case(r, k, cin, cout, b, seed=b + r + k + cin + 1, weight_scale=0.05)
        _calibrate(p, x, b, r)
        big = _check_conv(p, x, b, r, cout, f"calibrated wide conv b={b} r={r} k={k} {cin}->{cout} mode={m}", "cuda")
        assert big > 10, big
    finally:
        ops.set_mlp_mode(0)


@pytest.mark.parametrize("b,r,k,cin,cout", [(3, 5, 3, 128, 64), (64, 5, 1, 384, 256), (128, 5, 5, 256, 128)])
def test_conv3d_range_guard_reruns_on_bf16x3(b, r, k, cin, cout):
    """inputs scaled past 65504: the fp16x2 pass raises its flag, mode 0 returns bit for bit what mode 2 computes (the rerun's
    image is built over the fp16x2 image's bytes), and both are right (64- and 128-wide column tiles)"""
    p, x = _conv_case(r, k, cin, cout, b, seed=5 + b)
    x = x * 1e5
    W, sc, sh, _ = p.folded("c")
    got = {}
    for m in (0, 2):
        ops.set_mlp_mode(m)
        try:
            got[m] = ops.conv3d(x, r, W, sc, sh)
        finally:
            ops.set_mlp_mode(0)
    assert torch.equal(got[0], got[2])
    G.contract_close(_grid(got[0], b, r).numpy(), G.npy(mo.conv3d(_grid(x, b, r, "cuda"), p, "c")), f"x1e5 b={b} k={k} {cin}->{cout}")


def test_conv3d_misaligned_affine_takes_the_fma_kernel():
    """scale / shift that are contiguous but not 8-byte aligned (an odd-offset slice) must not reach the tensor path's float2
    loads: the call is served by the FMA kernel and is still right"""
    b, r, k, cin, cout = 3, 5, 3, 128, 64
    p, x = _conv_case(r, k, cin, cout, b, seed=9)
    W, sc, sh, _ = p.folded("c")
    buf = torch.zeros((2, cout + 1), device="cuda")
    buf[0, 1:], buf[1, 1:] = sc, sh
    out = ops.conv3d(x, r, W, buf[0, 1:], buf[1, 1:])
    assert buf[0, 1:].data_ptr() % 8 == 4
    G.contract_close(_grid(out, b, r).numpy(), mo.conv3d(_grid(x, b, r), p, "c").numpy(), "misaligned scale / shift")


def test_conv3d_workspace_follows_the_path():
    from scanobjectnn_b200 import _lib
    lib = _lib.load()
    big = lib.psa_conv3d_workspace_bytes(32, 3, 5, 512, 256)
    assert big > 0
    assert lib.psa_conv3d_workspace_bytes(32, 5, 1, 20, 64) == 0           # c = 20: the FMA kernel
    ops.set_mlp_mode(1)
    try:
        assert lib.psa_conv3d_workspace_bytes(32, 3, 5, 512, 256) == 0
    finally:
        ops.set_mlp_mode(0)
    # mode 0 holds one weight image (the bf16x3 rerun reuses the fp16x2 image's bytes): under 7 bytes per weight with the partials
    assert big < 125 * 512 * 256 * 7 + 16 * 32 * 27 * 256 * 4


@pytest.mark.parametrize("r", [5, 3])
def test_pool3d_matches_float64(r):
    b, c = 3, 96
    gen = torch.Generator(device="cuda").manual_seed(r)
    x = torch.randn((b * r ** 3, c), generator=gen, device="cuda")
    x[5, :] = x[6, :]                                                          # ties in the max
    avg = ops.pool3d(x, r, "avg")
    mx = ops.pool3d(x, r, "max")
    ro = (r + 1) // 2
    assert tuple(mx.shape) == (b * ro ** 3, c)
    assert float((_grid(avg, b, r) - mo.avg_pool3(_grid(x, b, r))).abs().max()) < 1e-6
    assert torch.equal(_grid(mx, b, ro), mo.max_pool2(_grid(x, b, r)))


@pytest.fixture(scope="module")
def params():
    return M.init_params(seed=11, randomize_bn=True)


@pytest.mark.parametrize("b", [32, 64])
def test_model_matches_float64_on_its_own_fisher_vector(params, b):
    """B=32 and B=64 (ScanObjectNN's batch, where inception3's 1^3 layers take 128-wide column tiles)"""
    n = 1024
    if b == 64:
        assert _tile_width(64, 5, 256) == 128
    pts = torch.from_numpy(make_clouds("ball", b, n, seed=21)).cuda()
    gmm = _gmm(5)
    logits, fv = M.get_model(pts, *gmm, False, params=params)
    assert tuple(fv.shape) == (b, 20, 125) and tuple(logits.shape) == (b, 15)
    want_fv = mo.fisher_vector(G.npy(pts), *(G.npy(t) for t in gmm))
    assert float(np.abs(G.npy(fv).astype(np.float64) - want_fv.transpose(0, 2, 1)).max()) < 1e-6
    want, _ = mo.forward_from_fv(fv.transpose(1, 2), params)                  # float64, on the GPU
    G.contract_close(G.npy(logits), G.npy(want), "3dmfv logits")
    again, _ = M.get_model(pts, *gmm, False, params=params)
    assert torch.equal(logits, again)
    eng = InferenceEngine(lambda x: M.get_model(x, *gmm, False, params=params)[0], (b, n, 3), (b, 15), slots=1)
    slot = eng.submit(pts)
    assert torch.equal(eng.result(slot), logits)


def test_refusals_on_the_gpu(params):
    pts = torch.zeros((2, 64, 3), device="cuda")
    gmm = _gmm(5)
    with pytest.raises(NotImplementedError):
        M.get_model(pts, *gmm, True, params=params)
    with pytest.raises(NotImplementedError):
        M.get_model(pts.clone().requires_grad_(True), *gmm, False, params=params)
    with pytest.raises(NotImplementedError):
        M.get_model(pts, *gmm, False, add_noise=True, params=params)
    with pytest.raises(ValueError):
        M.get_model(pts, *gmm, False, num_classes=40, params=params)
    with pytest.raises(ValueError):                                            # G = 100 is not a cube
        M.get_model(pts, gmm[0][:100], gmm[1][:100], gmm[2][:100], False, params=params)
    with pytest.raises(ValueError):
        ops.conv3d(torch.zeros((125, 64), device="cuda"), 5, torch.zeros((2, 2, 2, 64, 32), device="cuda"), None, torch.zeros(32, device="cuda"))
    with pytest.raises(ValueError):
        ops.pool3d(torch.zeros((100, 8), device="cuda"), 5, "max")
    with pytest.raises(ValueError):
        ops.fisher_vector(pts, gmm[0], gmm[1][:, :2], gmm[2])


def test_allocation_peak_is_below_the_composition(params):
    spec = importlib.util.spec_from_file_location("mfv_timing", os.path.join(ROOT, "tools", "mfv_timing.py"))
    T = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(T)
    pts = torch.from_numpy(make_clouds("ball", 32, 1024, seed=9)).cuda()
    gmm = _gmm(5)
    comp = T.Composed(params)
    with torch.no_grad():
        M.get_model(pts, *gmm, False, params=params)                          # warm-up: folded weights cached
        comp.forward(pts, *gmm)
        fused, lf = T.peak(lambda: M.get_model(pts, *gmm, False, params=params)[0])
        composed, lc = T.peak(lambda: comp.forward(pts, *gmm))
    print(f"[peak] B=32 N=1024: fused {fused / 2**20:.1f} MiB, torch composition {composed / 2**20:.1f} MiB above the inputs and weights")
    assert fused < composed
    assert float((lf - lc).abs().max()) < 1e-3
