"""Training-mode fused EdgeConv (training.edgeconv_training, csrc/edgeconv_train.cu) against a float64 restatement of the materialised
formula and against the materialising composition (group_point -> [x_i, x_j - x_i] -> mlp_training -> amax) it replaces in dgcnn.

Inputs on coarse dyadic grids (x on 1/16, weights on 1/64) make every edge value y_ij exact in fp32 whatever the summation order, so
the fused op, the composition and float64 all see the same tied maxima.  With generic floats two fp32 evaluations in different orders
can disagree on a near-tie at the last bit and route the max's gradient differently; that is a property of the max, not an error."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from scanobjectnn_b200 import _lib, ops
from scanobjectnn_b200.tf_util import VariableStore
from scanobjectnn_b200.training import EdgeConvTrainer, edgeconv_training, mlp_training

from .restate import edgeconv_store, edges, flat_grad, grid_x, rel

OTOL, GTOL = 1e-5, 1e-4          # outputs / gradients, relative to the largest entry (the bound of test_train_gpu.py)
MODEL = (32, 2048, 20)           # DGCNN: B, N, k


def _ref64(x, idx, W, bias, gamma, beta):
    """[x_i, x_j - x_i] . W + b -> batch norm over all edges (biased variance, eps 1e-3) -> relu -> amax over k, in float64"""
    y = edges(x, idx) @ W + bias
    mean, var = y.mean((0, 1, 2)), y.var((0, 1, 2), unbiased=False)
    z = torch.relu((y - mean) / torch.sqrt(var + 1e-3) * gamma + beta)
    return z.amax(dim=2), mean, var


def _old_path(x, idx, scope, params):
    """the materialising composition dgcnn used for single-layer EdgeConvs (and still uses for the T-net)"""
    b, n, c = x.shape
    k = idx.shape[-1]
    centre = x.unsqueeze(2).expand(b, n, k, c)
    edge = torch.cat([centre, ops.group_point(x.contiguous(), idx) - centre], dim=-1)
    y = mlp_training(edge.reshape(b * n * k, 2 * c), [(scope, True)], 0.5, params)
    return y.view(b, n, k, -1).amax(dim=2)


def test_edgeconv_train_rejects_bad_arguments_without_a_gpu():
    lib = _lib.load()
    fake = C.c_void_p(1 << 20)                  # never dereferenced: every check below fails before any launch
    null = C.c_void_p(0)
    big = C.c_size_t(1 << 40)

    def fwd(b, n, c, k, cout, ws=fake, ws_bytes=big, x=fake):
        return lib.psa_edgeconv_train_fwd(b, n, c, k, cout, x, fake, fake, null, fake, fake, ws, ws_bytes, null)

    def bwd(b, n, c, k, cout, ws=fake, ws_bytes=big):
        return lib.psa_edgeconv_train_bwd(b, n, c, k, cout, *([fake] * 15), ws, ws_bytes, null)

    assert fwd(0, 16, 4, 20, 64) == -1 and fwd(2, 16, 0, 20, 64) == -1 and fwd(2, 16, 4, 0, 64) == -1
    assert b"bad dims" in lib.psa_last_error()
    assert fwd(2, 16, 4, 20, 64, x=null) == -1                                    # null buffer
    need = lib.psa_edgeconv_train_workspace_bytes(2, 16, 4, 20, 64)
    assert need > 0
    assert fwd(2, 16, 4, 20, 64, ws_bytes=C.c_size_t(need - 1)) == -1            # short workspace
    assert b"workspace" in lib.psa_last_error()
    assert fwd(2, 16, 4, 20, 64, ws=C.c_void_p((1 << 20) + 16)) == -1             # misaligned workspace
    assert b"aligned" in lib.psa_last_error()
    assert fwd(2, 16, 4, 20, 48) == -2 and bwd(2, 16, 4, 20, 48) == -2            # C_out not a multiple of 32
    assert fwd(2, 16, 4, 20, 288) == -2                                          # C_out > 256
    assert lib.psa_edgeconv_train_pool(2, 16, 20, 48, *([fake] * 6), null) == -2
    assert lib.psa_edgeconv_train_workspace_bytes(2, 16, 4, 20, 48) == 0
    assert bwd(1, 51201, 4, 20, 64) == -2                                        # beyond the reverse neighbour lists
    assert bwd(2, 16, 4, 20, 64, ws=null) == -1
    # a weight of the wrong shape is refused before anything is allocated on a device
    p = VariableStore(device="cpu")
    p.add_conv2d("e", 6, 64)
    with pytest.raises(ValueError, match=r"\(8, C_out\)"):
        EdgeConvTrainer(p, 2, 16, 4, 20, "e", device="cpu")


@pytest.mark.gpu
@pytest.mark.parametrize("c,cout,k", [(3, 64, 20), (64, 64, 20), (64, 128, 20), (64, 64, 1), (64, 32, 40)])
def test_edgeconv_training_matches_float64(c, cout, k):
    """outputs, moving averages and every gradient against torch autograd over the float64 formula; random graphs with self-loops,
    and one cloud made of duplicated points, so tied maxima and their even split occur"""
    b, n = 3, 300
    p = edgeconv_store(c, cout, seed=c + cout + k)
    x_np = grid_x(b, n, c, seed=k)
    x_np[1, n // 2:] = x_np[1, :n // 2]                                             # cloud 1: every point twice
    rng = np.random.default_rng(7)
    idx_np = rng.integers(0, n, (b, n, k)).astype(np.int32)
    idx_np[:, :, 0] = np.arange(n)                                                  # self-loops, as kNN has them
    idx_np[1, :, 1 % k] = (np.arange(n) + n // 2) % n                               # ... and the point's duplicate
    x = torch.tensor(x_np, device="cuda", requires_grad=True)
    idx = torch.tensor(idx_np, device="cuda")
    s = "e"
    w64, b64 = p[f"{s}/weights"].double().reshape(2 * c, cout).clone().requires_grad_(True), p[f"{s}/biases"].double().clone().requires_grad_(True)
    g64, be64 = p[f"{s}/bn/gamma"].double().clone().requires_grad_(True), p[f"{s}/bn/beta"].double().clone().requires_grad_(True)
    mm0, mv0 = p[f"{s}/bn/moving_mean"].double().clone(), p[f"{s}/bn/moving_variance"].double().clone()

    out = edgeconv_training(x, idx, s, 0.9, p)
    assert out.shape == (b, n, cout) and out.grad_fn is not None
    R = torch.tensor(np.random.default_rng(11).standard_normal((b, n, cout)).astype(np.float32), device="cuda")
    fp = p._flat
    gflat, gx = torch.autograd.grad(out, [fp.flat, x], R)

    x64 = x.detach().double().requires_grad_(True)
    o64, mean, var = _ref64(x64, idx, w64, b64, g64, be64)
    want = torch.autograd.grad(o64, [x64, w64, b64, g64, be64], R.double())
    assert rel(out.detach().cpu(), o64.detach().cpu()) < OTOL
    assert rel(p[f"{s}/bn/moving_mean"].cpu(), (0.9 * mm0 + 0.1 * mean.detach()).cpu()) < OTOL
    assert rel(p[f"{s}/bn/moving_variance"].cpu(), (0.9 * mv0 + 0.1 * var.detach()).cpu()) < OTOL
    assert rel(gx.cpu(), want[0].cpu()) < GTOL
    assert rel(flat_grad(p, f"{s}/weights", gflat).reshape(2 * c, cout).cpu(), want[1].cpu()) < GTOL
    assert rel(flat_grad(p, f"{s}/bn/gamma", gflat).cpu(), want[3].cpu()) < GTOL
    assert rel(flat_grad(p, f"{s}/bn/beta", gflat).cpu(), want[4].cpu()) < GTOL
    assert not bool(flat_grad(p, f"{s}/biases", gflat).any()) and not bool(fp.grad_of(f"{s}/biases").any())     # exactly zero under BN
    ties = p._trainers[("edgeconv", s, b, n, c, k)].ties
    assert k == 1 or int(ties.max()) > 1                                           # the even split was exercised


@pytest.mark.gpu
def test_edgeconv_training_matches_the_materialising_composition_at_the_model_shape():
    """B=32, N=2048, k=20, 128 -> 64 (dgcnn2..3), on the real kNN graph of the input"""
    b, n, k = MODEL
    c, cout = 64, 64
    x = torch.tensor(grid_x(b, n, c, seed=3), device="cuda", requires_grad=True)
    idx = ops.knn_graph(x.detach(), k)
    R = torch.tensor(np.random.default_rng(5).standard_normal((b, n, cout)).astype(np.float32), device="cuda")
    res = []
    for fn in (lambda p: edgeconv_training(x, idx, "dgcnn2", 0.5, p), lambda p: _old_path(x, idx, "dgcnn2", p)):
        p = edgeconv_store(c, cout, seed=21, scope="dgcnn2")
        out = fn(p)
        gflat, gx = torch.autograd.grad(out, [p._flat.flat, x], R)
        fp = p._flat
        res.append((out.detach(), gx, *(flat_grad(p, f"dgcnn2/{v}", gflat).clone() for v in ("weights", "bn/gamma", "bn/beta", "biases"))))
        del out, gflat, gx, p
        torch.cuda.empty_cache()
    errs = {name: rel(a.cpu(), bb.cpu()) for name, a, bb in zip(("out", "dx", "dW", "dgamma", "dbeta"), res[0], res[1])}
    print("[edgeconv vs composition] max error relative to the largest entry:", {k_: f"{v:.2e}" for k_, v in errs.items()})
    assert errs["out"] < OTOL
    assert max(errs["dx"], errs["dW"], errs["dgamma"], errs["dbeta"]) < GTOL
    assert not bool(res[0][5].any())


@pytest.mark.gpu
def test_edgeconv_training_is_bit_reproducible_and_stores_no_edge_tensor():
    b, n, k = MODEL
    c, cout = 64, 64
    rng = np.random.default_rng(8)
    x = torch.tensor(rng.standard_normal((b, n, c)).astype(np.float32), device="cuda", requires_grad=True)
    idx = ops.knn_graph(x.detach(), k)
    R = torch.tensor(rng.standard_normal((b, n, cout)).astype(np.float32), device="cuda")
    p = VariableStore(device="cuda", seed=4)
    p.add_conv2d("dgcnn2", 2 * c, cout, randomize_bn=True)
    gc.collect()                     # earlier tests' trainers must not be freed inside the measured window
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    runs = []
    for _ in range(2):
        out = edgeconv_training(x, idx, "dgcnn2", 0.5, p)
        gflat, gx = torch.autograd.grad(out, [p._flat.flat, x], R)
        runs.append((out.detach(), gflat, gx))
        if len(runs) == 1:
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - base
    edge_bytes = b * n * k * cout * 4
    print(f"[edgeconv] forward + backward raised the allocation peak by {peak / 2**20:.1f} MiB (one per-edge tensor: {edge_bytes / 2**20:.1f} MiB)")
    assert peak < edge_bytes
    for a, bb in zip(runs[0], runs[1]):
        assert torch.equal(a, bb)
