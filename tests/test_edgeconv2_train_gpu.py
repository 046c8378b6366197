"""Training-mode two-layer EdgeConv (training.edgeconv_training with two scopes, csrc/edgeconv2_train.cu) against a float64 restatement
of the materialised formula and against the materialising composition (group_point -> [x_i, x_j - x_i] -> mlp_training over the
edge rows -> amax) that DGCNN's input transform net used before.

y2 goes through batch norm 1, whose scale is irrational, so no input grid makes it exact: a maximum whose runner-up (a different value,
not a bit-identical duplicate edge) lies within 1e-5 of it may be won by another edge in fp32.  The tests find those maxima on the
float64 side and give them a zero incoming gradient, so the routing of their gradient does not matter; exact ties (self-loops,
duplicated points) keep theirs and exercise the even split."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from scanobjectnn_b200 import _lib, dgcnn, ops
from scanobjectnn_b200.tf_util import VariableStore
from scanobjectnn_b200.training import EdgeConv2Trainer, MlpTrainer, edgeconv_training, mlp_training

from .restate import EC2, ambiguous, edgeconv2_store, edges, flat_grad, layer, params_as, rel

OTOL, GTOL = 1e-5, 1e-4
MODEL = (32, 2048, 20)
S1, S2 = EC2


def _ref64(x, idx, P):
    """[x_i, x_j - x_i] -> (conv + batch norm over all edges (biased variance, eps 1e-3) + relu) twice -> (max over k, z2, batch
    stats by scope)"""
    stats = {}
    h = layer(layer(edges(x, idx), P, S1, False, stats=stats), P, S2, False, stats=stats)
    return h.amax(dim=2), h, stats


def _composition(x, idx, bn_decay, params):
    b, n, c = x.shape
    k = idx.shape[-1]
    centre = x.unsqueeze(2).expand(b, n, k, c)
    edge = torch.cat([centre, ops.group_point(x.contiguous(), idx) - centre], dim=-1)
    y = mlp_training(edge.reshape(b * n * k, 2 * c), [(S1, True), (S2, True)], bn_decay, params)
    return y.view(b, n, k, -1).amax(dim=2)


def test_edgeconv2_train_rejects_bad_arguments_without_a_gpu():
    lib = _lib.load()
    fake = C.c_void_p(1 << 20)                  # never dereferenced: every check below fails before any launch
    null = C.c_void_p(0)
    big = C.c_size_t(1 << 40)

    def fwd(b, n, c, k, c1=64, c2=128, ws=fake, ws_bytes=big, nn=fake):
        return lib.psa_edgeconv2_train_fwd(b, n, c, k, c1, c2, nn, *([fake] * 6), ws, ws_bytes, null)

    def pool(b, n, c, k, c1=64, c2=128, ws=fake):
        return lib.psa_edgeconv2_train_pool(b, n, c, k, c1, c2, *([fake] * 11), ws, big, null)

    def bwd(b, n, c, k, c1=64, c2=128, ws=fake, ws_bytes=big):
        return lib.psa_edgeconv2_train_bwd(b, n, c, k, c1, c2, *([fake] * 23), ws, ws_bytes, null)

    assert fwd(0, 16, 3, 20) == -1 and fwd(2, 16, 0, 20) == -1 and fwd(2, 16, 3, 0) == -1
    assert b"bad dims" in lib.psa_last_error()
    assert fwd(2, 16, 3, 20, nn=null) == -1 and b"null" in lib.psa_last_error()
    assert pool(2, 16, 3, 20, ws=null) == -1 and bwd(2, 16, 3, 20, ws=null) == -1
    need = lib.psa_edgeconv2_train_workspace_bytes(2, 16, 3, 20, 64, 128)
    assert need >= lib.psa_edgeconv_train_workspace_bytes(2, 16, 3, 20, 64) > 0      # the layer-1 call shares the workspace
    assert fwd(2, 16, 3, 20, ws_bytes=C.c_size_t(need - 1)) == -1 and b"workspace" in lib.psa_last_error()
    assert fwd(2, 16, 3, 20, ws=C.c_void_p((1 << 20) + 16)) == -1 and b"aligned" in lib.psa_last_error()
    for c1, c2 in ((32, 128), (64, 64), (128, 128), (64, 256)):
        assert fwd(2, 16, 3, 20, c1, c2) == -2 and pool(2, 16, 3, 20, c1, c2) == -2 and bwd(2, 16, 3, 20, c1, c2) == -2
        assert lib.psa_edgeconv2_train_workspace_bytes(2, 16, 3, 20, c1, c2) == 0
    assert fwd(2, 16, 3, 33) == -2 and b"mask" in lib.psa_last_error()               # k > 32
    assert lib.psa_edgeconv2_train_workspace_bytes(2, 16, 3, 33, 64, 128) == 0
    assert bwd(1, 51201, 3, 20) == -2                                                # beyond the reverse neighbour lists
    # weights of the wrong shape are refused before anything is allocated on a device
    p = VariableStore(device="cpu")
    p.add_conv2d(S1, 6, 64)
    p.add_conv2d(S2, 64, 128)
    with pytest.raises(ValueError, match=r"\(8, C1\)"):
        EdgeConv2Trainer(p, 2, 16, 4, 20, (S1, S2), device="cpu")
    q = VariableStore(device="cpu")
    q.add_conv2d(S1, 6, 64)
    q.add_conv2d(S2, 32, 128)
    with pytest.raises(ValueError, match=r"\(64, C2\)"):
        EdgeConv2Trainer(q, 2, 16, 3, 20, (S1, S2), device="cpu")
    r = VariableStore(device="cpu")
    r.add_conv2d(S1, 6, 64)
    r.add_conv2d(S2, 64, 64)
    with pytest.raises(_lib.PsaError, match="C2 = 64"):
        EdgeConv2Trainer(r, 2, 16, 3, 20, (S1, S2), device="cpu")


@pytest.mark.gpu
@pytest.mark.parametrize("k", [20, 1, 32])
def test_edgeconv2_training_matches_float64(k):
    """outputs, both layers' moving averages and every gradient against torch autograd over the float64 formula; random graphs with
    self-loops, and one cloud made of duplicated points, so exact ties and their even split occur"""
    b, n, c = 3, 300, 3
    p = edgeconv2_store(c, seed=k)
    rng = np.random.default_rng(k)
    x_np = rng.standard_normal((b, n, c)).astype(np.float32)
    x_np[1, n // 2:] = x_np[1, :n // 2]                                             # cloud 1: every point twice
    idx_np = rng.integers(0, n, (b, n, k)).astype(np.int32)
    idx_np[:, :, 0] = np.arange(n)                                                  # self-loops, as kNN has them
    idx_np[1, :, 1 % k] = (np.arange(n) + n // 2) % n                               # ... and the point's duplicate
    x = torch.tensor(x_np, device="cuda", requires_grad=True)
    idx = torch.tensor(idx_np, device="cuda")
    P = params_as(p, torch.float64, grad=True)
    names = [f"{s}/{v}" for s in (S1, S2) for v in ("weights", "biases", "bn/gamma", "bn/beta")]
    mov0 = {s: (p[f"{s}/bn/moving_mean"].double().clone(), p[f"{s}/bn/moving_variance"].double().clone()) for s in (S1, S2)}

    x64 = x.detach().double().requires_grad_(True)
    o64, z64, stats = _ref64(x64, idx, P)
    amb = ambiguous(z64, 2)
    R = torch.tensor(rng.standard_normal((b, n, 128)).astype(np.float32), device="cuda")
    R[amb] = 0.0
    print(f"[edgeconv2 k={k}] ambiguous maxima masked: {int(amb.sum())} of {amb.numel()}")
    assert float(amb.double().mean()) < 0.01

    out = edgeconv_training(x, idx, (S1, S2), 0.9, p)
    assert out.shape == (b, n, 128) and out.grad_fn is not None
    fp = p._flat
    gflat, gx = torch.autograd.grad(out, [fp.flat, x], R)
    want = dict(zip(["x"] + names, torch.autograd.grad(o64, [x64] + [P[v] for v in names], R.double())))

    assert rel(out.detach().cpu(), o64.detach().cpu()) < OTOL
    for s, (mean, var) in stats.items():
        mm0, mv0 = mov0[s]
        assert rel(p[f"{s}/bn/moving_mean"].cpu(), (0.9 * mm0 + 0.1 * mean.detach()).cpu()) < OTOL
        assert rel(p[f"{s}/bn/moving_variance"].cpu(), (0.9 * mv0 + 0.1 * var.detach()).cpu()) < OTOL
    assert rel(gx.cpu(), want["x"].cpu()) < GTOL
    for s in (S1, S2):
        assert rel(flat_grad(p, f"{s}/weights", gflat).cpu(), want[f"{s}/weights"].cpu()) < GTOL, s
        assert rel(flat_grad(p, f"{s}/bn/gamma", gflat).cpu(), want[f"{s}/bn/gamma"].cpu()) < GTOL, s
        assert rel(flat_grad(p, f"{s}/bn/beta", gflat).cpu(), want[f"{s}/bn/beta"].cpu()) < GTOL, s
        assert not bool(flat_grad(p, f"{s}/biases", gflat).any()) and not bool(fp.grad_of(f"{s}/biases").any())   # exactly zero under BN
    mask = p._trainers[("edgeconv2", (S1, S2), b, n, c, k)].mask
    cnt = np.unpackbits(mask.cpu().numpy().view(np.uint8)).reshape(tuple(mask.shape) + (32,)).sum(-1).astype(np.int64)
    assert cnt.min() >= 1
    assert k == 1 or cnt.max() > 1                                                  # the even split was exercised


@pytest.mark.gpu
def test_edgeconv2_training_matches_the_materialising_composition_at_the_model_shape():
    """B=32, N=2048, k=20, c=3 -> 64 -> 128 (the T-net) on the real kNN graph of the input"""
    b, n, k = MODEL
    c = 3
    rng = np.random.default_rng(3)
    x = torch.tensor(rng.standard_normal((b, n, c)).astype(np.float32), device="cuda", requires_grad=True)
    idx = ops.knn_graph(x.detach(), k)
    with torch.no_grad():
        _, z64, _ = _ref64(x.detach().double(), idx, params_as(edgeconv2_store(c, seed=21), torch.float64))
        amb = ambiguous(z64, 2)
        del z64
    torch.cuda.empty_cache()
    R = torch.tensor(rng.standard_normal((b, n, 128)).astype(np.float32), device="cuda")
    R[amb] = 0.0
    print(f"[edgeconv2 model shape] ambiguous maxima masked: {int(amb.sum())} of {amb.numel()}")
    assert float(amb.double().mean()) < 0.01
    res = []
    for fn in (lambda p: edgeconv_training(x, idx, (S1, S2), 0.5, p), lambda p: _composition(x, idx, 0.5, p)):
        p = edgeconv2_store(c, seed=21)
        out = fn(p)
        gflat, gx = torch.autograd.grad(out, [p._flat.flat, x], R)
        fp = p._flat
        res.append((out.detach(), gx) + tuple(flat_grad(p, f"{s}/{v}", gflat).clone() for s in (S1, S2) for v in ("weights", "bn/gamma", "bn/beta")))
        del out, gflat, gx, p
        torch.cuda.empty_cache()
    names = ("out", "dx", "dW1", "dgamma1", "dbeta1", "dW2", "dgamma2", "dbeta2")
    errs = {name: rel(a.cpu(), bb.cpu()) for name, a, bb in zip(names, res[0], res[1])}
    print("[edgeconv2 vs composition] max error relative to the largest entry:", {k_: f"{v:.2e}" for k_, v in errs.items()})
    assert errs["out"] < OTOL
    assert max(v for k_, v in errs.items() if k_ != "out") < GTOL


@pytest.mark.gpu
def test_edgeconv2_training_is_bit_reproducible_and_stores_no_edge_tensor():
    b, n, k = MODEL
    c = 3
    rng = np.random.default_rng(8)
    x = torch.tensor(rng.standard_normal((b, n, c)).astype(np.float32), device="cuda", requires_grad=True)
    idx = ops.knn_graph(x.detach(), k)
    R = torch.tensor(rng.standard_normal((b, n, 128)).astype(np.float32), device="cuda")
    p = edgeconv2_store(c, seed=4)
    gc.collect()                     # earlier tests' trainers must not be freed inside the measured window
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    runs = []
    for _ in range(2):
        out = edgeconv_training(x, idx, (S1, S2), 0.5, p)
        gflat, gx = torch.autograd.grad(out, [p._flat.flat, x], R)
        runs.append((out.detach(), gflat, gx))
        if len(runs) == 1:
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - base
    del out, gflat, gx
    q = edgeconv2_store(c, seed=4)
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base_c = torch.cuda.memory_allocated()
    oc = _composition(x, idx, 0.5, q)
    torch.autograd.grad(oc, [q._flat.flat, x], R)
    torch.cuda.synchronize()
    peak_c = torch.cuda.max_memory_allocated() - base_c
    edge_bytes = b * n * k * 128 * 4
    print(f"[edgeconv2] forward + backward raised the allocation peak by {peak / 2**20:.1f} MiB (composition: {peak_c / 2**20:.1f} MiB; "
          f"one E x C2 tensor: {edge_bytes / 2**20:.1f} MiB)")
    assert peak < edge_bytes
    for a, bb in zip(runs[0], runs[1]):
        assert torch.equal(a, bb)


@pytest.mark.gpu
def test_dgcnn_training_runs_the_t_net_without_an_edge_row_trainer():
    b, n = 2, 256
    p = dgcnn.init_params(seed=1)
    xyz = torch.randn(b, n, 3, device="cuda")
    logits, ep = dgcnn.get_model(xyz, True, bn_decay=0.5, params=p)
    dgcnn.get_loss(logits, torch.zeros(b, dtype=torch.int64, device="cuda"), ep).backward()
    trainers = p._trainers.values()
    assert not any(isinstance(t, MlpTrainer) and t.rows == b * n * dgcnn.K_NEIGHBORS for t in trainers)
    assert any(isinstance(t, EdgeConv2Trainer) for t in trainers)
    assert bool(torch.isfinite(p._flat.flat.grad).all())
