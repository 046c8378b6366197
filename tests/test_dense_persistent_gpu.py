"""tc_dense_kernel at shapes where each persistent CTA processes several tiles: parity against the fp64 restatement, and
results that do not depend on which CTA claimed which tile (dynamic claiming at inference, a static order in training)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import mlp_oracle as mo
from scanobjectnn_b200 import _lib, ops
from scanobjectnn_b200._lib import PsaActIn, ptr, stream
from scanobjectnn_b200.tf_util import VariableStore

from . import gpu_util as G

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["tensor", "tensor_bf16x3"])
def mlp_mode(request):
    ops.set_mlp_mode({"tensor": 0, "tensor_bf16x3": 2}[request.param])
    yield request.param
    ops.set_mlp_mode(0)


@pytest.mark.parametrize("rows,pool_k,chans,offset", [(65536, 2048, [320, 1024], 0), (65536, 1, [256, 512], 0),
                                                      (16384, 64, [131, 256], 0),       # odd K: element-wise x staging
                                                      (16384, 1, [128, 256], 1)])       # x not 16-byte aligned
def test_multi_tile_shared_mlp_matches_fp64(rows, pool_k, chans, offset, mlp_mode):
    p = VariableStore(device="cuda", seed=rows + chans[0])
    scopes = []
    for i in range(len(chans) - 1):
        p.add_conv2d(f"m/conv{i}", chans[i], chans[i + 1], bn=True, randomize_bn=True)
        scopes.append(f"m/conv{i}")
    relus = [True] * len(scopes)
    rng = np.random.default_rng(rows + chans[0])
    x = rng.standard_normal((rows, chans[0])).astype(np.float32)
    buf = torch.empty(rows * chans[0] + offset, device="cuda")
    xd = buf[offset:].view(rows, chans[0])
    xd.copy_(G.cu(x))
    mlp = p.mlp(scopes, relus)
    got = ops.shared_mlp(xd, mlp, pool_k=pool_k)
    again = ops.shared_mlp(xd, mlp, pool_k=pool_k)
    assert torch.equal(got, again), "the result depends on the tile schedule"
    want = mo.mlp_chain(x, p, scopes, relus)
    if pool_k > 1:
        want = want.reshape(rows // pool_k, pool_k, -1).max(1)
    G.contract_close(G.npy(got), want, f"shared_mlp {chans} pool {pool_k} rows {rows}")


def test_training_forward_is_bitwise_repeatable():
    """The training forward takes its tiles in a static order: output and column statistics are bitwise the same run to run."""
    lib = _lib.load()
    rows, K, N = 16384, 256, 512
    rng = np.random.default_rng(5)
    xd, sd, td = G.cu(rng.standard_normal((rows, K)).astype(np.float32)), G.cu(rng.uniform(0.5, 1.5, K).astype(np.float32)), \
        G.cu(rng.standard_normal(K).astype(np.float32) * 0.3)
    Wd, bd = G.cu((rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)), G.cu(rng.standard_normal(N).astype(np.float32) * 0.1)
    need = lib.psa_train_dense_workspace_bytes(rows, K, N)
    ws = torch.empty(need // 4 + 16, device="cuda")
    a = PsaActIn()
    a.x = xd.data_ptr(); a.ld = K; a.mask = None; a.relu = 1; a.scale = sd.data_ptr(); a.shift = td.data_ptr()
    outs = []
    for _ in range(2):
        y = torch.empty((rows, N), device="cuda")
        stats = torch.empty((2, N), device="cuda")
        assert lib.psa_train_dense_fwd(rows, K, N, C.byref(a), ptr(Wd), ptr(bd), ptr(y), ptr(stats), ptr(ws), C.c_size_t(need), stream()) == 0
        outs.append((y, stats))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    h = np.maximum(G.npy(xd).astype(np.float64) * G.npy(sd) + G.npy(td), 0)
    want = h @ G.npy(Wd).astype(np.float64) + G.npy(bd)
    assert float(np.abs(G.npy(outs[0][0]) - want).max() / np.abs(want).max()) < 1e-5
