"""Tensor-core path: the arithmetic-mode switch, and one dense tensor-core layer in isolation against fp64 (descriptor / fragment layout /
swizzle check: structured rows and columns that a layout mix-up would move)."""
import numpy as np
import pytest
import torch

from scanobjectnn_b200 import ops

from . import gpu_util as G

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kd,n", [(64, 64), (64, 128), (128, 64), (128, 128), (512, 256)])
def test_tc_single_layer_matches_fp64(kd, n):
    rng = np.random.default_rng(kd * 1000 + n)
    a = np.maximum(rng.standard_normal((128, kd)), 0).astype(np.float32)
    a[5] = 0.0
    a[:, 3] = np.arange(128, dtype=np.float32) / 128         # a structured column / row pattern: catches layout mix-ups
    w = (rng.uniform(-1, 1, (kd, n)) * np.sqrt(6.0 / (kd + n))).astype(np.float32)
    w[7, :] = np.linspace(-1, 1, n, dtype=np.float32)
    mlp = ops.MlpParams([(G.cu(w), None, torch.zeros(n, device="cuda"), False)])
    d = G.npy(ops.shared_mlp(G.cu(a), mlp))
    want = a.astype(np.float64) @ w.astype(np.float64)
    G.contract_close(d, want, f"tensor-core layer {kd}x{n}")


def test_tc_identity_weight_is_exact_passthrough():
    a = np.random.default_rng(0).standard_normal((128, 128)).astype(np.float32)
    mlp = ops.MlpParams([(torch.eye(128, device="cuda"), None, torch.zeros(128, device="cuda"), False)])
    d = G.npy(ops.shared_mlp(G.cu(a), mlp))
    # w = 1 is one exact piece; a = a1 + a2 drops what lies below 2^-22 |a| (fp16x2): the product reproduces a to that rounding
    assert np.abs(d - a).max() <= np.abs(a).max() * 2.0 ** -22


def test_mlp_mode_switch():
    assert ops.get_mlp_mode() == 0
    ops.set_mlp_mode(1)
    assert ops.get_mlp_mode() == 1
    ops.set_mlp_mode(2)              # tensor cores with bf16x3 operands (what the fp16 range guard reruns on)
    assert ops.get_mlp_mode() == 2
    ops.set_mlp_mode(0)
    with pytest.raises(ValueError):
        ops.set_mlp_mode(3)
