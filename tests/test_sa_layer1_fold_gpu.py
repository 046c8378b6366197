"""Layer 1 of a set-abstraction level with input features runs as V[j] + c . s (Wc - Wx), with V = s (points . W1[3:] +
xyz . W1[:3]) + t computed once per source point by the dense layer in front of the level.  That reassociation has edges of
its own, checked here against float64 at PointNet++ SA2's widths (131 -> 128 -> 128 -> 256, 64 neighbours):
  * clouds far from the origin: V and the centre term are large and cancel to the small (x_j - c) . W1x of the level;
  * a neighbour equal to its centre (every neighbourhood's first entry is the centre itself);
  * V beyond the fp16 range: the fp16x2 level raises its flag and the bf16x3 rerun, which reads the same V, gives the result."""
import numpy as np
import pytest
import torch

from scanobjectnn_b200 import ops

pytestmark = pytest.mark.gpu

B, N, M, K, C = 4, 512, 128, 64, 128
WIDTHS = [3 + C, 128, 128, 256]


def _case(offset, feat_scale, seed):
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(-1.0, 1.0, (B, N, 3)) + offset
    new_xyz = xyz[:, :M].copy()                                   # centres are points of the cloud
    idx = rng.integers(0, N, (B, M, K)).astype(np.int32)
    idx[:, :, 0] = np.arange(M)                                   # the first neighbour is the centre itself
    pts = np.maximum(rng.standard_normal((B, N, C)), 0.0) * feat_scale
    layers = []
    for l in range(3):
        w = rng.standard_normal((WIDTHS[l], WIDTHS[l + 1])) / np.sqrt(WIDTHS[l])
        layers.append((w, rng.uniform(0.5, 2.0, WIDTHS[l + 1]), rng.standard_normal(WIDTHS[l + 1]) * 0.1))
    return [a.astype(np.float32) for a in (xyz, new_xyz, pts)], idx, [tuple(a.astype(np.float32) for a in L) for L in layers]


def _reference(xyz, new_xyz, pts, idx, layers):
    x, c, f = (a.astype(np.float64) for a in (xyz, new_xyz, pts))
    bi = np.arange(B)[:, None, None]
    h = np.concatenate([x[bi, idx] - c[:, :, None, :], f[bi, idx]], axis=-1)
    for w, s, t in layers:
        h = np.maximum(h @ w.astype(np.float64) * s + t, 0.0)
    return h.max(axis=2)


@pytest.mark.parametrize("offset, feat_scale", [(0.0, 1.0), (10.0, 1.0), (0.0, 3e5)], ids=["origin", "far", "overflow"])
def test_folded_layer1_matches_float64(offset, feat_scale):
    (xyz, new_xyz, pts), idx, layers = _case(offset, feat_scale, seed=7)
    dev = lambda a: torch.from_numpy(a).cuda()
    mlp = ops.MlpParams([(dev(w), dev(s), dev(t), True) for w, s, t in layers])
    got = ops.sa_module_infer(dev(xyz), dev(new_xyz), dev(pts), 0.4, K, mlp, idx=dev(idx)).cpu().numpy()
    want = _reference(xyz, new_xyz, pts, idx, layers)
    if feat_scale > 1.0:
        assert np.abs(want).max() > 65504.0, "the case must leave the fp16 range"
    err = np.abs(got - want).max()
    assert np.isfinite(got).all() and err <= 1e-5 * max(1.0, np.abs(want).max()), f"max |err| {err:.3e}, max |want| {np.abs(want).max():.3e}"
