"""The set-abstraction kernel max-pools its last layer into one shared row per neighbourhood of the chunk a unit is computing,
with atomicMax on an order-preserving int code of the float, and stores the rows once per chunk.  Checked against float64 at
1e-5 where the existing tests do not reach:
  * a last layer without ReLU whose outputs are nearly all negative (the code flips the magnitude bits of negative values),
    the rest positive;
  * neighbourhoods of every size, several spanning passes, and ones of a single repeated point (`cnt = 0`);
  * a level whose neighbourhood count is not a multiple of the chunk, so the last chunk's rows past the end are not stored;
  * warpgroup units (K = 32, 64), joint units (K = 128), and a last layer 768 wide, which at fp16x2 is resident but leaves no
    room for a joint buffer of all its columns and is therefore streamed, pooled 64 columns at a time."""
import numpy as np
import pytest
import torch

from scanobjectnn_b200 import ops

from . import restate

pytestmark = pytest.mark.gpu

B, M = 3, 37                                              # 111 neighbourhoods: 15 past the last full 16-chunk, 7 past the 8-chunk


def _case(n, k, widths, c, seed):
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(-1.0, 1.0, (B, n, 3)).astype(np.float32)
    new_xyz = xyz[:, :M].copy()
    pts = rng.standard_normal((B, n, c)).astype(np.float32) if c else None
    # neighbourhood sizes cycle through the 16-row slot edges, a single point (the ball query's cnt = 0) and full
    sizes = [1, 0, 2, 15, 16, 17, k - 1, k, 31, 33] * (B * M)
    idx = np.empty((B * M, k), np.int32)
    for g in range(B * M):
        cnt = min(sizes[g], k)
        row = rng.choice(n, size=max(cnt, 1), replace=False).astype(np.int32)
        idx[g] = np.concatenate([row, np.full(k - len(row), row[0], np.int32)])
    layers = []
    for l in range(len(widths) - 1):
        w = rng.standard_normal((widths[l], widths[l + 1])) / np.sqrt(widths[l])
        s, t = rng.uniform(0.5, 2.0, widths[l + 1]), rng.standard_normal(widths[l + 1]) * 0.1
        if l == len(widths) - 2:
            t = t - 4.0                                   # the last layer, without ReLU: nearly every output negative
        layers.append((w.astype(np.float32), s.astype(np.float32), t.astype(np.float32)))
    return xyz, new_xyz, pts, idx.reshape(B, M, k), layers


def _reference(xyz, new_xyz, pts, idx, layers):
    t64 = lambda a: None if a is None else torch.from_numpy(a).double()
    x = t64(xyz)
    ar = torch.arange(B)[:, None, None]
    h = torch.cat([x[ar, torch.from_numpy(idx).long()] - t64(new_xyz)[:, :, None, :]]
                  + ([t64(pts)[ar, torch.from_numpy(idx).long()]] if pts is not None else []), -1)
    for l, (w, s, t) in enumerate(layers):
        h = h @ t64(w) * t64(s) + t64(t)
        if l < len(layers) - 1:
            h = torch.clamp_min(h, 0.0)
    return h.amax(dim=2).numpy()


@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("n,k,c,widths", [(512, 32, 0, [3, 64, 64, 128]),          # SA1's widths, warpgroup units
                                          (512, 64, 128, [131, 128, 128, 256]),    # SA2's widths, warpgroup units
                                          (512, 128, 0, [3, 64, 64, 128]),         # joint units
                                          (512, 32, 0, [3, 64, 64, 768])],         # joint, the last layer streamed
                         ids=["sa1", "sa2", "k128", "wide"])
def test_pooled_last_layer_without_relu_matches_float64(n, k, c, widths, mode):
    assert restate.sa_tc_layers(widths, c, k, mode) is not None, "the level must run on the set-abstraction kernel"
    xyz, new_xyz, pts, idx, layers = _case(n, k, widths, c, seed=k + len(widths) + widths[-1])
    dev = lambda a: None if a is None else torch.from_numpy(a).cuda()
    mlp = ops.MlpParams([(dev(w), dev(s), dev(t), l < len(layers) - 1) for l, (w, s, t) in enumerate(layers)])
    ops.set_mlp_mode(mode)
    try:
        got = ops.sa_module_infer(dev(xyz), dev(new_xyz), dev(pts), 0.4, k, mlp, idx=dev(idx)).cpu().numpy()
    finally:
        ops.set_mlp_mode(0)
    want = _reference(xyz, new_xyz, pts, idx, layers)
    assert got.shape == want.shape and 0.9 < (want < 0).mean() < 1.0
    err = np.abs(got - want).max()
    assert np.isfinite(got).all() and err <= 1e-5 * max(1.0, np.abs(want).max()), f"max |err| {err:.3e}, max |want| {np.abs(want).max():.3e}"
