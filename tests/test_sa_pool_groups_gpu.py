"""A level whose last layer is too wide to pool all its 64-channel chunks at once pools them in groups: a 128 -> 64 -> 640
level at fp16x2 leaves room for a pooling buffer of five chunks, so it runs two groups of five, an odd group size that ends
in a single chunk.  Every chunk of the last layer sees the same A fragment, weight block and wgmma order whatever the
layer's width, so the wide level's columns must equal, bitwise, those of the same level cut to its first 512 and last 128
output channels, which pool all their chunks in one group.  The gathers of the next pass run whatever the grouping: a
pass that kept the previous pass's coordinates or U rows would break the equality."""
import numpy as np
import pytest
import torch

from scanobjectnn_b200 import ops
from scanobjectnn_b200.synthetic import make_clouds

pytestmark = pytest.mark.gpu


def _layer(rng, cin, cout, relu=True):
    w = torch.from_numpy((rng.standard_normal((cin, cout)) / np.sqrt(cin)).astype(np.float32)).cuda()
    scale = torch.from_numpy(rng.uniform(-1.5, 1.5, cout).astype(np.float32)).cuda()
    shift = torch.from_numpy(rng.uniform(-0.2, 0.2, cout).astype(np.float32)).cuda()
    return w, scale, shift, relu


@pytest.mark.parametrize("k,r", [(32, 0.2), (64, 0.4)])
def test_grouped_pooling_matches_single_group_bitwise(k, r):
    b, n, m, c = 4, 512, 128, 128
    rng = np.random.default_rng(k)
    l0, l1, (w2, s2, t2, _) = _layer(rng, 3 + c, 128), _layer(rng, 128, 64), _layer(rng, 64, 640)
    xyz = torch.from_numpy(make_clouds("ball", b, n, seed=n)).cuda()
    pts = torch.from_numpy(rng.standard_normal((b, n, c)).astype(np.float32)).cuda()
    _, new_xyz = ops.farthest_point_sample_and_gather(m, xyz)
    idx, _ = ops.query_ball_point(r, k, xyz, new_xyz)

    def run(cols):
        last = (w2[:, cols].contiguous(), s2[cols].contiguous(), t2[cols].contiguous(), True)
        return ops.sa_module_infer(xyz, new_xyz, pts, r, k, ops.MlpParams([l0, l1, last]), idx=idx)

    wide = run(slice(0, 640))
    lo, hi = run(slice(0, 512)), run(slice(512, 640))
    torch.cuda.synchronize()
    wide, want = wide.cpu().numpy(), torch.cat([lo, hi], dim=-1).cpu().numpy()
    assert np.isfinite(want).all() and (want != 0).mean() > 0.2
    assert np.array_equal(wide.view(np.uint32), want.view(np.uint32)), f"max|diff| = {np.abs(wide - want).max()}"
