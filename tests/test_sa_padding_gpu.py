"""The set-abstraction tensor-core kernel computes only the rows of each neighbourhood before its ball-query padding (the
entries from L on repeat idx[0], and a max does not change when a row is repeated).  Here the same level is run on the ball
query's tail-padded idx, which compacts, and on the same idx with each neighbourhood's entries permuted so that the last one
differs from the first, which forces every row to be computed.  The two outputs must be bitwise equal: a real row dropped,
or pooled into the wrong neighbourhood, breaks it.  Neighbourhood sizes on the 16-row slot boundaries are forced into idx."""
import numpy as np
import pytest
import torch

from scanobjectnn_b200 import ops
from scanobjectnn_b200.pointnet_util import _mlp_scopes, add_sa_module_params
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import VariableStore

pytestmark = pytest.mark.gpu


def _force_counts(idx, n, counts, rng):
    """rows of idx (G, K) rewritten as `count` distinct points followed by copies of the first (count 0: all zeros),
    spread over the array so that they fall at different positions of chunks and passes"""
    rows = idx.shape[0]
    picks = rng.choice(rows, size=3 * len(counts), replace=False)
    picks[-1] = rows - 1                                   # the last neighbourhood of the level
    for i, r in enumerate(picks):
        cnt = counts[i % len(counts)]
        row = np.zeros(idx.shape[1], np.int32)
        if cnt:
            row[:cnt] = rng.choice(n, size=cnt, replace=False)
            row[cnt:] = row[0]
        idx[r] = row
    return idx


def _permute_to_full(idx, rng):
    """each row's entries permuted so that the last differs from the first (rows with a single distinct value stay as they are)"""
    out = idx.copy()
    for r in range(out.shape[0]):
        row = rng.permutation(out[r])
        if row[-1] == row[0]:
            other = np.nonzero(row != row[0])[0]
            if len(other):
                j = other[0]
                row[-1], row[j] = row[j], row[-1]
        out[r] = row
    return out


@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("n,m,r,k,c,mlp", [(2048, 512, 0.2, 32, 0, [64, 64, 128]),        # PointNet++ SA1
                                           (512, 128, 0.4, 64, 128, [128, 128, 256])])    # PointNet++ SA2
def test_padding_rows_skipped_bitwise(n, m, r, k, c, mlp, mode):
    b = 4
    p = VariableStore(device="cuda", seed=k)
    add_sa_module_params(p, "sa", 3 + c, mlp, randomize_bn=True)
    params = p.mlp(_mlp_scopes("sa", mlp))
    rng = np.random.default_rng(k)
    xyz = torch.from_numpy(make_clouds("ball", b, n, seed=n)).cuda()
    pts = torch.from_numpy(rng.standard_normal((b, n, c)).astype(np.float32)).cuda() if c else None
    _, new_xyz = ops.farthest_point_sample_and_gather(m, xyz)
    idx, cnt = ops.query_ball_point(r, k, xyz, new_xyz)
    counts = [0, 1, 16, 17, k] + ([33, 48] if k == 64 else [])
    padded = _force_counts(idx.cpu().numpy().reshape(b * m, k), n, counts, rng)
    full = _permute_to_full(padded, rng)
    distinct = np.array([len(np.unique(row)) for row in padded])
    assert (distinct < k).mean() > 0.5, "the ball query should leave most neighbourhoods padded"
    assert all(np.any(distinct == max(cc, 1)) for cc in counts)
    assert np.all((full[:, -1] != full[:, 0]) | (distinct == 1))
    ops.set_mlp_mode(mode)
    try:
        got = ops.sa_module_infer(xyz, new_xyz, pts, r, k, params, idx=torch.from_numpy(padded.reshape(b, m, k)).cuda())
        want = ops.sa_module_infer(xyz, new_xyz, pts, r, k, params, idx=torch.from_numpy(full.reshape(b, m, k)).cuda())
        torch.cuda.synchronize()
    finally:
        ops.set_mlp_mode(0)
    got, want = got.cpu().numpy(), want.cpu().numpy()
    assert np.isfinite(want).all()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"max|diff| = {np.abs(got - want).max()}"
