"""The host readers of the segmentation scripts (data_utils.py:188-229, 271-277): masks and part labels follow their points."""
import numpy as np
import pytest

from scanobjectnn_b200 import data_utils as du


def _clouds(m=5, n=12):
    # point j of cloud i sits at (i, j, i * 100 + j); its mask / part label is i * 100 + j as well
    ii, jj = np.meshgrid(np.arange(m), np.arange(n), indexing="ij")
    pcs = np.stack([ii, jj, ii * 100 + jj], axis=-1).astype(np.float32)
    return pcs, np.arange(m) * 10, (ii * 100 + jj).astype(np.int64)


@pytest.mark.parametrize("fn", ["withmask", "parts"])
def test_per_point_labels_follow_the_sampled_points(fn):
    pcs, labels, per_point = _clouds()
    rng = np.random.default_rng(3)
    if fn == "withmask":
        sampled, lab, sp = du.get_current_data_withmask_h5(pcs, labels, per_point, 7, rng=rng)
    else:
        sampled, lab, sp = du.get_current_data_parts_h5(pcs, labels, per_point, 7, rng=rng)
    assert sampled.shape == (5, 7, 3) and sp.shape == (5, 7) and lab.shape == (5,)
    assert np.array_equal(sampled[:, :, 2], sp)                       # each label travels with its point
    assert np.array_equal(lab, sampled[:, 0, 0].astype(int) * 10)      # and each cloud label with its cloud
    # one point subset shared by every cloud (data_utils.py:190-197), distinct points, and a permutation of the clouds
    assert (sampled[:, :, 1] == sampled[:1, :, 1]).all()
    assert len(set(sampled[0, :, 1].tolist())) == 7
    assert sorted(sampled[:, 0, 0].astype(int).tolist()) == list(range(5))


def test_injected_rng_is_deterministic_and_matches_the_plain_reader():
    pcs, labels, per_point = _clouds()
    a = du.get_current_data_withmask_h5(pcs, labels, per_point, 6, rng=np.random.default_rng(9))
    b = du.get_current_data_parts_h5(pcs, labels, per_point, 6, rng=np.random.default_rng(9))
    c = du.get_current_data_h5(pcs, labels, 6, np.random.default_rng(9))
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    assert np.array_equal(a[0], c[0]) and np.array_equal(a[1], c[1])


def test_withmask_without_shuffle_keeps_the_first_points_in_order():
    pcs, labels, per_point = _clouds()
    sampled, lab, sp = du.get_current_data_withmask_h5(pcs, labels, per_point, 4, shuffle=False)
    assert np.array_equal(sampled, pcs[:, :4]) and np.array_equal(lab, labels) and np.array_equal(sp, per_point[:, :4])


def test_parts_reader_reports_missing_dependency(tmp_path):
    try:
        import h5py  # noqa: F401
    except ImportError:
        with pytest.raises(ImportError, match="h5py"):
            du.load_parts_h5(str(tmp_path / "x.h5"))
        return
    with h5py.File(tmp_path / "p.h5", "w") as f:
        f["data"], f["label"], f["parts"] = np.zeros((2, 4, 3), np.float32), np.arange(2), np.ones((2, 4), np.int64)
    d, lab, parts = du.load_parts_h5(str(tmp_path / "p.h5"))
    assert d.shape == (2, 4, 3) and lab.tolist() == [0, 1] and parts.shape == (2, 4)
