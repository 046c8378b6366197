"""Host-side readers of the reference (data_utils.py), same names and return values, so that real ScanObjectNN files
can be fed to the kernels when they are available (SURVEY 8f rank 3).  Pure numpy; h5py is optional (absent in the
build image: ``load_h5`` then raises ImportError with the reason instead of failing at import).

Raw object files (README.md:27-57, data_utils.py:50-75): float32 ``[count, count x (x y z nx ny nz r g b inst sem)]``.
h5 files (data_utils.py:249-261): ``data (M,2048,3) float32``, ``label (M,)``, ``mask (M,2048)`` with -1 = background."""
from __future__ import annotations

import os

import numpy as np


def load_pc_file(filename, suncg: bool = False, with_bg: bool = True, data_path: str = ""):
    """data_utils.py:50-75.  Returns the (count,3) xyz array; ``with_bg=False`` keeps only the points of the most frequent
    instance label among those whose last attribute is not 0/1/2 (the reference's background filter)."""
    pc = np.fromfile(os.path.join(data_path, filename), dtype=np.float32)
    if pc.size < 1:
        raise ValueError(f"{filename}: empty object file")
    count = int(pc[0])
    per = 3 if suncg else 11
    if pc.size - 1 != count * per:
        raise ValueError(f"{filename}: header says {count} points, file holds {(pc.size - 1) / per:g}")
    pc = pc[1:].reshape((-1, per))
    if with_bg or suncg:
        return np.array(pc[:, 0:3])
    keep = np.where((pc[:, -1] != 0) & (pc[:, -1] != 1) & (pc[:, -1] != 2))[0]
    values, counts = np.unique(pc[keep, -1], return_counts=True)
    idx = np.where(pc[:, -1] == values[np.argmax(counts)])[0]
    return np.array(pc[idx, 0:3])


def _h5py():
    try:
        import h5py
    except ImportError as e:          # pragma: no cover - depends on the image
        raise ImportError("h5py is not installed: ScanObjectNN .h5 files cannot be read in this environment") from e
    return h5py


def load_h5(h5_filename):
    """data_utils.py:249-253 -> (data (M,N,3) float32, label (M,))."""
    with _h5py().File(h5_filename, "r") as f:
        return f["data"][:], f["label"][:]


def load_withmask_h5(h5_filename):
    """data_utils.py:255-261 -> (data, label, mask (M,N); -1 = background)."""
    with _h5py().File(h5_filename, "r") as f:
        return f["data"][:], f["label"][:], f["mask"][:]


def load_parts_h5(h5_filename):
    """data_utils.py:271-277 -> (data, label, parts (M,N) per-point part labels)."""
    with _h5py().File(h5_filename, "r") as f:
        return f["data"][:], f["label"][:], f["parts"][:]


def convert_to_binary_mask(masks):
    """data_utils.py:280-290: 1 = object, 0 = background (mask == -1), float64 like the reference."""
    masks = np.asarray(masks)
    out = np.ones(masks.shape)
    out[masks == -1] = 0
    return out


def get_current_data_h5(pcs, labels, num_points, rng: np.random.Generator | None = None, return_indices: bool = False):
    """data_utils.py:171-186: one random point subset shared by all clouds, then a random cloud order.  Returns the
    reference's (sampled, labels); with ``return_indices`` also (idx_pts[:num_points], cloud_order) -- the index lists
    ``ops.augment_batch(perm=...)`` takes when the subset is applied on the device instead."""
    rng = np.random.default_rng() if rng is None else rng
    idx_pts = rng.permutation(pcs.shape[1])
    order = rng.permutation(len(labels))
    sampled = pcs[:, idx_pts[:num_points], :][order]
    if return_indices:
        return sampled, np.asarray(labels)[order], idx_pts[:num_points].astype(np.int32), order
    return sampled, np.asarray(labels)[order]


def get_current_data_withmask_h5(pcs, labels, masks, num_points, shuffle: bool = True, rng: np.random.Generator | None = None):
    """data_utils.py:188-210: get_current_data_h5 that carries the per-point masks (M,N) along with the points.  ``shuffle=False``
    keeps the first num_points points and the cloud order.  Returns (sampled, labels, sampled_mask)."""
    idx_pts = np.arange(pcs.shape[1])
    order = np.arange(len(labels))
    if shuffle:
        rng = np.random.default_rng() if rng is None else rng
        idx_pts = rng.permutation(pcs.shape[1])
        order = rng.permutation(len(labels))
    return pcs[:, idx_pts[:num_points], :][order], np.asarray(labels)[order], masks[:, idx_pts[:num_points]][order]


def get_current_data_parts_h5(pcs, labels, parts, num_points, rng: np.random.Generator | None = None):
    """data_utils.py:212-229: get_current_data_h5 that carries the per-point part labels (M,N).  Returns (sampled, labels,
    sampled_parts)."""
    return get_current_data_withmask_h5(pcs, labels, parts, num_points, True, rng)
