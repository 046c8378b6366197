"""Generate tests/golden/*.npz from the REFERENCE's own code.

Runs on the GPU box (the reference's CUDA kernels need a device):
    python tests/golden/make_golden.py OUT_DIR        # on a GPU machine with oracle/_ref built
  * ref_gpu_*.npz   outputs of pointnet2/tf_ops/{sampling/tf_sampling_g.cu, grouping/tf_grouping_g.cu} compiled
                    for sm_90a (oracle/_ref/libref_tfops.so, built by `make -C oracle ref` from the reference checkout)
  * ref_cpu_*.npz   outputs of the reference's CPU code (oracle/_ref/libref_cpu.so): threenn_cpu,
                    threeinterpolate_cpu, query_ball_point_cpu, selection_sort_cpu
Inputs are NOT stored: they are regenerated from seeds by scanobjectnn_b200.synthetic.make_clouds / numpy
default_rng exactly as written here (tests/test_golden*.py repeat the same calls).
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np

from oracle import oracle as orc
from scanobjectnn_b200.synthetic import make_clouds

CASES = [("ball", 1001), ("shell", 1002), ("dup", 1003)]
B, N = 4, 2048


def inputs(kind, seed):
    return make_clouds(kind, B, N, seed=seed)


def main(outdir):
    os.makedirs(outdir, exist_ok=True)
    import torch

    from tests import gpu_util as G
    for kind, seed in CASES:
        xyz = inputs(kind, seed)
        t = G.cu(xyz)
        fps1 = G.ref_fps(t, 512)
        l1 = G.ref_gather_point(t, fps1)
        bq1, cnt1 = G.ref_query_ball_point(0.2, 32, t, l1)
        fps2 = G.ref_fps(l1, 128)
        l2 = G.ref_gather_point(l1, fps2)
        bq2, cnt2 = G.ref_query_ball_point(0.4, 64, l1, l2)
        np.savez_compressed(os.path.join(outdir, f"ref_gpu_{kind}.npz"),
                            fps1=G.npy(fps1).astype(np.int16), bq1=G.npy(bq1).astype(np.int16), cnt1=G.npy(cnt1).astype(np.int16),
                            fps2=G.npy(fps2).astype(np.int16), bq2=G.npy(bq2).astype(np.int16), cnt2=G.npy(cnt2).astype(np.int16))
    # SelectionSort on a seeded matrix with ties
    rng = np.random.default_rng(77)
    d = rng.random((2, 8, 200), dtype=np.float32)
    d[0, 0, 10:40] = d[0, 0, 3]
    d[1, 1, :] = 0.25
    oi, ov = G.ref_selection_sort(16, G.cu(d))
    np.savez_compressed(os.path.join(outdir, "ref_gpu_selection_sort.npz"), outi=G.npy(oi).astype(np.int16), out=G.npy(ov))
    # CPU-only reference ops
    xyz1 = make_clouds("shell", 2, 2048, seed=2001)
    xyz2 = make_clouds("ball", 2, 512, seed=2002)
    dist, idx = orc.refcpu_three_nn(xyz1, xyz2)
    pts = np.random.default_rng(2003).standard_normal((2, 512, 16)).astype(np.float32)
    w = orc.three_weights(dist)          # pointnet_util.py:212-215 (TF ops in the reference; restated)
    out = orc.refcpu_three_interpolate(pts, idx, w)
    np.savez_compressed(os.path.join(outdir, "ref_cpu_three_nn.npz"), dist=dist, idx=idx.astype(np.int16), interp=out)
    qb = orc.refcpu_query_ball_point(0.2, 32, xyz2, xyz2[:, ::4].copy(), fill=-1)
    np.savez_compressed(os.path.join(outdir, "ref_cpu_ball_query.npz"), idx=qb.astype(np.int16))
    print("golden written to", outdir, sorted(os.listdir(outdir)))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "gpurun_out", "golden"))
