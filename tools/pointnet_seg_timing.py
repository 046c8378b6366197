"""Cost of pointnet_seg (PointNet's classification + background-mask model) with the tiled global feature folded into conv6, against
the tile + concat composition the reference writes (pointnet/models/pointnet_seg.py:81-88), at B=32 and N in {1024, 2048}:

  inference       get_model(xyz, False) under no_grad
  training step   get_model(xyz, True) + get_loss + backward (variable gradients in the flat bucket; no optimizer step)

  grouped   conv6's point rows over the points (K = 64) plus one row per cloud (ops.shared_mlp_grouped / mlp_training(group=))
  concat    conv6 over concat([point_feat, tile(global_feat)]) (K = 1088), as a shared_mlp chain / an mlp_training node

The two are alternated call by call; medians of --iters CUDA-event timings after --warmup.  Also prints the allocation peak of one
inference call of each above what was allocated before it, and the card's name and power limit.

  python tools/pointnet_seg_timing.py [--batch 32] [--npoints 1024 2048] [--iters 20] [--warmup 5]
"""
from __future__ import annotations

import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scanobjectnn_b200 import ops, pointnet_seg, training  # noqa: E402
from scanobjectnn_b200.synthetic import make_clouds  # noqa: E402

GROUPED = (pointnet_seg.seg_head, pointnet_seg.seg_head_training)
LAYERS = [(s, True) for s in pointnet_seg.HEAD] + [("conv10", False)]


def _tiled(point_feat, global_feat):
    b, n, _ = point_feat.shape
    return torch.cat([point_feat, global_feat[:, None, :].expand(b, n, global_feat.shape[-1])], dim=2)


def concat_head(point_feat, global_feat, params):
    h = ops.shared_mlp(_tiled(point_feat, global_feat), params.mlp(pointnet_seg.HEAD))
    return ops.shared_mlp(h, params.mlp(["conv10"], [False]))


def concat_head_training(point_feat, global_feat, bn_decay, params, frozen=False):
    return training.mlp_training(_tiled(point_feat, global_feat), LAYERS, bn_decay, params, frozen=frozen)


CONCAT = (concat_head, concat_head_training)


def _use(head):
    pointnet_seg.seg_head, pointnet_seg.seg_head_training = head


def _alternate(fns, iters, warmup):
    for _ in range(warmup):
        for fn in fns:
            fn()
    torch.cuda.synchronize()
    ms = [[] for _ in fns]
    for _ in range(iters):
        for i, fn in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ms[i].append(a.elapsed_time(b))
    return [statistics.median(m) for m in ms]


def _peak_mib(fn):
    fn()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2**20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--npoints", type=int, nargs="+", default=[1024, 2048])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_properties(0).name
    print(f"# {card}, B={a.batch}, median of {a.iters} after {a.warmup} warm-up iterations (CUDA events), grouped and concat alternated")
    B = a.batch
    for N in a.npoints:
        p = pointnet_seg.init_params(seed=1, randomize_bn=True)
        xyz = torch.from_numpy(make_clouds("ball", B, N, seed=7)).cuda()
        labels = torch.arange(B, device="cuda") % pointnet_seg.NUM_CLASSES
        mask = (torch.arange(B * N, device="cuda") % 3 == 0).long().view(B, N)

        def infer(head):
            def fn():
                _use(head)
                with torch.no_grad():
                    return pointnet_seg.get_model(xyz, False, params=p)
            return fn

        def step(head):
            def fn():
                _use(head)
                cls, seg, ep = pointnet_seg.get_model(xyz, True, bn_decay=0.5, params=p)
                pointnet_seg.get_loss(cls, seg, labels, mask, ep)[0].backward()
                p._flat.flat.grad = None
            return fn

        seg_g, seg_c = infer(GROUPED)()[1], infer(CONCAT)()[1]
        diff = float((seg_g - seg_c).abs().max())
        del seg_g, seg_c
        tg, tc = _alternate([infer(GROUPED), infer(CONCAT)], a.iters, a.warmup)
        print(f"N={N:5d} inference      grouped {tg:8.3f} ms   concat {tc:8.3f} ms   (max|seg_pred diff| {diff:.2e})")
        pg, pc = _peak_mib(infer(GROUPED)), _peak_mib(infer(CONCAT))
        print(f"N={N:5d} inference peak grouped {pg:8.1f} MiB  concat {pc:8.1f} MiB")
        tg, tc = _alternate([step(GROUPED), step(CONCAT)], a.iters, a.warmup)
        print(f"N={N:5d} training step  grouped {tg:8.3f} ms   concat {tc:8.3f} ms")
        _use(GROUPED)
        del p


if __name__ == "__main__":
    main()
