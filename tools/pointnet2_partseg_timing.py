"""Cost of pointnet2_cls_partseg (PointNet++ part segmentation) with fa_layer1 as a grouped first layer, against fa_layer1 as the
reference writes it (pointnet_fp_module: three_nn + interpolation, i.e. tile(l3_points, 128), + concat with l2_points, K = 1280), at
B=32 and N in {1024, 2048}:

  inference       get_model(xyz, False) under no_grad
  training step   get_model(xyz, True) + get_loss + backward (variable gradients in the flat bucket; no optimizer step)

  grouped   pointnet_fp_module_broadcast: l3_points . W[0:1024] once per cloud, W[1024:1280] over the 128 points of each cloud
  concat    pointnet_fp_module on the materialised (B, 128, 1280) input

The two are alternated call by call; medians of --iters CUDA-event timings after --warmup.  Also prints the allocation peak of one
inference call of each above what was allocated before it, and the card's name and power limit.

  python tools/pointnet2_partseg_timing.py [--batch 32] [--npoints 1024 2048] [--iters 20] [--warmup 5]
"""
from __future__ import annotations

import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scanobjectnn_b200 import pointnet2_cls_partseg as M  # noqa: E402
from scanobjectnn_b200.pointnet_util import pointnet_fp_module, pointnet_fp_module_broadcast  # noqa: E402
from scanobjectnn_b200.synthetic import make_clouds  # noqa: E402

GROUPED, CONCAT = pointnet_fp_module_broadcast, pointnet_fp_module


def _use(fa_layer1):
    M.pointnet_fp_module_broadcast = fa_layer1


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
        p = M.init_params(seed=1, randomize_bn=True)
        xyz = torch.from_numpy(make_clouds("ball", B, N, seed=7)).cuda()
        parts = (torch.arange(B * N, device="cuda") % M.NUM_CLASSES).view(B, N)

        def infer(fa_layer1):
            def fn():
                _use(fa_layer1)
                with torch.no_grad():
                    return M.get_model(xyz, False, params=p)
            return fn

        def step(fa_layer1):
            def fn():
                _use(fa_layer1)
                M.get_loss(M.get_model(xyz, True, bn_decay=0.5, params=p), parts).backward()
                p._flat.flat.grad = None
            return fn

        seg_g, seg_c = infer(GROUPED)(), infer(CONCAT)()
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
