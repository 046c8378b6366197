"""Cost of the gradient with respect to the input point coordinates at B=32, N=2048 (CUDA events, median of --iters after --warmup),
for pointnet2_cls_ssg (--model ssg, the default), dgcnn (--model dgcnn) or vanilla PointNet (--model pointnet):

  fused inference forward          get_model(xyz, False) without requires_grad (fused kernels, BN folded)
  frozen forward + input backward  get_model(xyz, False) with xyz.requires_grad: training kernels, moving-average BN, d loss / d xyz
  training step                    get_model(xyz, True) + cross-entropy + backward, without and with xyz.requires_grad

  python tools/input_grad_timing.py [--model ssg|dgcnn|pointnet] [--batch 32] [--npoints 2048] [--iters 30] [--warmup 10]
"""
from __future__ import annotations

import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scanobjectnn_b200 import dgcnn, pointnet2_cls_ssg, pointnet_cls  # noqa: E402
from scanobjectnn_b200.synthetic import make_clouds  # noqa: E402

MODELS = {"ssg": pointnet2_cls_ssg, "dgcnn": dgcnn, "pointnet": pointnet_cls}


def _time(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=sorted(MODELS), default="ssg")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--npoints", type=int, default=2048)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    B, N = a.batch, a.npoints
    xyz = torch.from_numpy(make_clouds("ball", B, N, seed=7)).cuda()
    labels = torch.arange(B, device="cuda") % 15
    model = MODELS[a.model]
    p_inf = model.init_params(seed=1, randomize_bn=True)
    p_tr = model.init_params(seed=1, randomize_bn=True)
    ce = torch.nn.functional.cross_entropy

    def fused():
        with torch.no_grad():
            model.get_model(xyz, False, params=p_inf)

    def frozen():
        x = xyz.detach().requires_grad_(True)
        logits, _ = model.get_model(x, False, params=p_inf)
        ce(logits, labels).backward()

    def step(want_xyz):
        def run():
            x = xyz.detach().requires_grad_(want_xyz)
            logits, _ = model.get_model(x, True, bn_decay=0.5, params=p_tr)
            ce(logits, labels).backward()
            p_tr._flat.flat.grad = None
        return run

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_properties(0).name
    tag = "" if a.model == "ssg" else f"{a.model}, "          # the default's header is the one DESIGN.md quotes
    print(f"# {card}, {tag}B={B}, N={N}, median of {a.iters} after {a.warmup} warm-up iterations (CUDA events)")
    rows = [("fused inference forward", fused), ("frozen forward + input backward", frozen),
            ("training step, no xyz gradient", step(False)), ("training step, with xyz gradient", step(True))]
    for name, fn in rows:
        print(f"{name:36s} {_time(fn, a.iters, a.warmup):8.3f} ms")


if __name__ == "__main__":
    main()
