"""DGCNN training at B=32, N=2048, k=20: the fused training-mode EdgeConvs (training.edgeconv_training, csrc/edgeconv_train.cu
and csrc/edgeconv2_train.cu) against the materialising composition they replaced in dgcnn.py (group_point -> [x_i, x_j - x_i] ->
mlp_training over B*N*k edge rows -> amax over k), in one process, alternating the two.

  per layer   for each EdgeConv shape of dgcnn1..4 (2C -> C_out = 6 -> 64, 128 -> 64, 128 -> 128) and the T-net's two-layer one
              (6 -> 64 -> 128): forward and forward + backward time (CUDA events, median of repeats after warm-up), the rise of
              torch.cuda.max_memory_allocated over one forward + backward, and the largest output / input-gradient difference
  whole step  dgcnn.get_model(is_training=True) + get_loss + backward, clouds/s; the composition is substituted for every EdgeConv
              (T-net included) inside this script only

Prints the card name and power limit, then one JSON line.  Usage: python tools/dgcnn_train_timing.py [--reps 15] [--steps 10]"""
import argparse
import gc
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from scanobjectnn_b200 import dgcnn, ops
from scanobjectnn_b200.synthetic import make_clouds
from scanobjectnn_b200.tf_util import VariableStore
from scanobjectnn_b200.training import edgeconv_training, mlp_training

B, N, K = 32, 2048, 20
TNET = ("transform_net1/tconv1", "transform_net1/tconv2")
SHAPES = [(("dgcnn1",), 3, [64]), (("dgcnn2",), 64, [64]), (("dgcnn4",), 64, [128]), (TNET, 3, [64, 128])]   # (scopes, C, widths)


def composition(x, idx, scopes, bn_decay, params):
    b, n, c = x.shape
    k = idx.shape[-1]
    scopes = (scopes,) if isinstance(scopes, str) else scopes
    centre = x.unsqueeze(2).expand(b, n, k, c)
    edge = torch.cat([centre, ops.group_point(x.contiguous(), idx) - centre], dim=-1)
    y = mlp_training(edge.reshape(b * n * k, 2 * c), [(s, True) for s in scopes], bn_decay, params)
    return y.view(b, n, k, -1).amax(dim=2)


def fused(x, idx, scopes, bn_decay, params):
    return edgeconv_training(x, idx, scopes[0] if len(scopes) == 1 else scopes, bn_decay, params)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def event_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def per_layer(reps):
    res = {}
    rng = np.random.default_rng(0)
    for scope, c, widths in SHAPES:
        cout = widths[-1]
        x = torch.tensor(rng.standard_normal((B, N, c)).astype(np.float32), device="cuda", requires_grad=True)
        idx = ops.knn_graph(x.detach(), K)
        R = torch.tensor(rng.standard_normal((B, N, cout)).astype(np.float32), device="cuda")
        stores = {}
        for name in ("composition", "fused"):
            stores[name] = VariableStore(device="cuda", seed=1)
            for s_, cin, w_ in zip(scope, [2 * c] + widths[:-1], widths):
                stores[name].add_conv2d(s_, cin, w_, randomize_bn=True)
        paths = {"composition": composition, "fused": fused}

        def fwd(name):
            with torch.no_grad():
                paths[name](x, idx, scope, 0.5, stores[name])

        def fwd_bwd(name):
            p = stores[name]
            out = paths[name](x, idx, scope, 0.5, p)
            return out, torch.autograd.grad(out, [p._flat.flat, x], R)

        outs, mem = {}, {}
        for name in paths:                                        # warm-up (buffers, algorithm choice) + memory + results
            for _ in range(2):
                fwd_bwd(name)
            gc.collect()
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            out, (_, gx) = fwd_bwd(name)
            torch.cuda.synchronize()
            mem[name] = (torch.cuda.max_memory_allocated() - base) / 2**20
            outs[name] = (out.detach().clone(), gx.clone())
            del out, gx
        t = {name: {"fwd": [], "fwd_bwd": []} for name in paths}
        for _ in range(reps):                                     # alternate the two paths
            for name in paths:
                t[name]["fwd"].append(event_ms(lambda: fwd(name)))
                t[name]["fwd_bwd"].append(event_ms(lambda: fwd_bwd(name)))
        rel = lambda a, b: float((a - b).abs().max() / b.abs().max())                     # noqa: E731
        res["->".join(str(v) for v in [2 * c] + widths)] = {
            **{name: {"fwd_ms": float(np.median(t[name]["fwd"])), "fwd_bwd_ms": float(np.median(t[name]["fwd_bwd"])),
                      "peak_alloc_rise_mib": mem[name]} for name in paths},
            "speedup_fwd_bwd": float(np.median(t["composition"]["fwd_bwd"]) / np.median(t["fused"]["fwd_bwd"])),
            "max_rel_diff_out": rel(outs["fused"][0], outs["composition"][0]),
            "max_rel_diff_dx": rel(outs["fused"][1], outs["composition"][1]),
            # points whose dx differs by more than 1e-4 of the largest entry: where the two fp32 evaluations of y_ij round a
            # near-tie of the max differently and so route its gradient to different edges
            "points_dx_diff_over_1e-4": int(((outs["fused"][1] - outs["composition"][1]).abs().amax(-1) > 1e-4 * outs["composition"][1].abs().max()).sum()),
        }
        del stores, outs
        torch.cuda.empty_cache()
    return res


def whole_step(steps):
    xyz = torch.from_numpy(make_clouds("ball", B, N, seed=3)).cuda()
    labels = torch.from_numpy(np.random.default_rng(0).integers(0, 15, B)).cuda()
    fused_edge = dgcnn._edge_conv_training

    def composition_edge(x, k, layers, bn_decay, params, idx=None):
        if idx is None:
            with torch.no_grad():
                idx = ops.knn_graph(x.detach().contiguous(), k)
        return composition(x, idx, tuple(s for s, _ in layers), bn_decay, params), idx

    stores = {name: dgcnn.init_params(seed=2) for name in ("composition", "fused")}
    edge_fns = {"composition": composition_edge, "fused": fused_edge}

    def step(name):
        dgcnn._edge_conv_training = edge_fns[name]
        try:
            p = stores[name]
            logits, ep = dgcnn.get_model(xyz, True, bn_decay=0.5, params=p)
            p._flat.flat.grad = None
            dgcnn.get_loss(logits, labels, ep).backward()
        finally:
            dgcnn._edge_conv_training = fused_edge

    for name in edge_fns:
        for _ in range(3):
            step(name)
    ms = {name: [] for name in edge_fns}
    for _ in range(steps):
        for name in edge_fns:
            ms[name].append(event_ms(lambda: step(name)))
    return {name: {"ms_per_step": float(np.median(v)), "clouds_per_s": B / (float(np.median(v)) * 1e-3)} for name, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    info = card()
    print("card:", info, flush=True)
    out = {"card": info, "B": B, "N": N, "k": K, "per_layer": per_layer(args.reps), "whole_step": whole_step(args.steps)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
