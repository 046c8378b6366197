"""Cost of SpiderCNN's fused spiderConv layers (spidercnn_cls_xyz) against the materialising composition the reference runs, at
B=32 and N in {1024, 2048}, k=20, T=5:

  fused     ops.spider_conv (the product A[p][(j,t,c)] = h[nn(p,j)][c] g_t(delta_pj) is gathered and scaled inside the GEMM)
            + ops.group_norm_affine
  composed  group_point of the activated features, the Taylor filter and the (B,N,k,C,T) product in torch, the [1,k] conv as an fp32
            matmul (TF32 off), torch group_norm + ReLU

Per layer: the median time of each (CUDA events, the two alternated call by call), the fused layer's achieved FLOP/s with FLOPs
from shapes (2 B N k C_in T C_out), each side's allocation peak above what was allocated before it, and the largest difference of
the pre-norm outputs relative to their largest magnitude.  Also the whole inference forward.  Prints the card's name and power
limit, read in the same run.

  python tools/spidercnn_timing.py [--batch 32] [--npoints 1024 2048] [--iters 20] [--warmup 5]
"""
from __future__ import annotations

import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scanobjectnn_b200 import ops  # noqa: E402
from scanobjectnn_b200 import spidercnn_cls_xyz as M  # noqa: E402
from scanobjectnn_b200.synthetic import make_clouds  # noqa: E402
from scanobjectnn_b200.tf_util import GN_EPS  # noqa: E402


def _taylor_filter(delta, taylor):
    X, Y, Z = (delta[..., i:i + 1] for i in range(3))
    mono = [X, Y, Z, X * Y * Z, X * Y, Y * Z, X * Z, torch.ones_like(X), X * X, Y * Y, Z * Z, X * X * Y, X * Y * Y, X * X * Z, X * Z * Z,
            Y * Y * Z, Y * Z * Z, X * X * X, Y * Y * Y, Z * Z * Z]
    return sum(m * taylor[i] for i, m in enumerate(mono))                          # (B,N,k,T)


def _composed(delta, idx, feat, s, u, taylor, w, bias, gamma, beta, groups):
    h = feat if s is None else torch.relu(feat * s[:, None, :] + u[:, None, :])
    grouped = ops.group_point(h.contiguous(), idx)                                  # (B,N,k,C)
    b, n, k, c = grouped.shape
    g = _taylor_filter(delta, taylor)
    prod = (grouped.unsqueeze(-1) * g.unsqueeze(3)).reshape(b * n, k * c * taylor.shape[1])
    y = (prod @ w.reshape(-1, w.shape[-1]) + bias).reshape(b, n, -1)
    out = torch.relu(torch.nn.functional.group_norm(y.permute(0, 2, 1), groups, gamma, beta, GN_EPS).permute(0, 2, 1))
    return y, out


def _time(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return ts


def _peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--npoints", type=int, nargs="+", default=[1024, 2048])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spidercnn_timing: no CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_properties(0).name
    print(f"# {card}, B={a.batch}, median of {a.iters} after {a.warmup} warm-up iterations (CUDA events), fused and composed alternated")
    B = a.batch
    p = M.init_params(seed=1, randomize_bn=True)
    with torch.no_grad():
        for N in a.npoints:
            xyz = torch.from_numpy(make_clouds("ball", B, N, seed=7)).cuda()
            _, ep = M.get_model(xyz, False, params=p, return_end_points=True)
            idx = ep["idx"]
            delta = (ops.group_point(xyz, idx) - xyz.unsqueeze(2)).contiguous()
            feat, s, u = xyz, None, None
            cin = 3
            for l, cout in enumerate(M.CHANNELS, start=1):
                taylor, w, bias, gamma, beta = p.spider(f"fanConv{l}/taylor")
                groups = min(M.GROUPS, cout)
                args = (delta, idx, feat, s, u)
                fused = lambda: ops.spider_conv(delta, idx, args[2], taylor, w, bias, args[3], args[4])
                comp = lambda: _composed(*args, taylor, w, bias, gamma, beta, groups)
                tf, tc = [], []
                for _ in range(a.warmup):
                    fused(); comp()
                for _ in range(a.iters):
                    tf += _time(fused, 1, 0)
                    tc += _time(comp, 1, 0)
                mf, y = _peak(fused)
                mc, (yc, _) = _peak(comp)
                diff = float((y - yc).abs().max() / yc.abs().max())
                flops = 2.0 * B * N * M.NSAMPLE * cin * M.TAYLOR_CHANNEL * cout
                med_f, med_c = statistics.median(tf), statistics.median(tc)
                print(f"N={N} fanConv{l} {cin:>3}->{cout:<3}  fused {med_f:8.3f} ms ({flops / med_f / 1e9:7.1f} TFLOP/s, peak {mf / 2**20:7.1f} MiB)"
                      f"  composed {med_c:8.3f} ms (peak {mc / 2**20:8.1f} MiB)  max|dy|/max|y| = {diff:.2e}")
                sc, sh = ops.group_norm_affine(y, gamma, beta, groups, GN_EPS)
                feat, s, u, cin = y, sc, sh, cout
            fwd = lambda: M.get_model(xyz, False, params=p)
            t = _time(fwd, a.iters, a.warmup)
            mpk, _ = _peak(fwd)
            print(f"N={N} forward  {statistics.median(t):8.3f} ms  ({B / statistics.median(t) * 1e3:8.0f} clouds/s, peak {mpk / 2**20:.1f} MiB)")


if __name__ == "__main__":
    main()
