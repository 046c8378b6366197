"""Cost of PointCNN's fused inference path (pointcnn_cls) against a materialising torch composition of what the reference runs:

  fused     ops.knn_dilated (no distance matrix), ops.xconv_core (everything up to the depthwise stage per query tile; only the
            (B*P, C_in*dm) depthwise output reaches memory), ops.dense_elu_affine (tensor cores, ELU / batch-norm epilogue, slices of
            the 480-wide row written in place), ops.pool_rows and ops.shared_mlp for the mean and the logits
  composed  the expanded (B,P,N) distance matrix by torch.bmm, torch.topk, gathers of the (B,P,K,3) and (B,P,K,C_prev) neighbour
            tensors, F.conv2d for the lifting, X_0 and the pointwise convs, F.conv2d with groups= for X_1, X_2 and the depthwise stage,
            torch.matmul for X . F, torch.cat, all fp32 with TF32 off

Times are GPU time per call: each side is captured as a CUDA graph and replayed ten times back to back between two CUDA events; the
median of --iters such windows, the two sides alternated window by window.  Per X-Conv layer (on the same input features), for each
dense GEMM of the model alone (TFLOP/s from 2 rows K N), and for the whole forward with each side's allocation peak on an eager call.
Prints the card's name, power limit and max SM clock, read in the same run.

  python tools/pointcnn_timing.py [--batch 32] [--npoints 1024 2048] [--iters 20] [--warmup 5]
"""
from __future__ import annotations

import argparse
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scanobjectnn_b200 import ops  # noqa: E402
from scanobjectnn_b200 import pointcnn_cls as M  # noqa: E402
from scanobjectnn_b200.synthetic import make_clouds  # noqa: E402


class Composed:
    """the reference's layer in torch, NCHW with the neighbour axis as the width; weights in torch layouts prepared once"""

    def __init__(self, p):
        self.p = p

    def aff(self, layer, y, dim=1):
        s, t = self.p.elu_bn(layer)
        shape = [1] * y.dim()
        shape[dim] = -1
        return F.elu(y) * s.view(shape) + t.view(shape)

    def pw(self, x, layer, var="kernel", act=True):
        """1x1 conv on NCHW x, ELU (unless act=False), batch norm"""
        w = self.p[f"{layer}/{var}"]
        y = F.conv2d(x, w.reshape(-1, w.shape[-1]).t()[:, :, None, None])
        if act:
            return self.aff(layer, y)
        s, t = self.p.elu_bn(layer)
        return y * s.view(1, -1, 1, 1) + t.view(1, -1, 1, 1)

    def knn(self, pts, qrs, k, d):
        D = (qrs * qrs).sum(-1, keepdim=True) - 2 * torch.bmm(qrs, pts.transpose(1, 2)) + (pts * pts).sum(-1)[:, None, :]
        return torch.topk(-D, k * d, dim=-1, sorted=True)[1][:, :, ::d]

    def xconv(self, tag, k, d, dm, glob, pts, qrs, fts):
        B, P = qrs.shape[:2]
        idx = self.knn(pts, qrs, k, d)
        bi = torch.arange(B, device=pts.device)[:, None, None]
        local = (pts[bi, idx] - qrs[:, :, None, :]).permute(0, 3, 1, 2).contiguous()            # (B,3,P,K)
        lifted = self.pw(self.pw(local, f"{tag}nn_fts_from_pts_0"), f"{tag}nn_fts_from_pts")
        Fin = lifted if fts is None else torch.cat([lifted, fts[bi, idx].permute(0, 3, 1, 2)], 1)
        X0 = self.aff(f"{tag}X_0", F.conv2d(local, self.p[f"{tag}X_0/kernel"].permute(3, 2, 0, 1)))   # (B,K*K,P,1)
        X = X0[..., 0].permute(0, 2, 1).reshape(B, P, k, k)
        for name, act in (("X_1", True), ("X_2", False)):
            w = self.p[f"{tag}{name}/depthwise_weights"].permute(2, 3, 0, 1).reshape(k * k, 1, 1, k)
            y = F.conv2d(X.permute(0, 3, 1, 2), w, groups=k)                                      # (B,K*K,P,1)
            if act:
                y = self.aff(f"{tag}{name}", y)
            else:
                s, t = self.p.elu_bn(f"{tag}{name}")
                y = y * s.view(1, -1, 1, 1) + t.view(1, -1, 1, 1)
            X = y[..., 0].permute(0, 2, 1).reshape(B, P, k, k)
        fts_X = torch.matmul(X, Fin.permute(0, 2, 3, 1))                                          # (B,P,K,C_in)
        cin = fts_X.shape[-1]
        wdw = self.p[f"{tag}fts_conv/depthwise_kernel"].permute(2, 3, 0, 1).reshape(cin * dm, 1, 1, k)
        dw = F.conv2d(fts_X.permute(0, 3, 1, 2), wdw, groups=cin)                                  # (B,C_in*dm,P,1)
        out = self.pw(dw, f"{tag}fts_conv", "pointwise_kernel")
        if glob:
            g = self.pw(self.pw(qrs.permute(0, 2, 1)[..., None], f"{tag}fts_global_0"), f"{tag}fts_global")
            out = torch.cat([g, out], 1)
        return out[..., 0].permute(0, 2, 1)                                                       # (B,P,C)

    def forward(self, points):
        n = points.shape[1]
        pts, fts = points, None
        for tag, k, d, P, _, _, _, dm, glob in M.layer_table():
            P = n if P == -1 else P
            qrs = pts[:, :P]
            fts, pts = self.xconv(tag, k, d, dm, glob, pts, qrs, fts), qrs
        net = fts
        for i in range(len(M.FC)):
            net = self.aff(f"fc{i}", net @ self.p[f"fc{i}/kernel"], dim=-1)
        return net.mean(1, keepdim=True) @ self.p["logits/kernel"] + self.p["logits/bias"]


def fused_layer(p, l, pts, qrs, fts):
    """one X-Conv layer of pointcnn_cls.get_model: kNN, core, the global branch and the pointwise GEMM"""
    tag, k, d, _, c, _, _, dm, glob = M.layer_table()[l]
    b, P = qrs.shape[:2]
    idx = ops.knn_dilated(pts, qrs, k, d)
    dw = ops.xconv_core(pts, qrs, idx, fts, M.xconv_weights(p, tag), dm)
    out = torch.empty((b * P, glob + c), dtype=torch.float32, device=pts.device)
    if glob:
        g0 = M._dense(p, f"{tag}fts_global_0", "kernel", qrs.reshape(b * P, 3))
        M._dense(p, f"{tag}fts_global", "kernel", g0, out=out, offset=0)
    M._dense(p, f"{tag}fts_conv", "pointwise_kernel", dw, out=out, offset=glob)
    return out.view(b, P, -1)


def _graph(fn):
    """fn captured as a CUDA graph (after two eager calls on a side stream, which also fill the weight caches)"""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn(); fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def _time_pair(fa, fb, iters, warmup, reps=10):
    """GPU time per call of each side in ms: CUDA-graph replays, `reps` back to back between two events, median of `iters` windows,
    the two sides alternated window by window"""
    ga, gb = _graph(fa), _graph(fb)
    for _ in range(warmup):
        ga.replay(); gb.replay()
    ta, tb = [], []
    for _ in range(iters):
        for g, ts in ((ga, ta), (gb, tb)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                g.replay()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) / reps)
    del ga, gb
    return statistics.median(ta), statistics.median(tb)


def peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[32])
    ap.add_argument("--npoints", type=int, nargs="+", default=[1024, 2048])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pointcnn_timing: no CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_properties(0).name
    print(f"# {card}; GPU time per call: CUDA-graph replay, 10 replays between CUDA events, median of {a.iters} windows after "
          f"{a.warmup} warm-up replays, fused and composed alternated window by window; fp32, TF32 off")
    p = M.init_params(seed=1, randomize_bn=True)
    comp = Composed(p)
    with torch.no_grad():
        for B in a.batch:
            for N in a.npoints:
                x = torch.from_numpy(make_clouds("ball", B, N, seed=N)).cuda()
                _, ep = M.get_model(x, False, params=p, return_end_points=True)
                pts, fts = x, None
                for l, (tag, k, d, P, c, _, _, dm, glob) in enumerate(M.layer_table()):
                    P = N if P == -1 else P
                    qrs = x[:, :P].contiguous()
                    mf, mc = _time_pair(lambda: fused_layer(p, l, pts, qrs, fts), lambda: comp.xconv(tag, k, d, dm, glob, pts, qrs, fts),
                                        a.iters, a.warmup)
                    pf, yf = peak(lambda: fused_layer(p, l, pts, qrs, fts))
                    pc, yc = peak(lambda: comp.xconv(tag, k, d, dm, glob, pts, qrs, fts))
                    print(f"B={B} N={N} xconv_{l + 1} K={k} D={d} P={P} C={c}  fused {mf * 1e3:8.1f} us (peak {pf / 2**20:7.1f} MiB)  "
                          f"composed {mc * 1e3:8.1f} us (peak {pc / 2**20:8.1f} MiB)  max|diff| {float((yf - yc).abs().max()):.2e}")
                    pts, fts = qrs, ep[f"fts{l + 1}"]
                gemms = []
                for l, (tag, _, _, P, c, c_pts, c_prev, dm, glob) in enumerate(M.layer_table()):
                    P = N if P == -1 else P
                    gemms.append((f"xconv_{l + 1} pointwise", f"{tag}fts_conv", "pointwise_kernel", B * P, (c_pts + c_prev) * dm, c))
                    if glob:
                        gemms.append(("xconv_4 global", f"{tag}fts_global", "kernel", B * P, glob, glob))
                cin = ep["fts4"].shape[-1]
                for i, c in enumerate(M.FC):
                    gemms.append((f"fc{i}", f"fc{i}", "kernel", B * 128, cin, c))
                    cin = c
                gen = torch.Generator(device="cuda").manual_seed(N)
                for name, layer, var, rows, K, Nc in gemms:
                    xin = torch.randn((rows, K), generator=gen, device="cuda")
                    w = p[f"{layer}/{var}"].reshape(K, Nc)
                    s, t = p.elu_bn(layer)
                    mf, mc = _time_pair(lambda: ops.dense_elu_affine(xin, w, s, t), lambda: F.elu(xin @ w) * s + t, a.iters, a.warmup)
                    fl = 2.0 * rows * K * Nc
                    print(f"B={B} N={N} gemm {name:<20} {rows:>6} x {K:>3} -> {Nc:<3} fused {mf * 1e3:7.1f} us ({fl / mf / 1e9:6.1f} TFLOP/s)  "
                          f"composed {mc * 1e3:7.1f} us ({fl / mc / 1e9:6.1f} TFLOP/s)")
                fwd = lambda: M.get_model(x, False, params=p)
                cfw = lambda: comp.forward(x)
                mf, mc = _time_pair(fwd, cfw, a.iters, a.warmup)
                pf, lf = peak(fwd)
                pc, lc = peak(cfw)
                print(f"B={B} N={N} forward  fused {mf:7.3f} ms ({B / mf * 1e3:7.0f} clouds/s, peak {pf / 2**20:7.1f} MiB)  composed {mc:7.3f} ms "
                      f"({B / mc * 1e3:7.0f} clouds/s, peak {pc / 2**20:8.1f} MiB)  max|dlogits| {float((lf - lc).abs().max()):.2e}")


if __name__ == "__main__":
    main()
