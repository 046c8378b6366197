"""Cost of 3DmFV-Net's fused inference path (mfv_net_cls) against a torch composition of what the reference runs:

  fused     ops.fisher_vector (one fp64 kernel, no (B,N,G,3) tiles), ops.conv3d (tensor cores, taps outside the grid skipped, voxel-major
            rows, branches written in place), ops.pool3d, ops.shared_mlp for the head
  composed  a literal tiled torch transcription of get_3dmfv in fp32 (tf_util.py:578-652), F.conv3d in fp32 with TF32 off plus the
            folded batch norm and ReLU, torch.cat, F.avg_pool3d / F.max_pool3d, ops.shared_mlp for the head

Times are GPU time per call: each side is captured as a CUDA graph and replayed ten times back to back between two CUDA events (no
Python or host enqueue inside the window); the median of --iters such windows, the two sides alternated window by window.

At B in {32, 64} (--batch) on the 5^3 grid: every conv layer (time of each side, with TFLOP/s against
the nominal FLOP 2 B r^3 k^3 C_in C_out and against the in-grid FLOP, which counts only taps inside the grid), the Fisher vector at N in
{1024, 2048} (--npoints), and the whole forward with each side's allocation peak; also the Fisher vector alone on the 8^3 grid.  The
MMAs the tensor-core kernel issues (taps active for some row of a 128-row tile) are printed against the in-grid MACs per layer.
Prints the card's name and power limit, read in the same run.

  python tools/mfv_timing.py [--batch 32 64] [--npoints 1024 2048] [--iters 20] [--warmup 5]
"""
from __future__ import annotations

import argparse
import math
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scanobjectnn_b200 import mfv_net_cls as M  # noqa: E402
from scanobjectnn_b200 import ops  # noqa: E402
from scanobjectnn_b200.synthetic import make_clouds  # noqa: E402


def composed_fv(points, w, mu, sigma):
    """get_3dmfv(flatten=False) with the reference's (B,N,G,D) tiles, fp32 -> (B,G,20)"""
    B, N, D = points.shape
    G = mu.shape[0]
    batch_sig = sigma[None, None].repeat(B, N, 1, 1)
    batch_mu = mu[None, None].repeat(B, N, 1, 1)
    batch_w = w[None, None].repeat(B, N, 1)
    batch_points = points[:, :, None, :].repeat(1, 1, G, 1)
    w_per_batch_per_d = w[None, :, None].repeat(B, 1, 3 * D)
    z = (batch_points - batch_mu) / batch_sig
    p_per_point = torch.exp(-0.5 * (z * z).sum(-1)) / ((2 * math.pi) ** 1.5 * batch_sig.prod(-1))
    w_p = p_per_point * batch_w
    Q = w_p / w_p.sum(-1, keepdim=True).repeat(1, 1, G)
    Q_per_d = Q[..., None].repeat(1, 1, 1, D)
    d_pi_all = ((Q - batch_w) / (torch.sqrt(batch_w) * N))[..., None]
    d_pi = torch.cat([d_pi_all.amax(1), d_pi_all.sum(1)], 2)
    d_mu_all = Q_per_d * (batch_points - batch_mu) / batch_sig
    d_mu = (1 / (N * torch.sqrt(w_per_batch_per_d))) * torch.cat([d_mu_all.amax(1), d_mu_all.amin(1), d_mu_all.sum(1)], 2)
    d_sig_all = Q_per_d * (((batch_points - batch_mu) / batch_sig) ** 2 - 1)
    d_sigma = (1 / (N * torch.sqrt(2 * w_per_batch_per_d))) * torch.cat([d_sig_all.amax(1), d_sig_all.amin(1), d_sig_all.sum(1)], 2)
    out = []
    for v in (d_pi, d_mu, d_sigma):
        v = torch.sign(v) * torch.abs(v) ** 0.5
        out.append(F.normalize(v, dim=1, eps=1e-6))           # v / max(||v||, 1e-6) = v / sqrt(max(sum v^2, 1e-12))
    return torch.cat(out, 2)


class Composed:
    """the torch composition of the network; torch-layout weights prepared once"""

    def __init__(self, params):
        self.p = params
        self.w = {}
        for scope, k, cin, cout in M._module_widths():
            W, sc, sh, _ = params.folded(scope)
            self.w[scope] = (W.reshape(k, k, k, cin, cout).permute(4, 3, 0, 1, 2).contiguous(), sc, sh)
        self.head = params.mlp(["fc1", "fc2", "fc3", "fc4"], [True, True, True, False])

    def conv(self, x, scope):
        W, sc, sh = self.w[scope]
        return torch.relu(F.conv3d(x, W, padding=W.shape[-1] // 2) * sc[None, :, None, None, None] + sh[None, :, None, None, None])

    def inception(self, x, scope):
        one = self.conv(x, f"{scope}_conv1")
        avg = F.avg_pool3d(x, 3, stride=1, padding=1, count_include_pad=False)
        return torch.cat([one, self.conv(one, f"{scope}_conv2"), self.conv(one, f"{scope}_conv3"), self.conv(avg, f"{scope}_conv4")], 1)

    def forward(self, points, w, mu, sigma):
        fv = composed_fv(points, w, mu, sigma)
        b, g, _ = fv.shape
        r = round(g ** (1 / 3))
        net = fv.permute(0, 2, 1).reshape(b, 20, r, r, r)
        for l in (1, 2, 3):
            net = self.inception(net, f"inception{l}")
        net = F.max_pool3d(net, 2, 2, ceil_mode=True)
        for l in (4, 5):
            net = self.inception(net, f"inception{l}")
        net = F.max_pool3d(net, 2, 2, ceil_mode=True)
        return ops.shared_mlp(net.permute(0, 2, 3, 4, 1).reshape(b, -1).contiguous(), self.head)


def in_grid_taps(r, k):
    """sum over the r^3 voxels of the taps of a k^3 kernel that land inside the grid"""
    h = k // 2
    per_axis = sum(min(r - 1, i + h) - max(0, i - h) + 1 for i in range(r))
    return per_axis ** 3


def issued_taps(b, r, k):
    """sum over 128-row tiles (voxel-major rows) of 128 x the taps active for some row of the tile (the tensor-core kernel's rule)"""
    rows, h, total = b * r ** 3, k // 2, 0
    for t0 in range(0, rows, 128):
        vox = range(t0 // b, (min(rows, t0 + 128) - 1) // b + 1)
        cells = [(v // (r * r), v // r % r, v % r) for v in vox]
        act = sum(1 for dz in range(-h, h + 1) for dy in range(-h, h + 1) for dx in range(-h, h + 1)
                  if any(0 <= z + dz < r and 0 <= y + dy < r and 0 <= x + dx < r for z, y, x in cells))
        total += 128 * act
    return total


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
    """GPU time per call of each side, in ms: each side is replayed as a CUDA graph, `reps` replays back to back between two
    events, so the window holds the launches' GPU time and the gaps between them but no Python or host enqueue; median of
    `iters` windows, the two sides alternated window by window"""
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
    ap.add_argument("--batch", type=int, nargs="+", default=[32, 64])
    ap.add_argument("--npoints", type=int, nargs="+", default=[1024, 2048])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mfv_timing: no CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_properties(0).name
    print(f"# {card}; GPU time per call: CUDA-graph replay, 10 replays between CUDA events, median of {a.iters} windows after "
          f"{a.warmup} warm-up replays, fused and composed alternated window by window")
    p = M.init_params(seed=1, randomize_bn=True)
    comp = Composed(p)
    gmm = [torch.from_numpy(t).cuda() for t in M.get_3d_grid_gmm((5, 5, 5))]
    with torch.no_grad():
        for B in a.batch:
            gen = torch.Generator(device="cuda").manual_seed(B)
            for scope, k, cin, cout in M._module_widths():
                r = 3 if scope.startswith(("inception4", "inception5")) else 5
                xin = torch.relu(torch.randn((B * r ** 3, cin), generator=gen, device="cuda"))
                W, sc, sh, _ = p.folded(scope)
                xg = xin.reshape(r ** 3, B, cin).permute(1, 2, 0).reshape(B, cin, r, r, r).contiguous()
                fused = lambda: ops.conv3d(xin, r, W, sc, sh)
                tcomp = lambda: comp.conv(xg, scope)
                mf, mc = _time_pair(fused, tcomp, a.iters, a.warmup)
                nominal = 2.0 * B * r ** 3 * k ** 3 * cin * cout
                ingrid = 2.0 * B * in_grid_taps(r, k) * cin * cout
                issued = issued_taps(B, r, k) / (B * in_grid_taps(r, k))
                print(f"B={B} {scope:<17} r={r} k={k} {cin:>3}->{cout:<3} fused {mf * 1e3:8.1f} us "
                      f"({nominal / mf / 1e9:6.1f} nominal / {ingrid / mf / 1e9:6.1f} in-grid TFLOP/s)  composed {mc * 1e3:8.1f} us "
                      f"({nominal / mc / 1e9:6.1f} / {ingrid / mc / 1e9:6.1f})  issued/in-grid MACs {issued:.2f}")
            for N in a.npoints:
                pts = torch.from_numpy(make_clouds("ball", B, N, seed=7)).cuda()
                mf, mc = _time_pair(lambda: ops.fisher_vector(pts, *gmm), lambda: composed_fv(pts, *gmm), a.iters, a.warmup)
                pf, fv = peak(lambda: ops.fisher_vector(pts, *gmm))
                pc, fvc = peak(lambda: composed_fv(pts, *gmm))
                print(f"B={B} N={N} fisher_vector G=125  fused {mf * 1e3:8.1f} us (peak {pf / 2**20:7.1f} MiB)  composed {mc * 1e3:8.1f} us "
                      f"(peak {pc / 2**20:8.1f} MiB)  max|diff| {float((fv - fvc).abs().max()):.2e}")
                fwd = lambda: M.get_model(pts, *gmm, False, params=p)[0]
                cfw = lambda: comp.forward(pts, *gmm)
                mf, mc = _time_pair(fwd, cfw, a.iters, a.warmup)
                pf, lf = peak(fwd)
                pc, lc = peak(cfw)
                print(f"B={B} N={N} forward  fused {mf:7.3f} ms ({B / mf * 1e3:7.0f} clouds/s, peak {pf / 2**20:7.1f} MiB)  composed {mc:7.3f} ms "
                      f"({B / mc * 1e3:7.0f} clouds/s, peak {pc / 2**20:8.1f} MiB)  max|dlogits| {float((lf - lc).abs().max()):.2e}")
        gmm8 = [torch.from_numpy(t).cuda() for t in M.get_3d_grid_gmm((8, 8, 8))]
        for B in a.batch:
            for N in a.npoints:
                pts = torch.from_numpy(make_clouds("ball", B, N, seed=8)).cuda()
                mf, mc = _time_pair(lambda: ops.fisher_vector(pts, *gmm8), lambda: composed_fv(pts, *gmm8), a.iters, a.warmup)
                pc, _ = peak(lambda: composed_fv(pts, *gmm8))
                print(f"B={B} N={N} fisher_vector G=512  fused {mf * 1e3:8.1f} us  composed {mc * 1e3:8.1f} us (peak {pc / 2**20:8.1f} MiB)")


if __name__ == "__main__":
    main()
