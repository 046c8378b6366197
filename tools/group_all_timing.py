"""Where the time of the group-all cluster kernel (tc_group_all_kernel) goes, at SSG's SA3 shape: c = 256, mlp [256, 512, 1024],
128 points per cloud.

  level    the whole group-all level (memset, cluster kernel, no-op bf16x3 reruns) captured as a CUDA graph of ten calls and
           replayed between two CUDA events; the median of --iters windows, per call
  kernel   tc_group_all_kernel alone, mean over --iters * 10 launches in a torch.profiler run of its own
  stamps   one launch of a separate build of libpsa.so with -DPSA_GA_STAMPS (compiled into a temporary directory; the library
           the package loads has no stamps): thread 0 of every consumer warpgroup records clock64() per K block when the weight
           block is ready, when the group is issued, when the next K block's A operand is in registers and when the group has
           retired.  Printed per layer as the mean over CTAs and warpgroups, in SM cycles.

At b = 32 the level needs more clusters than fit at once (DESIGN.md §3.3); b = 30 runs inside one wave.  Prints the card's name,
power limit and max SM clock, read in the same run.

  python tools/group_all_timing.py [--batch 30 32] [--iters 20] [--no-stamps]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N, CIN, MLP = 128, 256, [256, 512, 1024]
STAMP_CTAS, STAMP_USES = 256, 64          # kGaStampCtas, kGaStampUses in csrc/tc_mlp.cu


def level(b, seed=5):
    from scanobjectnn_b200.pointnet_util import add_sa_module_params, pointnet_sa_module
    from scanobjectnn_b200.synthetic import make_clouds
    from scanobjectnn_b200.tf_util import VariableStore
    p = VariableStore(device="cuda", seed=seed)
    add_sa_module_params(p, "sa", 3 + CIN, MLP, randomize_bn=True)
    xyz = torch.from_numpy(make_clouds("ball", b, N, seed=seed)).cuda()
    rng = np.random.default_rng(seed)
    pts = torch.from_numpy(np.maximum(rng.standard_normal((b, N, CIN)), 0.0).astype(np.float32)).cuda()
    return lambda: pointnet_sa_module(xyz, pts, None, None, None, MLP, None, True, False, None, "sa", params=p)[1]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or "nvidia-smi unavailable"


def time_level(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        fn()
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            for _ in range(10):
                fn()
    torch.cuda.synchronize()
    g.replay()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    out = []
    for _ in range(iters):
        ev[0].record()
        g.replay()
        ev[1].record()
        ev[1].synchronize()
        out.append(ev[0].elapsed_time(ev[1]) * 1e3 / 10)
    return statistics.median(out)


def time_kernel(fn, iters):
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters * 10):
            fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if "tc_group_all_kernel" in e.key]
    if not ev:
        raise RuntimeError("tc_group_all_kernel did not run (the level is not eligible for the cluster kernel)")
    attr = "device_time" if hasattr(ev[0], "device_time") else "cuda_time"
    return sum(getattr(e, attr) * e.count for e in ev) / sum(e.count for e in ev)


def build_stamped(tmp):
    """libpsa.so with tc_mlp.cu compiled with -DPSA_GA_STAMPS, in `tmp`"""
    from scanobjectnn_b200 import build
    build.build_library()
    obj = os.path.join(tmp, "tc_mlp.o")
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-DPSA_GA_STAMPS", "-c", os.path.join(build.CSRC, "tc_mlp.cu"), "-o", obj]
    subprocess.run(cmd, check=True)
    objs = [os.path.join(build.OBJDIR, f) for f in sorted(os.listdir(build.OBJDIR)) if f.endswith(".o") and f != "tc_mlp.o"]
    lib = os.path.join(tmp, "libpsa.so")
    subprocess.run([build._nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", lib, obj, *objs, "-lcudart"], check=True)
    return lib


def stamps_child(lib_path, b):
    """runs in a process of its own, on the stamped library"""
    from scanobjectnn_b200 import _lib
    _lib.LIB_PATH = lib_path
    lib = _lib.load()
    fn = level(b)
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    buf = np.zeros((STAMP_CTAS, 2, STAMP_USES, 4), np.int64)
    fn()
    torch.cuda.synchronize()
    assert lib.psa_group_all_stamps(buf.ctypes.data_as(C.c_void_p)) == 0
    kc = [CIN // 64, MLP[0] // 64, MLP[1] // 64]
    passes = [1, 1, MLP[2] // 4 // 128]
    bounds, u = [], 0
    for l in range(3):
        bounds.append((u, u + kc[l] * passes[l]))
        u += kc[l] * passes[l]
    st = buf[: 4 * b]                                     # (cta, wg, use, 4)
    start = st[:, :, STAMP_USES - 1, 0]
    res = {"b": b, "uses": u, "cycles_total": float(np.mean(st[:, :, u - 1, 3] - start))}
    for l, (u0, u1) in enumerate(bounds):
        w, i, a, r = (st[:, :, u0:u1, k].astype(np.float64) for k in range(4))
        prev_r = np.concatenate([st[:, :, u0 - 1: u0, 3] if u0 else start[:, :, None], st[:, :, u0:u1 - 1, 3]], axis=2)
        res[f"layer{l}"] = {
            "blocks": u1 - u0,
            "step": float(np.mean(r - prev_r)),                 # retire to retire
            "weight_wait": float(np.mean(w - prev_r)),          # previous retire (or layer start) to weight block ready
            "issue": float(np.mean(i - w)),                     # weight ready to group committed
            "a_next": float(np.mean(a[:, :, :-1] - i[:, :, :-1])) if u1 - u0 > 1 else 0.0,   # committed to next A in registers
            "tail": float(np.mean(r - np.maximum(a, i))),       # from there to retired
            "first_block_wait": float(np.mean(w[:, :, 0] - prev_r[:, :, 0])),   # epilogue + cross-CTA handshake + weights
        }
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[30, 32])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--no-stamps", action="store_true")
    ap.add_argument("--stamped-lib", help="a stamped libpsa.so built earlier (default: build one into a temporary directory)")
    ap.add_argument("--stamps-child", nargs=2, metavar=("LIB", "B"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.stamps_child:
        stamps_child(args.stamps_child[0], int(args.stamps_child[1]))
        return
    assert torch.cuda.is_available(), "group_all_timing needs a GPU"
    print(f"card: {card()}")
    for b in args.batch:
        fn = level(b)
        lv = time_level(fn, args.iters)
        kt = time_kernel(fn, args.iters)
        print(json.dumps({"b": b, "level_us": round(lv, 2), "kernel_us": round(kt, 2)}))
    if args.no_stamps:
        return
    with tempfile.TemporaryDirectory() as tmp:
        lib = args.stamped_lib or build_stamped(tmp)
        for b in args.batch:
            subprocess.run([sys.executable, os.path.abspath(__file__), "--stamps-child", lib, str(b)], check=True)


if __name__ == "__main__":
    main()
