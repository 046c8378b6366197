"""Where the time of the set-abstraction kernel (tc_sa_kernel) goes, at PointNet++ SSG's SA1 and SA2 shapes (B = 32, N = 2048):
SA1 = 2048 -> 512 centres, 32 neighbours, mlp [64, 64, 128], no input features; SA2 = 512 -> 128 centres, 64 neighbours,
mlp [128, 128, 256] over 128 features (SA1's output).  The ball queries are computed once; only the MLP part of a level is timed.

  kernel   tc_sa_kernel (fp16x2) alone, mean over --iters launches in a torch.profiler run of its own
  stamps   one launch of a separate build of libpsa.so with -DPSA_SA_STAMPS (compiled into a temporary directory; the library
           the package loads has no stamps): lane 0 of the first warp of every warpgroup records clock64() at the phase
           boundaries of each 64-row pass (pass top; layer 1's gathered inputs in registers; layer 1 built; layer 2 issued,
           retired, epilogue done; each last-layer chunk issued, retired, epilogue done; in a pass that ends a chunk of
           neighbourhoods, both barriers of its store passed; the next pass's gather stages A and B issued).  Printed as the
           mean cycles from one phase to the next, in the order the phases run, over every pass of every warpgroup that
           reached the phase, in SM cycles; then the same apart for the passes that end a chunk and for those that do not.
           The stamps add global stores and registers of their own (the stamped build spills a few words), so the table is
           a breakdown of a pass, not its exact length in libpsa.so.

Prints the card's name, power limit and max SM clock, read in the same run.

  python tools/sa_timing.py [--levels sa1 sa2] [--iters 50] [--no-stamps]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, N = 32, 2048
STAMP_CTAS, STAMP_PASSES = 264, 64        # kSaStampCtas, kSaStampPasses in csrc/tc_mlp.cu
PHASES = ["top", "inputs landed", "layer 1 built", "layer 2 issued", "layer 2 retired", "layer 2 epilogue",
          "chunk end barrier 1", "chunk end barrier 2", "next stage A issued", "next stage B issued"]
CHUNKS = 4
NPHASE = len(PHASES) + 3 * CHUNKS         # kSaStampPhases


def phase_names():
    names = list(PHASES)
    for nc in range(CHUNKS):
        names += [f"chunk {nc} issued", f"chunk {nc} retired", f"chunk {nc} epilogue"]
    return names


def levels(seed=1001):
    from scanobjectnn_b200 import ops, pointnet2_cls_ssg
    from scanobjectnn_b200.synthetic import make_clouds
    p = pointnet2_cls_ssg.init_params(seed=1, randomize_bn=True)
    x = torch.from_numpy(make_clouds("ball", B, N, seed=seed)).cuda()
    mlp1 = p.mlp([f"layer1/conv{i}" for i in range(3)])
    mlp2 = p.mlp([f"layer2/conv{i}" for i in range(3)])
    _, l1_xyz = ops.farthest_point_sample_and_gather(512, x)
    l1_pts, idx1, _ = ops.sa_module_infer(x, l1_xyz, None, 0.2, 32, mlp1, return_idx=True)
    _, l2_xyz = ops.farthest_point_sample_and_gather(128, l1_xyz)
    _, idx2, _ = ops.sa_module_infer(l1_xyz, l2_xyz, l1_pts, 0.4, 64, mlp2, return_idx=True)
    return {"sa1": lambda: ops.sa_module_infer(x, l1_xyz, None, 0.2, 32, mlp1, idx=idx1),
            "sa2": lambda: ops.sa_module_infer(l1_xyz, l2_xyz, l1_pts, 0.4, 64, mlp2, idx=idx2)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or "nvidia-smi unavailable"


def time_kernel(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if "tc_sa_kernel<2" in e.key]
    if not ev:
        raise RuntimeError("tc_sa_kernel<2, ..> did not run (the level is not on the fp16x2 set-abstraction kernel)")
    attr = "device_time" if hasattr(ev[0], "device_time") else "cuda_time"
    return sum(getattr(e, attr) * e.count for e in ev) / sum(e.count for e in ev)


def build_stamped(tmp):
    """libpsa.so with tc_mlp.cu compiled with -DPSA_SA_STAMPS, in `tmp`"""
    from scanobjectnn_b200 import build
    build.build_library()
    obj = os.path.join(tmp, "tc_mlp.o")
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-DPSA_SA_STAMPS", "-c", os.path.join(build.CSRC, "tc_mlp.cu"), "-o", obj]
    subprocess.run(cmd, check=True)
    objs = [os.path.join(build.OBJDIR, f) for f in sorted(os.listdir(build.OBJDIR)) if f.endswith(".o") and f != "tc_mlp.o"]
    lib = os.path.join(tmp, "libpsa.so")
    subprocess.run([build._nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", lib, obj, *objs, "-lcudart"], check=True)
    return lib


def table(st, top, rel, passes):
    """the mean cycles from one phase to the next over the passes selected by `passes`, in the order the phases run"""
    names = phase_names()
    mean = {}
    for k in range(1, NPHASE):
        ok = passes & (st[:, :-1, k] > 0)
        if ok.sum() > 0:
            mean[names[k]] = float(rel[:, :, k][ok].mean())
    rows, prev, prev_t = [], "top", 0.0
    for n in sorted(mean, key=mean.get):
        rows.append({"phase": f"{prev} -> {n}", "cycles": round(mean[n] - prev_t, 1)})
        prev, prev_t = n, mean[n]
    length = float((top[:, 1:] - top[:, :-1])[passes].mean())
    rows.append({"phase": f"{prev} -> next top", "cycles": round(length - prev_t, 1)})
    return {"passes": int(passes.sum()), "pass_cycles": round(length, 1), "phases": rows}


def summarise(st):
    """st: (ctas, 2, passes, phases) clock64 stamps, 0 where a pass did not reach a phase -> per-phase means over every pass,
    and apart over the passes that end a chunk of neighbourhoods and those that do not"""
    st = st.reshape(-1, STAMP_PASSES, NPHASE).astype(np.float64)
    top = st[:, :, 0]
    done = (top[:, :-1] > 0) & (top[:, 1:] > 0)            # passes followed by another: their length is known
    rel = st[:, :-1, :] - top[:, :-1, None]
    ends = done & (st[:, :-1, PHASES.index("chunk end barrier 1")] > 0)
    out = table(st, top, rel, done)
    for name, m in (("chunk_end", ends), ("inside_chunk", done & ~ends)):
        if m.any():
            out[name] = table(st, top, rel, m)
    return out


def stamps_child(lib_path, name):
    """runs in a process of its own, on the stamped library"""
    from scanobjectnn_b200 import _lib
    _lib.LIB_PATH = lib_path
    lib = _lib.load()
    fn = levels()[name]
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    assert lib.psa_sa_stamps_clear() == 0
    fn()
    torch.cuda.synchronize()
    buf = np.zeros((STAMP_CTAS, 2, STAMP_PASSES, NPHASE), np.int64)
    assert lib.psa_sa_stamps(buf.ctypes.data_as(C.c_void_p)) == 0
    print(json.dumps({"level": name, **summarise(buf)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", nargs="+", default=["sa1", "sa2"], choices=["sa1", "sa2"])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--no-stamps", action="store_true")
    ap.add_argument("--stamped-lib", help="a stamped libpsa.so built earlier (default: build one into a temporary directory)")
    ap.add_argument("--stamps-child", nargs=2, metavar=("LIB", "LEVEL"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.stamps_child:
        stamps_child(*args.stamps_child)
        return
    assert torch.cuda.is_available(), "sa_timing needs a GPU"
    print(f"card: {card()}")
    fns = levels()
    for name in args.levels:
        print(json.dumps({"level": name, "kernel_us": round(time_kernel(fns[name], args.iters), 2)}))
    if args.no_stamps:
        return
    with tempfile.TemporaryDirectory() as tmp:
        lib = args.stamped_lib or build_stamped(tmp)
        for name in args.levels:
            subprocess.run([sys.executable, os.path.abspath(__file__), "--stamps-child", lib, name], check=True)


if __name__ == "__main__":
    main()
