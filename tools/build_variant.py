"""Build an instrumented copy of the library next to libpsa.so:  python tools/build_variant.py <name> [-DFLAG ...]
-> scanobjectnn_b200/libpsa_<name>.so (objects under csrc/build_<name>/); use it with PSA_LIB_PATH=..."""
import concurrent.futures as cf
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scanobjectnn_b200 import build as B  # noqa: E402

name, flags = sys.argv[1], sys.argv[2:]
objdir = os.path.join(B.CSRC, f"build_{name}")
os.makedirs(objdir, exist_ok=True)
lib = os.path.join(B.HERE, f"libpsa_{name}.so")
nvcc = B._nvcc()
jobs, objs = [], []
for src in B.sources():
    obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
    objs.append(obj)
    jobs.append([nvcc, *B.NVCC_FLAGS, *flags, "-c", src, "-o", obj])
with cf.ThreadPoolExecutor(max_workers=8) as ex:
    for r in ex.map(lambda c: subprocess.run(c, capture_output=True, text=True), jobs):
        if r.returncode != 0:
            sys.exit(r.stdout + r.stderr)
r = subprocess.run([nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", lib, *objs, "-lcudart"], capture_output=True, text=True)
if r.returncode != 0:
    sys.exit(r.stdout + r.stderr)
print(lib)
