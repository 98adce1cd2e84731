"""Build libmmg.so (hand-written sm_90a kernels + C-ABI) in-tree with nvcc.  No torch headers, no pybind:
the library is a plain C-ABI shared object (include/mmg.h) loaded with ctypes."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libmmg.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr"]


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(verbose=False, force=False):
    os.makedirs(OBJ, exist_ok=True)
    srcs = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")]
    hdrs.append(os.path.join(os.path.dirname(HERE), "include", "mmg.h"))
    jobs = []
    for s in srcs:
        src, obj = os.path.join(CSRC, s), os.path.join(OBJ, s[:-3] + ".o")
        if force or _newer(obj, [src] + hdrs):
            jobs.append([NVCC] + FLAGS + ["-c", src, "-o", obj])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        if verbose and (r.stdout or r.stderr):
            print(r.stdout + r.stderr)

    with ThreadPoolExecutor(max_workers=8) as ex:
        list(ex.map(run, jobs))
    objs = [os.path.join(OBJ, s[:-3] + ".o") for s in srcs]
    if force or jobs or _newer(LIB, objs):
        run([NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"])
    return LIB


if __name__ == "__main__":
    print(build(verbose=True, force="--force" in sys.argv))
