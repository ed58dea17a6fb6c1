"""In-tree build of the CUDA library (sm_90a only).  `python -m rainbow_iqn_apex_b200._build`."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libriqn_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = [*ARCH, "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr"]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps():
    extra = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    extra.append(os.path.join(os.path.dirname(HERE), "include", "riqn_b200.h"))
    return extra


def build(force=False, verbose=False):
    """Compile every csrc/*.cu to an object (cached by mtime) and link libriqn_b200.so in-tree."""
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    dep_mtime = max(os.path.getmtime(p) for p in _deps())
    objs, procs = [], []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), dep_mtime):
            cmd = [NVCC, *FLAGS, "-c", src, "-o", obj]
            if verbose:
                print(" ".join(cmd))
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{out.decode()}")
    if procs or force or not os.path.exists(LIB) or any(os.path.getmtime(o) > os.path.getmtime(LIB) for o in objs):
        cmd = [NVCC, "-shared", "-o", LIB, *objs, *ARCH, "-lcudart_static",
               "-ldl", "-lrt", "-lpthread"]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout.decode())
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
