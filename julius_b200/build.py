"""Build libjb200.so (CUDA, sm_90a only) in-tree with nvcc.  No JIT cache: the library is loaded from the tree."""
from __future__ import annotations

import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB = os.path.join(HERE, "libjb200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = [*GENCODE, "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def sources():
    return sorted(glob.glob(os.path.join(HERE, "csrc", "*.cu")))


def up_to_date() -> bool:
    if not os.path.exists(LIB):
        return False
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(HERE, "csrc", "*.cuh")) + glob.glob(os.path.join(ROOT, "include", "*.h"))
    return all(os.path.getmtime(d) <= t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and up_to_date():
        return LIB
    objdir = os.path.join(HERE, "csrc", "_obj")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        # the beam kernel's float decisions must not be FMA-contracted
        extra = ["--fmad=false"] if os.path.basename(src) in ("beam.cu",) else []
        cmd = [NVCC, *FLAGS, *extra, "-I", os.path.join(ROOT, "include"), "-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append(out)
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f"nvcc failed on {src}")
    with open(os.path.join(objdir, "ptxas.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    subprocess.run([NVCC, "-shared", "-o", LIB, *objs, *GENCODE], check=True)
    return LIB


if __name__ == "__main__":
    args = sys.argv[1:]
    print(build(force="--force" in args, verbose="-v" in args))
