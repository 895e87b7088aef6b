"""Builds libvqb200.so (all CUDA kernels + the C ABI of include/vqb200.h) in-tree with nvcc for sm_90a (H100).

Usage: python build_native.py [--force]
The library and the object files under build/ are build products (git-ignored).

--use_fast_math (approximate division / sqrt, flush-to-zero) is limited to the attention translation unit, whose online
softmax is written for it; GroupNorm statistics, the VQ distance, the optimizer and everything else compile with IEEE
division / sqrt and denormals (the VQ argmin must be bit-exact against a NumPy oracle that keeps denormals).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libvqb200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xptxas", "-v",
]
FAST_MATH_UNITS = {"attention.cu"}


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def needs_build(out=OUT):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "vqb200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    out = OUT
    if not force and not needs_build(out):
        return out
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)

    def compile_one(src):
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        flags = list(FLAGS)
        if os.path.basename(src) in FAST_MATH_UNITS:
            flags.append("--use_fast_math")
        r = subprocess.run([NVCC, *flags, "-c", src, "-o", obj], capture_output=True, text=True)
        return src, obj, r

    with ThreadPoolExecutor(max_workers=8) as ex:
        results = list(ex.map(compile_one, sources()))
    objs = []
    for src, obj, r in results:
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError(f"nvcc failed for {src}")
        if verbose:
            sys.stderr.write(r.stderr)
        objs.append(obj)
    tmp = out + ".tmp"
    r = subprocess.run([NVCC, "-shared", "-o", tmp, *objs, "-gencode", "arch=compute_90a,code=sm_90a"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    os.replace(tmp, out)  # atomic: a concurrent snapshot never sees a half-written library
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
