"""Builds libwarprnnt.so (the C-ABI drop-in) in-tree for sm_90a (H100) with nvcc.

    python warp-transducer_b200/build.py [--force] [--verbose]

The shared object lands in warp-transducer_b200/lib/ (git-ignored).  cudart is linked statically so the library has no run-time dependency beyond the
driver; it shares the primary context (and therefore streams and device pointers) with PyTorch.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "lib", "libwarprnnt.so")
SOURCES = ["rnnt_entry.cu", "rnnt_joiner.cu"]
# every source/header under csrc/ plus the public header: editing any of them marks the .so stale
DEPS = sorted(f for f in os.listdir(SRC) if f.endswith((".cu", ".cuh", ".h"))) + \
       [os.path.join("..", "..", "include", "rnnt.h")]
# ptxas --split-compile=0: ptxas compiles the kernels of the translation unit on as many threads as the host has CPUs
# (each kernel's code is the same as from one thread; only the wall time changes).
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "-cudart", "static", "-Xptxas", "--split-compile=0",
]


def stale():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(os.path.join(SRC, d)) > t for d in DEPS)


def build(force=False, verbose=False):
    if not force and not stale():
        return OUT
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
          [os.path.join(SRC, s) for s in SOURCES] + ["-o", OUT]
    env = dict(os.environ)
    # the image exports CC/CXX pointing at a gcc without its spec files; nvcc must use the system one
    env.pop("CC", None), env.pop("CXX", None)
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n%s\n%s" % (" ".join(cmd), r.stdout + r.stderr))
    if verbose:
        print(r.stdout + r.stderr)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
