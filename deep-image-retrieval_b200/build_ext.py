"""Build libdirb200.so (the C-ABI CUDA library) and libdirb200_blocktest.so (test-only wrappers of csrc/block.cuh)
in-tree with nvcc for sm_90a."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SOURCES = ["common.cu", "conv.cu", "ops.cu", "search.cu", "net.cu", "api.cu", "resize.cu", "label_count.cu", "jpeg.cu", "pca.cu",
           "aploss.cu", "diffusion.cu", "diffusion_trunc.cu", "join.cu", "kmeans.cu", "pq.cu", "graph.cu"]
LIB = os.path.join(HERE, "libdirb200.so")
BLOCKTEST_SRC = os.path.join(os.path.dirname(HERE), "tests", "block_harness.cu")
BLOCKTEST_LIB = os.path.join(HERE, "libdirb200_blocktest.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _newer(a, b):
    return (not os.path.exists(b)) or os.path.getmtime(a) > os.path.getmtime(b)


def build(force=False, verbose=False):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "dirb200.h"))
    objs, procs = [], []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _newer(s, o) or any(_newer(h, o) for h in headers):
            cmd = [nvcc] + NVCC_FLAGS + ["-c", s, "-o", o]
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            print("==== nvcc", src, "->", p.returncode)
            print(out)
        with open(os.path.join(objdir, src + ".log"), "w") as f:
            f.write(out)
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    if procs or not os.path.exists(LIB):
        cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
        subprocess.check_call(cmd)
    # the test-only wrappers of block.cuh's primitives (tests/test_gpu_block.py), a library of their own
    if force or _newer(BLOCKTEST_SRC, BLOCKTEST_LIB) or any(_newer(h, BLOCKTEST_LIB) for h in headers):
        cmd = [nvcc] + NVCC_FLAGS + ["-shared", BLOCKTEST_SRC, "-o", BLOCKTEST_LIB, "-cudart", "static"]
        p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if p.returncode != 0 or verbose:
            print("==== nvcc block_harness.cu ->", p.returncode)
            print(p.stdout)
        with open(os.path.join(objdir, "block_harness.cu.log"), "w") as f:
            f.write(p.stdout)
        if p.returncode != 0:
            raise RuntimeError("nvcc failed")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
