"""Builds libphk.so (hand-written sm_90a CUDA + the C ABI of include/phk.h) in-tree with nvcc."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libphk.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-warn-spills"]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")]
    deps.append(os.path.join(os.path.dirname(HERE), "include", "phk.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    objs = []
    procs = []
    for src in sources():
        obj = src[:-3] + ".o"
        objs.append(obj)
        cmd = [NVCC, *FLAGS, "-c", src, "-o", obj] + (["-Xptxas", "-v"] if verbose else [])
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if out.strip():
            print(out)
        if p.returncode != 0:
            print(f"nvcc failed on {src}", file=sys.stderr)
            failed = True
    if failed:
        raise RuntimeError("libphk build failed")
    subprocess.check_call([NVCC, *FLAGS[:2], "-shared", "-o", LIB, *objs, "-lcudart", "-lcuda"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
