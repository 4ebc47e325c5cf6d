"""Builds libcoclr_b200.so (the C-ABI library of sm_90a kernels) in-tree with nvcc.

The library is compiled only for sm_90a (`-gencode arch=compute_90a,code=sm_90a`, NVIDIA H100); nvcc
cross-compiles without a GPU, so this also is the "does it build" check of `__graft_entry__.build()`.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libcoclr_b200.so")
STAMP = os.path.join(HERE, ".libcoclr_b200.stamp")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "-I", os.path.join(ROOT, "include"),
    "-I", CSRC,
]


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest():
    h = hashlib.sha256()
    files = _sources() + sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h")))
    files.append(os.path.join(ROOT, "include", "coclr_b200.h"))
    for f in files:
        h.update(f.encode())
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ and link libcoclr_b200.so. Returns the library path."""
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP):
        with open(STAMP) as fh:
            if fh.read().strip() == dig:
                return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    objs = []
    for src in _sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [nvcc] + NVCC_FLAGS + ["-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, out.decode()))
    cmd = [nvcc, "-shared", "-o", LIB] + objs  # cudart linked statically (nvcc default)
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if out.returncode != 0:
        raise RuntimeError("link failed:\n%s" % out.stdout.decode())
    with open(STAMP, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
