"""Build librnc.so (the sm_90a kernels + C ABI) in-tree with nvcc.

    python raft-ncup_b200/rnc/build.py [--force] [--verbose]

nvcc cross-compiles for sm_90a without a GPU.  The .so lands next to this file (git-ignored), so the package imports
straight from the source tree.
"""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
OBJ = os.path.join(PKG, "build")
LIB = os.path.join(HERE, "librnc.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
              "--expt-relaxed-constexpr", "-Xptxas", "-warn-spills"]


def nvcc_path():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: librnc.so cannot be built")


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest():
    h = hashlib.sha256()
    for f in sorted(os.listdir(CSRC)) + ["../../include/rnc.h"]:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(f.encode())
            h.update(fh.read())
    h.update(" ".join(ARCH + NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ for sm_90a and link librnc.so.  Returns the path."""
    stamp = os.path.join(OBJ, "stamp")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB
    nvcc = nvcc_path()
    os.makedirs(OBJ, exist_ok=True)
    inc = ["-I", os.path.join(ROOT, "include"), "-I", CSRC]
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(OBJ, src[:-3] + ".o")
        objs.append(obj)
        cmd = [nvcc, *ARCH, *NVCC_FLAGS, *inc, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"--- nvcc failed on {src}\n{out}\n")
        elif out.strip() and (verbose or "warning" in out.lower() or "spill" in out.lower()):
            sys.stderr.write(f"--- {src}\n{out}\n")
    if failed:
        raise RuntimeError("librnc.so build failed")
    cmd = [nvcc, *ARCH, "-shared", "-o", LIB, *objs, "-lcuda"]
    subprocess.check_call(cmd)
    with open(stamp, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
