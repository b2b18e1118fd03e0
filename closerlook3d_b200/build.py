"""Build libcl3d.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python -m closerlook3d_b200.build [--force]

nvcc cross-compiles without a GPU.  The .so and the objects are build products (git-ignored).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
SO_PATH = os.path.join(PKG_DIR, "libcl3d.so")
OBJ_DIR = os.path.join(PKG_DIR, "csrc", "_obj")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "--expt-relaxed-constexpr", "--extended-lambda", "-Xcompiler", "-fPIC"]


EXTRA_FLAGS = {}  # per-file additions to NVCC_FLAGS, e.g. {"x.cu": ["-fmad=false"]}


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _newest_src_mtime():
    m = 0.0
    for f in os.listdir(CSRC):
        if f.endswith((".cu", ".cuh", ".h")):
            m = max(m, os.path.getmtime(os.path.join(CSRC, f)))
    m = max(m, os.path.getmtime(os.path.join(PKG_DIR, "..", "include", "cl3d.h")))
    return m


def build(force=False, verbose=False):
    if not force and os.path.exists(SO_PATH) and os.path.getmtime(SO_PATH) >= _newest_src_mtime():
        return SO_PATH
    os.makedirs(OBJ_DIR, exist_ok=True)
    nvcc = os.environ.get("NVCC", "nvcc")
    objs = []
    cmds = []
    hdr_m = max(os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h")))
    hdr_m = max(hdr_m, os.path.getmtime(os.path.join(PKG_DIR, "..", "include", "cl3d.h")))
    for s in sources():
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ_DIR, s[:-3] + ".o")
        objs.append(obj)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_m):
            cmds.append([nvcc] + NVCC_FLAGS + EXTRA_FLAGS.get(s, []) + ["-c", src, "-o", obj])

    def run(cmd):
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        return r

    with ThreadPoolExecutor(max_workers=max(1, min(8, len(cmds) or 1))) as ex:
        list(ex.map(run, cmds))
    run([nvcc, "-shared", "-o", SO_PATH] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"])
    return SO_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
