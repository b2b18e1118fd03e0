#!/usr/bin/env python
"""Build recipe for oracle/_ref: the reference's own CUDA extension, compiled unmodified.

TEST INFRASTRUCTURE ONLY.  Nothing in the product path (closerlook3d_b200/) imports this.

The reference's native ops (pytorch/ops/pt_custom_ops/_ext_src, 4 .cu + 5 .cpp files) are compiled
*from where they lie* in a checkout of the reference (CL3D_REFERENCE, default /root/reference) with a
hand-written nvcc/g++ recipe (the reference's own setup.py is not run), for sm_90 (plain, as the reference
would be built by TORCH_CUDA_ARCH_LIST=9.0), with the reference's own flags (-O2, no fast-math).  Outputs go
only into oracle/_ref/ (git-ignored).  Where it is built, the result is used as

  * the GPU-side pin for the C restatement in oracle/cl3d_oracle.c (bit-exact idx / idx_mask / sub_xyz), and
  * the "reference GPU path" timing in bench.py (extra, informational).

No reference source is copied into the repository.
"""
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = os.path.join(os.environ.get("CL3D_REFERENCE", "/root/reference"), "pytorch/ops/pt_custom_ops/_ext_src")
OUT_DIR = os.path.join(HERE, "_ref", "pt_custom_ops")
SO_NAME = "_ext" + sysconfig.get_config_var("EXT_SUFFIX")


def ref_available():
    return os.path.isdir(os.path.join(REF_SRC, "src"))


def built_path():
    p = os.path.join(OUT_DIR, SO_NAME)
    return p if os.path.exists(p) else None


def build(force=False, verbose=True):
    """Compile the reference extension.  Returns the .so path, or None when the reference checkout is absent
    (a previously built file is used if there is one)."""
    if not ref_available():
        return built_path()
    if built_path() and not force:
        return built_path()
    import torch  # noqa: F401
    from torch.utils import cpp_extension as ce

    os.makedirs(OUT_DIR, exist_ok=True)
    obj_dir = os.path.join(HERE, "_ref", "obj")
    os.makedirs(obj_dir, exist_ok=True)
    incs = ce.include_paths("cuda") + [sysconfig.get_paths()["include"], os.path.join(REF_SRC, "include")]
    inc_flags = [f"-I{p}" for p in incs]
    common = ["-DTORCH_EXTENSION_NAME=_ext", "-DTORCH_API_INCLUDE_EXTENSION_H",
              "-D_GLIBCXX_USE_CXX11_ABI=1", "-std=c++17"]
    srcs = sorted(os.listdir(os.path.join(REF_SRC, "src")))
    jobs = []
    objs = []
    for s in srcs:
        src = os.path.join(REF_SRC, "src", s)
        obj = os.path.join(obj_dir, s + ".o")
        objs.append(obj)
        if s.endswith(".cu"):
            cmd = ["nvcc", "-c", src, "-o", obj, "-O2", "-gencode", "arch=compute_90,code=sm_90",
                   "--compiler-options", "-fPIC", "--expt-relaxed-constexpr"] + common + inc_flags
        elif s.endswith(".cpp"):
            cmd = ["g++", "-c", src, "-o", obj, "-O2", "-fPIC"] + common + inc_flags
        else:
            objs.pop()
            continue
        jobs.append(cmd)

    def run(cmd):
        if verbose:
            print(" ".join(cmd[:4]), "...", flush=True)
        subprocess.check_call(cmd)

    with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
        list(ex.map(run, jobs))
    lib_dirs = ce.library_paths("cuda")
    so = os.path.join(OUT_DIR, SO_NAME)
    link = ["g++", "-shared", "-o", so] + objs + [f"-L{d}" for d in lib_dirs] + \
           ["-lc10", "-ltorch", "-ltorch_cpu", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda", "-lcudart"] + \
           [f"-Wl,-rpath,{d}" for d in lib_dirs]
    run(link)
    with open(os.path.join(OUT_DIR, "__init__.py"), "w") as f:
        f.write("# built by oracle/build_ref.py from the unmodified reference sources (test infrastructure)\n")
    return so


def load():
    """Import the compiled reference extension as module `pt_custom_ops._ext` (needs a GPU to be useful)."""
    so = built_path()
    if so is None:
        raise ImportError("oracle/_ref is not built (run oracle/build_ref.py where the reference checkout exists)")
    import importlib.util
    import torch  # noqa: F401  (must be loaded first: the .so links against libtorch)
    spec = importlib.util.spec_from_file_location("_ext", so)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    p = build(force="--force" in sys.argv)
    print("oracle/_ref:", p)
