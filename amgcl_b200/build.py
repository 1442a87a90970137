"""Build recipes for the native parts of amgcl_b200 (all in-tree, no JIT cache).

  libamgcl_b200.so         CUDA kernels + C ABI (nvcc, sm_90a only; csrc/api_*.cu)
  libamgcl_b200_dropin.so  AMGCL's own make_solver/amg/cg/bicgstab templates
                           instantiated on backend::b200 (g++; needs the AMGCL
                           headers, i.e. only buildable where /root/reference or
                           $AMGCL_ROOT exists -- the prebuilt .so travels to the GPU box)
  poisson_b200             examples/poisson_b200.cpp: the reference tutorial program with the
                           backend typedef switched (plain g++, links libamgcl_b200.so)
"""
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "amgcl_b200")
LIBDIR = os.path.join(PKG, "lib")
CSRC = os.path.join(PKG, "csrc")
HOST = os.path.join(PKG, "host")
INCLUDE = os.path.join(ROOT, "include")

LIB_CUDA = os.path.join(LIBDIR, "libamgcl_b200.so")
LIB_DROPIN = os.path.join(LIBDIR, "libamgcl_b200_dropin.so")
EXAMPLE = os.path.join(LIBDIR, "poisson_b200")
EXAMPLE_SRC = os.path.join(ROOT, "examples", "poisson_b200.cpp")

NVCC_COMPILE = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fopenmp", "-I", INCLUDE,
]
# portable x86-64 flags: the GPU box may have a different CPU than the build box
CXX_FLAGS = ["-O2", "-mavx2", "-mfma", "-std=c++17", "-fopenmp", "-fPIC", "-shared", "-DAMGCL_NO_BOOST"]


def amgcl_root():
    """Directory holding the AMGCL headers (amgcl/amg.hpp), or None."""
    for cand in (os.environ.get("AMGCL_ROOT"), "/root/reference"):
        if cand and os.path.isfile(os.path.join(cand, "amgcl", "amg.hpp")):
            return cand
    return None


def _newer(target, sources):
    if not os.path.isfile(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _run(cmd):
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if proc.returncode != 0:
        raise RuntimeError("build failed: %s\n%s" % (" ".join(cmd), proc.stdout))
    return proc.stdout


def nvcc_path():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.isfile(cand):
            return cand
    return None


def cuda_sources():
    """The translation units of libamgcl_b200.so (api_*.cu) and everything they include."""
    units = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    headers = sorted(f for f in os.listdir(CSRC) if f.endswith(".cuh"))
    return units, headers


def build_cuda(force=False, verbose=False):
    """Compile the CUDA kernels + C ABI for sm_90a into libamgcl_b200.so (one object per
    api_*.cu, compiled concurrently, objects kept under lib/obj/)."""
    os.makedirs(LIBDIR, exist_ok=True)
    units, headers = cuda_sources()
    deps = [os.path.join(CSRC, f) for f in headers] + [os.path.join(INCLUDE, "amgcl_b200.h"),
                                                         os.path.join(INCLUDE, "amgcl_b200_formats.h"),
                                                         os.path.join(INCLUDE, "amgcl_b200_coarse.h")]
    if not force and not _newer(LIB_CUDA, deps + [os.path.join(CSRC, u) for u in units]):
        return LIB_CUDA
    nvcc = nvcc_path()
    if nvcc is None:
        raise RuntimeError("nvcc not found: cannot build libamgcl_b200.so")
    objdir = os.path.join(LIBDIR, "obj")
    os.makedirs(objdir, exist_ok=True)
    jobs = []
    for u in units:
        src = os.path.join(CSRC, u)
        obj = os.path.join(objdir, u[:-3] + ".o")
        if force or _newer(obj, deps + [src]):
            cmd = [nvcc] + NVCC_COMPILE + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
            jobs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = []
    for cmd, proc in jobs:
        out = proc.communicate()[0]
        if proc.returncode != 0:
            failed.append("build failed: %s\n%s" % (" ".join(cmd), out))
        elif verbose:
            print(out)
    if failed:
        raise RuntimeError("\n".join(failed))
    objs = [os.path.join(objdir, u[:-3] + ".o") for u in units]
    # --no-undefined: a launch the dispatcher reaches but no unit instantiates fails here, not at
    # the first call that reaches it
    _run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fopenmp",
          "-Xlinker", "--no-undefined", "-o", LIB_CUDA] + objs + ["-lgomp"])
    return LIB_CUDA


def build_dropin(force=False):
    """Instantiate AMGCL's unmodified solver templates on the b200 backend."""
    os.makedirs(LIBDIR, exist_ok=True)
    sources = [os.path.join(HOST, "dropin.cpp"),
               os.path.join(INCLUDE, "amgcl", "backend", "b200.hpp"),
               os.path.join(INCLUDE, "amgcl_b200.h")]
    if not force and not _newer(LIB_DROPIN, sources + [LIB_CUDA] if os.path.isfile(LIB_CUDA) else sources):
        return LIB_DROPIN
    root = amgcl_root()
    if root is None:
        if os.path.isfile(LIB_DROPIN):
            return LIB_DROPIN          # prebuilt copy shipped with the snapshot
        raise RuntimeError("AMGCL headers not found (set AMGCL_ROOT) and no prebuilt drop-in library")
    cmd = ["g++"] + CXX_FLAGS + ["-I", INCLUDE, "-I", root,
                                 os.path.join(HOST, "dropin.cpp"), "-o", LIB_DROPIN,
                                 "-L", LIBDIR, "-lamgcl_b200", "-Wl,-rpath,$ORIGIN"]
    _run(cmd)
    return LIB_DROPIN


def build_example(force=False):
    """Compile the tutorial-style user program exactly as INTEGRATION.md section 1 says a user would."""
    sources = [EXAMPLE_SRC, os.path.join(INCLUDE, "amgcl", "backend", "b200.hpp"),
               os.path.join(INCLUDE, "amgcl_b200.h")]
    if not force and not _newer(EXAMPLE, sources):
        return EXAMPLE
    root = amgcl_root()
    if root is None:
        if os.path.isfile(EXAMPLE):
            return EXAMPLE
        raise RuntimeError("AMGCL headers not found (set AMGCL_ROOT) and no prebuilt example")
    _run(["g++", "-std=c++17", "-O2", "-mavx2", "-mfma", "-fopenmp", "-DAMGCL_NO_BOOST",
          "-I", root, "-I", INCLUDE, EXAMPLE_SRC, "-o", EXAMPLE,
          "-L", LIBDIR, "-lamgcl_b200", "-Wl,-rpath,$ORIGIN"])
    return EXAMPLE


def build_all(force=False, verbose=False):
    build_cuda(force=force, verbose=verbose)
    build_dropin(force=force)
    build_example(force=force)


if __name__ == "__main__":
    import sys
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("built:", LIB_CUDA, LIB_DROPIN)
