"""In-tree build of the native pieces (no JIT cache: the built files travel with the repo snapshot).

  medpy_b200/lib/libmedpy_b200_gc.so      C ABI + CUDA kernels   (nvcc, sm_90a only)
  medpy_b200/_mgc<EXT_SUFFIX>             pybind11 binding       (g++, links the C-ABI library via $ORIGIN/lib)

``python -m medpy_b200.build`` or ``medpy_b200.build.build_all()``; __graft_entry__.build() calls the latter.
"""
import concurrent.futures
import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libmedpy_b200_gc.so")
EXT = os.path.join(HERE, "_mgc" + sysconfig.get_config_var("EXT_SUFFIX"))
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CXX = os.environ.get("CXX", "g++")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
    # IEEE everywhere: denormals kept, exact div/sqrt, and no FMA contraction so the float64 weights equal
    # numpy's (SURVEY.md §7.2 item 2)
    "-ftz=false", "-prec-div=true", "-prec-sqrt=true", "-fmad=false",
]


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _includes(path, seen=None):
    """The file plus every local header it includes (transitively)."""
    seen = seen if seen is not None else set()
    if path in seen or not os.path.exists(path):
        return seen
    seen.add(path)
    with open(path) as fh:
        for line in fh:
            line = line.strip()
            if line.startswith("#include \""):
                name = line.split('"')[1]
                _includes(os.path.normpath(os.path.join(os.path.dirname(path), name)), seen)
    return seen


def build_lib(force=False, verbose=False):
    """One object per translation unit (rebuilt only when the unit or a header it includes changed), linked into one
    shared library: the lattice C ABI (gc_api.cu, gc_build_api.cu, gc_solve.cu, gc_fold.cu, gc_slab.cu, gc_batch.cu;
    gc_handle.cuh), gc_sparse_api.cu (sparse graphs) and gc_labels_api.cu (label images).  Every .cu file in csrc/ is a
    unit; they compile concurrently, one nvcc process each."""
    units = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith(".cu")]
    objdir = os.path.join(LIBDIR, "obj")
    os.makedirs(objdir, exist_ok=True)
    header = os.path.join(INCLUDE, "medpy_b200_graphcut.h")
    compile_flags = [f for f in NVCC_FLAGS if f != "-shared"]
    objs = []
    stale = []
    for unit in units:
        obj = os.path.join(objdir, os.path.basename(unit)[:-3] + ".o")
        objs.append(obj)
        deps = sorted(_includes(unit)) + [header, os.path.abspath(__file__)]
        if force or _newer(obj, deps):
            stale.append([NVCC] + compile_flags + (["-Xptxas", "-v"] if verbose else []) + ["-I", INCLUDE, "-c", unit, "-o", obj])
    if stale:
        with concurrent.futures.ThreadPoolExecutor(max_workers=min(len(stale), os.cpu_count() or 1)) as pool:
            list(pool.map(subprocess.check_call, stale))
    if force or stale or not os.path.exists(LIB) or _newer(LIB, objs):
        subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fPIC",
                               "-o", LIB] + objs)
    return LIB


def build_ext(force=False):
    src = os.path.join(CSRC, "gc_pybind.cpp")
    if not force and not _newer(EXT, [src, LIB, os.path.join(INCLUDE, "medpy_b200_graphcut.h"), os.path.join(CSRC, "host_pack.hpp")]):
        return EXT
    import pybind11
    cmd = [CXX, "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden",
           "-I", sysconfig.get_paths()["include"], "-I", pybind11.get_include(), "-I", INCLUDE,
           src, "-o", EXT, "-L", LIBDIR, "-lmedpy_b200_gc", "-Wl,-rpath,$ORIGIN/lib"]
    subprocess.check_call(cmd)
    return EXT


def build_all(force=False, verbose=False):
    build_lib(force=force, verbose=verbose)
    build_ext(force=force)
    return LIB, EXT


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(LIB)
    print(EXT)
