"""In-tree build of the native libraries (nvcc cross-compiles sm_90a without a GPU).

  anakin_b200/lib/libb200saber.so   C-ABI CUDA device layer   (include/b200_saber.h)
  anakin_b200/lib/libanakin_b200.so host framework + C API     (include/anakin_b200.h)

`python -m anakin_b200.build` or __graft_entry__.build() call build_all(). Objects are
rebuilt only when a source or header is newer. Build products are git-ignored.
"""
import concurrent.futures as cf
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "build")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-fvisibility=hidden",
                     "--expt-relaxed-constexpr", "-ccbin", "g++"]
# experimental device code paths are compiled in only on request (B200_BUILD_DEFINES="B200_TIMELINE ...")
NVCC_FLAGS += ["-D" + d for d in os.environ.get("B200_BUILD_DEFINES", "").split() if d]
CXX_FLAGS = ["-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-Wall", "-pthread"]


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def _headers():
    hs = glob.glob(os.path.join(CSRC, "**", "*.cuh"), recursive=True)
    hs += glob.glob(os.path.join(CSRC, "**", "*.h"), recursive=True)
    hs += glob.glob(os.path.join(ROOT, "include", "*.h"))
    return hs


def _run(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("build failed: %s\n%s" % (" ".join(cmd), r.stdout))
    return r.stdout


def _compile(src, flags_extra=()):
    rel = os.path.relpath(src, CSRC).replace(os.sep, "_")
    obj = os.path.join(OBJDIR, rel + ".o")
    if _newer(obj, [src] + _headers()):
        if src.endswith(".cu"):
            _run([NVCC] + NVCC_FLAGS + list(flags_extra) + ["-c", src, "-o", obj])
        else:
            _run(["g++"] + CXX_FLAGS + ["-I/usr/local/cuda/include", "-I" + os.path.join(ROOT, "include"),
                                         "-I" + CSRC] + list(flags_extra) + ["-c", src, "-o", obj])
        return obj, True
    return obj, False


def build_saber(verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    srcs = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        res = list(ex.map(_compile, srcs))
    objs = [o for o, _ in res]
    lib = os.path.join(LIBDIR, "libb200saber.so")
    if any(ch for _, ch in res) or not os.path.exists(lib):
        _run([NVCC] + ARCH + ["-shared", "-o", lib] + objs + ["-ccbin", "g++"])
        if verbose:
            print("linked", lib)
    return lib


def build_framework(verbose=False):
    fdir = os.path.join(CSRC, "framework")
    srcs = sorted(glob.glob(os.path.join(fdir, "*.cpp")))
    if not srcs:
        return None
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        res = list(ex.map(_compile, srcs))
    objs = [o for o, _ in res]
    lib = os.path.join(LIBDIR, "libanakin_b200.so")
    if any(ch for _, ch in res) or not os.path.exists(lib) or _newer(lib, [os.path.join(LIBDIR, "libb200saber.so")]):
        _run(["g++", "-shared", "-o", lib] + objs +
             ["-L" + LIBDIR, "-lb200saber", "-Wl,-rpath,$ORIGIN", "-L/usr/local/cuda/lib64", "-lcudart",
              "-Wl,-rpath,/usr/local/cuda/lib64", "-pthread"])
        if verbose:
            print("linked", lib)
    return lib


def build_all(verbose=False):
    a = build_saber(verbose)
    b = build_framework(verbose)
    return a, b


if __name__ == "__main__":
    print(build_all(verbose=True))
