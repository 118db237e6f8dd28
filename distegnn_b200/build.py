"""Build the CUDA libraries in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m distegnn_b200.build [--force] [--verbose]

  libdistegnn_b200.so          the product: every entry point of include/distegnn_b200.h (csrc/*.cu)
  libdistegnn_b200_testing.so  cross-check twins of include/distegnn_b200_testing.h (csrc/testing/*.cu); loaded only by
                               tests/twin_backend.py, never by the package

The shared libraries and objects are build products (git-ignored); `build()` rebuilds them whenever a source, header or
this file is newer.
"""
from __future__ import annotations

import argparse
import concurrent.futures as cf
import os
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
TSRC = os.path.join(CSRC, "testing")
ROOT = os.path.dirname(PKG)
INC = os.path.join(ROOT, "include")
LIB = os.path.join(PKG, "libdistegnn_b200.so")
LIB_TESTING = os.path.join(PKG, "libdistegnn_b200_testing.so")
OBJ = os.path.join(CSRC, "build")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
          "-Xptxas", "-v", "--expt-relaxed-constexpr", "-I", CSRC]
# shared by both libraries (error string, parameter layout, device queries)
COMMON = ["api.cu"]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def testing_sources():
    return sorted(os.path.join("testing", f) for f in os.listdir(TSRC) if f.endswith(".cu"))


def _deps_mtime():
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs += [os.path.join(INC, f) for f in os.listdir(INC) if f.endswith(".h")]
    return max(os.path.getmtime(h) for h in hdrs)


def _compile(src, verbose):
    obj = os.path.join(OBJ, src.replace(os.sep, "_")[:-3] + ".o")
    extra = []
    if src.startswith("testing" + os.sep):        # the twins' declarations (default visibility) come from the testing header
        extra += ["-include", os.path.join(INC, "distegnn_b200_testing.h")]
    cmd = [NVCC, *ARCH, *CFLAGS, *extra, "-c", os.path.join(CSRC, src), "-o", obj]
    p = subprocess.run(cmd, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{p.stdout}\n{p.stderr}")
    with open(obj + ".ptxas.log", "w") as f:
        f.write(p.stderr)
    if verbose:
        print(p.stderr)
    return obj


def _link(lib, objs):
    tmp = lib + ".tmp"                      # link aside, then rename: a snapshot of the tree never sees a half-written .so
    p = subprocess.run([NVCC, *ARCH, "-shared", "-o", tmp, *objs, "-cudart", "shared",
                        "-Xlinker", "-rpath,/usr/local/cuda/lib64"], capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError(f"link failed:\n{p.stdout}\n{p.stderr}")
    os.replace(tmp, lib)
    return lib


def build(force: bool = False, verbose: bool = False) -> str:
    srcs, tsrcs = sources(), testing_sources()
    newest = max([os.path.getmtime(os.path.join(CSRC, s)) for s in srcs + tsrcs]
                 + [_deps_mtime(), os.path.getmtime(__file__)])
    if not force and all(os.path.exists(l) and os.path.getmtime(l) >= newest for l in (LIB, LIB_TESTING)):
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs) + len(tsrcs))) as ex:
        objs = dict(zip(srcs + tsrcs, ex.map(lambda s: _compile(s, verbose), srcs + tsrcs)))
    _link(LIB, [objs[s] for s in srcs])
    _link(LIB_TESTING, [objs[s] for s in COMMON] + [objs[s] for s in tsrcs])
    return LIB


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    a = ap.parse_args()
    print(build(a.force, a.verbose))
