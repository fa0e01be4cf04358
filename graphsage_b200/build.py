"""In-tree build of libgraphsage_b200.so for the H100 (sm_90a; nvcc cross-compiles without a GPU).

    python -m graphsage_b200.build [--force]

The .so lands next to the sources (graphsage_b200/csrc/libgraphsage_b200.so, git-ignored), so the
package is importable from the source tree.
"""
import concurrent.futures
import os
import subprocess
import sys

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc")
LIB = os.path.join(CSRC, "libgraphsage_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-DGS_NO_FAST_MATH"] + os.environ.get("GS_EXTRA_NVCC_FLAGS", "").split()


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers():
    inc = os.path.join(os.path.dirname(os.path.dirname(CSRC)), "include")
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs += [os.path.join(inc, f) for f in os.listdir(inc) if f.endswith(".h")]
    return hs


def _compile(src, verbose):
    obj = src[:-3] + ".o"
    cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    return obj, r.stderr


def build_library(force=False, verbose=False):
    srcs = _sources()
    newest = max(os.path.getmtime(p) for p in srcs + _headers() + [os.path.abspath(__file__)])
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= newest:
        return LIB
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile(s, verbose), srcs))
    if verbose:
        for _, log in results:
            sys.stderr.write(log)
    objs = [o for o, _ in results]
    cmd = [NVCC, "-shared", "-o", LIB] + objs + ARCH + ["-lcudart_static", "-lpthread", "-ldl", "-lrt"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
