"""Build libsamplenet_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python samplenet_b200/csrc/build.py [--force] [--verbose]

Sources: every *.cu in this directory.  Output: samplenet_b200/lib/libsamplenet_b200.so (git-ignored).  Objects are cached under
samplenet_b200/csrc/build/sm_90a/ keyed on mtimes.
"""
import glob
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
OUT = os.path.join(PKG, "lib", "libsamplenet_b200.so")
ARCH = "sm_90a"
OBJ = os.path.join(HERE, "build", ARCH)   # per target: objects of another architecture are never linked in
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=" + ARCH, "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr",
]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    srcs = sorted(glob.glob(os.path.join(HERE, "*.cu")))
    hdrs = sorted(glob.glob(os.path.join(HERE, "*.cuh"))) + [os.path.join(os.path.dirname(PKG), "include", "samplenet_b200.h")]
    objs = [os.path.join(OBJ, os.path.basename(s)[:-3] + ".o") for s in srcs]

    def compile_one(pair):
        src, obj = pair
        if not force and not _stale(obj, [src] + hdrs):
            return None
        cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        return (src, r.stderr)

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(compile_one, zip(srcs, objs)))
    if verbose:
        for r in results:
            if r:
                print("====", r[0]); print(r[1])
    if force or _stale(OUT, objs):
        cmd = [NVCC, "-shared", "-o", OUT] + objs + ["-gencode", "arch=compute_90a,code=" + ARCH, "-lcudart_static", "-Xcompiler", "-fPIC"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
