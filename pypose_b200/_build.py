"""In-tree build of libb200pose.so (sm_90a, H100, only).

`python -m pypose_b200._build` or `__graft_entry__.build()`.  nvcc cross-compiles without a GPU.
Objects are cached under pypose_b200/csrc/build/ keyed on source mtimes and the compile flags; the shared
library is written to pypose_b200/lib/, where pypose_b200._C loads it from the source tree.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "build")
LIB = os.path.join(HERE, "lib", "libb200pose.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr"]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers_mtime():
    m = 0.0
    for f in os.listdir(CSRC):
        if f.endswith((".cuh", ".h")):
            m = max(m, os.path.getmtime(os.path.join(CSRC, f)))
    inc = os.path.join(os.path.dirname(HERE), "include")
    if os.path.isdir(inc):
        for f in os.listdir(inc):
            m = max(m, os.path.getmtime(os.path.join(inc, f)))
    return m


def _compile(src, hm, verbose):
    s = os.path.join(CSRC, src)
    o = os.path.join(OBJ, src[:-3] + ".o")
    if os.path.exists(o) and os.path.getmtime(o) >= max(os.path.getmtime(s), hm):
        return o, False
    cmd = [NVCC] + FLAGS + ["-I", CSRC, "-I", os.path.join(os.path.dirname(HERE), "include"), "-c", s, "-o", o]
    if verbose:
        print(" ".join(cmd), flush=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    return o, True


def build(verbose=False, force=False):
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    stamp = os.path.join(OBJ, "flags.txt")
    key = " ".join([NVCC] + FLAGS)
    if not force and (not os.path.exists(stamp) or open(stamp).read() != key):
        force = True                       # objects built with other flags (another architecture) are not reused
    if force:
        for f in os.listdir(OBJ):
            os.remove(os.path.join(OBJ, f))
        if os.path.exists(LIB):
            os.remove(LIB)
        with open(stamp, "w") as f:
            f.write(key)
    hm = _headers_mtime()
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        res = list(ex.map(lambda s: _compile(s, hm, verbose), srcs))
    objs = [o for o, _ in res]
    changed = any(c for _, c in res)
    if changed or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(o) for o in objs):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ARCH
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(verbose=True, force="--force" in sys.argv))
