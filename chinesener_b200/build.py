"""Build libner_b200.so (sm_90a only) in-tree with nvcc.

`python -m chinesener_b200.build` or `__graft_entry__.build()`.  Objects are rebuilt only
when a source/header is newer; translation units compile in parallel.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
OBJDIR = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libner_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--use_fast_math=false",
]
NVCC_FLAGS = [f for f in NVCC_FLAGS if f != "--use_fast_math=false"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _newest_header():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")]
    hs += [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE) if f.endswith(".h")]
    return max(os.path.getmtime(h) for h in hs)


def source_hash():
    """sha256 over every source the library is built from (csrc/*.cu, csrc/*.cuh, include/*.h, in name order): compiled
    into capi.cu and echoed by `ner_build_info()`, so a loaded .so can be matched against the tree it claims to come from."""
    import hashlib
    h = hashlib.sha256()
    files = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh"))]
    files += [os.path.join(INCLUDE, f) for f in sorted(os.listdir(INCLUDE)) if f.endswith(".h")]
    for p in files:
        h.update(os.path.basename(p).encode() + b"\0")
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()[:16]


def _compile(src, verbose):
    obj = os.path.join(OBJDIR, src[:-3] + ".o")
    srcp = os.path.join(CSRC, src)
    extra = []
    if src == "capi.cu":            # carries the source hash: recompiled whenever any source changed
        digest = source_hash()
        stamp = os.path.join(OBJDIR, "capi.hash")
        extra = ['-DNER_SOURCE_HASH="%s"' % digest]
        if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == digest:
            return obj, False
        with open(stamp, "w") as f:
            f.write(digest)
    elif os.path.exists(obj) and os.path.getmtime(obj) >= max(os.path.getmtime(srcp), _newest_header()):
        return obj, False
    cmd = [_nvcc()] + NVCC_FLAGS + extra + ["-I", INCLUDE, "-c", srcp, "-o", obj]
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.run(cmd, check=True)
    return obj, True


def build(verbose=True, force=False):
    os.makedirs(OBJDIR, exist_ok=True)
    if force:
        for f in os.listdir(OBJDIR):
            os.remove(os.path.join(OBJDIR, f))
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 2)) as ex:
        res = list(ex.map(lambda s: _compile(s, verbose), sources()))
    objs = [o for o, _ in res]
    if any(c for _, c in res) or not os.path.exists(LIB):
        cmd = [_nvcc(), "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.run(cmd, check=True)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
    print(LIB)
