"""In-tree build of libb200zk.so (CUDA kernels + C ABI) for sm_90a (H100) with plain nvcc.

`python -m distributed_groth16_b200.build` or `build()` from __graft_entry__.py.  nvcc
cross-compiles without a GPU."""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libb200zk.so")
SOURCES = ["api.cu", "ntt.cu", "msm.cu", "prove.cu", "qap.cu", "setup.cu", "codec.cu", "verify.cu", "packexp.cu", "group.cu",
           "selftest.cu"]
ARCH = "sm_90a"
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = GENCODE + ["-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-O2"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _deps_mtime() -> float:
    t = os.path.getmtime(os.path.abspath(__file__))          # flags live here: a flag change rebuilds
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for f in os.listdir(root):
            t = max(t, os.path.getmtime(os.path.join(root, f)))
    return t


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= _deps_mtime():
        sys.stderr.write("distributed_groth16_b200.build: %s is newer than every source under csrc/ and include/: reused "
                         "(build(force=True) recompiles)\n" % os.path.relpath(LIB))
        return LIB
    sys.stderr.write("distributed_groth16_b200.build: compiling %d translation units for %s with %s\n" % (len(SOURCES), ARCH, _nvcc()))
    os.makedirs(OBJ, exist_ok=True)
    nvcc = _nvcc()
    extra = ["-Xptxas", "-v"] if verbose else []

    def compile_one(src):
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + extra + ["-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    r = subprocess.run([nvcc, "-shared", "-o", LIB] + objs + GENCODE,
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
