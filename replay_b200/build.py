"""Build replay_b200/librp_b200.so from csrc/*.cu with nvcc for sm_90a (cross-compiles without a GPU).

    python -m replay_b200.build [--force]

The .so is built in the source tree (git-ignored).  cudart is linked statically; the only
driver symbol (cuTensorMapEncodeTiled) is resolved at run time through cudaGetDriverEntryPoint.
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "librp_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--use_fast_math",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "-I", os.path.join(os.path.dirname(HERE), "include"),
] + os.environ.get("RP_NVCC_EXTRA", "").split()   # diagnostic builds only (e.g. -DRP_ATTN_TRACE), never the shipped library


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(path):
    h = hashlib.sha1()
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cuh", ".h")) or os.path.join(CSRC, f) == path:
            with open(os.path.join(CSRC, f), "rb") as fh:
                h.update(fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _compile(src):
    path = os.path.join(CSRC, src)
    obj = os.path.join(OBJ, src[:-3] + ".o")
    stamp = obj + ".sha1"
    dig = _digest(path)
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
        return obj, False
    cmd = [NVCC, *FLAGS, "-c", path, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as fh:
        fh.write(dig)
    return obj, True


def build(force: bool = False, verbose: bool = True) -> str:
    os.makedirs(OBJ, exist_ok=True)
    if force:
        for f in os.listdir(OBJ):
            os.remove(os.path.join(OBJ, f))
    srcs = _sources()
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        res = list(ex.map(_compile, srcs))
    objs = [o for o, _ in res]
    changed = any(c for _, c in res)
    if changed or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB, *objs, "-cudart", "static", "-Xlinker", "--no-undefined", "-lpthread", "-ldl", "-lrt"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(f"[replay_b200.build] built {LIB} from {len(srcs)} sources", file=sys.stderr)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
