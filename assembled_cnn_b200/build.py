"""In-tree build of libacnn.so (sm_90a only) with plain nvcc -- no JIT cache, no torch extension.

`python -m assembled_cnn_b200.build` or `__graft_entry__.build()`.  nvcc cross-compiles without a
GPU; the resulting .so sits next to this file, so the package imports from the source tree.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ_DIR = os.path.join(HERE, "build")
LIB_PATH = os.path.join(HERE, "libacnn.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr", "--extended-lambda",
]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libacnn.so cannot be built")


def _sources() -> list[str]:
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(path: str) -> str:
    h = hashlib.sha1()
    h.update(" ".join(NVCC_FLAGS).encode())
    # every header change rebuilds everything that can include it (few files, seconds each); the
    # model-level headers are only seen by csrc/model_*.cu
    model_src = os.path.basename(path).startswith("model_")
    inc = os.path.join(HERE, "..", "include")
    headers = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".h", ".cuh"))]
    headers += [os.path.join(inc, f) for f in sorted(os.listdir(inc)) if f.endswith(".h")]
    for f in headers:
        if os.path.basename(f) in ("model_plan.h", "acnn_model.h") and not model_src:
            continue
        with open(f, "rb") as fh:
            h.update(fh.read())
    with open(path, "rb") as fh:
        h.update(fh.read())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every csrc/*.cu and link libacnn.so.  Returns the library path."""
    os.makedirs(OBJ_DIR, exist_ok=True)
    nvcc = _nvcc()
    srcs = _sources()
    objs, jobs = [], []
    for s in srcs:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ_DIR, s[:-3] + ".o")
        stamp = obj + ".sha1"
        dig = _digest(src)
        objs.append(obj)
        fresh = (not force and os.path.exists(obj) and os.path.exists(stamp)
                 and open(stamp).read() == dig)
        if not fresh:
            jobs.append((src, obj, stamp, dig))

    def compile_one(job):
        src, obj, stamp, dig = job
        cmd = [nvcc] + NVCC_FLAGS + ["-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        with open(stamp, "w") as fh:
            fh.write(dig)

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(compile_one, jobs))
    if jobs or not os.path.exists(LIB_PATH):
        cmd = [nvcc, "-shared", "-o", LIB_PATH] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
