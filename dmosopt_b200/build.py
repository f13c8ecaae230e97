"""Build libdmosopt_b200.so in-tree with nvcc for sm_90a (H100).

    python -m dmosopt_b200.build            # incremental
    python -m dmosopt_b200.build --force    # rebuild everything

nvcc cross-compiles without a GPU; the resulting .so sits next to this file (git-ignored).
"""

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "build")
LIB = os.path.join(HERE, "libdmosopt_b200.so")

SOURCES = ["ctx.cu", "prims.cu", "rank.cu", "sortmo.cu", "variation.cu", "gp.cu", "gp_fit.cu", "gp_tensor.cu", "gp_multitask.cu", "gp_multitask_fit.cu", "gp_variational.cu", "gp_variational_fit.cu", "gp_deep.cu", "gp_deep_fit.cu", "hv.cu", "hv3_tree.cu", "hv_many.cu", "hv_mc.cu", "epsilon.cu", "sa.cu", "design.cu", "feasibility.cu", "moea_ext.cu", "smpso.cu", "cmaes_step.cu", "benchmarks.cu", "step.cu"]

NVCC_FLAGS = [
    "-gencode",
    "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "-O3",
    "-std=c++17",
    "-Xcompiler",
    "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas",
    "-v",
]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _digest(paths):
    h = hashlib.sha256()
    h.update(" ".join(NVCC_FLAGS).encode())
    for p in paths:
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _headers():
    hs = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(os.path.dirname(HERE), "include", "dmosopt_b200.h"))
    return hs


def _compile(src, force, log):
    obj = os.path.join(OBJ, src.replace(".cu", ".o"))
    stamp = obj + ".sha"
    dg = _digest([os.path.join(CSRC, src)] + _headers())
    if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dg:
        return obj, False
    cmd = [_nvcc()] + NVCC_FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    with open(os.path.join(OBJ, src + ".log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(dg)
    if log:
        print(f"[dmosopt_b200.build] compiled {src}", flush=True)
    return obj, True


def build(force=False, verbose=True):
    os.makedirs(OBJ, exist_ok=True)
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        res = list(ex.map(lambda s: _compile(s, force, verbose), srcs))
    objs = [o for o, _ in res]
    changed = any(c for _, c in res)
    if changed or not os.path.exists(LIB):
        cmd = [_nvcc(), "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(f"[dmosopt_b200.build] linked {LIB}", flush=True)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
