"""Build libdasp_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m dasp_pytorch_b200.build [--force] [--verbose]

The shared library lands next to this file, so the package imports from the repository tree
without an install step (the library and the object files under build/ are git-ignored).
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
# experiments: DASP_NVCC_DEFS="-DDASP_EQ_E=7" DASP_LIB_SUFFIX=_e7 python -m dasp_pytorch_b200.build --force
LIB = os.path.join(HERE, f"libdasp_b200{os.environ.get('DASP_LIB_SUFFIX', '')}.so")
SOURCES = ["abi.cu", "pointwise.cu", "stereo.cu", "dynamics.cu", "biquad.cu", "reverb.cu"]

ARCH = "arch=compute_90a,code=sm_90a"
NVCC_FLAGS = [
    "-gencode", ARCH,
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC,-O3,-Wall",
    "-Xptxas", "-v",
]


def _nvcc() -> str:
    cand = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")
    return cand


def _stale(objs_srcs) -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(INCLUDE, "dasp_b200.h"), __file__]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    if not force and not _stale(srcs):
        return LIB
    nvcc = _nvcc()
    cuda_lib = os.path.join(os.path.dirname(os.path.dirname(nvcc)), "lib64")
    objs = []
    logs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in srcs:
        obj = os.path.join(HERE, "build", os.path.basename(src) + os.environ.get("DASP_LIB_SUFFIX", "") + ".o")
        cmd = [nvcc, *NVCC_FLAGS, *os.environ.get("DASP_NVCC_DEFS", "").split(), "-I", INCLUDE, "-I", CSRC, "-c", src, "-o", obj]
        procs.append((src, cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, cmd, p in procs:
        out, _ = p.communicate()
        logs.append(f"$ {' '.join(cmd)}\n{out}")
        if p.returncode != 0:
            sys.stderr.write(logs[-1])
            raise RuntimeError(f"nvcc failed on {src}")
    link = [nvcc, "-gencode", ARCH, "-shared", "-o", LIB, *objs, "-L", cuda_lib, "-lcufft", "-lcudart",
            "-Xlinker", f"-rpath={cuda_lib}"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    logs.append(f"$ {' '.join(link)}\n{r.stdout}")
    if r.returncode != 0:
        sys.stderr.write(logs[-1])
        raise RuntimeError("link failed")
    with open(os.path.join(HERE, "build", "build.log"), "w") as f:
        f.write("\n".join(logs))
    if verbose:
        print("\n".join(logs))
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
