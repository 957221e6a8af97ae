"""In-tree build of libswapnet_b200.so (sm_90a, H100) with plain nvcc.

The library is a C-ABI shared object (include/swapnet_b200.h); nothing here links against
torch.  Object files live under swapnet_b200/csrc/build/, the .so next to this file so that it
travels with the source snapshot to the GPU box.
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
OUT = os.path.join(HERE, "libswapnet_b200.so")
SOURCES = ["api.cu", "gemm_tc.cu", "elementwise.cu", "roi_align.cu", "perceptual.cu", "patch_logits.cu", "augment.cu",
           "pixel_disc.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libswapnet_b200.so")


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = True) -> str:
    """Compile (if stale) and return the path of the shared library."""
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h"))]
    deps.append(os.path.join(HERE, "..", "include", "swapnet_b200.h"))
    stamp = os.path.join(CSRC, "build", "stamp")
    dig = _digest(deps)
    if not force and os.path.exists(OUT) and os.path.exists(stamp) and open(stamp).read() == dig:
        return OUT
    nvcc = _nvcc()
    os.makedirs(os.path.join(CSRC, "build"), exist_ok=True)
    objs = [os.path.join(CSRC, "build", src.replace(".cu", ".o")) for src in SOURCES]
    cmds = [[nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj] for src, obj in zip(SOURCES, objs)]
    if verbose:
        for cmd in cmds:
            print("[swapnet_b200.build]", " ".join(cmd), file=sys.stderr)
    # the sources are independent translation units: compile them side by side
    with ThreadPoolExecutor(max_workers=min(len(cmds), os.cpu_count() or 1)) as pool:
        for _ in pool.map(lambda cmd: subprocess.run(cmd, check=True), cmds):
            pass
    cmd = [nvcc, "-shared", "-o", OUT, *objs, "-Wno-deprecated-gpu-targets"]
    if verbose:
        print("[swapnet_b200.build]", " ".join(cmd), file=sys.stderr)
    subprocess.run(cmd, check=True)
    with open(stamp, "w") as f:
        f.write(dig)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
