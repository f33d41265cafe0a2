"""Build libidiff_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

No torch / pybind dependency: plain `nvcc -shared`.  The .so lands next to the sources
(instancediffusion_b200/csrc/libidiff_b200.so) so it travels with the repo snapshot.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc")
LIB = os.path.join(CSRC, "libidiff_b200.so")
LIB_BF16 = os.path.join(CSRC, "libidiff_b200_bf16.so")  # same sources, -DIDIFF_STORAGE_BF16=1 (include/idiff_b200.h)
SOURCES = ["host.cu", "gemm2.cu", "attention.cu", "norm.cu", "scaleu.cu", "elementwise.cu", "convnext.cu", "vae.cu", "clip.cu"]
HEADERS = ["common.cuh", "host.cuh", "wgmma.cuh", os.path.join("..", "..", "include", "idiff_b200.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found; cannot build libidiff_b200.so")
    return cand


def _digest() -> str:
    h = hashlib.sha256()
    for f in SOURCES + HEADERS:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every .cu to an object (in parallel), once per storage type, and link the two shared libraries."""
    stamp = os.path.join(CSRC, ".build_stamp")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(LIB_BF16) and os.path.exists(stamp):
        with open(stamp) as fh:
            if fh.read().strip() == dig:
                return LIB
    nvcc = _nvcc()
    objs = {LIB: [], LIB_BF16: []}
    procs = []
    for lib, suffix, defs in ((LIB, ".o", []), (LIB_BF16, ".bf16.o", ["-DIDIFF_STORAGE_BF16=1"])):
        for src in SOURCES:
            obj = os.path.join(CSRC, src.replace(".cu", suffix))
            objs[lib].append(obj)
            cmd = [nvcc, *NVCC_FLAGS, *defs, "-c", os.path.join(CSRC, src), "-o", obj]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            procs.append((src + suffix, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"[build] {src} failed:\n{out}\n")
        elif verbose or out.strip():
            sys.stderr.write(f"[build] {src}:\n{out}\n")
    if failed:
        raise RuntimeError("nvcc compilation failed")
    for lib, lobjs in objs.items():
        link = [nvcc, "-shared", "-o", lib, *lobjs, "-gencode", "arch=compute_90a,code=sm_90a"]
        r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout)
    with open(stamp, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
