"""Build libmugd.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m mug_diffusion_b200.build [--force]

The .so and the object files are build products (git-ignored); build() of __graft_entry__.py runs this.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmugd.so")
STAMP = os.path.join(HERE, "build", "libmugd.stamp")
SOURCES = ["api.cu", "norm.cu", "gemm_simt.cu", "gemm_tc.cu", "attention.cu", "attention_tc.cu", "s4.cu", "elementwise.cu", "plan_io.cu", "melspec.cu", "gridscan.cu", "chartpost.cu", "plms.cu", "ddpm.cu", "remix.cu", "dpm.cu", "randn.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=default", "--use_fast_math=false",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _digest() -> str:
    h = hashlib.sha256()
    files = sorted(os.listdir(CSRC)) + [os.path.join("..", "..", "include", "mugd.h")]
    for f in files:
        p = os.path.join(CSRC, f)
        if os.path.isfile(p):
            h.update(f.encode())
            with open(p, "rb") as fh:
                h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read().strip() == dig:
        return LIB
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    nvcc = _nvcc()
    flags = [f for f in NVCC_FLAGS if f != "--use_fast_math=false"]
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc, *flags, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0:
            failed = True
            sys.stderr.write(f"--- nvcc failed for {src} ---\n{out}\n")
        elif verbose or out.strip():
            sys.stderr.write(f"--- {src} ---\n{out}\n")
    if failed:
        raise RuntimeError("libmugd build failed")
    cmd = [nvcc, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
    subprocess.check_call(cmd)
    with open(STAMP, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
