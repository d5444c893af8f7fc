"""Build the C-ABI shared library (capital_b200/libcapital_b200.so) with nvcc for sm_90a (H100), in-tree.

    python -m capital_b200.build [--force]

No GPU is needed (nvcc cross-compiles).  Also used by __graft_entry__.build().
"""
from __future__ import annotations
import os, subprocess, sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "csrc", "_obj")
LIB = os.path.join(HERE, "libcapital_b200.so")
SOURCES = ["api.cu", "gemm_tn.cu", "leaf.cu", "layout.cu", "cholinv_local.cu", "dist.cu", "peer.cu", "gemm_tf32.cu", "solve.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
# -dlcm=cg: plain global loads are cached in L2 only.  Buffers of the multi-GPU path are written by OTHER processes' copy engines and
# kernels (peer DMA into mirror / gather slots, remote epilogue stores into exchange buffers and C replicas) and re-used every few
# products; an L1 line that survives from the previous use would be read back stale (seen as a handful of wrong 128-byte lines when
# kernels of two streams overlap, i.e. when "kernel boundaries" no longer flush an SM's L1).  L2 is the coherence point for those
# writes.  The hot loops do not depend on L1 (TMA -> shared memory, or explicit __ldcg), and the layout kernels are streaming.
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "-Xcompiler", "-fvisibility=hidden", "-Xptxas", "-v", "-Xptxas", "-dlcm=cg"]


def _newer(a: str, b: str) -> bool:
    return (not os.path.exists(b)) or os.path.getmtime(a) > os.path.getmtime(b)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(HERE, "..", "include", "capital_b200.h"))
    jobs = []
    for s in SOURCES:
        src, obj = os.path.join(CSRC, s), os.path.join(OBJ, s.replace(".cu", ".o"))
        if force or _newer(src, obj) or any(_newer(h, obj) for h in headers):
            jobs.append((src, obj))

    def cc(job):
        src, obj = job
        r = subprocess.run([NVCC, *FLAGS, "-c", src, "-o", obj], capture_output=True, text=True)
        return src, r

    with ThreadPoolExecutor(max_workers=8) as ex:
        for src, r in ex.map(cc, jobs):
            if verbose or r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed on {src}")
    objs = [os.path.join(OBJ, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or not os.path.exists(LIB):
        r = subprocess.run([NVCC, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-ldl",
                            "-Xcompiler", "-fPIC"], capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
