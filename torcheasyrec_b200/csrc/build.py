"""Builds libtzk.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

No torch dependency: plain `nvcc -shared`.  Objects are rebuilt only when a source is newer.
"""

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SOURCES = ["tzk_core.cu", "tzk_gather.cu", "tzk_bwd.cu", "tzk_dist.cu", "tzk_dense.cu", "tzk_tower.cu", "tzk_din.cu", "tzk_peer.cu", "tzk_interact_wide.cu",
           "tzk_interact_bf16.cu", "tzk_metrics.cu", "tzk_wukong.cu",
           "tzk_masknet.cu", "tzk_ple.cu", "tzk_pepnet.cu"]
HEADERS = ["tzk_common.cuh", "tzk_tower_bwd2.cuh", "tzk_interact_tc.cuh", "tzk_tower_tail.cuh", "tzk_interact_bf16.cuh",
           "tzk_metrics.cuh", "tzk_wukong.cuh", "tzk_masknet.cuh", "tzk_ple.cuh", "tzk_pepnet.cuh", "tzk_launch.cuh",
           "tzk_batch_sum.cuh",
"tzk_sm90_ptx.h", "tzk_tma.h", "tzk_wgrad3x.cuh", "tzk_wgmma.cuh", os.path.join("..", "..", "include", "tzk.h")]
LIB = os.path.join(HERE, "libtzk.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _mtime(p):
    return os.path.getmtime(p) if os.path.exists(p) else 0.0


def build(verbose: bool = False, force: bool = False) -> str:
    hdr_time = max(_mtime(os.path.join(HERE, h)) for h in HEADERS)
    objs = []
    procs = []
    for src in SOURCES:
        s = os.path.join(HERE, src)
        o = os.path.join(HERE, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _mtime(o) < max(_mtime(s), hdr_time):
            cmd = [NVCC, *FLAGS, "-c", s, "-o", o]
            if verbose:
                cmd.insert(1, "-Xptxas")
                cmd.insert(2, "-v")
                print(" ".join(cmd), flush=True)
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"nvcc failed for {src}:\n{out}\n")
        elif verbose and out:
            print(out)
    if failed:
        raise RuntimeError("libtzk build failed")
    if force or procs or _mtime(LIB) < max(_mtime(o) for o in objs):
        # link next to the target and rename: a reader (another process) never sees a torn library
        cmd = [NVCC, "-shared", "-Wno-deprecated-gpu-targets", "-o", LIB + ".tmp", *objs]
        subprocess.run(cmd, check=True)
        os.replace(LIB + ".tmp", LIB)
    build_gemm(force)
    build_gemm3x(force)
    return LIB


def build_gemm3x(force: bool = False) -> str:
    """libtzk_gemm3x.so: hand-written TMA + mma.sync 3xTF32 GEMMs of the wide tower layer (forward, dgrad, wgrad)."""
    src = os.path.join(HERE, "tzk_gemm3x.cu")
    lib = os.path.join(HERE, "libtzk_gemm3x.so")
    deps = [src] + [os.path.join(HERE, h) for h in ("tzk_launch.cuh", "tzk_sm90_ptx.h", "tzk_tma.h", "tzk_wgrad3x.cuh")]
    if force or _mtime(lib) < max(_mtime(d) for d in deps):
        subprocess.run([NVCC, *FLAGS, "-shared", src, "-o", lib + ".tmp"], check=True)
        os.replace(lib + ".tmp", lib)
    return lib


def build_gemm(force: bool = False) -> str:
    """libtzk_gemm.so: the cuBLASLt-12.9 BF16x9 wrapper for the dense towers (host C++, dlopen at run time)."""
    src = os.path.join(HERE, "tzk_gemm.cpp")
    lib = os.path.join(HERE, "libtzk_gemm.so")
    if force or _mtime(lib) < _mtime(src):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I/usr/local/cuda/include", src, "-o", lib,
                        "-ldl"], check=True)
    return lib


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
