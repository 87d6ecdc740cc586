"""Where the time of the fused interaction + wide-layer input gradient (interact_wide_bwd_kernel in
torcheasyrec_b200/csrc/tzk_interact_wide.cu) goes, per 64-sample tile: the kernel is built with TZK_FB_TIMING, which
records %globaltimer at four points of every tile (start, dZ split, ring drained = end of the GEMM phase, end of the
per-sample phase; the last one is the latest warp's), and run at B = 65536 on the DLRM-Criteo shape.

Prints one JSON line: per phase the median and mean ns per tile, the kernel's span (first start to last end) and the
card's name and power limit.  The instrumented build goes to a temporary directory; the tree is not written.

    python scripts/phase_split_interact_wide.py [--batch 65536] [--reps 20] [--src path/to/tzk_interact_wide.cu]
"""
import argparse
import ctypes
import json
import os
import subprocess
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "torcheasyrec_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--src", default=os.path.join(CSRC, "tzk_interact_wide.cu"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    with tempfile.TemporaryDirectory() as d:
        so = os.path.join(d, "libfb_timing.so")
        subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC", "-shared", "-DTZK_FB_TIMING", "-I", os.path.dirname(os.path.abspath(a.src)),
                        "-I", CSRC, a.src, "-o", so], check=True)
        # tzk_common.cuh's error reporting lives in the package's libtzk.so
        ctypes.CDLL(os.path.join(CSRC, "libtzk.so"), mode=ctypes.RTLD_GLOBAL)
        lib = ctypes.CDLL(so)
    P, I64 = ctypes.c_void_p, ctypes.c_int64
    lib.tzk_interact_wide_bwd.argtypes = [P, I64, P, I64, P, I64, P, I64, I64, P, I64, P, I64, P, P, P]
    lib.tzk_interact_wide_bwd_timing.argtypes = [P]

    B = a.batch
    g = torch.Generator(device="cuda").manual_seed(0)
    dense = torch.randn(B, 16, device="cuda", generator=g)
    sparse = torch.randn(B, 416, device="cuda", generator=g)
    dz = torch.randn(B, 64, device="cuda", generator=g) / 8
    w = torch.randn(64, 784, device="cuda", generator=g) / 28
    dd, ds = torch.empty(B, 16, device="cuda"), torch.empty(B, 416, device="cuda")
    wh, wl = torch.empty(784, 64, device="cuda"), torch.empty(784, 64, device="cuda")
    tiles = (B + 63) // 64
    buf = torch.zeros(tiles, 4, dtype=torch.int64, device="cuda")
    assert lib.tzk_interact_wide_bwd_timing(buf.data_ptr()) == 0
    stream = torch.cuda.current_stream().cuda_stream

    def run():
        assert lib.tzk_interact_wide_bwd(dz.data_ptr(), 64, w.data_ptr(), 784, dense.data_ptr(), 16, sparse.data_ptr(),
                                         416, B, dd.data_ptr(), 16, ds.data_ptr(), 416, wh.data_ptr(), wl.data_ptr(),
                                         stream) == 0

    for _ in range(3):
        run()
    phases = {"start_to_dz_split": [], "gemm_phase": [], "per_sample_phase": [], "tile": []}
    spans = []
    for _ in range(a.reps):
        buf.zero_()
        run()
        torch.cuda.synchronize()
        t = buf.double()
        assert (t > 0).all(), "a tile recorded no time"
        for name, d in zip(phases, (t[:, 1] - t[:, 0], t[:, 2] - t[:, 1], t[:, 3] - t[:, 2], t[:, 3] - t[:, 0])):
            phases[name].append(d)
        spans.append((t[:, 3].max() - t[:, 0].min()).item())
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    out = {"gpu": smi, "batch": B, "tiles": tiles, "src": os.path.relpath(os.path.abspath(a.src), ROOT),
           "kernel_span_us_median": round(sorted(spans)[len(spans) // 2] / 1e3, 1), "ns_per_tile": {}}
    for name, ds_ in phases.items():
        v = torch.cat(ds_)
        out["ns_per_tile"][name] = {"median": round(v.median().item()), "mean": round(v.mean().item())}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
