"""Times the input-gradient side of DLRM-Criteo's interaction + first final-MLP layer at B = 65536 with CUDA events:
the layer-by-layer chain (gemm3x input gradient dZ -> dX [B, 784], then the tensor-core interaction backward dX -> dE)
against the fused kernel (tzk_interact_wide_bwd), and checks that both give the same bits.

Prints, per variant, the time per call, the algorithmic bytes per sample and GB/s, TF32-equivalent FLOP/s (3 MMAs per
product, as the 3xTF32 split issues them) and the share of the H100 SXM data-sheet bound that applies.

    python scripts/bench_interact_wide.py [--batch 65536] [--iters 200]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torcheasyrec_b200 import dense_gemm as G  # noqa: E402
from torcheasyrec_b200.kernels import default_kernels  # noqa: E402

HBM_BPS = 3.35e12          # H100 SXM data sheet
TF32_FLOPS = 495e12        # dense


def timed(fn, iters):
    for _ in range(5):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) * 1e3 / iters      # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    B = a.batch
    lib = G._gemm3x_lib()
    if lib is None or not torch.cuda.is_available():
        raise SystemExit("needs a GPU and libtzk_gemm3x.so")
    g = torch.Generator(device="cuda").manual_seed(0)
    dense = torch.randn(B, 16, device="cuda", generator=g)
    sparse = torch.randn(B, 416, device="cuda", generator=g)
    dz = torch.randn(B, 64, device="cuda", generator=g) / 8
    w = torch.randn(64, 784, device="cuda", generator=g) / 28
    w[:, 351] = 0
    K = default_kernels()

    def chain():
        dx = G.gemm3x(lib, dz, w.t().contiguous(), None, False)
        return K.dot_interact_bwd(dense, sparse, dx, 26, 16, True, True, p_pad=1)

    def fused():
        return K.interact_wide_bwd(dz, w, dense, sparse)

    c_d, c_s = chain()
    f_d, f_s = fused()
    same = bool(torch.equal(c_d, f_d) and torch.equal(c_s, f_s))
    maxdiff = max((c_d - f_d).abs().max().item(), (c_s - f_s).abs().max().item())

    mma_flop = 2 * 3 * B * (64 * 784 + 27 * 27 * 16)        # dgrad + S E (padded MMA work is not counted)
    variants = {
        # dZ 256 + dX write 3136 | dX 3136 + E 1728 + dE 1728
        "chain (gemm3x dgrad + interaction bwd)": (chain, 256 + 3136 + 3136 + 1728 + 1728),
        # dZ 256 + E 1728 + dE 1728, plus the pass-through part of dE written and read back through L2 (not counted)
        "fused (tzk_interact_wide_bwd)": (fused, 256 + 1728 + 1728),
    }
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = {"gpu": smi, "batch": B, "bitwise_equal": same, "max_abs_diff": maxdiff, "variants": {}}
    for name, (fn, bps) in variants.items():
        us = timed(fn, a.iters)
        t_mem, t_mma = bps * B / HBM_BPS, mma_flop / TF32_FLOPS
        bound = "HBM" if t_mem >= t_mma else "TF32"
        out["variants"][name] = {
            "us": round(us, 1), "bytes_per_sample": bps, "GB_per_s": round(bps * B / us / 1e3, 1),
            "TF32_equiv_TFLOP_per_s": round(mma_flop / us / 1e6, 1), "bound": bound,
            "share_of_bound": round(max(t_mem, t_mma) * 1e6 / us, 3)}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
