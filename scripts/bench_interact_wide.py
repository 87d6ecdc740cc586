"""Times DLRM-Criteo's interaction + first final-MLP layer at B = 65536 with CUDA events, each pass against the
layer-by-layer chain it replaces, and checks that both give the same bits:
  forward          interaction forward -> X [B, 784], then gemm3x  vs  tzk_interact_wide_fwd (Y and the pair columns)
  input gradient   gemm3x dgrad dZ -> dX [B, 784], then the interaction backward  vs  tzk_interact_wide_bwd
  weight gradient  wgrad3x on the materialised X  vs  tzk_interact_wide_wgrad on pairs, dense and sparse

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
    bias = torch.randn(64, device="cuda", generator=g) / 4
    K = default_kernels()
    x = K.dot_interact_fwd(dense, sparse, 26, 16, True, True, 4, 1)
    pairs = x[:, :352].contiguous()

    def fwd_chain():
        xx = K.dot_interact_fwd(dense, sparse, 26, 16, True, True, 4, 1)
        return G.gemm3x(lib, xx, w, bias, True), xx[:, :352]

    def fwd_fused():
        return K.interact_wide_fwd(dense, sparse, w, bias)

    def wgrad_x():
        return (G.wgrad3x(lib, x, dz),)

    def wgrad_sources():
        return (K.interact_wide_wgrad(dz, pairs, dense, sparse, G.SLABS),)

    def chain():
        dx = G.gemm3x(lib, dz, w.t().contiguous(), None, False)
        return K.dot_interact_bwd(dense, sparse, dx, 26, 16, True, True, p_pad=1)

    def fused():
        return K.interact_wide_bwd(dz, w, dense, sparse)

    # per pass: MMA work (3 MMAs per product; padded MMA work is not counted) and, per variant, algorithmic B/sample
    passes = {
        "forward": (2 * 3 * B * (64 * 784 + 351 * 16), {
            # E 1728 + X write 3136 | X 3136 + Y 256
            "chain (interaction fwd + gemm3x)": (fwd_chain, 1728 + 3136 + 3136 + 256),
            # E 1728 + pairs 1408 + Y 256
            "fused (tzk_interact_wide_fwd)": (fwd_fused, 1728 + 1408 + 256)}),
        "input gradient": (2 * 3 * B * (64 * 784 + 27 * 27 * 16), {
            # dZ 256 + dX write 3136 | dX 3136 + E 1728 + dE 1728
            "chain (gemm3x dgrad + interaction bwd)": (chain, 256 + 3136 + 3136 + 1728 + 1728),
            # dZ 256 + E 1728 + dE 1728, plus the pass-through part of dE written and read back through L2 (not counted)
            "fused (tzk_interact_wide_bwd)": (fused, 256 + 1728 + 1728)}),
        "weight gradient": (2 * 3 * B * 64 * 784, {
            # X 3136 + dZ 256
            "wgrad3x on X": (wgrad_x, 3136 + 256),
            # pairs 1408 + E 1728 + dZ 256
            "tzk_interact_wide_wgrad on pairs, dense, sparse": (wgrad_sources, 1408 + 1728 + 256)}),
    }
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = {"gpu": smi, "batch": B, "passes": {}}
    for pname, (mma_flop, variants) in passes.items():
        (ref_fn, _), (new_fn, _) = variants.values()
        ref, new = ref_fn(), new_fn()
        res = {"bitwise_equal": all(bool(torch.equal(r, n)) for r, n in zip(ref, new)),
               "max_abs_diff": max((r - n).abs().max().item() for r, n in zip(ref, new)), "variants": {}}
        for name, (fn, bps) in variants.items():
            us = timed(fn, a.iters)
            t_mem, t_mma = bps * B / HBM_BPS, mma_flop / TF32_FLOPS
            bound = "HBM" if t_mem >= t_mma else "TF32"
            res["variants"][name] = {
                "us": round(us, 1), "bytes_per_sample": bps, "GB_per_s": round(bps * B / us / 1e3, 1),
                "TF32_equiv_TFLOP_per_s": round(mma_flop / us / 1e6, 1), "bound": bound,
                "share_of_bound": round(max(t_mem, t_mma) * 1e6 / us, 3)}
        out["passes"][pname] = res
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
