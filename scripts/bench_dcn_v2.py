"""DCN-v2's fused cross network (csrc/tzk_dcn_v2.cuh) against the reference's torch loop, and the graphed dcn_v2_taobao
training step with each (DESIGN.md §8).

    python scripts/bench_dcn_v2.py [--iters 50] [--out /tmp/bench_dcn_v2.json]

Cross network shapes (D, L, r): (128, 2, 32) the docs example after its backbone, (256, 2, 32) the docs config without
the backbone, (256, 3, 64) the widest rank at D = 256; each at B = 8192 and 65536.  "fused" is functional.cross_v2,
"torch" functional.torch_cross_v2 with the same weights (TF32 off: fp32 GEMMs).  CUDA events, warm-up first, the two
paths alternated round by round in one process.  A torch.profiler pass per shape at B = 65536 then gives each kernel's
own time, set against the least time its algorithmic bytes and FLOPs allow:
  fwd          reads x0, writes y and v:                    4 B (2 D + L r) bytes,   4 B D r L FLOPs
  bwd_data     reads x0, dy, v, writes dx0 and dv:          4 B (3 D + 2 L r) bytes, 6 B D r L FLOPs
  bwd_weight   reads x0, dy, v, dv:                         4 B (2 D + 2 L r) bytes, 8 B D r L FLOPs
The 3xTF32 split issues three TF32 MMAs per product, so the compute bound is 3 x FLOPs at the data sheet's dense TF32
rate.  The steps: dcn_v2_taobao graphed at B = 8192 and 65536, the torch path picked by patching
Fn.cross_v2_usable.  The card's name and power limit are read in the same run.  Fails without a GPU.
"""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200.rank_models import CrossV2  # noqa: E402

SHAPES = [(128, 2, 32), (256, 2, 32), (256, 3, 64)]
TF32_TFLOPS, HBM_TBS = 495.0, 3.35        # H100 SXM data sheet, dense TF32 and HBM3
MAX_ROWS = 1_000_000                      # the graphed steps cap every table (the cross network does not read them)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q[0] if q else ""}


def timed(fns, iters, warm=5):
    for f in fns.values():
        for _ in range(warm):
            f()
    torch.cuda.synchronize()
    tot = {k: 0.0 for k in fns}
    for _ in range(iters):
        for k, f in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            tot[k] += a.elapsed_time(b)
    return {k: v / iters for k, v in tot.items()}


def bounds(B, D, L, r):
    """Least time (ms) of each kernel from its algorithmic bytes (HBM) and 3xTF32 FLOPs, and which of the two binds."""
    byts = {"fwd": 4.0 * B * (2 * D + L * r), "bwd_data": 4.0 * B * (3 * D + 2 * L * r),
            "bwd_weight": 4.0 * B * (2 * D + 2 * L * r)}
    flops = {"fwd": 4.0 * B * D * r * L, "bwd_data": 6.0 * B * D * r * L, "bwd_weight": 8.0 * B * D * r * L}
    out = {}
    for k in byts:
        t_hbm = byts[k] / (HBM_TBS * 1e12) * 1e3
        t_tc = 3 * flops[k] / (TF32_TFLOPS * 1e12) * 1e3
        out[k] = {"bytes": byts[k], "flops": flops[k], "hbm_ms": t_hbm, "tf32x3_ms": t_tc,
                  "least_ms": max(t_hbm, t_tc), "bound": "HBM" if t_hbm >= t_tc else "3xTF32"}
    return out


def kernel_times(fn, iters=20):
    """ms per call of every CUDA kernel `fn` launches, from torch.profiler (a run of its own)."""
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and getattr(e, "self_device_time_total", 0) > 0:
            out[e.key] = e.self_device_time_total / iters / 1e3
    return out


def cross_calls(iters):
    out = {}
    for D, L, r in SHAPES:
        torch.manual_seed(0)
        cross = CrossV2(D, L, r).cuda()
        for B in (8192, 65536):
            x = torch.randn(B, D, device="cuda").requires_grad_(True)
            dy = torch.randn(B, D, device="cuda")
            # (256, 3, 64) is past Fn.DCN_V2_MAX_DR: the model runs it on the torch path; timed here on both
            assert Fn.cross_v2_usable(x, cross.u_kernels, cross.v_kernels) == (D * r <= Fn.DCN_V2_MAX_DR)

            def fwd_bwd(f):
                def go():
                    f(x, cross.u_kernels, cross.v_kernels).backward(dy)
                return go

            def fwd(f):
                def go():
                    with torch.no_grad():
                        f(x, cross.u_kernels, cross.v_kernels)
                return go

            rec = {"fwd_ms": timed({"fused": fwd(Fn.cross_v2), "torch": fwd(Fn.torch_cross_v2)}, iters),
                   "fwd_bwd_ms": timed({"fused": fwd_bwd(Fn.cross_v2), "torch": fwd_bwd(Fn.torch_cross_v2)}, iters)}
            if B == 65536:
                ks = kernel_times(fwd_bwd(Fn.cross_v2))
                b = bounds(B, D, L, r)
                mine = {}
                for name, ms in ks.items():
                    for k in ("fwd", "bwd_data", "bwd_weight", "prep", "reduce"):
                        if f"{k}_kernel" in name:
                            mine[k] = mine.get(k, 0.0) + ms
                rec["kernels_ms"] = mine
                rec["bounds"] = b
                rec["fraction_of_least_time"] = {k: b[k]["least_ms"] / mine[k] for k in b if mine.get(k)}
            out[f"D{D}_L{L}_r{r}_B{B}"] = rec
            del x, dy
    return out


def steps(iters):
    from torcheasyrec_b200.engine import GraphedTrainStep, Pipeline

    out = {}
    real = Fn.cross_v2_usable
    for B in (8192, 65536):
        for name in ("fused", "torch"):
            if name == "torch":
                Fn.cross_v2_usable = lambda *a, **k: False
            try:
                p = Pipeline("dcn_v2_taobao", device="cuda", seed=3, max_rows=MAX_ROWS)
                batch = p.synthetic_batch(B, seed=1)
                step = GraphedTrainStep(p, batch, warmup=3)
                step.load(batch.pin_memory())
                out[f"graphed_B{B}_{name}_ms"] = timed({"g": step.replay}, iters)["g"]
            finally:
                Fn.cross_v2_usable = real
            del step, p
            gc.collect()
            torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dcn_v2 needs a GPU")
    res = {"card": card(), "cross": cross_calls(a.iters), "steps": steps(a.iters)}
    txt = json.dumps(res, indent=1, default=str)
    print(txt)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(txt)


if __name__ == "__main__":
    main()
