"""PEPNet's fused gate-product kernels against the torch chains they replace, for pepnet_taobao's EPNet gate and each
PPNet depth, the graphed pepnet_taobao training step on both formulations, and the GEMMs' share of the step
(DESIGN.md §8).

    python scripts/bench_pepnet.py [--batches 8192 65536] [--iters 50] [--out /tmp/bench_pepnet.json]

CUDA events, warm-up first, the variants alternated round by round inside one process.  Shapes are pepnet_taobao's
(2 tasks): the EPNet product over main (N = 256, identity, no bias); PPNet depth 0 (2 segments of N = 512, ReLU with the
main linear's bias) and depth 1 (2 x 256).  The torch chain is the reference's element-wise formulation on the same GEMM
outputs, act(x + bx) * (gamma * sigmoid(z + bz)), and its autograd backward (input and bias gradients).  Algorithmic
bytes count each [B, N] tensor a pass must read or write once (fp32): forward x, z, y; backward x, z, dy, dx, dz.  The
graphed steps of both formulations are captured first and then replayed alternately.  The GEMM share is the device time
of the GEMM kernels over the device time of all kernels in one eager fp32 step, from torch.profiler in a run of its
own.  The card's name, power limit and SM clock are read in the same run.  Fails without a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200.kernels import default_kernels  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
GAMMA = 2.0
# name: (segment widths, ReLU with the linear's bias)
PASSES = {"epnet": ([256], False), "ppnet_depth0": ([512, 512], True), "ppnet_depth1": ([256, 256], True)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q[0] if q else ""}


def timed(fns, iters, warm=5):
    """Mean ms per call of each fn, alternating the fns round by round."""
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


def product_pass(B, name, iters):
    widths, relu = PASSES[name]
    T, N = len(widths), widths[0]
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(B)
    r = lambda *s: torch.randn(*s, device=dev, generator=g)  # noqa: E731
    x, z, dy = r(B, T * N), r(B, T * N), r(B, T * N)
    bxs = [0.1 * r(N) if relu else None for _ in range(T)]
    bzs = [0.1 * r(N) for _ in range(T)]
    y, dx, dz = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    cols = [slice(i * N, (i + 1) * N) for i in range(T)]
    segs = [(x[:, c], bxs[i], z[:, c], bzs[i], y[:, c], relu, GAMMA) for i, c in enumerate(cols)]
    bsegs = [(x[:, c], bxs[i], z[:, c], bzs[i], None, relu, GAMMA) for i, c in enumerate(cols)]
    K = default_kernels()
    # the torch chain per task on leaf copies (the reference's element-wise ops after its GEMMs)
    xt = [x[:, c].clone().requires_grad_(True) for c in cols]
    zt = [z[:, c].clone().requires_grad_(True) for c in cols]
    bxt = [b.clone().requires_grad_(True) if b is not None else None for b in bxs]
    bzt = [b.clone().requires_grad_(True) for b in bzs]

    def chain():
        out = []
        for i in range(T):
            a = xt[i] + bxt[i] if relu else xt[i]
            h = torch.relu(a) if relu else a
            out.append(h * (GAMMA * torch.sigmoid(zt[i] + bzt[i])))
        return out

    with torch.no_grad():
        fwd = timed({"fused": lambda: K.pepnet_gate_fwd(segs), "torch": chain}, iters)
    ys = chain()
    leaves = xt + zt + [b for b in bxt if b is not None] + bzt
    dys = [dy[:, c].contiguous() for c in cols]
    bwd = timed({"fused": lambda: K.pepnet_gate_bwd(bsegs, [dy[:, c] for c in cols], [dx[:, c] for c in cols],
                                                    [dz[:, c] for c in cols]),
                 "torch": lambda: torch.autograd.grad(ys, leaves, dys, retain_graph=True)}, iters)
    byts = {"fwd": 4 * B * T * N * 3, "bwd": 4 * B * T * N * 5}
    out = {}
    for nm, tab in (("fwd", fwd), ("bwd", bwd)):
        fu, to = tab["fused"], tab["torch"]
        bps = byts[nm] / (fu * 1e-3)
        out[nm] = {"fused_ms": round(fu, 4), "torch_ms": round(to, 4), "speedup": round(to / fu, 2),
                   "bytes": byts[nm], "fused_GBps": round(bps / 1e9, 1),
                   "fused_share_of_3.35TBps": round(bps / HBM_BYTES_PER_S, 3)}
    return out


def graphed_steps(B, iters):
    """Both formulations captured (the torch one with Fn.pepnet_usable forced off while it is built and captured),
    then replayed alternately."""
    from torcheasyrec_b200.engine import GraphedTrainStep, Pipeline

    steps = {}
    real = Fn.pepnet_usable
    for name in ("fused", "torch"):
        if name == "torch":
            Fn.pepnet_usable = lambda *a, **k: False
        try:
            p = Pipeline("pepnet_taobao", device="cuda", max_rows=1_000_000, seed=1)
            batches = [p.synthetic_batch(B, seed=i) for i in range(2)]
            step = GraphedTrainStep(p, batches[0], warmup=3)
            step.load(batches[1].pin_memory())
            steps[name] = (p, step)
        finally:
            Fn.pepnet_usable = real
    res = timed({k: v[1].replay for k, v in steps.items()}, iters)
    del steps
    torch.cuda.empty_cache()
    return {"fused_ms": round(res["fused"], 3), "torch_ms": round(res["torch"], 3),
            "speedup": round(res["torch"] / res["fused"], 3)}


def gemm_share(B):
    """Device time of GEMM kernels / of every kernel, in one eager fp32 pepnet_taobao step (fused gates)."""
    from torch.profiler import ProfilerActivity, profile

    from torcheasyrec_b200.engine import Pipeline

    p = Pipeline("pepnet_taobao", device="cuda", max_rows=1_000_000, seed=1, capturable=False)
    batch = p.synthetic_batch(B, seed=0).to("cuda")
    for _ in range(3):
        p.eager_step(batch)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        p.eager_step(batch)
        torch.cuda.synchronize()
    tot, gemm, pep = 0.0, 0.0, 0.0
    for ev in prof.key_averages():
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        if t <= 0 or ev.key.startswith("cuda") or ev.key.startswith("Memcpy") or ev.key.startswith("Memset"):
            continue
        tot += t
        k = ev.key.lower()
        if "gemm" in k or "xmma" in k or "cutlass" in k:
            gemm += t
        if "tzk_pepnet" in k:
            pep += t
    del p
    torch.cuda.empty_cache()
    return {"kernels_ms": round(tot / 1e3, 3), "gemm_ms": round(gemm / 1e3, 3), "pepnet_gate_ms": round(pep / 1e3, 3),
            "gemm_share": round(gemm / tot, 3) if tot else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[8192, 65536])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_pepnet.py measures on the GPU; no CUDA device is visible")
    torch.backends.cuda.matmul.allow_tf32 = False
    res = {"card": card(), "passes": {k: {"widths": v[0], "relu_with_bias": v[1]} for k, v in PASSES.items()}}
    for B in args.batches:
        res[f"B{B}"] = {"passes": {nm: product_pass(B, nm, args.iters) for nm in PASSES},
                        "graphed_step": graphed_steps(B, max(10, args.iters // 5)), "eager_step_kernels": gemm_share(B)}
        print(json.dumps({f"B{B}": res[f"B{B}"]}), flush=True)
    res["card_after"] = card()
    print(json.dumps(res["card"]), json.dumps(res["card_after"]))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
