"""PLE's fused gate passes against the torch chains they replace, per ple_taobao extraction layer, the graphed ple_taobao
training step on both paths, and the GEMMs' share of the step (DESIGN.md §8).

    python scripts/bench_ple.py [--batches 8192 65536] [--iters 50] [--out /tmp/bench_ple.json]

CUDA events, warm-up first, the variants alternated inside one process.  Layer shapes are ple_taobao's (2 tasks):
layer 1 K = 256 (one input for all gates), H = 256, gates over 4 / 4 / 6 experts; layer 2 K = 256 (three inputs),
H = 64, gates over 6 / 6 / 9; layer 3 K = 64 (two inputs), H = 32, gates over 8 / 8.  The torch chain is the
reference's `_gate_forward` per gate (Linear, softmax, stack, matmul) and its autograd backward.  Algorithmic bytes
count each tensor a pass must read or write once (fp32).  The GEMM share is the device time of the GEMM kernels over
the device time of all kernels in one eager fp32 step, from torch.profiler in a run of its own.  The card's name,
power limit and SM clock are read in the same run.  Fails without a GPU.
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

T = 2
# name: (K, H, experts per task, shared experts, final, one input tensor for every gate)
LAYERS = {"layer1": (256, 256, 2, 2, False, True), "layer2": (256, 64, 3, 3, False, False),
          "layer3": (64, 32, 4, 4, True, False)}


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


def layer_pass(B, name, iters):
    K_, H, per, S, final, one = LAYERS[name]
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(B)
    r = lambda *s: torch.randn(*s, device=dev, generator=g)  # noqa: E731
    shared = list(range(T * per, T * per + S))
    ge = [list(range(i * per, (i + 1) * per)) + shared for i in range(T)] + ([] if final else [list(range(T * per + S))])
    n_in = 1 if one else (T if final else T + 1)
    gi = [0] * len(ge) if one else ([i for i in range(T)] + ([] if final else [T]))
    inputs = [r(B, K_) for _ in range(n_in)]
    experts = [r(B, H) for _ in range(T * per + S)]
    weights = [0.1 * r(len(ids), K_) for ids in ge]
    biases = [0.1 * r(len(ids)) for ids in ge]
    dy = r(len(ge), B, H)
    Kn = default_kernels()
    _, p = Kn.ple_gate_fwd(inputs, gi, weights, biases, experts, ge)
    # the torch chain on leaf copies
    x_t = [x.clone().requires_grad_(True) for x in inputs]
    e_t = [e.clone().requires_grad_(True) for e in experts]
    w_t = [w.clone().requires_grad_(True) for w in weights]
    b_t = [b.clone().requires_grad_(True) for b in biases]

    def chain():
        out = []
        for j, ids in enumerate(ge):
            vec = torch.stack([e_t[x] for x in ids], dim=1)
            gate = torch.softmax(torch.nn.functional.linear(x_t[gi[j]], w_t[j], b_t[j]), dim=1).unsqueeze(1)
            out.append(torch.matmul(gate, vec).squeeze(1))
        return out

    with torch.no_grad():
        fwd = timed({"fused": lambda: Kn.ple_gate_fwd(inputs, gi, weights, biases, experts, ge), "torch": chain}, iters)
    ys = chain()
    leaves = x_t + e_t + w_t + b_t
    dys = list(dy.unbind(0))
    bwd = timed({"fused": lambda: Kn.ple_gate_bwd(inputs, gi, weights, biases, experts, ge, p, dy),
                 "torch": lambda: torch.autograd.grad(ys, leaves, dys, retain_graph=True)}, iters)
    f4, G, sumE = 4 * B, len(ge), sum(len(ids) for ids in ge)
    byts = {"fwd": f4 * (n_in * K_ + len(experts) * H + G * H + sumE),
            "bwd": f4 * (n_in * K_ + len(experts) * H + G * H + sumE + len(experts) * H + n_in * K_)}
    out = {}
    for nm, tab in (("fwd", fwd), ("bwd", bwd)):
        fu, to = tab["fused"], tab["torch"]
        out[nm] = {"fused_ms": round(fu, 4), "torch_ms": round(to, 4), "speedup": round(to / fu, 2),
                   "bytes": byts[nm], "fused_GBps": round(byts[nm] / fu / 1e6, 1)}
    return out


def graphed_step(B, iters):
    from torcheasyrec_b200.engine import GraphedTrainStep, Pipeline

    res = {}
    real = Fn.ple_gate_usable
    for name in ("fused", "torch"):
        if name == "torch":
            Fn.ple_gate_usable = lambda *a, **k: False
        try:
            p = Pipeline("ple_taobao", device="cuda", max_rows=1_000_000, seed=1)
            batches = [p.synthetic_batch(B, seed=i) for i in range(2)]
            step = GraphedTrainStep(p, batches[0], warmup=3)
            step.load(batches[1].pin_memory())
            res[name] = timed({"s": step.replay}, iters)["s"]
            del step, p
            torch.cuda.empty_cache()
        finally:
            Fn.ple_gate_usable = real
    return {"fused_ms": round(res["fused"], 3), "torch_ms": round(res["torch"], 3),
            "speedup": round(res["torch"] / res["fused"], 3)}


def gemm_share(B):
    """Device time of GEMM kernels / of every kernel, in one eager fp32 ple_taobao step (fused gates)."""
    from torch.profiler import ProfilerActivity, profile

    from torcheasyrec_b200.engine import Pipeline

    p = Pipeline("ple_taobao", device="cuda", max_rows=1_000_000, seed=1, capturable=False)
    batch = p.synthetic_batch(B, seed=0).to("cuda")
    for _ in range(3):
        p.eager_step(batch)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        p.eager_step(batch)
        torch.cuda.synchronize()
    tot, gemm, ple = 0.0, 0.0, 0.0
    for ev in prof.key_averages():
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        if t <= 0 or ev.key.startswith("cuda") or ev.key.startswith("Memcpy") or ev.key.startswith("Memset"):
            continue
        tot += t
        k = ev.key.lower()
        if "gemm" in k or "xmma" in k or "cutlass" in k:
            gemm += t
        if "tzk_ple" in k:
            ple += t
    del p
    torch.cuda.empty_cache()
    return {"kernels_ms": round(tot / 1e3, 3), "gemm_ms": round(gemm / 1e3, 3), "ple_gates_ms": round(ple / 1e3, 3),
            "gemm_share": round(gemm / tot, 3) if tot else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[8192, 65536])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ple.py measures on the GPU; no CUDA device is visible")
    res = {"card": card(), "layers": {k: dict(zip(("K", "H", "per_task", "shared", "final", "one_input"), v))
                                      for k, v in LAYERS.items()}}
    for B in args.batches:
        res[f"B{B}"] = {"layers": {nm: layer_pass(B, nm, args.iters) for nm in LAYERS},
                        "graphed_step": graphed_step(B, max(10, args.iters // 5)), "eager_step_kernels": gemm_share(B)}
        print(json.dumps({f"B{B}": res[f"B{B}"]}), flush=True)
    res["card_after"] = card()
    print(json.dumps(res["card"]), json.dumps(res["card_after"]))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
