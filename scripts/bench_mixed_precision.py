"""DLRM-Criteo with train_config.mixed_precision "BF16" against fp32 on one GPU.

    python scripts/bench_mixed_precision.py [--batch 65536] [--steps 20] [--rounds 5] [--max-rows 0]

Reports, as one JSON line:
  * step: GraphedTrainStep time per step of DLRM-Criteo (full hash sizes unless --max-rows), fp32 against BF16;
  * interact: the BF16 interaction kernels (tzk_dot_interact27_fwd_bf16 / _bwd_bf16) against the torch autocast chain
    they replace (bmm + triu gather + cats, and its autograd backward), in microseconds.
Every number is the median over --rounds rounds with the two sides alternating inside each round, with the range; CUDA
events around --steps back-to-back calls after a warm-up.  The GPU's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e!r})"}


def _time(fn, n):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / n


def _summary(xs, scale=1.0):
    xs = [x * scale for x in xs]
    return {"median": round(statistics.median(xs), 3), "min": round(min(xs), 3), "max": round(max(xs), 3), "n": len(xs)}


def bench_steps(args):
    from torcheasyrec_b200.engine import GraphedTrainStep, Pipeline

    sides = {}
    for mp in ("", "BF16"):
        pipe = Pipeline("dlrm_criteo", device="cuda:0", max_rows=args.max_rows or None, seed=1,
                        edits={"train_config.mixed_precision": mp} if mp else None)
        batches = [pipe.synthetic_batch(args.batch, seed=20260923 + i).pin_memory() for i in range(2)]
        step = GraphedTrainStep(pipe, batches[0], warmup=3)
        step.load(batches[1])
        sides[mp or "fp32"] = step
    times = {k: [] for k in sides}
    for _ in range(args.rounds):
        for k, step in sides.items():
            step.replay()
            torch.cuda.synchronize()
            times[k].append(_time(step.replay, args.steps))
    out = {k: _summary(v) for k, v in times.items()}
    out["unit"] = "ms/step"
    out["loss_last"] = {k: float(s.loss) for k, s in sides.items()}
    return out


def bench_interact(args):
    from torcheasyrec_b200 import functional as Fn
    from torcheasyrec_b200.kernels import default_kernels

    k = default_kernels()
    B = args.batch
    torch.manual_seed(0)
    dense = torch.randn(B, 16, device="cuda").to(torch.bfloat16).requires_grad_()
    sparse = torch.randn(B, 416, device="cuda", requires_grad=True)
    dx_b = torch.randn(B, 784, device="cuda").to(torch.bfloat16)
    dx_t = torch.cat([dx_b[:, :351], dx_b[:, 352:]], dim=1).float()

    def torch_fwd():
        with torch.autocast("cuda", torch.bfloat16):
            return Fn.dlrm_interaction(dense, sparse, 26, 16, aligned=True)[0]

    with torch.autocast("cuda", torch.bfloat16):
        xt = Fn.dlrm_interaction(dense, sparse, 26, 16, aligned=True)[0]

    def torch_bwd():
        torch.autograd.grad(xt, (dense, sparse), dx_t, retain_graph=True)

    d, s = dense.detach(), sparse.detach()
    sides = {"kernel_fwd": lambda: k.dot_interact27_fwd_bf16(d, s),
             "torch_fwd": lambda: torch_fwd(),
             "kernel_bwd": lambda: k.dot_interact27_bwd_bf16(dx_b, d, s),
             "torch_bwd": torch_bwd}
    for fn in sides.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {n: [] for n in sides}
    for _ in range(args.rounds):
        for n, fn in sides.items():
            times[n].append(_time(fn, args.steps))
    out = {n: _summary(v, 1000.0) for n, v in times.items()}
    out["unit"] = "us/call"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--max-rows", type=int, default=0, help="cap every table at this many rows (0: full hash sizes)")
    ap.add_argument("--skip-steps", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mixed_precision.py measures on a GPU; none is visible")
    res = {"what": "DLRM-Criteo, train_config.mixed_precision BF16 vs fp32", "batch": args.batch, **_gpu_info()}
    res["interact"] = bench_interact(args)
    if not args.skip_steps:
        res["step"] = bench_steps(args)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
