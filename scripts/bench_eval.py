"""Evaluation on one GPU: the graphed eval step of DLRM-Criteo, and tzk_binned_auc_update against torchmetrics' update.

    python scripts/bench_eval.py [--batch 65536] [--steps 20] [--rounds 5] [--max-rows 0]

Reports, as one JSON line:
  * step: GraphedEvalStep of DLRM-Criteo (full hash sizes unless --max-rows) in ms per step and samples/s, with the
    GraphedTrainStep of the same model and batch in ms per step for context;
  * auc_update: tzk_binned_auc_update at --batch predictions and T = 200 / 1000 / 10000 thresholds, in microseconds,
    against the torch formulation of torchmetrics' binned update (`(p[:, None] >= thr).long()` -> one bincount over
    (threshold, label, above) cells), run in chunks of predictions so that the [chunk, T] comparison fits in memory.
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
    return {"median": round(statistics.median(xs), 3), "min": round(min(xs), 3), "max": round(max(xs), 3)}


def torch_binned_update(p, y, thr, confmat, chunk):
    """torchmetrics' _binary_precision_recall_curve_update_vectorized, chunked over the predictions."""
    T = thr.numel()
    base = 4 * torch.arange(T, device=p.device)
    for s in range(0, p.numel(), chunk):
        pt = (p[s:s + chunk, None] >= thr[None, :]).long()
        idx = pt + 2 * y[s:s + chunk, None].long() + base
        confmat += torch.bincount(idx.flatten(), minlength=4 * T).reshape(T, 2, 2)


def bench_auc(B, steps, rounds):
    from torcheasyrec_b200.kernels import default_kernels

    k = default_kernels()
    g = torch.Generator(device="cuda").manual_seed(0)
    p = torch.rand(B, device="cuda", generator=g)
    y = (torch.rand(B, device="cuda", generator=g) < 0.25).float()
    out = {}
    for T in (200, 1000, 10000):
        thr = torch.linspace(0, 1, T, device="cuda")
        counts = torch.zeros((T + 1, 2), dtype=torch.int64, device="cuda")
        invalid = torch.zeros(1, dtype=torch.int64, device="cuda")
        confmat = torch.zeros((T, 2, 2), dtype=torch.int64, device="cuda")
        chunk = max(1, (256 << 20) // (8 * T))          # [chunk, T] int64 cells: at most 256 MB per pass
        ours = lambda: k.binned_auc_update(p, y, thr, counts, invalid)
        ref = lambda: torch_binned_update(p, y, thr, confmat, chunk)
        ours(), ref()
        torch.cuda.synchronize()
        ta, tb = [], []
        for _ in range(rounds):
            ta.append(_time(ours, steps))
            tb.append(_time(ref, max(1, steps // 4)))
        # same counts: tps[k] of the confusion matrix = samples with bin > k
        counts.zero_(), confmat.zero_()
        ours(), ref()
        above = counts.flip(0).cumsum(0).flip(0)[1:]
        assert torch.equal(above, confmat[:, :, 1]), f"T={T}: histogram and confusion matrix disagree"
        out[f"T{T}"] = {"tzk_us": _summary(ta, 1000.0), "torch_us": _summary(tb, 1000.0),
                        "speedup": round(statistics.median(tb) / statistics.median(ta), 1)}
    return out


def bench_step(B, steps, rounds, max_rows):
    from torcheasyrec_b200.engine import GraphedEvalStep, GraphedTrainStep, Pipeline

    pipe = Pipeline("dlrm_criteo", device="cuda:0", max_rows=max_rows or None, seed=1)
    batch = pipe.synthetic_batch(B, seed=1)
    train = GraphedTrainStep(pipe, batch, warmup=3)
    ev = GraphedEvalStep(pipe, batch)
    for _ in range(3):
        train.replay(), ev.replay()
    torch.cuda.synchronize()
    te, tt = [], []
    for _ in range(rounds):
        te.append(_time(ev.replay, steps))
        tt.append(_time(train.replay, steps))
    pipe.model.compute_metric()
    return {"eval_ms": _summary(te), "eval_samples_per_s": round(B / (statistics.median(te) / 1000.0)),
            "train_ms": _summary(tt), "batch": B, "max_rows": max_rows or "full"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--max-rows", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py measures on a CUDA device; none is visible")
    res = {**_gpu_info(), "auc_update": bench_auc(args.batch, args.steps, args.rounds),
           "step": bench_step(args.batch, args.steps, args.rounds, args.max_rows)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
