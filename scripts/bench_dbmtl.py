"""The fused JRC loss (csrc/tzk_jrc.cuh) against the reference's [B, B] formulation, its kernels one by one, and the
dbmtl_taobao_jrc training step graphed and eager (DESIGN.md §8).

    python scripts/bench_dbmtl.py [--iters 50] [--out /tmp/bench_dbmtl.json]

CUDA events, warm-up first, the variants alternated round by round inside one process.  Loss calls: forward and
backward of one tower's loss on B samples with mean session sizes 1, 8, 64 and B (ids uniform over B / size sessions,
labels 1 with probability 0.3).  "fused" is functional.jrc_loss (tzk_jrc_loss, 64 key bits); "bxb" restates the
reference's formulation (tzrec/loss/jrc_loss.py:68-117: a [B, B] session mask, [P, B] / [N, B] tiles of logits, masks
and labels, two cross-entropies) with its autograd backward; it reads the positive count on the host.  Algorithmic bytes
of the fused call: the inputs once (logits 8, label 4, session id 8 B per sample) and the gradient once (8 B), the
sort (keys 8 + index 4 B per sample, read and written by each of its passes over 64 bits: 8 passes of 8 bits), and the
three passes (each reads the sorted key and index and its per-sample operands: 12 + 12, 12 + 20, 12 + 16 B).  At
B = 65536 the [B, B] formulation's bytes are printed (>= 36 B^2 by its shapes) and it is not run.  Per-kernel times
come from torch.profiler in a run of its own.  Steps: the graphed dbmtl_taobao_jrc step at B = 8192 and 65536; at
8192 also eager steps on the fused loss, on functional.torch_jrc_loss (O(B), syncs) and on the [B, B] formulation.  The
card's name and power limit are read in the same run.  Fails without a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from torcheasyrec_b200 import functional as Fn  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
SIZES = (1, 8, 64, "B")


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


def bxb_jrc(logits, labels, session_ids, alpha=0.5):
    """The reference's [B, B] formulation (mean reduction), restated."""
    y = labels.long()
    ce = F.cross_entropy(logits, y)
    B = y.shape[0]
    mask = torch.eq(session_ids.unsqueeze(1), session_ids.unsqueeze(0)).float()
    diag_index = torch.arange(B, device=logits.device)
    diag = torch.eye(B, dtype=torch.int64, device=logits.device)
    pos_num = int(y.sum())
    neg_num = B - pos_num
    out = []
    for cls, num, col in ((1, pos_num, 1), (0, neg_num, 0)):
        idx = torch.where(y == cls)[0]
        lg = logits[:, col].unsqueeze(0).tile([num, 1])
        yy = (y if cls == 1 else 1 - y).unsqueeze(0).tile([num, 1])
        lg = lg + ((1 - mask.index_select(0, idx)) + (1 - diag.index_select(0, idx)) * yy) * -1e9
        out.append(F.cross_entropy(lg, diag_index.index_select(0, idx)) * num / B)
    return alpha * ce + (1 - alpha) * (out[0] + out[1])


def case(B, size, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    L = B if size == "B" else size
    logits = (torch.randn(B, 2, device="cuda", generator=g) * 2).requires_grad_(True)
    y = (torch.rand(B, device="cuda", generator=g) < 0.3).float()
    s = torch.randint(0, max(1, B // L), (B,), device="cuda", generator=g)
    return logits, y, s


def fused_bytes(B):
    return B * (8 + 4 + 8 + 8) + 8 * B * (12 * 2) + B * (24 + 32 + 28)


def loss_calls(iters):
    rows = []
    for B in (8192, 16384):
        for size in SIZES:
            logits, y, s = case(B, size)

            def fused():
                Fn.jrc_loss(logits, y, s, 0.5).backward()

            def bxb():
                bxb_jrc(logits, y, s).backward()

            t = timed({"fused": fused, "bxb": bxb}, iters)
            nb = fused_bytes(B)
            rows.append({"B": B, "session_size": size, "fused_ms": t["fused"], "bxb_ms": t["bxb"],
                         "speedup": t["bxb"] / t["fused"], "fused_bytes": nb,
                         "fused_GBps": nb / t["fused"] / 1e6, "fused_frac_hbm": nb / (t["fused"] * 1e-3) / HBM_BYTES_PER_S,
                         "bxb_bytes_lower_bound": 36 * B * B})
    for size in SIZES:
        logits, y, s = case(65536, size)
        t = timed({"fused": lambda: Fn.jrc_loss(logits, y, s, 0.5).backward()}, iters)
        rows.append({"B": 65536, "session_size": size, "fused_ms": t["fused"], "bxb_ms": "not run",
                     "bxb_bytes_lower_bound": 36 * 65536 * 65536, "fused_bytes": fused_bytes(65536),
                     "fused_frac_hbm": fused_bytes(65536) / (t["fused"] * 1e-3) / HBM_BYTES_PER_S})
    return rows


def kernel_split(B=65536, size=8):
    """Device time per kernel of one fused call (forward + backward), from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    logits, y, s = case(B, size)
    for _ in range(3):
        Fn.jrc_loss(logits, y, s, 0.5).backward()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            Fn.jrc_loss(logits, y, s, 0.5).backward()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0):
            t = getattr(e, "self_device_time_total", 0) or getattr(e, "self_cuda_time_total", 0)
            if t:
                out[e.key[:80]] = t / 10 / 1000.0     # ms per call
    return {"B": B, "session_size": size, "ms_per_call": dict(sorted(out.items(), key=lambda kv: -kv[1]))}


def steps(iters):
    from torcheasyrec_b200.engine import GraphedTrainStep, Pipeline

    path = os.path.join(ROOT, "tests", "golden", "ref_examples", "dbmtl_taobao_jrc.config")
    out = {}
    for B in (8192, 65536):
        p = Pipeline(path, device="cuda", seed=3)
        batch = p.synthetic_batch(B, seed=1)
        step = GraphedTrainStep(p, batch, warmup=3)
        step.load(batch.pin_memory())
        out[f"graphed_B{B}_ms"] = timed({"g": step.replay}, iters)["g"]
        del step, p
        torch.cuda.empty_cache()
    p = Pipeline(path, device="cuda", seed=3, capturable=False)
    dev = p.synthetic_batch(8192, seed=1).to("cuda")
    real = Fn.jrc_loss

    def torch_path(logits, labels, sid, alpha, weights=None, key_bits=64):
        return Fn.torch_jrc_loss(logits.float(), labels, sid, alpha)

    def bxb_path(logits, labels, sid, alpha, weights=None, key_bits=64):
        return bxb_jrc(logits.float(), labels, sid, alpha)

    t = {}
    for name, fn in (("fused", real), ("torch_O(B)", torch_path), ("bxb", bxb_path)):
        Fn.jrc_loss = fn
        try:
            t[name] = timed({"s": lambda: p.eager_step(dev)}, iters)["s"]
        finally:
            Fn.jrc_loss = real
    out["eager_B8192_ms"] = t
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dbmtl needs a GPU")
    res = {"card": card(), "loss_calls": loss_calls(a.iters), "kernels": kernel_split(), "steps": steps(a.iters)}
    txt = json.dumps(res, indent=1, default=str)
    print(txt)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(txt)


if __name__ == "__main__":
    main()
