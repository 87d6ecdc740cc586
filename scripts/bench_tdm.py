"""TDM's fused multi-window DIN attention (csrc/tzk_tdm.cuh) against the torch jagged chain and the reference's padded
formulation, and `bench.py --model tdm_taobao` (DESIGN.md §8).

    python scripts/bench_tdm.py [--iters 50] [--out /tmp/bench_tdm.json]

Forward + backward of the tdm_taobao encoder (C = Dq = 48, windows 1,1,1,2,2,2,5,6,10,20, attn_mlp [36] PReLU) at
B = 8192 and 65536 with lengths drawn from the synthetic mix {0, 1, U[2, 50], 50} (about 19 rows per sample).
"fused" is functional.multiwindow_din, "torch" functional.torch_multiwindow_din over the same jagged rows, "padded"
the encoder's padded [B, T, C] path (the reference's formulation; the padding is done outside the timed region).
Then the example's eager training step at B = 8192 with each path, and `bench.py --model tdm_taobao --batch-size
8192` in a subprocess.  CUDA events, warm-up first, the variants alternated round by round in one process.

FLOPs and bytes come from the shapes: the attention MLP's forward is 2 (3C H + H) FLOP per row, the backward
recomputes it and adds about twice that; the fused kernels' essential bytes are the rows read twice forward (MLP and
pooling) and backward plus d rows written, z, the outputs and the upstream gradient.  The card's name and power limit
are read in the same run.  Fails without a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200.rank_models import MultiWindowDINEncoder  # noqa: E402

WINDOWS = [1, 1, 1, 2, 2, 2, 5, 6, 10, 20]
C, H = 48, 36
FP32_TFLOPS, HBM_TBS = 67.0, 3.35         # H100 SXM data sheet, dense FP32 and HBM3


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


def inputs(B, seed):
    g = torch.Generator().manual_seed(seed)
    kind = torch.randint(0, 4, (B,), generator=g)
    lens = torch.where(kind == 0, 0, torch.where(kind == 1, 1, torch.where(
        kind == 2, torch.randint(2, 51, (B,), generator=g), 50)))
    off = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(lens, 0)])
    q = torch.randn(B, C, generator=g) * 0.5
    seq = torch.randn(int(off[-1]), C, generator=g) * 0.5
    return q.cuda(), seq.cuda(), off.cuda(), lens.cuda()


def model(B, N):
    L = len(WINDOWS)
    mlp_fwd = 2.0 * N * (3 * C * H + H) + 2.0 * N * C          # attention MLP and pooling
    flops = {"fwd": mlp_fwd, "bwd": 3.0 * mlp_fwd}
    byts = {"fwd": 4.0 * (2 * N * C + N + B * (L + 1) * C + B * C),
            "bwd": 4.0 * (2 * N * C + N + N * C + B * (L + 1) * C + 2 * B * C)}
    t_min = {k: max(flops[k] / (FP32_TFLOPS * 1e12), byts[k] / (HBM_TBS * 1e12)) * 1e3 for k in flops}
    bound = {k: "FP32" if flops[k] / (FP32_TFLOPS * 1e12) > byts[k] / (HBM_TBS * 1e12) else "HBM" for k in flops}
    return flops, byts, t_min, bound


def encoder_calls(iters):
    torch.manual_seed(0)
    enc = MultiWindowDINEncoder(C, C, "seq", WINDOWS, dict(hidden_units=[H], activation="nn.PReLU")).cuda()
    out = {}
    for B in (8192, 65536):
        q, seq, off, lens = inputs(B, B)
        N = seq.shape[0]
        assert Fn.multiwindow_din_usable(q, seq, enc.mlp, WINDOWS)
        qq, ss = q.clone().requires_grad_(True), seq.clone().requires_grad_(True)
        T = int(lens.max())
        pad = torch.zeros(B, T, C, device="cuda")
        pos = torch.arange(N, device="cuda") - torch.repeat_interleave(off[:-1], lens)
        pad[torch.repeat_interleave(torch.arange(B, device="cuda"), lens), pos] = seq
        pp = pad.requires_grad_(True)
        emb_p = {"seq.query": qq, "seq.sequence": pp, "seq.sequence_length": lens}

        def run(f):
            def go():
                y = f()
                y.backward(torch.ones_like(y))
            return go

        fns = {"fused": run(lambda: Fn.multiwindow_din(qq, ss, off, enc.mlp, enc.linear, enc.active, WINDOWS)),
               "torch": run(lambda: Fn.torch_multiwindow_din(qq, ss, off, enc.mlp, enc.linear, enc.active, WINDOWS)),
               "padded": run(lambda: enc(emb_p))}
        both = timed(fns, iters)
        fwd = timed({"fused": lambda: Fn.multiwindow_din(qq, ss, off, enc.mlp, enc.linear, enc.active, WINDOWS)}, iters)
        flops, byts, t_min, bound = model(B, N)
        out[f"B{B}"] = {"rows": N, "rows_per_sample": N / B, "fwd_bwd_ms": both, "fused_fwd_ms": fwd["fused"],
                        "fused_bwd_ms_by_difference": both["fused"] - fwd["fused"], "flops": flops, "bytes": byts,
                        "least_time_ms": t_min, "bound": bound}
    return out


def train_step(iters):
    """The tdm_taobao example's eager training step (sequence workloads step eagerly) at B = 8192, full tables, with
    the fused attention and with it forced onto the torch jagged chain, alternated."""
    from torcheasyrec_b200.engine import Pipeline

    example = os.path.join(ROOT, "tests", "golden", "ref_examples", "tdm_taobao.config")
    pipe = Pipeline(example, device="cuda", seed=3, capturable=False)
    batch = pipe.synthetic_batch(8192, seed=1).to("cuda")
    real = Fn.multiwindow_din_usable

    def step(fused):
        def go():
            Fn.multiwindow_din_usable = real if fused else (lambda *a, **k: False)
            try:
                pipe.eager_step(batch)
            finally:
                Fn.multiwindow_din_usable = real
        return go

    return timed({"fused": step(True), "torch": step(False)}, iters)


def bench_py():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--model", "tdm_taobao",
                        "--batch-size", "8192", "--steps", "50", "--warmup", "10"], capture_output=True, text=True,
                       cwd=ROOT)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    return json.loads(lines[-1]) if lines else {"returncode": r.returncode, "stderr": r.stderr[-3000:]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default="")
    ap.add_argument("--no-bench-py", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tdm needs a GPU")
    res = {"card": card(), "encoder": encoder_calls(a.iters), "train_step_B8192_ms": train_step(a.iters)}
    if not a.no_bench_py:
        res["bench_py"] = bench_py()
    txt = json.dumps(res, indent=1, default=str)
    print(txt)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(txt)


if __name__ == "__main__":
    main()
