"""RocketLaunching's fused head (csrc/tzk_rocket.cuh) against the reference's torch chain, and the
rocket_launching_criteo training step with each (DESIGN.md §8).

    python scripts/bench_rocket.py [--iters 50] [--out /tmp/bench_rocket.json]

CUDA events, warm-up first, the variants alternated round by round inside one process.  Head calls: forward and
backward of everything after the two MLPs of rocket_launching_criteo (light and booster hidden 32, two classes, the
pairs light 64 / booster 64 and light 32 / booster 32, COSINE) at B = 8192 and 65536; "fused" is functional.rocket_head,
"torch" functional.torch_rocket_head with the reference's nn.Linear heads.  Steps: the graphed rocket_launching_criteo
step at B = 8192 and 65536 (tables capped at 10^6 rows) with the fused head, and with the head forced onto torch_rocket_head; then
`bench.py --model rocket_launching_criteo --batch-size 8192` in a subprocess.  The card's name and power limit are read
in the same run.  Fails without a GPU.
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

MAX_ROWS = 1_000_000           # the graphed steps cap every table (the head does not depend on the tables)
EXAMPLE = os.path.join(ROOT, "tests", "golden", "ref_examples", "rocket_launching_criteo.config")


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


def head_calls(iters):
    out = {}
    for B in (8192, 65536):
        g = torch.Generator(device="cuda").manual_seed(B)
        def r(*s):
            return torch.randn(*s, generator=g, device="cuda")
        hl, hb = torch.relu(r(B, 32)).requires_grad_(), torch.relu(r(B, 32)).requires_grad_()
        lin_l, lin_b = torch.nn.Linear(32, 2).cuda(), torch.nn.Linear(32, 2).cuda()
        pairs = [(torch.relu(r(B, 64)).requires_grad_(), torch.relu(r(B, 64))), (hl, hb)]
        labels = torch.randint(0, 2, (B,), generator=g, device="cuda").float()

        def fused():
            _, _, losses = Fn.rocket_head([(hl, lin_l.weight, lin_l.bias), (hb, lin_b.weight, lin_b.bias)], labels,
                                          0.0, pairs, Fn.ROCKET_COSINE)
            torch.stack(losses).sum().backward()

        def chain():
            _, _, losses = Fn.torch_rocket_head([(hl, lin_l), (hb, lin_b)], labels, 0.0, pairs, Fn.ROCKET_COSINE)
            torch.stack(losses).sum().backward()

        out[f"B{B}_fwd_bwd_ms"] = timed({"fused": fused, "torch": chain}, iters)
    return out


def steps(iters):
    from torcheasyrec_b200.engine import GraphedTrainStep, Pipeline

    out = {}
    real = Fn.rocket_head_usable
    for B in (8192, 65536):
        for name in ("fused", "torch"):
            if name == "torch":
                Fn.rocket_head_usable = lambda *a, **k: False
            try:
                p = Pipeline(EXAMPLE, device="cuda", seed=3, max_rows=MAX_ROWS)
                batch = p.synthetic_batch(B, seed=1)
                step = GraphedTrainStep(p, batch, warmup=3)
                step.load(batch.pin_memory())
                out[f"graphed_B{B}_{name}_ms"] = timed({"g": step.replay}, iters)["g"]
            finally:
                Fn.rocket_head_usable = real
            del step, p
            gc.collect()
            torch.cuda.empty_cache()
    return out


def bench_py():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--model",
                        "rocket_launching_criteo", "--batch-size", "8192", "--steps", "50", "--warmup", "10"],
                       capture_output=True, text=True, cwd=ROOT)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    return json.loads(lines[-1]) if lines else {"returncode": r.returncode, "stderr": r.stderr[-2000:]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rocket needs a GPU")
    res = {"card": card(), "head_calls": head_calls(a.iters), "steps": steps(a.iters), "bench_py": bench_py()}
    txt = json.dumps(res, indent=1, default=str)
    print(txt)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(txt)


if __name__ == "__main__":
    main()
