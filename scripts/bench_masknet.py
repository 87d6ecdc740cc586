"""MaskNet's fused passes against the torch chains they replace, the step's GEMM time, and the graphed masknet_criteo
training step on both paths (DESIGN.md §8).

    python scripts/bench_masknet.py [--batches 8192 65536] [--iters 50] [--out /tmp/bench_masknet.json]

CUDA events, warm-up first, the variants alternated inside one process.  Shapes are masknet_criteo's: E = 429 (pitch
432), A = 1287 (pitch 1288), H = 512, 3 parallel blocks.  Algorithmic bytes count each tensor a pass must read or write
once (fp32).  The card's name, power limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from torcheasyrec_b200 import dense_gemm  # noqa: E402
from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200.kernels import default_kernels  # noqa: E402

E, A, H, NB = 429, 1287, 512, 3
EP, AP = 432, 1288


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


def passes(B, iters):
    K = default_kernels()
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(B)
    r = lambda *s: torch.randn(*s, device=dev, generator=g)  # noqa: E731
    e = torch.zeros(B, EP, device=dev)
    e[:, :E] = r(B, E)
    m, dv = r(B, NB * EP), r(B, NB * EP)
    b2, lw, lb = r(NB * E), 1 + 0.1 * r(E), 0.1 * r(E)
    z, dy = r(B, NB * H), r(B, NB * H)
    b3, fw, fb = r(NB * H), 1 + 0.1 * r(NB * H), 0.1 * r(NB * H)
    _, st = K.masknet_mask_fwd(e, m, b2, lw, lb, E, NB)
    _, st2 = K.masknet_ffn_fwd(z, b3, fw, fb, NB)
    # the torch formulation's tensors: unpadded [B, E] / [B, H] per block
    e_t = e[:, :E].contiguous().requires_grad_(True)
    m_t = [m[:, i * EP:i * EP + E].contiguous().requires_grad_(True) for i in range(NB)]
    b2_t = [b2[i * E:(i + 1) * E].clone().requires_grad_(True) for i in range(NB)]
    lw_t, lb_t = lw.clone().requires_grad_(True), lb.clone().requires_grad_(True)
    dv_t = [dv[:, i * EP:i * EP + E].contiguous() for i in range(NB)]
    z_t = [z[:, i * H:(i + 1) * H].contiguous().requires_grad_(True) for i in range(NB)]
    b3_t = [b3[i * H:(i + 1) * H].clone().requires_grad_(True) for i in range(NB)]
    fw_t = [fw[i * H:(i + 1) * H].clone().requires_grad_(True) for i in range(NB)]
    fb_t = [fb[i * H:(i + 1) * H].clone().requires_grad_(True) for i in range(NB)]

    def mask_torch():
        ln = F.layer_norm(e_t, (E,), lw_t, lb_t)
        return [ln * (m_t[i] + b2_t[i]) for i in range(NB)]

    def ffn_torch():
        return torch.cat([torch.relu(F.layer_norm(z_t[i] + b3_t[i], (H,), fw_t[i], fb_t[i])) for i in range(NB)], 1)

    with torch.no_grad():
        fwd = timed({"mask_fused": lambda: K.masknet_mask_fwd(e, m, b2, lw, lb, E, NB), "mask_torch": mask_torch,
                     "ffn_fused": lambda: K.masknet_ffn_fwd(z, b3, fw, fb, NB), "ffn_torch": ffn_torch}, iters)
    vs = mask_torch()
    hid = ffn_torch()
    mask_in = [e_t, lw_t, lb_t] + m_t + b2_t
    ffn_in = z_t + b3_t + fw_t + fb_t
    bwd = timed({
        "mask_fused": lambda: K.masknet_mask_bwd(e, m, b2, lw, lb, st, dv, E, NB),
        "mask_torch": lambda: torch.autograd.grad(vs, mask_in, dv_t, retain_graph=True),
        "ffn_fused": lambda: K.masknet_ffn_bwd(z, b3, fw, fb, st2, dy, NB),
        "ffn_torch": lambda: torch.autograd.grad(hid, ffn_in, dy, retain_graph=True)}, iters)
    f4 = 4 * B
    byts = {"mask_fwd": f4 * (E + 2 * NB * E), "mask_bwd": f4 * (E + 3 * NB * E + E),
            "ffn_fwd": f4 * (2 * NB * H), "ffn_bwd": f4 * (3 * NB * H)}
    out = {}
    for name, tab, key in (("mask_fwd", fwd, "mask"), ("mask_bwd", bwd, "mask"), ("ffn_fwd", fwd, "ffn"),
                           ("ffn_bwd", bwd, "ffn")):
        fu, to = tab[f"{key}_fused"], tab[f"{key}_torch"]
        out[name] = {"fused_ms": round(fu, 4), "torch_ms": round(to, 4), "speedup": round(to / fu, 2),
                     "bytes": byts[name], "fused_GBps": round(byts[name] / fu / 1e6, 1)}
    # the fused path's GEMMs alone (forward and backward), on the padded layout
    x, h = e, r(B, NB * AP).relu_()
    w1, w2, w3 = r(NB * AP, EP), r(NB, EP, AP), r(NB, H, EP)
    mm, zz, dvv, dh = torch.empty(B, NB * EP, device=dev), torch.empty(B, NB * H, device=dev), \
        torch.empty(B, NB * EP, device=dev), torch.empty(B, NB * AP, device=dev)

    def gemms():
        dense_gemm.gemm(x, False, w1, True)
        for i in range(NB):
            dense_gemm.gemm(h[:, i * AP:(i + 1) * AP], False, w2[i], True, out=mm[:, i * EP:(i + 1) * EP])
            dense_gemm.gemm(mm[:, i * EP:(i + 1) * EP], False, w3[i], True, out=zz[:, i * H:(i + 1) * H])
        for i in range(NB):
            dense_gemm.gemm(zz[:, i * H:(i + 1) * H], False, w3[i], False, out=dvv[:, i * EP:(i + 1) * EP])
            dense_gemm.gemm(zz[:, i * H:(i + 1) * H], True, mm[:, i * EP:(i + 1) * EP], False)
            dense_gemm.gemm(mm[:, i * EP:(i + 1) * EP], False, w2[i], False, out=dh[:, i * AP:(i + 1) * AP])
            dense_gemm.gemm(mm[:, i * EP:(i + 1) * EP], True, h[:, i * AP:(i + 1) * AP], False)
        dense_gemm.gemm(dh, True, x, False)
        dense_gemm.gemm(dh, False, w1, False, out=x, beta=1.0)

    out["gemms_ms"] = round(timed({"g": gemms}, iters)["g"], 4)
    return out


def graphed_step(B, iters):
    from torcheasyrec_b200.engine import GraphedTrainStep, Pipeline

    res = {}
    real = Fn.masknet_usable
    for name in ("fused", "torch"):
        if name == "torch":
            Fn.masknet_usable = lambda *a, **k: False
        try:
            p = Pipeline("masknet_criteo", device="cuda", max_rows=1_000_000, seed=1)
            batches = [p.synthetic_batch(B, seed=i) for i in range(2)]
            step = GraphedTrainStep(p, batches[0], warmup=3)
            step.load(batches[1].pin_memory())
            res[name] = timed({"s": step.replay}, iters)["s"]
            del step, p
            torch.cuda.empty_cache()
        finally:
            Fn.masknet_usable = real
    return {"fused_ms": round(res["fused"], 3), "torch_ms": round(res["torch"], 3),
            "speedup": round(res["torch"] / res["fused"], 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[8192, 65536])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    res = {"card": card(), "shape": {"E": E, "A": A, "H": H, "n_mask_blocks": NB}}
    for B in args.batches:
        res[f"B{B}"] = {"passes": passes(B, args.iters), "graphed_step": graphed_step(B, max(10, args.iters // 5))}
        print(json.dumps({f"B{B}": res[f"B{B}"]}), flush=True)
    res["card_after"] = card()
    print(json.dumps(res["card"]), json.dumps(res["card_after"]))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
