"""Times the WuKong layer's fused kernels (csrc/tzk_wukong.cuh) with CUDA events against the reference's torch chain for
the same work, at the wukong_criteo layers (layer 1: n = 27 with the residual projection; layer 2: n = 32 with the
identity residual; d = 16, k = 24, f = l = 16), and the graphed wukong_criteo training step.

  mix_fwd   vs  permute, matmul, matmul, view, LayerNorm(n k); LCB permute / matmul / permute; residual ditto; add
  out_fwd   vs  concat(fmb, lcb) + residual, LayerNorm(d)
  mix_bwd / out_bwd  vs  autograd of the same chains (the FMB MLP excluded on both sides)

Per kernel: time per call, the algorithmic bytes (each input read once, each output written once) and the GB/s they
give, and the FP32 FFMA rate.  The card's name, power limit and SM clock are read in the same run.

    python scripts/bench_wukong.py [--batches 8192,65536] [--iters 100] [--out PATH.json]
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

HBM_BPS = 3.35e12          # H100 SXM data sheet
FP32_FLOPS = 67e12


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


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        q = f"unavailable: {e!r}"
    return q


def layer_bench(B, n, proj, iters):
    d, k, f, l = 16, 24, 16, 16
    m = f + l
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(B, n, d, device=dev, generator=g)
    wf = torch.randn(n, k, device=dev, generator=g) * 0.2
    wl = torch.randn(n, l, device=dev, generator=g) * 0.2
    wr = torch.randn(n, m, device=dev, generator=g) * 0.2 if proj else None
    gf, bf = torch.ones(n * k, device=dev), torch.zeros(n * k, device=dev)
    gam, bet = torch.ones(d, device=dev), torch.zeros(d, device=dev)
    fmb = torch.randn(B, f * d, device=dev, generator=g)
    d_ln_f = torch.randn(B, n * k, device=dev, generator=g)
    dy = torch.randn(B, m, d, device=dev, generator=g)
    K = default_kernels()
    ln_f, st, base = K.wukong_mix_fwd(x, wf, gf, bf, wl, wr, f)
    y, ost = K.wukong_out_fwd(fmb, base, gam, bet, f)
    nk, nd, md = n * k, n * d, m * d
    res = {}
    # bytes per sample of each pass (fp32), each tensor touched once; FLOPs per sample (2 per multiply-add)
    flop_mix = 2 * (n * d * k * 2 + (m if proj else 0) * n * d + l * n * d)
    model = {
        "mix_fwd": (4 * (nd + nk + 2 + md), flop_mix),
        "out_fwd": (4 * (f * d + 2 * md + 2 * m), 0),
        "mix_bwd": (4 * (nd + nk + 2 + md + nd), 2 * flop_mix + 2 * n * d * k * 2),
        "out_bwd": (4 * (f * d + md + 2 * m + md + f * d + md), 0),
    }
    fused = {
        "mix_fwd": lambda: K.wukong_mix_fwd(x, wf, gf, bf, wl, wr, f),
        "out_fwd": lambda: K.wukong_out_fwd(fmb, base, gam, bet, f),
        "mix_bwd": lambda: K.wukong_mix_bwd(x, wf, gf, wl, wr, f, st, d_ln_f, dy),
        "out_bwd": lambda: K.wukong_out_bwd(fmb, base, gam, f, ost, dy),
    }
    # the reference's chain for the same work (tzrec/modules/interaction.py:255-378 without the FMB MLP)
    xr = x.clone().requires_grad_(True)
    params = [t.clone().requires_grad_(True) for t in (wf, gf, bf, wl, gam, bet)] + (
        [wr.clone().requires_grad_(True)] if proj else [])
    wf_, gf_, bf_, wl_, gam_, bet_ = params[:6]
    wr_ = params[6] if proj else None
    fmb_r = fmb.clone().requires_grad_(True)

    def ref_mix():
        t = torch.matmul(xr.permute(0, 2, 1), wf_)
        fm = torch.matmul(xr, t).view(-1, nk)
        lnf = torch.nn.functional.layer_norm(fm, (nk,), gf_, bf_)
        lcb = Fn.torch_linear_compress(xr, wl_)
        r = Fn.torch_linear_compress(xr, wr_) if proj else xr
        return lnf, lcb, r

    def ref_out(lcb, r):
        z = torch.concat((fmb_r.view(-1, f, d), lcb), dim=1) + r
        return torch.nn.functional.layer_norm(z, (d,), gam_, bet_)

    lnf_r, lcb_r, r_r = ref_mix()
    out_r = ref_out(lcb_r, r_r)
    d_lcb, d_r = torch.randn_like(lcb_r), torch.randn_like(r_r) if proj else None

    def ref_mix_bwd():
        outs = [lnf_r, lcb_r] + ([r_r] if proj else [])
        grads = [d_ln_f, d_lcb] + ([d_r] if proj else [])
        torch.autograd.grad(outs, [xr, wf_, gf_, bf_, wl_] + ([wr_] if proj else []), grads, retain_graph=True)

    def ref_out_bwd():
        torch.autograd.grad([out_r], [fmb_r, lcb_r, r_r, gam_, bet_] if proj else [fmb_r, lcb_r, gam_, bet_], [dy],
                            retain_graph=True)

    chain = {"mix_fwd": lambda: ref_mix(), "out_fwd": lambda: ref_out(lcb_r.detach(), r_r.detach()),
             "mix_bwd": ref_mix_bwd, "out_bwd": ref_out_bwd}
    for name in fused:
        t_f = timed(fused[name], iters)
        with torch.set_grad_enabled(name.endswith("bwd")):
            t_c = timed(chain[name], iters)
        nbytes, flops = model[name]
        res[name] = {"fused_us": round(t_f, 2), "torch_chain_us": round(t_c, 2), "speedup": round(t_c / t_f, 2),
                     "bytes_per_sample": nbytes, "fused_GBps": round(nbytes * B / t_f / 1e3, 1),
                     "hbm_share": round(nbytes * B / (t_f * 1e-6) / HBM_BPS, 3)}
        if flops:
            res[name]["fused_fp32_TFLOPs"] = round(flops * B / (t_f * 1e-6) / 1e12, 2)
            res[name]["fp32_share"] = round(flops * B / (t_f * 1e-6) / FP32_FLOPS, 3)
    return res


def step_bench(B, iters):
    from torcheasyrec_b200.engine import GraphedTrainStep, Pipeline

    p = Pipeline("wukong_criteo", device="cuda:0", max_rows=1_000_000, seed=1)
    batches = [p.synthetic_batch(B, seed=50 + i) for i in range(4)]
    step = GraphedTrainStep(p, batches[0], warmup=3)
    pinned = [b.pin_memory() for b in batches]
    for bt in pinned:
        step.load(bt)
        step.replay()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for i in range(iters):
        step.load(pinned[i % len(pinned)])
        step.replay()
    end.record()
    torch.cuda.synchronize()
    return {"batch": B, "tables_capped_rows": 1_000_000, "graphed_step_ms": round(start.elapsed_time(end) / iters, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="8192,65536")
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    out = {"card": card(), "layers": {}}
    for B in (int(s) for s in a.batches.split(",")):
        for tag, n, proj in (("layer1_n27_proj", 27, True), ("layer2_n32_identity", 32, False)):
            out["layers"][f"{tag}_B{B}"] = layer_bench(B, n, proj, a.iters)
    out["step"] = [step_bench(8192, a.iters)]
    out["card_after"] = card()
    print(json.dumps(out, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
