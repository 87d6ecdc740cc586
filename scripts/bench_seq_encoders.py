"""SelfAttentionEncoder's fused attention core (csrc/tzk_seq_attn.cuh) against the torch jagged chain and the reference's
padded formulation, and the eager dbmtl_taobao_seq_encoders step (DESIGN.md §8).

    python scripts/bench_seq_encoders.py [--iters 20] [--out /tmp/bench_seq_encoders.json]

Forward + backward of the attention core at B = 8192, sequence dim 48, lengths drawn from SURVEY's cfg4 mixture
{0, 1, U[2, 100], 100} (a quarter each, about 38 rows per sample), at E / H = 512 / 8 and 64 / 4.  "fused" is
functional.self_attn_pool, "torch" functional.torch_self_attn_pool over the same in-projected jagged rows, "padded"
the reference's nn.MultiheadAttention over [B, T, E] with its [B H, T, T] mask (the padding is done outside the timed
region), then out_proj and the row sum.  Each variant alone is also timed for the attention core only
(fused: the two kernels).  CUDA events, warm-up first, the variants alternated round by round in one process.

FLOPs and bytes come from the shapes.  Per (sample, head) with L kept rows and head width hd the formula needs
2 L^2 hd FLOP for the scores and 2 L hd for the pooling forward; the backward needs the scores again, 2 L^2 hd each for
dq and dk and L^2 for D.  The kernels recompute the scores (twice forward, three times backward), so the essential
FLOPs are the formula's: 2 L^2 hd + 2 L hd forward and 6 L^2 hd + 4 L hd backward.  Essential bytes: q, k, v read
once and lse written forward; q, k, v, lse read and dq, dk, dv written backward.  Least time = max(FLOP / 67 TFLOP/s,
bytes / 3.35 TB/s) (H100 SXM data sheet, dense FP32 and HBM3).  The card's name and power limit are read in the same
run.  Fails without a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200.engine import Pipeline  # noqa: E402
from torcheasyrec_b200.kernels import default_kernels  # noqa: E402
from torcheasyrec_b200.rank_models import SelfAttentionEncoder, _attention_mask  # noqa: E402

FP32_TFLOPS, HBM_TBS = 67.0, 3.35
B, D = 8192, 48


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q[0] if q else ""}


def timed(fns, iters, warm=3):
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


def lengths(seed=0):
    rng = np.random.default_rng(seed)
    kind = rng.integers(0, 4, B)
    return np.where(kind == 0, 0, np.where(kind == 1, 1, np.where(kind == 2, rng.integers(2, 101, B), 100)))


def least_ms(lens, E, H):
    hd = E // H
    l1, l2 = float(lens.sum()), float((lens.astype(np.float64) ** 2).sum())
    N = l1
    fl_f = H * (2 * l2 * hd + 2 * l1 * hd)
    fl_b = H * (6 * l2 * hd + 4 * l1 * hd)
    by_f = 4 * (3 * N * E + N * H + B * E)
    by_b = 4 * (3 * N * E + N * H + B * E + 3 * N * E)
    t = lambda fl, by: max(fl / (FP32_TFLOPS * 1e12), by / (HBM_TBS * 1e12)) * 1e3  # noqa: E731
    return {"fwd": t(fl_f, by_f), "bwd": t(fl_b, by_b), "flop_fwd": fl_f, "flop_bwd": fl_b,
            "bound_fwd": "flop" if fl_f / FP32_TFLOPS > by_f / HBM_TBS * 1e0 else "bytes"}


def core(E, H, iters):
    lens = lengths()
    N = int(lens.sum())
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)).cuda()
    g = torch.Generator(device="cuda").manual_seed(1)
    q, k, v = (torch.randn(N, E, device="cuda", generator=g) for _ in range(3))
    dout = torch.randn(B, E, device="cuda", generator=g)
    kk = default_kernels()
    state = {}

    def kern_fwd():
        state["f"] = kk.self_attn_pool_fwd(q, k, v, off, H, 0)

    kern_fwd()

    def kern_bwd():
        kk.self_attn_pool_bwd(q, k, v, off, H, 0, state["f"][1], dout)

    leaves = [t.clone().requires_grad_(True) for t in (q, k, v)]

    def fused():
        Fn.self_attn_pool(*leaves, off, H, 0).backward(dout)

    def torch_chain():
        Fn.torch_self_attn_pool(*leaves, off, H, 0).backward(dout)

    # the reference's formulation at the same in-projected rows: MHA with identity in-projection weights is the
    # attention core plus out_proj, which the fused path applies to [B, E] instead of [B T, E]
    torch.manual_seed(0)
    enc = SelfAttentionEncoder(D, "s", E, num_heads=H).cuda()
    T = int(lens.max())
    seg = torch.repeat_interleave(torch.arange(B, device="cuda"), torch.from_numpy(lens).cuda())
    pos = torch.arange(N, device="cuda") - off[:-1][seg]
    seqp = torch.zeros(B, T, D, device="cuda")
    seqp[seg, pos] = torch.randn(N, D, device="cuda", generator=g)
    seqr = seqp[seg, pos].clone()
    lens_t = torch.from_numpy(lens).cuda()
    dout_e = torch.randn(B, E, device="cuda", generator=g)

    def padded_encoder():
        enc({"s.sequence": seqp, "s.sequence_length": lens_t}).backward(dout_e)

    def jagged_encoder():
        enc({"s.sequence": seqr, "s.sequence_length": lens_t, "s.sequence_offsets": off}).backward(dout_e)

    mask = _attention_mask(seqp, H, lens_t)
    assert mask.shape == (B * H, T, T)
    ms = timed({"kernel_fwd": kern_fwd, "kernel_bwd": kern_bwd, "fused_core": fused, "torch_core": torch_chain,
                "encoder_jagged_fused": jagged_encoder, "encoder_padded_reference": padded_encoder}, iters)
    lb = least_ms(lens, E, H)
    return {"E": E, "H": H, "N": N, "T": T, "ms": ms, "least_ms": lb,
            "kernel_share_of_least": {"fwd": lb["fwd"] / ms["kernel_fwd"], "bwd": lb["bwd"] / ms["kernel_bwd"]}}


def step(iters):
    res = {}
    pipe = Pipeline("dbmtl_taobao_seq_encoders", device="cuda:0", max_rows=100000, seed=3, capturable=False)
    batch = pipe.synthetic_batch(B, seed=1).to("cuda:0")
    usable = Fn.self_attn_pool_usable
    fns = {"fused": lambda: pipe.eager_step(batch)}

    def torch_step():
        Fn.self_attn_pool_usable = lambda *a: False
        try:
            pipe.eager_step(batch)
        finally:
            Fn.self_attn_pool_usable = usable

    fns["torch"] = torch_step
    res["eager_step_ms"] = timed(fns, iters)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    out = {"card": card(), "B": B, "D": D, "core": [core(512, 8, args.iters), core(64, 4, args.iters)]}
    torch.cuda.empty_cache()
    out["dbmtl_taobao_seq_encoders"] = step(max(5, args.iters // 2))
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text)


if __name__ == "__main__":
    main()
