"""Times weighted bags against unweighted ones on the three kernels they touch, with CUDA events: the pooled gather,
the id half of the fused backward (linearize + radix sort + run lists; weighted: + the pass that turns sorted positions
back into bags and sorts the weights) and the gradient half (run reduction + Adagrad update on the interleaved arena).

Two collections:
  criteo  DLRM-Criteo's 26 tables (D = 16, one id per bag) at B = 65536, uniform ids;
  ccp     the Ali-CCP MMoE config's tables (D = 8 / 12 / 16), every bag multi-hot with 1..2 L ids (mean L = 5 by
          default; Ali-CCP's weighted kv features are lists), at B = 8192 (its data_config.batch_size).
Three inputs each: unweighted, weighted with all-ones weights, weighted with random weights.  The modes are timed in
turn, round after round; each line reports the median over rounds and the min-max spread.  Algorithmic bytes:
gather = nnz * (8 B id + 4 D B row) + B * sum(D) * 4 B out (+ 4 B per id weighted); gradient half = per touched row
4 D 4 B (row + accumulator, read + write) + nnz * 4 B (+ 4 B per id weighted).  The card's name and power limit are
printed with the numbers.

    python scripts/bench_weighted_lookup.py [--iters 50] [--rounds 5] [--max-rows 0] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from torcheasyrec_b200 import kernels as K  # noqa: E402
from torcheasyrec_b200.embedding_modules import SparseOptimizerSpec  # noqa: E402
from torcheasyrec_b200.engine import Pipeline  # noqa: E402

CCP = os.path.join(ROOT, "tests", "golden", "ref_examples", "mmoe_taobao_ccp.config")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def timed(fn, iters):
    for _ in range(3):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e3 / iters


def collection_input(name, B, mean_len, max_rows, dev, gen):
    if name == "criteo":
        pipe = Pipeline("dlrm_criteo", device="cuda:0", max_rows=max_rows or None, seed=0)
    else:
        pipe = Pipeline(CCP, device="cuda:0", max_rows=max_rows or None, seed=0)
    coll = pipe.model.sparse_collections()[0]
    lay = coll.layout
    F = lay.num_features
    if name == "criteo":
        lengths = torch.ones(F * B, dtype=torch.int32, device=dev)
    else:
        lengths = torch.randint(1, 2 * mean_len, (F * B,), dtype=torch.int32, device=dev, generator=gen)
    offsets = torch.zeros(F * B + 1, dtype=torch.int64, device=dev)
    offsets[1:] = torch.cumsum(lengths, 0)
    per = lengths.view(F, B).sum(1)
    rows = torch.tensor(lay.rows, device=dev)
    feat = torch.repeat_interleave(torch.arange(F, device=dev), per)
    ids = (torch.rand(int(offsets[-1]), device=dev, generator=gen) * rows[feat]).to(torch.int64)
    keys = torch.tensor(lay.key_base, device=dev)[feat] + ids
    U = int(torch.unique(keys).numel())
    return coll, ids, offsets, U


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--criteo-batch", type=int, default=65536)
    ap.add_argument("--ccp-batch", type=int, default=8192)
    ap.add_argument("--ccp-mean-len", type=int, default=5)
    ap.add_argument("--max-rows", type=int, default=0, help="cap every table (0: the configs' hash sizes)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    dev = torch.device("cuda:0")
    k = K.default_kernels()
    info = gpu_info()
    print(f"# {info}; {a.rounds} rounds x {a.iters} calls", flush=True)
    results = []
    gen = torch.Generator(device="cuda").manual_seed(1)
    for name, B in (("criteo", a.criteo_batch), ("ccp", a.ccp_batch)):
        coll, ids, offsets, U = collection_input(name, B, a.ccp_mean_len, a.max_rows, dev, gen)
        spec = SparseOptimizerSpec(kind=K.OPT_ADAGRAD, lr=0.01)
        coll.set_optimizer(spec)
        lay, nnz = coll.layout, ids.numel()
        D = lay.max_dim
        grad = torch.randn(B, lay.total_dim, device=dev, generator=gen) * 1e-3
        modes = {"unweighted": None, "weighted_ones": torch.ones(nnz, device=dev),
                 "weighted_random": torch.rand(nnz, device=dev, generator=gen) * 2}
        ws = {m: torch.empty(k.fused_bwd_workspace_bytes(lay, nnz, weighted=w is not None), dtype=torch.uint8,
                             device=dev) for m, w in modes.items()}
        t = {(m, p): [] for m in modes for p in ("gather", "id_half", "grad_half")}
        for r in range(a.rounds):
            for m, w in modes.items():
                kw = {} if w is None else {"per_sample_weights": w}
                t[(m, "gather")].append(timed(lambda: k.pooled_gather_fwd(coll.weights.data, lay, ids, offsets, B, **kw),
                                              a.iters))
                t[(m, "id_half")].append(timed(lambda: k.fused_bwd_sort(True, lay, ids, offsets, B, ws[m], **kw),
                                               a.iters))
                k.fused_bwd_sort(True, lay, ids, offsets, B, ws[m], **kw)
                t[(m, "grad_half")].append(timed(lambda: k.fused_bwd_apply(
                    spec.kind, True, grad, coll.weights.data, coll.opt_state, lay, offsets, nnz, B, spec.lr, spec.eps,
                    1.0, ws[m], **kw), a.iters))
        for (m, p), v in t.items():
            wb = 0 if m == "unweighted" else 4 * nnz
            if p == "gather":
                alg = nnz * 8 + sum(lay.dim[f] * 4 * int(offsets[(f + 1) * B] - offsets[f * B])
                                    for f in range(lay.num_features)) + B * lay.total_dim * 4 + wb
            elif p == "id_half":
                alg = nnz * 8 + wb                     # ids read (the sort's own traffic is not counted)
            else:
                alg = U * 4 * D * 4 + nnz * 4 + wb
            med = statistics.median(v)
            res = dict(collection=name, B=B, nnz=nnz, touched_rows=U, mode=m, phase=p, us=round(med, 2),
                       us_min=round(min(v), 2), us_max=round(max(v), 2), alg_bytes=alg,
                       alg_GBps=round(alg / med / 1e3, 1), gpu=info)
            results.append(res)
            print(json.dumps(res), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
