"""Times the gradient half of the fused sparse backward (fused_bwd_apply: run reduction + optimizer update) for every
sparse optimizer on DLRM-Criteo's embedding collection at B = 65536, uniform and Zipf(1.05) ids, with CUDA events.

The sort (fused_bwd_sort) runs once per batch outside the timed region; every timed call applies the same gradient to
the same sorted batch.  The optimizers are timed in turn, round after round, so that drifts of the shared machine
spread over all of them; each line reports the median over rounds and the min-max spread.  Algorithmic bytes follow
SURVEY §8(d): per touched row U, 2 D 4 B (SGD: read + write the row), 4 D 4 B (Adagrad, LARS: row + one state),
6 D 4 B (Adam, LAMB: row + two states), plus 8 B per row for a row-wise state (read + write).  Gradient reads are not
counted.  The card's name and power limit are printed with the numbers.

    python scripts/bench_sparse_optimizers.py [--batch 65536] [--iters 50] [--rounds 5] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torcheasyrec_b200 import kernels as K  # noqa: E402
from torcheasyrec_b200.embedding_modules import SparseOptimizerSpec  # noqa: E402
from torcheasyrec_b200.engine import Pipeline  # noqa: E402

# name -> (spec, interleaved arena, bytes per touched row in units of D * 4 B, extra bytes per row)
OPTIMIZERS = [
    ("sgd", SparseOptimizerSpec(kind=K.OPT_SGD, lr=0.01), False, 2, 0),
    ("adagrad_interleaved", SparseOptimizerSpec(kind=K.OPT_ADAGRAD, lr=0.01), True, 4, 0),
    ("adagrad", SparseOptimizerSpec(kind=K.OPT_ADAGRAD, lr=0.01), False, 4, 0),
    ("rowwise_adagrad", SparseOptimizerSpec(kind=K.OPT_ROWWISE_ADAGRAD, lr=0.01), False, 2, 8),
    ("rowwise_adagrad_l2", SparseOptimizerSpec(kind=K.OPT_ROWWISE_ADAGRAD, lr=0.01, weight_decay=0.01,
                                               weight_decay_mode=K.WD_L2), False, 2, 8),
    ("adam", SparseOptimizerSpec(kind=K.OPT_ADAM, lr=0.01, weight_decay=0.001), False, 6, 0),
    ("partial_rowwise_adam", SparseOptimizerSpec(kind=K.OPT_PARTIAL_ROWWISE_ADAM, lr=0.01), False, 4, 8),
    ("lamb", SparseOptimizerSpec(kind=K.OPT_LAMB, lr=0.01, weight_decay=0.001), False, 6, 0),
    ("partial_rowwise_lamb", SparseOptimizerSpec(kind=K.OPT_PARTIAL_ROWWISE_LAMB, lr=0.01), False, 4, 8),
    ("lars_sgd", SparseOptimizerSpec(kind=K.OPT_LARS_SGD, lr=1.0, weight_decay=0.0001), False, 4, 0),
]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--max-rows", type=int, default=0, help="cap every table (0: full Criteo hash sizes)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    dev = torch.device("cuda:0")
    pipe = Pipeline("dlrm_criteo", device="cuda:0", max_rows=a.max_rows or None, seed=0)
    coll = pipe.model.sparse_collections()[0]
    k = K.default_kernels()
    info = gpu_info()
    print(f"# {info}; B = {a.batch}; {a.rounds} rounds x {a.iters} calls", flush=True)
    results = []
    for dist in ("uniform", "zipf"):
        batch = pipe.synthetic_batch(a.batch, seed=7, id_dist=dist).to(dev)
        kjt = coll._select(next(iter(batch.sparse_features.values())))
        ids, offsets, B = kjt.values(), kjt.offsets(), kjt.stride()
        g = torch.Generator(device="cuda").manual_seed(1)
        grad = torch.randn(B, coll.layout.total_dim, device=dev, generator=g) * 1e-3
        # touched rows: distinct (table, row) keys
        F = coll.layout.num_features
        lens = offsets.diff().view(F, B).sum(1)
        feat = torch.repeat_interleave(torch.arange(F, device=dev), lens)
        rows = torch.tensor(coll.layout.rows, device=dev)[feat]
        kb = torch.tensor(coll.layout.key_base, device=dev)[feat]
        keys = kb + torch.where((ids >= 0) & (ids < rows), ids, torch.zeros_like(ids))
        U = int(torch.unique(keys).numel())
        D = coll.layout.max_dim
        times = {name: [] for name, *_ in OPTIMIZERS}
        setups = {}
        for r in range(a.rounds):
            for name, spec, inter, units, extra in OPTIMIZERS:
                os.environ["TZK_INTERLEAVE"] = "1" if inter else "0"
                coll.set_optimizer(spec)
                assert coll.layout.interleaved == inter, name
                if coll.opt_step is not None:
                    coll.opt_step.fill_(1.0)
                ws = coll._bwd_workspace(k, ids.numel())
                k.fused_bwd_sort(True, coll.layout, ids, offsets, B, ws)
                ex = coll.opt_extras(bump=False)

                def apply():
                    k.fused_bwd_apply(spec.kind, True, grad, coll.weights.data, coll.opt_state, coll.layout, offsets,
                                      ids.numel(), B, spec.lr, spec.eps, 1.0, ws, **ex)

                for _ in range(3):
                    apply()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                s.record()
                for _ in range(a.iters):
                    apply()
                e.record()
                torch.cuda.synchronize()
                times[name].append(s.elapsed_time(e) * 1e3 / a.iters)
                setups[name] = U * (units * D * 4 + extra)
        for name, *_ in OPTIMIZERS:
            t = times[name]
            med = statistics.median(t)
            res = dict(ids=dist, optimizer=name, us=round(med, 2), us_min=round(min(t), 2), us_max=round(max(t), 2),
                       touched_rows=U, alg_bytes=setups[name], alg_GBps=round(setups[name] / med / 1e3, 1), gpu=info)
            results.append(res)
            print(json.dumps(res), flush=True)
    os.environ.pop("TZK_INTERLEAVE", None)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
