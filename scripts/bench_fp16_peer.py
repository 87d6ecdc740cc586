"""Times the peer step with FP32 and with FP16 tables (data_type = FP16) at DLRM-Criteo shapes: 26 tables, D = 16, the
full hash sizes, one id per bag, B = 65536 per rank, uniform and Zipf ids.  CUDA events; each line is the median over
rounds (modes alternate round after round) with the min-max spread and the algorithmic bytes of the phase.

  kernels  W virtual ranks on ONE GPU (their arenas, wire and receive buffers are allocations of the same device, so
           every "remote" row and every pushed slice stays in local HBM; row-wise plan, small tables mirrored as
           PeerState does):
             gather        the requester's lookup, one launch;
             gather_split  the same as two launches (mirrored features, then the ones read from the owners' arenas);
             mirror        the per-step copy of the small tables;
             push_update   the push of this rank's gradient slices plus the owner's update over its receive buffer
                           (Adagrad; the small tables' partial-sum update is not included).
  step     (--step) the whole graphed training step of DLRM-Criteo on the peer exchange, one process per GPU: a single
           rank on one GPU, or W real ranks under torchrun.  The NVLink cost appears only in the torchrun run.

Algorithmic bytes per phase (table element e = 4 B for FP32, 2 B for FP16): gather = ids + offsets + rows (D e per id)
+ fp32 output; mirror = 2 x mirrored elements x e (read + write); push_update = slot index + fp32 slice read + written,
then per received slot the fp32 slice and the key, and per touched row D e read + written plus the fp32 state twice.
The card's name and power limit are read in the same run and printed with the numbers.

    python scripts/bench_fp16_peer.py [--world 4] [--iters 20] [--rounds 5] [--max-rows 0] [--step] [--out FILE]
    torchrun --nproc_per_node 8 scripts/bench_fp16_peer.py --step-only
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from torcheasyrec_b200 import kernels as K  # noqa: E402
from torcheasyrec_b200 import peer_exchange  # noqa: E402
from torcheasyrec_b200.distributed import _DimGroup, make_plan  # noqa: E402
from torcheasyrec_b200.embedding_modules import (DataType, EmbeddingBagConfig, SparseOptimizerSpec,  # noqa: E402
                                                 output_names_by_table)
from torcheasyrec_b200.example_configs import CRITEO_HASH_SIZES  # noqa: E402


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


class _Sym:
    def __init__(self, t, everyone, W):
        self.t, self.everyone, self.W = t, everyone, W

    @property
    def ptrs(self):
        return (ctypes.c_uint64 * self.W)(*[self.everyone[r].data_ptr() for r in range(self.W)])


def virtual_ranks(cfgs, W, B):
    plan = make_plan(cfgs, W, "row_wise")
    names = output_names_by_table(cfgs)
    registry = {}

    class St(peer_exchange.PeerState):
        def _alloc(self, numel, dtype):
            n = getattr(self, "_n_alloc", 0)
            self._n_alloc = n + 1
            slot = registry.setdefault(n, {})
            slot[self.me] = torch.zeros(max(int(numel), 1), dtype=dtype, device=self.device)
            return _Sym(slot[self.me], slot, self.W)

        def _host_barrier(self):
            pass

    sts = []
    for r in range(W):
        g = _DimGroup(cfgs, plan, r, W, torch.device("cuda:0"), True, names)
        g.static_alpha = 2.0
        if r == 0:
            g.local.set_optimizer(SparseOptimizerSpec.from_name("adagrad", lr=0.01))
        with torch.no_grad():       # (deterministic, cheap init: the values do not change the timings)
            g.local.weights.data.uniform_(-0.05, 0.05)
        sts.append(St(g, plan, None, B, [B] * g.F))
    return sts


def ids_for(g, B, dist_kind, gen):
    F, dev = g.F, g.device
    rows = torch.tensor([g.configs[t].num_embeddings for t in g.local._feat_table], device=dev,
                        dtype=torch.float64).repeat_interleave(B)
    u = torch.rand(F * B, device=dev, generator=gen, dtype=torch.float64)
    if dist_kind == "uniform":
        ids = (u * rows).to(torch.int64)
    else:                          # Zipf(1)-like: log-uniform ranks, scattered over the table by a multiplicative hash
        rank = (torch.pow(rows, u) - 1).to(torch.int64)
        ids = (rank * 2654435761) % rows.to(torch.int64)
    return ids, torch.arange(F * B + 1, dtype=torch.int64, device=dev)


def bench_kernels(a, k, info, results):
    W, B = a.world, a.batch
    gen = torch.Generator(device="cuda").manual_seed(1)
    hs = [min(h, a.max_rows) if a.max_rows else h for h in CRITEO_HASH_SIZES]
    for dt_name, dt in (("fp32", DataType.FP32), ("fp16", DataType.FP16)):
        cfgs = [EmbeddingBagConfig(num_embeddings=h, embedding_dim=16, name=f"t{i}", feature_names=[f"f{i}"],
                                   data_type=dt) for i, h in enumerate(hs)]
        sts = virtual_ranks(cfgs, W, B)
        st = sts[0]
        g, lay = st.g, st.g.local.layout
        e = 2 if dt == DataType.FP16 else 4
        assert st.tables.t.element_size() == e
        for dist_kind in ("uniform", "zipf"):
            per_rank = [ids_for(s.g, B, dist_kind, gen) for s in sts]
            ids, offsets = per_rank[0]
            nnz = ids.numel()
            grad = torch.randn(B, lay.total_dim, device="cuda", generator=gen)
            k.peer_mirror_refresh(st.tables, W, *st._seg, st.mirror)
            ft = g.local._feat_table
            loc = [f for f, t in enumerate(ft) if t in st._m_off]
            rem = [f for f, t in enumerate(ft) if t not in st._m_off]
            sel = (torch.tensor(loc, dtype=torch.int32, device="cuda"), torch.tensor(rem, dtype=torch.int32, device="cuda"))
            out = torch.empty(B, lay.total_dim, device="cuda")
            # wire + owner side: every virtual rank bucketizes and pushes into rank 0's receive buffer
            for r, s in enumerate(sts):
                k.peer_bucketize(*per_rank[r], g.F, B, W, s.feat_block_wire, s.g.feat_owner, s.feat_rows, s.rf_key_base,
                                 True, s.cap, s.wire_key.t, s.wire_idx.t, s.counts.t)
            torch.cuda.synchronize()
            assert all(int(s.counts.t[W]) == 0 for s in sts), "wire capacity overflowed"
            k.fused_bwd_sort_peer(st.wire_key, st.wire_idx, st.counts, 0, W, st.cap, 0, lay, g.overflow, st._workspace())
            for r, s in enumerate(sts):
                k.peer_push_grad(s.recv, grad, s.g.local.layout, per_rank[r][1], s.wire_idx.t, s.counts.t, r, W, s.cap,
                                 B, True)
            spec, extras = g.local.optimizer, g.local.opt_extras()

            def push_update():
                k.peer_push_grad(st.recv, grad, lay, offsets, st.wire_idx.t, st.counts.t, 0, W, st.cap, B, True)
                k.fused_bwd_apply(spec.kind, False, st.recv.t.view(W * st.cap, g.dim), g.local.weights.data,
                                  g.local.opt_state, lay, st._dummy_off, W * st.cap, 1, spec.lr, spec.eps, 1.0 / W,
                                  st._workspace(), **extras)

            def split():
                k.peer_pooled_gather_fwd(st.tables, st.rf_w_off, st.feat_rows, g.feat_block, g.feat_owner, lay, ids,
                                         offsets, B, W, out, st.mirror, st.feat_mirror_off, feat_sel=sel[1])
                k.peer_pooled_gather_fwd(st.tables, st.rf_w_off, st.feat_rows, g.feat_block, g.feat_owner, lay, ids,
                                         offsets, B, W, out, st.mirror, st.feat_mirror_off, feat_sel=sel[0])

            phases = {
                "gather": lambda: k.peer_pooled_gather_fwd(st.tables, st.rf_w_off, st.feat_rows, g.feat_block,
                                                           g.feat_owner, lay, ids, offsets, B, W, out, st.mirror,
                                                           st.feat_mirror_off),
                "gather_split": split,
                "mirror": lambda: k.peer_mirror_refresh(st.tables, W, *st._seg, st.mirror),
                "push_update": push_update,
            }
            t = {p: [] for p in phases}
            for _ in range(a.rounds):
                for p, fn in phases.items():
                    t[p].append(timed(fn, a.iters))
            slots = int(st.counts.t[:W].sum())
            recv_slots = int(sum(int(s.counts.t[0]) for s in sts))
            touched = recv_slots        # upper bound on the rows the owner touches (one row per received slot)
            n_mirror = int(st.mirror.numel())
            alg = {"gather": nnz * 8 + (F_B1 := (g.F * B + 1) * 8) + nnz * 16 * e + B * lay.total_dim * 4,
                   "gather_split": nnz * 8 + 2 * F_B1 + nnz * 16 * e + B * lay.total_dim * 4,
                   "mirror": 2 * n_mirror * e,
                   "push_update": slots * (4 + 2 * 16 * 4) + recv_slots * (16 * 4 + 8) + touched * (2 * 16 * e + 2 * 16 * 4)}
            for p, v in t.items():
                med = statistics.median(v)
                res = dict(part="kernels", tables=dt_name, ids=dist_kind, phase=p, W=W, B=B, nnz=nnz, us=round(med, 2),
                           us_min=round(min(v), 2), us_max=round(max(v), 2), alg_bytes=alg[p],
                           alg_GBps=round(alg[p] / med / 1e3, 1), gpu=info)
                results.append(res)
                print(json.dumps(res), flush=True)
        del sts, st, g
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def bench_step(a, info, results):
    """The whole graphed step on the peer exchange, FP32 and FP16 tables (one process per GPU)."""
    import torch.distributed as dist

    from torcheasyrec_b200.engine import GraphedTrainStep, Pipeline

    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29533")
        os.environ.setdefault("RANK", "0")
        os.environ.setdefault("WORLD_SIZE", "1")
        rank = int(os.environ.get("LOCAL_RANK", os.environ["RANK"]))
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", device_id=torch.device(f"cuda:{rank}"))
    rank, W = dist.get_rank(), dist.get_world_size()
    dev = f"cuda:{torch.cuda.current_device()}"
    from torcheasyrec_b200 import example_configs
    from torcheasyrec_b200.config import parse_text

    cfg = parse_text(example_configs.GENERATORS["dlrm_criteo"]())
    f16 = {f"feature_configs[{i}].id_feature.data_type": "FP16" for i, fc in enumerate(cfg.feature_configs)
           if fc.HasField("id_feature")}
    for dt_name, edits in (("fp32", None), ("fp16", f16)):
        p = Pipeline("dlrm_criteo", device=dev, max_rows=a.max_rows or None, seed=0, sharding="row_wise",
                     exchange="peer", static_capacity=2.0, edits=edits)
        batches = [p.synthetic_batch(a.batch, seed=100 + i + 1000 * rank) for i in range(4)]
        step = GraphedTrainStep(p, batches[0], warmup=3)
        batches = [bt.pin_memory() for bt in batches]
        v = []
        for _ in range(a.rounds):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            s.record()
            for i in range(a.iters):
                step.load(batches[i % 4])
                step.replay()
            e.record()
            torch.cuda.synchronize()
            v.append(s.elapsed_time(e) * 1e3 / a.iters)
        for sm in p.sharded:
            sm.check_overflow()
        med = statistics.median(v)
        res = dict(part="step", tables=dt_name, W=W, B=a.batch, us=round(med, 2), us_min=round(min(v), 2),
                   us_max=round(max(v), 2), gpu=info)
        if rank == 0:
            results.append(res)
            print(json.dumps(res), flush=True)
        del step, p
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    dist.barrier()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=4, help="virtual ranks of the kernel timings")
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--max-rows", type=int, default=0, help="cap every table (0: the full hash sizes)")
    ap.add_argument("--step", action="store_true", help="also time the whole graphed step")
    ap.add_argument("--step-only", action="store_true", help="only the graphed step (torchrun on real ranks)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    info = gpu_info()
    results = []
    if not a.step_only:
        torch.cuda.set_device(0)
        print(f"# {info}; W = {a.world} virtual ranks on one GPU; {a.rounds} rounds x {a.iters} calls", flush=True)
        bench_kernels(a, K.default_kernels(), info, results)
    if a.step or a.step_only:
        bench_step(a, info, results)
    if a.out and results:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
