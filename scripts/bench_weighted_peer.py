"""Times the weighted peer-step kernels against the unweighted ones with CUDA events: the requester's gather, the
bucketize (count + scan + scatter; weighted: + the slot weights) and the push of the gradient slices.

W virtual ranks live on ONE GPU: their arenas, wire and receive buffers are allocations of the same device and the
pointer tables point there, so rank 0's kernels run as they would on a node — except that every "remote" row and
every pushed slice stays in local HBM.  These numbers are the local instruction and byte cost of the weights only; the
NVLink cost and the step time at N > 1 are not measured here.

Two shapes (row-wise plan, W = 4 by default, the small tables mirrored as PeerState does):
  criteo  DLRM-Criteo's 26 tables (D = 16, one id per bag) at B = 65536;
  ccp     the Ali-CCP MMoE config's tables, multi-hot bags of 1..2L-1 ids (mean L = 5), B = 8192; one line per dim group.
Modes alternate round after round; each line is the median over rounds with the min-max spread.  Algorithmic bytes
added by the weights: +4 B per id for the gather (the weight), +8 B per id for the bucketize (weight read + slot
weight written) and +4 B per filled wire slot for the push (the slot weight).  The card's name and power limit are read
in the same call and printed with the numbers.

    python scripts/bench_weighted_peer.py [--world 4] [--iters 50] [--rounds 5] [--max-rows 0] [--out FILE]
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
from torcheasyrec_b200.embedding_modules import output_names_by_table  # noqa: E402
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


class _Sym:
    def __init__(self, t, everyone, W):
        self.t, self.everyone, self.W = t, everyone, W

    @property
    def ptrs(self):
        return (ctypes.c_uint64 * self.W)(*[self.everyone[r].data_ptr() for r in range(self.W)])


def virtual_ranks(coll, W, B, per_bag):
    """PeerState of every dim group for W virtual ranks on cuda:0 (built one after the other: no barrier is crossed)."""
    cfgs = coll._configs
    plan = make_plan(cfgs, W, "row_wise")
    names = dict(zip([c.name for c in cfgs], output_names_by_table(cfgs)))
    by_dim = {}
    for c in cfgs:
        by_dim.setdefault(c.embedding_dim, []).append(c)
    out = []
    for gi, cs in enumerate(by_dim.values()):
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
            g = _DimGroup(cs, plan, r, W, torch.device("cuda:0"), True, [names[c.name] for c in cs])
            g.static_alpha = 2.0
            sts.append(St(g, plan, None, B, [B * per_bag] * g.F))
        out.append(sts)
    return out


def batch(g, B, mean_len, gen):
    F, dev = g.F, g.device
    if mean_len <= 1:
        lengths = torch.ones(F * B, dtype=torch.int64, device=dev)
    else:
        lengths = torch.randint(1, 2 * mean_len, (F * B,), dtype=torch.int64, device=dev, generator=gen)
    offsets = torch.zeros(F * B + 1, dtype=torch.int64, device=dev)
    offsets[1:] = torch.cumsum(lengths, 0)
    rows = torch.tensor([g.configs[t].num_embeddings for t in g.local._feat_table], device=dev)
    feat = torch.repeat_interleave(torch.arange(F, device=dev), lengths.view(F, B).sum(1))
    ids = (torch.rand(int(offsets[-1]), device=dev, generator=gen) * rows[feat]).to(torch.int64)
    return ids, offsets


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=4)
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
    torch.cuda.set_device(0)
    k = K.default_kernels()
    info = gpu_info()
    W = a.world
    print(f"# {info}; W = {W} virtual ranks on one GPU; {a.rounds} rounds x {a.iters} calls", flush=True)
    gen = torch.Generator(device="cuda").manual_seed(1)
    results = []
    for name, cfg, B, L in (("criteo", "dlrm_criteo", a.criteo_batch, 1), ("ccp", CCP, a.ccp_batch, a.ccp_mean_len)):
        coll = Pipeline(cfg, device="cuda:0", max_rows=a.max_rows or None, seed=0).model.sparse_collections()[0]
        for sts in virtual_ranks(coll, W, B, 2 * L):
            st = sts[0]
            g, lay = st.g, st.g.local.layout
            ids, offsets = batch(g, B, L, gen)
            nnz = ids.numel()
            psw = torch.rand(nnz, device="cuda", generator=gen) * 2
            grad = torch.randn(B, lay.total_dim, device="cuda", generator=gen)
            st.wire_w = torch.zeros(W * st.cap, dtype=torch.float32, device="cuda")
            if st.mirror is not None:
                k.peer_mirror_refresh(st.tables, W, *st._seg, st.mirror)
            modes = {"unweighted": {}, "weighted": {"per_sample_weights": psw}}
            t = {(m, p): [] for m in modes for p in ("gather", "bucketize", "push")}
            for _ in range(a.rounds):
                for m, kw in modes.items():
                    t[(m, "gather")].append(timed(lambda: k.peer_pooled_gather_fwd(
                        st.tables, st.rf_w_off, st.feat_rows, g.feat_block, g.feat_owner, lay, ids, offsets, B, W, None,
                        st.mirror, st.feat_mirror_off, **kw), a.iters))
                    bkw = dict(kw, wire_w=st.wire_w) if kw else {}
                    t[(m, "bucketize")].append(timed(lambda: k.peer_bucketize(
                        ids, offsets, g.F, B, W, st.feat_block_wire, g.feat_owner, st.feat_rows, st.rf_key_base, True,
                        st.cap, st.wire_key.t, st.wire_idx.t, st.counts.t, **bkw), a.iters))
                    pkw = {"wire_w": st.wire_w} if kw else {}
                    t[(m, "push")].append(timed(lambda: k.peer_push_grad(
                        st.recv, grad, lay, offsets, st.wire_idx.t, st.counts.t, 0, W, st.cap, B, True, **pkw), a.iters))
            torch.cuda.synchronize()
            slots = int(st.counts.t[:W].sum())
            assert int(st.counts.t[W]) == 0, "wire capacity overflowed: raise static_alpha"
            rows_read = sum(lay.dim[f] * 4 * int(offsets[(f + 1) * B] - offsets[f * B]) for f in range(g.F))
            base = {"gather": nnz * 8 + rows_read + B * lay.total_dim * 4,
                    "bucketize": nnz * 8 * 2 + slots * 12,      # ids read twice (count, scatter), key + idx per slot
                    "push": slots * (4 + 2 * lay.dim[0] * 4)}    # idx + slice read + slice written
            extra = {"gather": 4 * nnz, "bucketize": 8 * nnz, "push": 4 * slots}
            for (m, p), v in t.items():
                alg = base[p] + (extra[p] if m == "weighted" else 0)
                med = statistics.median(v)
                res = dict(shape=name, dim=lay.dim[0], F=g.F, B=B, W=W, nnz=nnz, slots=slots, mode=m, phase=p,
                           us=round(med, 2), us_min=round(min(v), 2), us_max=round(max(v), 2), alg_bytes=alg,
                           alg_GBps=round(alg / med / 1e3, 1), gpu=info)
                results.append(res)
                print(json.dumps(res), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
