"""Sharded embedding collections: table-wise / row-wise / mixed placement over one NVSwitch domain.

Replaces what the reference obtains from torchrec's DistributedModelParallel (tzrec/main.py:783-804,
tzrec/utils/dist_util.py:164-195): ShardedEmbeddingBagCollection / ShardedEmbeddingCollection with their
input-dist (KJT bucketize + all-to-all, App. A.5/A.7), lookup, output-dist (A.6/A.8) and fused backward.

H100-first design (DESIGN.md §6) — ONE exchange pattern for every sharding type:
  forward   1. K1 bucketize: every id -> (owner rank, local row); table-wise = "block >= rows, owner = rank of
               the table", row-wise = "block = ceil(rows/W), owner 0" (tzk_bucketize_rw)
            2. all-to-all of the per-(dest, feature) id COUNTS [W,F] (a few hundred bytes, instead of torchrec's
               F*B lengths per peer) and of the ids themselves
            3. owner: un-pooled row gather straight from its shard arena (tzk_seq_gather_fwd)
            4. all-to-all of the rows back (the "return all-to-all" of north_star; for L=1 this is B*sum(D)*4
               bytes per rank instead of the reference's W-times larger dense reduce-scatter, SURVEY §7.2 H3)
            5. sample owner: pooled gather over the returned rows in ORIGINAL list order (tzk_pooled_gather_fwd
               on the row buffer) -> results are bit-identical for every W and every placement
  backward  5'. one gradient row per id at its wire slot (tzk_bag_grad_expand)  4'. all-to-all to the owners
            3'. owner: fused segmented optimizer update with grad_scale = 1/W (App. A.6) (tzk_fused_bwd)
NCCL (or gloo in CPU tests) carries the three all-to-alls; split sizes need one host read of the [2,W,F] count
matrix per collection per step.
Dense parameters are replicated; `DenseGradSync` averages their gradients (the reference wraps them in DDP).
"""

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

import torch
import torch.distributed as dist
from torch import nn

from . import functional as Fn
from .embedding_modules import (EmbeddingBagCollection, EmbeddingBagConfig, EmbeddingCollection, EmbeddingConfig,
                                PoolingType, SparseOptimizerSpec, _ArenaCollection)
from .kernels import POOL_MEAN, POOL_SUM, FeatureLayout, build_layout
from .sparse import JaggedTensor, KeyedJaggedTensor, KeyedTensor

TABLE_WISE, ROW_WISE = "table_wise", "row_wise"
BIG_BLOCK = 1 << 62


@dataclass
class TableShard:
    kind: str          # table_wise | row_wise
    owner: int = 0     # table_wise: rank that holds the whole table
    block: int = 0     # row_wise: rows per rank = ceil(rows / W)   (App. A.7)


def rw_block(rows: int, world: int) -> int:
    return max((rows + world - 1) // world, 1)


def make_plan(tables: Sequence, world: int, default: str = ROW_WISE,
              constraints: Optional[Dict[str, Sequence[str]]] = None, rw_min_rows: int = 0) -> Dict[str, TableShard]:
    """Constraint-driven placement (replaces the perf-model planner of tzrec/utils/plan_util.py:93-206).

    `constraints[table]` = allowed sharding types (embedding_constraints / global_embedding_constraints,
    feature.proto:6-13); first supported entry wins.  `default` may be "table_wise", "row_wise" or "mixed"
    (row-wise for tables with >= rw_min_rows rows, table-wise otherwise — BASELINE cfg5).
    Table-wise owners: largest tables first onto the rank with the fewest rows so far (deterministic)."""
    plan: Dict[str, TableShard] = {}
    load = [0] * world
    kinds = {}
    for c in tables:
        allowed = list((constraints or {}).get(c.name, []))
        kind = next((k for k in allowed if k in (TABLE_WISE, ROW_WISE)), None)
        if kind is None:
            kind = (ROW_WISE if c.num_embeddings >= rw_min_rows else TABLE_WISE) if default == "mixed" else default
        kinds[c.name] = kind
    for c in sorted(tables, key=lambda c: (-c.num_embeddings, c.name)):
        if kinds[c.name] == TABLE_WISE:
            r = min(range(world), key=lambda i: (load[i], i))
            load[r] += c.num_embeddings
            plan[c.name] = TableShard(TABLE_WISE, owner=r)
        else:
            plan[c.name] = TableShard(ROW_WISE, block=rw_block(c.num_embeddings, world))
    return {c.name: plan[c.name] for c in tables}


def local_rows(cfg, shard: TableShard, rank: int) -> int:
    if shard.kind == TABLE_WISE:
        return cfg.num_embeddings if shard.owner == rank else 0
    return max(0, min(shard.block, cfg.num_embeddings - rank * shard.block))


def _a2a(out: torch.Tensor, inp: torch.Tensor, out_splits, in_splits, group) -> torch.Tensor:
    dist.all_to_all_single(out, inp, out_splits, in_splits, group=group)
    return out


class _DimGroup:
    """All tables of one embedding_dim of a sharded collection: local shard arena + wire/return layouts."""

    def __init__(self, configs: List, plan: Dict[str, TableShard], rank: int, world: int, device, pooled: bool,
                 names: List[List[str]]):
        self.configs, self.rank, self.world, self.pooled = configs, rank, world, pooled
        from .embedding_modules import DataType

        if any(getattr(c, "data_type", DataType.FP32) != DataType.FP32 for c in configs):
            raise NotImplementedError("FP16 tables are supported on unsharded collections only")
        self.dim = configs[0].embedding_dim
        rows_local = [local_rows(c, plan[c.name], rank) for c in configs]
        cls = EmbeddingBagCollection if pooled else EmbeddingCollection
        # local shard arena + slot bookkeeping; output keys follow the WHOLE collection's naming
        self.local = cls(configs, device=device, local_rows=rows_local, names_by_table=names)
        self.local.allow_interleave = False      # peers read this arena (dense rows): csrc/tzk_peer.cu
        self.feature_names = self.local.feature_names()
        self.embedding_names = self.local._embedding_names
        F = len(self.feature_names)
        self.F = F
        lay = self.local.layout
        # bucketize parameters per feature slot
        blocks, owners = [], []
        for t in self.local._feat_table:
            sh = plan[configs[t].name]
            blocks.append(BIG_BLOCK if sh.kind == TABLE_WISE else sh.block)
            owners.append(sh.owner if sh.kind == TABLE_WISE else 0)
        self.feat_block = torch.tensor(blocks, dtype=torch.int64, device=device)
        self.feat_owner = torch.tensor(owners, dtype=torch.int32, device=device)
        # owner-side layout: slot (src, f) for src in range(W) -> same local table as f
        self.owner_layout = FeatureLayout(
            w_off=lay.w_off * world, rows=lay.rows * world, dim=lay.dim * world, col=[0] * (F * world),
            pool=[POOL_SUM] * (F * world), key_base=lay.key_base * world, total_keys=lay.total_keys,
            total_dim=self.dim, arena_elems=lay.arena_elems).to(device)
        # static-capacity variant (graph-capturable step): per source rank F feature slots + one padding slot
        padw = lambda xs, v: [x for r in range(world) for x in (list(xs) + [v])]
        self.owner_layout_static = FeatureLayout(
            w_off=padw(lay.w_off, 0), rows=padw(lay.rows, 0), dim=padw(lay.dim, self.dim),   # rows 0 = padding slot
            col=[0] * ((F + 1) * world), pool=[POOL_SUM] * ((F + 1) * world), key_base=padw(lay.key_base, 0),
            total_keys=lay.total_keys, total_dim=self.dim, arena_elems=lay.arena_elems).to(device)
        self.static_alpha: Optional[float] = None     # set by shard_model(static_capacity=...)
        self.static_cap: Optional[int] = None
        self.static_nnz: Optional[int] = None
        self.overflow = torch.zeros(1, dtype=torch.int32, device=device)
        # sample-owner layout over the returned row buffer ("table" = rows in wire order)
        self._ret_layout_cache: Dict[int, FeatureLayout] = {}
        self._pool = list(lay.pool)
        self._col = list(lay.col)
        self.total_dim = lay.total_dim
        self.device = device

    def ret_layout(self, nnz: int) -> FeatureLayout:
        lay = self._ret_layout_cache.get(nnz)
        if lay is None:
            F = self.F
            lay = FeatureLayout(w_off=[0] * F, rows=[max(nnz, 1)] * F, dim=[self.dim] * F, col=self._col,
                                pool=self._pool, key_base=[0] * F, total_keys=max(nnz, 1), total_dim=self.total_dim,
                                arena_elems=max(nnz, 1) * self.dim).to(self.device)
            if len(self._ret_layout_cache) > 64:
                self._ret_layout_cache.clear()
            self._ret_layout_cache[nnz] = lay
        return lay


class _Dispatch:
    """Steps 1-4 of the forward for one dim group; keeps what the backward needs."""

    def __init__(self, g: _DimGroup, kjt: KeyedJaggedTensor, group) -> None:
        k = Fn.backend()
        W, F, B = g.world, g.F, kjt.stride()
        self.g, self.B, self.group = g, B, group
        ids, offsets = kjt.values(), kjt.offsets()
        self.offsets = offsets
        self.nnz = ids.numel()
        _, oo, oids, _, inv = k.bucketize_rw(ids, offsets, F, B, W, g.feat_block, feat_owner=g.feat_owner,
                                             want_inv=True)
        self.inv = inv
        seg = oo[::B]                                    # [W*F+1] segment starts
        counts = (seg[1:] - seg[:-1]).view(W, F)         # ids per (dest, feature)
        recv_counts = torch.empty_like(counts)
        dist.all_to_all_single(recv_counts, counts, group=group)   # [src, F]
        both = torch.stack([counts, recv_counts]).cpu()  # the one host read per step
        self.in_splits = both[0].sum(1).tolist()         # what I send to each dest
        self.out_splits = both[1].sum(1).tolist()        # what I receive from each src
        n_recv = sum(self.out_splits)
        self.recv_ids = _a2a(torch.empty(n_recv, dtype=torch.int64, device=ids.device), oids, self.out_splits,
                             self.in_splits, group)
        self.bounds = k.lengths_to_offsets(recv_counts.reshape(-1).to(torch.int32))   # [W*F+1], B=1 "bags"
        self.n_recv = n_recv
        self.n_slots = self.nnz

    def rows_forward(self) -> torch.Tensor:
        g, k = self.g, Fn.backend()
        rows = k.seq_gather_fwd(g.local.weights.data, g.owner_layout, self.recv_ids, self.bounds, 1)
        ret = torch.empty((self.nnz, g.dim), dtype=torch.float32, device=rows.device)
        return _a2a(ret, rows, self.in_splits, self.out_splits, self.group)          # wire order

    def rows_backward(self, g_rows: torch.Tensor) -> None:
        g, k = self.g, Fn.backend()
        recv_g = torch.empty((self.n_recv, g.dim), dtype=torch.float32, device=g_rows.device)
        _a2a(recv_g, g_rows, self.out_splits, self.in_splits, self.group)
        spec = g.local.optimizer
        if spec is None:
            raise RuntimeError("sharded collection: no sparse optimizer set (call set_optimizer)")
        if self.n_recv:
            k.fused_bwd(spec.kind, False, recv_g, g.local.weights.data, g.local.opt_state, g.owner_layout,
                        self.recv_ids, self.bounds, 1, spec.lr, spec.eps, 1.0 / g.world,   # App. A.6: /W
                        **g.local.opt_extras())


class _StaticDispatch:
    """Same exchange with STATIC shapes (no host read, CUDA-graph capturable): every (src -> dest) message has a
    fixed capacity `cap` = ceil(alpha * nnz / W) ids; unused slots carry id 0 of a per-source padding slot and
    zero gradient rows, so they change nothing at the owner.  Counts travel as data; an overflow (a peer needs more
    than `cap`) raises the device flag `g.overflow`, which the caller checks after the step(s).
    Only for fixed-nnz workloads (one id per bag, like Criteo / Taobao non-sequence features)."""

    def __init__(self, g: _DimGroup, kjt: KeyedJaggedTensor, group) -> None:
        k = Fn.backend()
        W, F, B = g.world, g.F, kjt.stride()
        self.g, self.B, self.group = g, B, group
        ids, offsets = kjt.values(), kjt.offsets()
        dev = ids.device
        self.offsets = offsets
        self.nnz = nnz = ids.numel()
        if g.static_cap is None:
            g.static_nnz = nnz
            g.static_cap = (int(g.static_alpha * nnz / W) + 8) // 8 * 8
        if nnz != g.static_nnz:
            raise RuntimeError(f"static-capacity sharding was sized for {g.static_nnz} ids per step, got {nnz}")
        cap = g.static_cap
        self.n_slots = W * cap
        # bucketize straight into the fixed-capacity wire layout (destination r starts at slot r*cap)
        _, oo, send_ids, _, inv = k.bucketize_rw(ids, offsets, F, B, W, g.feat_block, feat_owner=g.feat_owner,
                                                 want_inv=True, wire_capacity=cap)
        seg = oo[::B]                                              # [W*F+1]
        dest_start = oo[::F * B]                                   # [W+1] compact start of every destination
        # ids beyond `cap` are dropped by the scatter, in compact (f, b) order per destination: the counts that travel
        # are clamped the same way, so the owner's per-source bounds always sum to <= cap and a later source's slots
        # never shift.  The overflowing step's update is lossy (the dropped ids get no gradient); every rank learns
        # about it in the same step because the flag rides along with the counts (column F).
        rel_s = (seg[:-1].view(W, F) - dest_start[:-1].unsqueeze(1)).clamp_(max=cap)
        rel_e = (seg[1:].view(W, F) - dest_start[:-1].unsqueeze(1)).clamp_(max=cap)
        over = ((dest_start[1:] - dest_start[:-1]) > cap).any().to(seg.dtype)
        counts = torch.cat([rel_e - rel_s, over.expand(W, 1)], dim=1)        # [dest, F + 1]
        self.inv = inv                                             # padded slot of every original id position
        recv = torch.empty_like(counts)
        dist.all_to_all_single(recv, counts, group=group)          # [src, F + 1], equal splits
        g.overflow.add_(recv[:, F].max().to(torch.int32))          # any source overflowed -> every rank raises together
        recv_counts = recv[:, :F].contiguous()
        self.recv_ids = torch.empty_like(send_ids)
        dist.all_to_all_single(self.recv_ids, send_ids, group=group)
        # owner-side "bags": per source its F feature runs, then the padding run up to cap
        tot = recv_counts.sum(1, keepdim=True)
        lens = torch.cat([recv_counts, (cap - tot).clamp_(min=0)], dim=1).reshape(-1).to(torch.int32)
        self.bounds = k.lengths_to_offsets(lens)                   # [W*(F+1)+1]

    def rows_forward(self) -> torch.Tensor:
        g, k = self.g, Fn.backend()
        rows = k.seq_gather_fwd(g.local.weights.data, g.owner_layout_static, self.recv_ids, self.bounds, 1)
        ret = torch.empty_like(rows)
        dist.all_to_all_single(ret, rows, group=self.group)
        return ret

    def rows_backward(self, g_rows: torch.Tensor) -> None:
        g, k = self.g, Fn.backend()
        recv_g = torch.empty_like(g_rows)
        dist.all_to_all_single(recv_g, g_rows, group=self.group)
        spec = g.local.optimizer
        if spec is None:
            raise RuntimeError("sharded collection: no sparse optimizer set (call set_optimizer)")
        k.fused_bwd(spec.kind, False, recv_g, g.local.weights.data, g.local.opt_state, g.owner_layout_static,
                    self.recv_ids, self.bounds, 1, spec.lr, spec.eps, 1.0 / g.world, **g.local.opt_extras())


def _dispatch(g: _DimGroup, kjt: KeyedJaggedTensor, group):
    return _StaticDispatch(g, kjt, group) if g.static_alpha else _Dispatch(g, kjt, group)


class _ShardedPooled(torch.autograd.Function):
    @staticmethod
    def forward(ctx, hook, g: _DimGroup, kjt: KeyedJaggedTensor, group):
        d = _dispatch(g, kjt, group)
        ret = d.rows_forward()
        out = Fn.backend().pooled_gather_fwd(ret.view(-1), g.ret_layout(d.n_slots), d.inv.to(torch.int64),
                                             d.offsets, d.B)
        ctx.d = d
        return out

    @staticmethod
    def backward(ctx, grad_out):
        d = ctx.d
        static = isinstance(d, _StaticDispatch)
        g_rows = Fn.backend().bag_grad_expand(Fn._rows_contig(grad_out), d.g.ret_layout(d.n_slots), d.offsets,
                                              d.inv.to(torch.int32), d.B, d.n_slots, zero=static)
        d.rows_backward(g_rows)
        return None, None, None, None


class _ShardedSeq(torch.autograd.Function):
    @staticmethod
    def forward(ctx, hook, g: _DimGroup, kjt: KeyedJaggedTensor, group):
        d = _Dispatch(g, kjt, group)
        ret = d.rows_forward()
        ctx.d = d
        return ret.index_select(0, d.inv.to(torch.int64)) if d.nnz else ret   # back to original id order

    @staticmethod
    def backward(ctx, grad_rows):
        d = ctx.d
        g_rows = torch.empty_like(grad_rows)
        if d.nnz:
            g_rows.index_copy_(0, d.inv.to(torch.int64), grad_rows.contiguous())
        d.rows_backward(g_rows)
        return None, None, None, None


class _ShardedBase(nn.Module):
    _pooled = True

    def __init__(self, tables: Sequence, plan: Dict[str, TableShard], device, group=None) -> None:
        super().__init__()
        self._group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self._configs = list(tables)
        self.plan = plan
        from .embedding_modules import output_names_by_table

        names = dict(zip([c.name for c in self._configs], output_names_by_table(self._configs)))
        by_dim: Dict[int, List] = {}
        for c in self._configs:
            by_dim.setdefault(c.embedding_dim, []).append(c)
        self.groups: List[_DimGroup] = [
            _DimGroup(cs, plan, self.rank, self.world, device, self._pooled, [names[c.name] for c in cs])
            for cs in by_dim.values()]
        self.shards = nn.ModuleList([g.local for g in self.groups])   # registers the local arenas
        for g in self.groups:            # checkpoints address the tables through this module's keys only
            g.local._load_via_owner = True
        self._hook = None

    def set_optimizer(self, spec: SparseOptimizerSpec) -> None:
        for g in self.groups:
            g.local.set_optimizer(spec)

    def _maybe_enable_peer(self, features: KeyedJaggedTensor) -> bool:
        """exchange="peer": on the first call move the shards into symmetric memory, size the wire buffers for this
        batch size and re-route forward() to the peer-memory kernels (collective: every rank gets here in its first
        step).  `_ids_budget` (KJT key -> ids per bag) sizes features with more than one id per bag."""
        if getattr(self, "_exchange", "nccl") != "peer" or getattr(self, "_peer_states", None) is not None:
            return False
        from .peer_exchange import enable_peer_exchange

        B = features.stride()
        per_bag = getattr(self, "_ids_budget", None) or {}
        enable_peer_exchange(self, B, {k: int(v) * B for k, v in per_bag.items()})
        return True

    def sparse_arenas(self) -> List[_ArenaCollection]:
        return [g.local for g in self.groups]

    def check_overflow(self) -> None:
        """Static-capacity mode: raises if any step since the last check needed more than the wire capacity.  The flag
        is exchanged inside the step, so every rank raises in the same call (no rank is left inside a collective)."""
        for g in self.groups:
            if g.static_alpha and int(g.overflow.item()):
                g.overflow.zero_()
                raise RuntimeError(f"static-capacity all-to-all overflowed (cap={g.static_cap} ids per peer); raise "
                                   "static_capacity or use the dynamic exchange")

    def _hook_tensor(self, device) -> Optional[torch.Tensor]:
        if not torch.is_grad_enabled():
            return None
        if self._hook is None or self._hook.device != device:
            self._hook = torch.zeros(1, device=device, requires_grad=True)
        return self._hook

    # ---- checkpoint keys (SURVEY §8f N2): the reference's per-table names, never `shards.*` -------------------------
    def _table_attr(self) -> str:
        return "embedding_bags" if self._pooled else "embeddings"

    def _table_shard(self, name: str):
        for g in self.groups:
            for t, c in enumerate(g.configs):
                if c.name == name:
                    sh = self.plan[name]
                    start = 0 if sh.kind == TABLE_WISE else self.rank * sh.block
                    n = g.local._table_rows[t]
                    return c, start, (g.local.table_weight(t) if n else None)
        raise KeyError(name)

    def state_dict(self, *args, destination=None, prefix="", keep_vars=False):
        """One entry per table, `<prefix>embedding_bags.<table>.weight`: a ShardedTensor of the table's global
        [rows, D] shape whose local shard views this rank's arena (what torchrec's sharded modules return and
        torch.distributed.checkpoint re-shards on load).  Collective."""
        from collections import OrderedDict

        from .checkpoint import sharded_rows_tensor

        if args:
            destination = args[0]
            prefix = args[1] if len(args) > 1 else prefix
        destination = OrderedDict() if destination is None else destination
        for c in self._configs:
            _, start, local = self._table_shard(c.name)
            destination[f"{prefix}{self._table_attr()}.{c.name}.weight"] = sharded_rows_tensor(
                local, start, (c.num_embeddings, c.embedding_dim), self._group)
        return destination

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        """Accepts, per table, the full [rows, D] tensor (a reference / W=1 checkpoint: this rank keeps its rows) or a
        ShardedTensor whose local shard matches this rank's (the in-place DCP flow)."""
        from torch.distributed._shard.sharded_tensor import ShardedTensor

        for c in self._configs:
            key = f"{prefix}{self._table_attr()}.{c.name}.weight"
            if key not in state_dict:
                if strict:
                    missing_keys.append(key)
                continue
            v = state_dict[key]
            _, start, local = self._table_shard(c.name)
            if isinstance(v, ShardedTensor):
                shards = v.local_shards()
                if local is None:
                    continue
                if len(shards) != 1 or list(shards[0].tensor.shape) != list(local.shape) or \
                        shards[0].metadata.shard_offsets[0] != start:
                    error_msgs.append(f"{key}: the ShardedTensor's local shard does not match this rank's rows "
                                      f"[{start}, {start + local.shape[0]})")
                    continue
                if shards[0].tensor.data_ptr() != local.data_ptr():
                    with torch.no_grad():
                        local.copy_(shards[0].tensor)
            else:
                if tuple(v.shape) != (c.num_embeddings, c.embedding_dim):
                    error_msgs.append(f"size mismatch for {key}: checkpoint {tuple(v.shape)}, table "
                                      f"{(c.num_embeddings, c.embedding_dim)}")
                    continue
                self.load_full_table(c.name, v)

    def load_full_table(self, name: str, full: torch.Tensor) -> None:
        """Copies this rank's rows of a full (unsharded) table into the local shard (parity tests, restore)."""
        for g in self.groups:
            for t, c in enumerate(g.configs):
                if c.name == name:
                    sh = self.plan[name]
                    n = g.local._table_rows[t]
                    if n:
                        start = 0 if sh.kind == TABLE_WISE else self.rank * sh.block
                        g.local.set_table_weight(t, full[start:start + n].to(g.local.weights.device))

    def gather_full_table(self, name: str) -> torch.Tensor:
        """All-gathers a table's shards back into [rows, D] (every rank gets it; tests / checkpoints)."""
        for g in self.groups:
            for t, c in enumerate(g.configs):
                if c.name == name:
                    sh = self.plan[name]
                    block = c.num_embeddings if sh.kind == TABLE_WISE else sh.block
                    pad = torch.zeros((block, c.embedding_dim), dtype=torch.float32, device=g.local.weights.device)
                    n = g.local._table_rows[t]
                    if n:
                        pad[:n] = g.local.table_weight(t)
                    parts = [torch.empty_like(pad) for _ in range(self.world)]
                    dist.all_gather(parts, pad, group=self._group)
                    if sh.kind == TABLE_WISE:
                        return parts[sh.owner]
                    return torch.cat(parts)[:c.num_embeddings]
        raise KeyError(name)


class ShardedEmbeddingBagCollection(_ShardedBase):
    """forward(KJT of the local batch) -> KeyedTensor [B, sum D], same values as the unsharded collection."""

    def embedding_bag_configs(self) -> List[EmbeddingBagConfig]:
        return self._configs

    def forward(self, features: KeyedJaggedTensor) -> KeyedTensor:
        if self._maybe_enable_peer(features):
            return self.forward(features)
        keys, lens, vals = [], [], []
        for g in self.groups:
            kjt = g.local._select(features)
            vals.append(_ShardedPooled.apply(self._hook_tensor(kjt.values().device), g, kjt, self._group))
            keys += g.embedding_names
            lens += [g.dim] * g.F
        return KeyedTensor(keys, lens, vals[0] if len(vals) == 1 else torch.cat(vals, dim=1))


class ShardedEmbeddingCollection(_ShardedBase):
    _pooled = False

    def embedding_configs(self) -> List[EmbeddingConfig]:
        return self._configs

    def embedding_names_by_table(self) -> List[List[str]]:
        return [n for g in self.groups for n in g.local.embedding_names_by_table()]

    def forward(self, features: KeyedJaggedTensor) -> Dict[str, JaggedTensor]:
        if self._maybe_enable_peer(features):
            return self.forward(features)
        out: Dict[str, JaggedTensor] = {}
        for g in self.groups:
            kjt = g.local._select(features)
            rows = _ShardedSeq.apply(self._hook_tensor(kjt.values().device), g, kjt, self._group)
            lpk, lengths, B = kjt.length_per_key(), kjt.lengths(), kjt.stride()
            s = 0
            for f, key in enumerate(g.embedding_names):
                out[key] = JaggedTensor(rows[s:s + lpk[f]], lengths=lengths[f * B:(f + 1) * B])
                s += lpk[f]
        return out


class DenseGradSync:
    """Average of the replicated dense gradients (the reference wraps dense params in DDP, dist_util.py:164-195):
    one flat buffer, one all-reduce per step."""

    def __init__(self, params: Sequence[torch.nn.Parameter], group=None) -> None:
        self.params = [p for p in params if p.requires_grad]
        self.group = group
        self.world = dist.get_world_size(group)
        n = sum(p.numel() for p in self.params)
        dev = self.params[0].device if self.params else "cpu"
        self.flat = torch.zeros(n, dtype=torch.float32, device=dev)
        o = 0
        for p in self.params:
            p.grad = self.flat[o:o + p.numel()].view_as(p)   # grads accumulate straight into the flat buffer
            o += p.numel()

    def zero(self) -> None:
        self.flat.zero_()
        o = 0
        for p in self.params:
            if p.grad is None or p.grad.data_ptr() != self.flat[o:o + p.numel()].data_ptr():
                p.grad = self.flat[o:o + p.numel()].view_as(p)
            o += p.numel()

    def sync(self) -> None:
        if self.world > 1:
            dist.all_reduce(self.flat, group=self.group)
            self.flat.div_(self.world)


def shard_model(model, device, default: str = ROW_WISE, group=None, rw_min_rows: int = 0, source=None,
                constraints: Optional[Dict[str, Sequence[str]]] = None, static_capacity: Optional[float] = None,
                exchange: str = "nccl", ids_per_bag: Optional[Dict[str, int]] = None):
    """Swaps every arena collection of `model.embedding_group` for its sharded twin (tzrec/main.py:799).

    `exchange="peer"`: the collections exchange through peer memory of the NVSwitch domain (csrc/tzk_peer.cu,
    peer_exchange.py) instead of NCCL all-to-alls; `static_capacity` is then the head-room factor of the wire buffers
    (default 1.5) and `ids_per_bag` (KJT key -> most ids per bag; sequence features: their sequence_length) sizes
    features with more than one id per bag (everything else: one id per bag).

    The model may have been built with its embedding collections on the meta device (as the reference does,
    embedding.py:187-188): shards are materialised directly on `device`, each rank initialising its own shard
    (like torchrec, App. A.4).  `source`: optional unsharded model with identical tables whose weights seed the
    shards instead (parity tests).  Returns the list of sharded modules."""
    eg = model.embedding_group
    world = dist.get_world_size(group)
    device = torch.device(device)
    sharded = []

    def convert(parent, attr, coll, src_coll):
        plan = make_plan(coll._configs, world, default, dict(constraints or {}), rw_min_rows)
        cls = ShardedEmbeddingBagCollection if isinstance(coll, EmbeddingBagCollection) else ShardedEmbeddingCollection
        new = cls(coll._configs, plan, device, group)
        pooled = isinstance(new, ShardedEmbeddingBagCollection)
        if exchange == "peer":         # peer-memory kernels instead of the NCCL all-to-alls (peer_exchange.py)
            # features without an entry in ids_per_bag carry one id per bag; a step with more ids than the budget
            # raises in the lookup (host-side size check) instead of overflowing silently
            new._exchange = "peer"
            new._ids_budget = {f: int((ids_per_bag or {})[f]) for g in new.groups for f in g.feature_names
                               if (ids_per_bag or {}).get(f)}
            for g in new.groups:
                g.static_alpha = float(static_capacity or 1.5)
        elif static_capacity and pooled:
            for g in new.groups:       # fixed-shape exchange (see _StaticDispatch); pooled collections only
                g.static_alpha = float(static_capacity)
        if coll.optimizer is not None:
            new.set_optimizer(coll.optimizer)
        seed = src_coll if src_coll is not None else (coll if coll.weights.device.type != "meta" else None)
        if seed is not None:
            for t, c in enumerate(seed._configs):
                new.load_full_table(c.name, seed.table_weight(t))
        if isinstance(parent, nn.ModuleDict):
            parent[attr] = new
        else:
            setattr(parent, attr, new)
        sharded.append(new)

    src_eg = source.embedding_group if source is not None else None
    for key, impl in eg.emb_impls.items():
        if impl.has_sparse:
            convert(impl, "ebc", impl.ebc, src_eg.emb_impls[key].ebc if src_eg is not None else None)
    for key, impl in eg.seq_emb_impls.items():
        for dim_key in list(impl.ec_dict.keys()):
            convert(impl.ec_dict, dim_key, impl.ec_dict[dim_key],
                    src_eg.seq_emb_impls[key].ec_dict[dim_key] if src_eg is not None else None)
    return sharded
