"""EmbeddingBagCollection / EmbeddingCollection with HBM-resident shard arenas and a fused backward.

This is the module object the reference builds at tzrec/modules/embedding.py:855 (EBC) and :1195 (EC) and
calls with one KeyedJaggedTensor at :930 / :1301.  In the reference these classes come from torchrec
([EXT] torchrec.modules.embedding_modules / embedding_configs) and the arithmetic from fbgemm TBE; here the
tables of a collection live back to back in ONE fp32 arena per rank, the forward is the tzk pooled / sequence
gather, and the backward applies the sparse optimizer in place (the reference installs the same behaviour
with apply_optimizer_in_backward, tzrec/main.py:774-781) — no dense gradient is ever materialised.
"""

import math
from dataclasses import dataclass, field
from enum import Enum
from typing import Callable, Dict, List, Optional, Sequence

import os
import weakref

import torch
from torch import nn

from . import functional as Fn
from .kernels import (OPT_ADAGRAD, OPT_ADAM, OPT_PARTIAL_ROWWISE_ADAM, OPT_ROWWISE_ADAGRAD, OPT_SGD, POOL_MEAN, POOL_SUM,
                      FeatureLayout, build_layout)
from .sparse import JaggedTensor, KeyedJaggedTensor, KeyedTensor


class PoolingType(Enum):
    SUM = "SUM"
    MEAN = "MEAN"
    NONE = "NONE"


class DataType(Enum):
    FP32 = "FP32"
    FP16 = "FP16"


@dataclass
class BaseEmbeddingConfig:
    num_embeddings: int
    embedding_dim: int
    name: str = ""
    data_type: DataType = DataType.FP32
    feature_names: List[str] = field(default_factory=list)
    init_fn: Optional[Callable[[torch.Tensor], Optional[torch.Tensor]]] = None

    def get_weight_init_max(self) -> float:
        return math.sqrt(1.0 / self.num_embeddings)


@dataclass
class EmbeddingBagConfig(BaseEmbeddingConfig):
    pooling: PoolingType = PoolingType.SUM


@dataclass
class EmbeddingConfig(BaseEmbeddingConfig):
    pass


@dataclass
class SparseOptimizerSpec:
    """What tzrec/optim/optimizer_builder.py:30-97 hands to apply_optimizer_in_backward."""

    kind: int = OPT_ADAGRAD
    lr: float = 0.001
    eps: float = 1e-8                      # fbgemm TBE default (App. A.10)
    initial_accumulator_value: float = 0.0  # optimizer_builder.py:57-61
    beta1: float = 0.9                      # Adam variants (optimizer.proto:89-131)
    beta2: float = 0.999
    weight_decay: float = 0.0
    max_gradient: float = 0.0               # > 0 <=> gradient_clipping: clamp the summed row gradient

    @staticmethod
    def from_name(name: str, **kw) -> "SparseOptimizerSpec":
        kinds = {"sgd": OPT_SGD, "adagrad": OPT_ADAGRAD, "rowwise_adagrad": OPT_ROWWISE_ADAGRAD,
                 "row_wise_adagrad": OPT_ROWWISE_ADAGRAD, "adam": OPT_ADAM,
                 "partial_rowwise_adam": OPT_PARTIAL_ROWWISE_ADAM}
        return SparseOptimizerSpec(kind=kinds[name.lower()], **kw)


def _default_init(cfg: BaseEmbeddingConfig, w: torch.Tensor) -> None:
    # [EXT] torchrec default init_fn: uniform(-1/sqrt(N), +1/sqrt(N))  (App. A.4)
    bound = cfg.get_weight_init_max()
    w.uniform_(-bound, bound)


def output_names_by_table(configs: Sequence[BaseEmbeddingConfig]) -> List[List[str]]:
    """Output key of every (table, feature) slot: `feature`, or `feature@table` when the feature is served by
    more than one table of the collection (App. A.2; tzrec/modules/embedding.py:826-827 relies on it)."""
    count: Dict[str, int] = {}
    for c in configs:
        for f in c.feature_names:
            count[f] = count.get(f, 0) + 1
    return [[f + "@" + c.name if count[f] > 1 else f for f in c.feature_names] for c in configs]


class _TableView(nn.Module):
    """`embedding_bags.<table>.weight` / `embeddings.<table>.weight` handle (a view into the arena)."""

    def __init__(self, owner: "_ArenaCollection", t: int) -> None:
        super().__init__()
        self._owner = [owner]
        self._t = t

    @property
    def weight(self) -> torch.Tensor:
        return self._owner[0].table_weight(self._t)

    def _load_from_state_dict(self, *args, **kwargs) -> None:
        return None      # `<table>.weight` is consumed by the owning collection (it writes into the arena)


class _ArenaCollection(nn.Module):
    """Shared machinery: arena, layout, optimizer state, key mapping."""

    _pooled = True

    def __init__(self, tables: Sequence[BaseEmbeddingConfig], device=None, local_rows: Optional[Sequence[int]] = None,
                 names_by_table: Optional[List[List[str]]] = None):
        super().__init__()
        self._configs = list(tables)
        names = [c.name for c in self._configs]
        assert len(set(names)) == len(names), f"duplicate table names {names}"
        self._device = torch.device(device) if device is not None else torch.device("cpu")
        # output keys: a feature served by >1 table of the (whole, unsharded) collection is feat@table (App. A.2)
        if names_by_table is None:
            names_by_table = output_names_by_table(self._configs)
        self._feature_names: List[str] = []     # KJT key consumed by each slot
        self._embedding_names: List[str] = []   # output key of each slot
        self._names_by_table: List[List[str]] = []
        feat_table, feat_pool = [], []
        for t, c in enumerate(self._configs):
            per = list(names_by_table[t])
            for f in c.feature_names:
                self._feature_names.append(f)
                feat_table.append(t)
                pool = getattr(c, "pooling", PoolingType.SUM)
                feat_pool.append(POOL_MEAN if pool == PoolingType.MEAN else POOL_SUM)
            self._embedding_names.extend(per)
            self._names_by_table.append(per)
        self._feat_table = feat_table
        rows = list(local_rows) if local_rows is not None else [c.num_embeddings for c in self._configs]
        self._table_rows = rows
        self._table_dim = [c.embedding_dim for c in self._configs]
        self.layout: FeatureLayout = build_layout(rows, self._table_dim, feat_table, feat_pool)
        self._table_off, self._table_key = {}, {}
        for f, t in enumerate(feat_table):
            self._table_off[t] = self.layout.w_off[f]
            self._table_key[t] = self.layout.key_base[f]
        # EmbeddingBagConfig.data_type (feature.proto `data_type`, features/feature.py:626,652): FP16 tables keep their
        # rows as halfs in the arena — half the gather bytes; pooling, outputs, gradients and optimizer state stay fp32,
        # the update rounds the new row to nearest (SURVEY §8f N4).  One dtype per collection.
        kinds = {getattr(c, "data_type", DataType.FP32) for c in self._configs}
        if len(kinds) > 1:
            raise NotImplementedError("a collection mixes FP32 and FP16 tables: group them by data_type")
        self.table_dtype = torch.float16 if kinds == {DataType.FP16} else torch.float32
        self.weights = nn.Parameter(torch.empty(self.layout.arena_elems, dtype=self.table_dtype, device=self._device),
                                    requires_grad=False)
        self._opt: Optional[SparseOptimizerSpec] = None
        self.register_buffer("opt_state", None, persistent=False)
        self.register_buffer("opt_state2", None, persistent=False)
        self.register_buffer("opt_step", None, persistent=False)
        self._hook = None
        self.grad_scale = 1.0  # sharded wrappers set 1/W here (App. A.6)
        # [weight row | Adagrad accumulator row] interleaving (set_optimizer): unsharded CUDA collections only; the local
        # shards of sharded collections keep dense rows (their arenas are read by peers: csrc/tzk_peer.cu)
        self.allow_interleave = True
        # the fused update runs on a side stream and is normally joined when the backward pass ends; a step driver that
        # promises to call join_pending() itself (engine.Pipeline.step_body: after the dense optimizer step) sets this and
        # gets the dense-gradient sync and the dense optimizer overlapped with the sparse update as well
        self.defer_join = False
        self._pending_join = None
        if self._device.type != "meta":
            self.reset_parameters()
            self.layout.to(self._device)

    # ---- parameters -----------------------------------------------------------------------------------
    def reset_parameters(self) -> None:
        with torch.no_grad():
            for t, c in enumerate(self._configs):
                if t not in self._table_off:
                    continue
                w = self.table_weight(t)
                if w.numel() == 0:
                    continue
                init = c.init_fn or (lambda x, c=c: _default_init(c, x))
                if w.dtype == torch.float32:
                    init(w)
                else:       # initialise in fp32 (same random stream as an FP32 table), then round once
                    tmp = torch.empty(w.shape, dtype=torch.float32, device=w.device)
                    init(tmp)
                    w.copy_(tmp)

    def table_weight(self, t: int) -> torch.Tensor:
        o, r, d = self._table_off[t], self._table_rows[t], self._table_dim[t]
        if self.layout.interleaved:       # [rows, 2 D] lines: weights in the first half (a strided view)
            return self.weights.data[o:o + r * 2 * d].view(r, 2 * d)[:, :d]
        return self.weights.data[o:o + r * d].view(r, d)

    def table_state(self, t: int) -> Optional[torch.Tensor]:
        if self.layout.interleaved:
            o, r, d = self._table_off[t], self._table_rows[t], self._table_dim[t]
            return self.weights.data[o:o + r * 2 * d].view(r, 2 * d)[:, d:]
        if self.opt_state is None:
            return None
        if self._opt.kind in (OPT_ADAGRAD, OPT_ADAM, OPT_PARTIAL_ROWWISE_ADAM):
            o = self._table_off[t]
            return self.opt_state[o:o + self._table_rows[t] * self._table_dim[t]].view(self._table_rows[t], -1)
        k = self._table_key[t]
        return self.opt_state[k:k + self._table_rows[t]]

    def set_table_weight(self, t: int, w: torch.Tensor) -> None:
        with torch.no_grad():
            self.table_weight(t).copy_(w)

    def dense_weights(self) -> torch.Tensor:
        """The tables back to back with dense rows (what `weights` holds unless the rows are interleaved with their
        optimizer state): layout-independent comparisons in tests, checkpoints of earlier versions."""
        if not self.layout.interleaved:
            return self.weights.data
        return torch.cat([self.table_weight(t).reshape(-1) for t in range(len(self._configs)) if t in self._table_off])

    def _relayout(self, interleaved: bool, fill: float) -> None:
        """Re-lays the arena with dense rows, or as [weight row | accumulator row] lines (kernels.build_layout)."""
        old = {t: self.table_weight(t) for t in range(len(self._configs)) if t in self._table_off}   # views of the old arena
        lay = build_layout(self._table_rows, self._table_dim, self._feat_table, list(self.layout.pool),
                           interleaved=interleaved)
        arena = torch.full((lay.arena_elems,), fill, dtype=torch.float32, device=self.weights.device)
        self.layout = lay.to(self.weights.device)
        for f, t in enumerate(self._feat_table):
            self._table_off[t] = lay.w_off[f]
            self._table_key[t] = lay.key_base[f]
        self.weights.data = arena
        for t, w in old.items():
            self.table_weight(t).copy_(w)

    # ---- checkpoint keys (SURVEY §8f N2) ------------------------------------------------------------------
    # The reference's state_dict holds one entry per table, `<prefix>embedding_bags.<table>.weight` (EBC) or
    # `<prefix>embeddings.<table>.weight` (EC) (tzrec/utils/checkpoint_util_test.py:375-396), and its fused optimizer
    # state is keyed `state.<that key>.<table>.momentum1`.  The arena is an implementation detail: it never appears
    # in a state_dict, and both directions go through per-table views.
    def _table_attr(self) -> str:
        return "embedding_bags" if self._pooled else "embeddings"

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        for t, c in enumerate(self._configs):
            if t in self._table_off:
                w = self.table_weight(t)
                destination[f"{prefix}{self._table_attr()}.{c.name}.weight"] = w if keep_vars else w.detach()

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        if getattr(self, "_load_via_owner", False):     # local shard of a sharded collection: its owner loaded it
            return
        arena_key = prefix + "weights"          # checkpoints written by earlier versions of this package
        if arena_key in state_dict:
            w = state_dict[arena_key]
            if self.layout.interleaved:
                with torch.no_grad():
                    o = 0
                    for t in range(len(self._configs)):
                        if t in self._table_off:
                            n = self._table_rows[t] * self._table_dim[t]
                            o = (o + 3) // 4 * 4
                            self.table_weight(t).copy_(w.reshape(-1)[o:o + n].view(self._table_rows[t], -1))
                            o += n
            elif w.numel() != self.weights.numel():
                error_msgs.append(f"size mismatch for {arena_key}: {tuple(w.shape)} vs {tuple(self.weights.shape)}")
            else:
                with torch.no_grad():
                    self.weights.data.copy_(w.reshape(-1))
            return
        for t, c in enumerate(self._configs):
            if t not in self._table_off:
                continue
            key = f"{prefix}{self._table_attr()}.{c.name}.weight"
            if key not in state_dict:
                if strict:
                    missing_keys.append(key)
                continue
            w = state_dict[key]
            want = (self._table_rows[t], self._table_dim[t])
            if tuple(w.shape) != want:
                error_msgs.append(f"size mismatch for {key}: checkpoint {tuple(w.shape)}, table {want}")
                continue
            self.set_table_weight(t, w.to(self.weights.device))

    def fused_optimizer_state_dict(self, prefix: str = "") -> Dict[str, torch.Tensor]:
        """`state.<param key>.<table>.momentum1` per table (the reference's `model.fused_optimizer.state_dict()` keys,
        checkpoint_util_test.py:387-390).  Element-wise Adagrad: [rows, dim]; row-wise Adagrad: [rows]; SGD: empty."""
        out: Dict[str, torch.Tensor] = {}
        for t, c in enumerate(self._configs):
            st = self.table_state(t) if t in self._table_off else None
            if st is not None:
                out[f"state.{prefix}{self._table_attr()}.{c.name}.weight.{c.name}.momentum1"] = st
        return out

    def load_fused_optimizer_state_dict(self, state: Dict[str, torch.Tensor], prefix: str = "",
                                        strict: bool = True) -> None:
        for t, c in enumerate(self._configs):
            dst = self.table_state(t) if t in self._table_off else None
            if dst is None:
                continue
            key = f"state.{prefix}{self._table_attr()}.{c.name}.weight.{c.name}.momentum1"
            if key not in state:
                if strict:
                    raise KeyError(key)
                continue
            with torch.no_grad():
                dst.copy_(state[key].to(dst.device).reshape(dst.shape))

    # ---- fused optimizer ------------------------------------------------------------------------------
    def set_optimizer(self, spec: SparseOptimizerSpec) -> None:
        """apply_optimizer_in_backward equivalent (tzrec/main.py:774-781)."""
        self._opt = spec
        dev = self.weights.device
        if self.layout.interleaved:        # a second set_optimizer: back to dense rows first (the old state is dropped)
            self._relayout(False, 0.0)
        # TZK_INTERLEAVE: "0": dense rows; "force": also off CUDA (host-logic tests); default on
        env = os.environ.get("TZK_INTERLEAVE", "1")
        if (spec.kind == OPT_ADAGRAD and self.allow_interleave and self.table_dtype == torch.float32
                and ((dev.type == "cuda" and env != "0") or env == "force")):
            # a D = 16 row and its accumulator in ONE 128-B line: the fused update reads and writes whole lines (two
            # half-line writes cost DRAM a read-modify-write each — profiles/README.md, round 2)
            self._relayout(True, spec.initial_accumulator_value)
            self.opt_state = None
        elif spec.kind == OPT_ADAGRAD:
            self.opt_state = torch.full((self.layout.arena_elems,), spec.initial_accumulator_value,
                                        dtype=torch.float32, device=dev)
        elif spec.kind == OPT_ROWWISE_ADAGRAD:
            self.opt_state = torch.full((self.layout.total_keys,), spec.initial_accumulator_value,
                                        dtype=torch.float32, device=dev)
        elif spec.kind in (OPT_ADAM, OPT_PARTIAL_ROWWISE_ADAM):
            self.opt_state = torch.zeros(self.layout.arena_elems, dtype=torch.float32, device=dev)    # momentum1
            n2 = self.layout.arena_elems if spec.kind == OPT_ADAM else self.layout.total_keys
            self.opt_state2 = torch.zeros(n2, dtype=torch.float32, device=dev)                        # momentum2
            self.opt_step = torch.zeros((), dtype=torch.float32, device=dev)                          # iteration t
        else:
            self.opt_state = None
        if spec.kind not in (OPT_ADAM, OPT_PARTIAL_ROWWISE_ADAM):
            self.opt_state2, self.opt_step = None, None

    def opt_extras(self, bump: bool = True) -> dict:
        """Keyword arguments of the extended update (tzk_opt_args) — empty for the classic kinds without clipping.
        `bump` advances the device-side step counter first (one call per backward)."""
        spec = self._opt
        if spec is None:
            return {}
        ex = {}
        if spec.kind in (OPT_ADAM, OPT_PARTIAL_ROWWISE_ADAM):
            if bump:
                self.opt_step.add_(1.0)
            ex.update(state2=self.opt_state2, step=self.opt_step, beta1=spec.beta1, beta2=spec.beta2,
                      weight_decay=spec.weight_decay)
        if spec.max_gradient > 0 or ex:
            ex["max_gradient"] = spec.max_gradient
        return ex

    @property
    def optimizer(self) -> Optional[SparseOptimizerSpec]:
        return self._opt

    # ---- introspection used by tzrec (models/model.py:162-201, embedding.py:670-671) --------------------
    def embedding_names_by_table(self) -> List[List[str]]:
        return self._names_by_table

    def feature_names(self) -> List[str]:
        return self._feature_names

    def _bwd_workspace(self, k, nnz: int) -> torch.Tensor:
        """Private fused-backward workspace (the sorted keys live here between forward and backward)."""
        need = k.fused_bwd_workspace_bytes(self.layout, nnz)
        ws = getattr(self, "_bwd_ws", None)
        if ws is None or ws.numel() < need or ws.device != self.weights.device:
            ws = torch.empty(max(need, 256), dtype=torch.uint8, device=self.weights.device)
            self._bwd_ws = ws
        return ws

    def _side_stream(self) -> "torch.cuda.Stream":
        st = getattr(self, "_side", None)
        if st is None:
            st = torch.cuda.Stream(device=self.weights.device)
            self._side = st
        return st

    def join_pending(self) -> None:
        """Orders the current stream after a fused update that is still running on the side stream (defer_join)."""
        pj = self._pending_join
        if pj is not None:
            torch.cuda.current_stream().wait_stream(pj)
            self._pending_join = None
            self._pending_apply = None

    def _hook_tensor(self) -> torch.Tensor:
        # autograd needs one differentiable input to schedule the fused backward
        if self._hook is None or self._hook.device != self.weights.device:
            self._hook = torch.zeros(1, device=self.weights.device, requires_grad=True)
        return self._hook

    def _select(self, kjt: KeyedJaggedTensor) -> KeyedJaggedTensor:
        """Bring the KJT into this collection's slot order (identity when it already is)."""
        keys = kjt.keys()
        if keys == self._feature_names:
            return kjt
        pos = {k: i for i, k in enumerate(keys)}
        return kjt.permute([pos[f] for f in self._feature_names])


def _early_sort(ctx, mod, pooled: bool, ids, offsets, B, want_grad: bool) -> None:
    """Enqueue the id-only half of the fused backward (linearize + radix sort) on the module's side stream right
    away: it overlaps the rest of the forward pass and the dense backward instead of sitting on the critical path
    (the role TrainPipelineSparseDist's data-dist stream plays in the reference, tzrec/utils/dist_util.py:221-303).
    The backward then only joins the stream and runs the gradient-dependent half."""
    ctx.early = None
    k = Fn.backend()
    owner = getattr(mod, "_early_owner", None)
    if getattr(mod, "_early_busy", False) and (owner is None or owner() is None):
        # the lookup that owns the workspace is gone without a backward (e.g. a prediction made with grad enabled, its
        # graph already freed): its sort is orphaned on the side stream — join it and release the workspace.  A
        # lookup that is still alive (second lookup of the same module inside one forward pass) keeps ownership and
        # this one takes the one-stream path.
        torch.cuda.current_stream().wait_stream(mod._side_stream())
        mod._early_busy = False
    # (`want_grad` comes from the caller: inside autograd.Function.forward grad mode is always off)
    if (mod.training and want_grad and ids.is_cuda and ids.numel() > 0
            and hasattr(k, "fused_bwd_sort") and mod.optimizer is not None
            and not getattr(mod, "_early_busy", False)      # one outstanding lookup per module owns the workspace
            and os.environ.get("TZK_EARLY_SORT", "1") != "0"):
        ws = mod._bwd_workspace(k, ids.numel())
        side = mod._side_stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            k.fused_bwd_sort(pooled, mod.layout, ids, offsets, B, ws)
        ctx.early = (ws, side)
        mod._early_busy = True
        mod._early_owner = weakref.ref(ctx)


def _fused_backward(ctx, mod, pooled: bool, grad, ids, offsets, who: str) -> None:
    spec = mod.optimizer
    if spec is None:
        raise RuntimeError(f"{who}.backward: no sparse optimizer set (call set_optimizer); tables are updated "
                           "inside the backward kernel like the reference's fused TBE")
    if not ids.numel():
        return
    k = Fn.backend()
    if ctx.early is not None:
        ws, side = ctx.early
        mod._early_busy = False
        cur = torch.cuda.current_stream()
        extras = mod.opt_extras()          # (advances the device step counter on `cur`)
        if os.environ.get("TZK_ASYNC_APPLY", "1") != "0":
            # The gradient half stays on the side stream (it is already ordered after the sort there) and the rest of
            # the backward pass — whatever autograd schedules after this node, e.g. the bottom MLP of DLRM — runs
            # next to it; the stream is joined when the backward pass ends.  Nothing between here and the join reads
            # or writes the tables.
            side.wait_stream(cur)          # the gradient (and the step counter) were produced on `cur`
            with torch.cuda.stream(side):
                k.fused_bwd_apply(spec.kind, pooled, grad, mod.weights.data, mod.opt_state, mod.layout, offsets,
                                  ids.numel(), ctx.B, spec.lr, spec.eps, mod.grad_scale, ws, **extras)
            # keeps the buffers the side-stream kernel reads away from the allocator until the join (autograd drops
            # the saved tensors as soon as this node returns)
            mod._pending_apply = (grad, offsets, ids)

            def _join(mod=mod, cur=cur, side=side):
                cur.wait_stream(side)
                mod._pending_apply = None

            if mod.defer_join:
                mod._pending_join = side      # the step driver joins after the dense optimizer step (join_pending)
            else:
                torch.autograd.Variable._execution_engine.queue_callback(_join)
        else:
            cur.wait_stream(side)
            k.fused_bwd_apply(spec.kind, pooled, grad, mod.weights.data, mod.opt_state, mod.layout, offsets,
                              ids.numel(), ctx.B, spec.lr, spec.eps, mod.grad_scale, ws, **extras)
    else:
        k.fused_bwd(spec.kind, pooled, grad, mod.weights.data, mod.opt_state, mod.layout, ids, offsets, ctx.B,
                    spec.lr, spec.eps, mod.grad_scale, **mod.opt_extras())


class _PooledLookup(torch.autograd.Function):
    @staticmethod
    def forward(ctx, hook, mod, ids, offsets, B):
        out = Fn.backend().pooled_gather_fwd(mod.weights.data, mod.layout, ids, offsets, B)
        ctx.mod, ctx.B = mod, B
        ctx.save_for_backward(ids, offsets)
        _early_sort(ctx, mod, True, ids, offsets, B, hook is not None)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        ids, offsets = ctx.saved_tensors
        _fused_backward(ctx, ctx.mod, True, Fn._rows_contig(grad_out), ids, offsets, "EmbeddingBagCollection")
        return None, None, None, None, None


class _SeqLookup(torch.autograd.Function):
    @staticmethod
    def forward(ctx, hook, mod, ids, offsets, B):
        out = Fn.backend().seq_gather_fwd(mod.weights.data, mod.layout, ids, offsets, B)
        ctx.mod, ctx.B = mod, B
        ctx.save_for_backward(ids, offsets)
        _early_sort(ctx, mod, False, ids, offsets, B, hook is not None)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        ids, offsets = ctx.saved_tensors
        _fused_backward(ctx, ctx.mod, False, grad_out.contiguous(), ids, offsets, "EmbeddingCollection")
        return None, None, None, None, None


class EmbeddingBagCollection(_ArenaCollection):
    """Pooled lookup: forward(KJT) -> KeyedTensor [B, sum_t sum_f D_t]  (embedding.py:855,930; App. A.2/A.3)."""

    def __init__(self, tables: Sequence[EmbeddingBagConfig], device=None, local_rows=None, names_by_table=None) -> None:
        super().__init__(tables, device, local_rows, names_by_table)
        self.embedding_bags = nn.ModuleDict({c.name: _TableView(self, t) for t, c in enumerate(self._configs)})
        self._lengths_per_key = [self._table_dim[t] for t in self._feat_table]

    def embedding_bag_configs(self) -> List[EmbeddingBagConfig]:
        return self._configs

    def pooled_values(self, kjt: KeyedJaggedTensor) -> torch.Tensor:
        kjt = self._select(kjt)
        B = kjt.stride()
        hook = self._hook_tensor() if torch.is_grad_enabled() else None
        return _PooledLookup.apply(hook, self, kjt.values(), kjt.offsets(), B)

    def forward(self, features: KeyedJaggedTensor) -> KeyedTensor:
        return KeyedTensor(self._embedding_names, self._lengths_per_key, self.pooled_values(features))


class EmbeddingCollection(_ArenaCollection):
    """Un-pooled lookup: forward(KJT) -> {key: JaggedTensor([sum len, D], lengths[B])} (embedding.py:1195,1301)."""

    _pooled = False

    def __init__(self, tables: Sequence[EmbeddingConfig], device=None, local_rows=None, names_by_table=None) -> None:
        super().__init__(tables, device, local_rows, names_by_table)
        dims = set(self._table_dim)
        assert len(dims) <= 1, f"EmbeddingCollection tables must share one embedding_dim, got {dims}"
        self._dim = self._table_dim[0] if self._table_dim else 0
        self.embeddings = nn.ModuleDict({c.name: _TableView(self, t) for t, c in enumerate(self._configs)})

    def embedding_configs(self) -> List[EmbeddingConfig]:
        return self._configs

    def embedding_dim(self) -> int:
        return self._dim

    def forward(self, features: KeyedJaggedTensor) -> Dict[str, JaggedTensor]:
        kjt = self._select(features)
        B = kjt.stride()
        hook = self._hook_tensor() if torch.is_grad_enabled() else None
        rows = _SeqLookup.apply(hook, self, kjt.values(), kjt.offsets(), B)
        lpk = kjt.length_per_key()
        lengths = kjt.lengths()
        out, s = {}, 0
        for f, key in enumerate(self._embedding_names):
            out[key] = JaggedTensor(rows[s:s + lpk[f]], lengths=lengths[f * B:(f + 1) * B])
            s += lpk[f]
        return out
