"""Step driver: builds a model from a tzrec pipeline config and runs train steps on one H100.

Replaces the part of tzrec/main.py that surrounds the hot path (model construction :763-781, optimizers
:814-876, the step loop :519-547) and torchrec's TrainPipelineSparseDist (tzrec/utils/dist_util.py:221-303)
with an H100-first design: the whole step (KJT scan, gather, interaction, dense towers, loss, backward incl.
the fused sparse update, dense optimizer) is captured ONCE in a CUDA graph over static device buffers and
replayed; a side stream stages the next host batch (pinned H2D) while the current graph runs.
Variable-shape workloads (sequence features) run the same code eagerly.
"""

import os
from typing import Any, Dict, List, Optional, Sequence

import torch

from .batch import Batch, synthetic_batch
from .config import Message, edit_config, load_pipeline_config
from .features import BaseFeature, create_features
from .rank_models import (RankModel, TrainWrapper, create_model, dense_optimizer_from_config,
                          mixed_precision_to_dtype, sparse_optimizer_from_config)
from .sparse import KeyedJaggedTensor, KeyedTensor


def override_num_buckets(cfg: Message, cap: int) -> None:
    """`num_buckets -> cap` for every id feature (BASELINE.json configs[0]: "1k-row tables")."""
    def fix(sub):
        for fld in ("num_buckets", "hash_bucket_size"):
            if sub._spec(fld) is not None and sub.HasField(fld):
                setattr(sub, fld, min(getattr(sub, fld), cap))
    for fc in cfg.feature_configs:
        kind = fc.WhichOneof("feature")
        sub = getattr(fc, kind)
        if sub._type == "SequenceFeature":
            for s in sub.features:
                fix(getattr(s, s.WhichOneof("feature")))
        else:
            fix(sub)


class Pipeline:
    """Everything needed to step one model: config, features, model, optimizers."""

    def __init__(self, config: str, device="cuda", max_rows: Optional[int] = None,
                 edits: Optional[Dict[str, Any]] = None, seed: int = 1234, capturable: bool = True,
                 sharding: Optional[str] = None, group=None, rw_min_rows: int = 0,
                 static_capacity: Optional[float] = None, exchange: str = "nccl") -> None:
        """`config`: path of a pipeline .config/.json, or the name of a built-in example
        (example_configs.GENERATORS: dlrm_criteo, deepfm_criteo, mmoe_taobao, multi_tower_din_taobao)."""
        from . import example_configs
        from .config import parse_text

        if config in example_configs.GENERATORS:
            self.cfg = parse_text(example_configs.GENERATORS[config]())
        else:
            self.cfg = load_pipeline_config(config)
        if edits:
            edit_config(self.cfg, edits)
        if max_rows:
            override_num_buckets(self.cfg, max_rows)
        self.device = torch.device(device)
        self.features: List[BaseFeature] = create_features(list(self.cfg.feature_configs),
                                                           fg_mode=self.cfg.data_config.fg_mode)
        self.labels = list(self.cfg.data_config.label_fields)
        if list(self.cfg.data_config.sample_weight_fields):
            raise NotImplementedError("data_config.sample_weight_fields: weighted losses are outside the hot-path scope")
        torch.manual_seed(seed)
        self.sharded, self.grad_sync = [], None
        if sharding is None:
            self.model: RankModel = create_model(self.cfg.model_config, self.features, self.labels,
                                                 device=self.device)
        else:
            # tables are built on the meta device and materialised per shard (embedding.py:187-188, main.py:799)
            from .distributed import DenseGradSync, shard_model

            self.model = create_model(self.cfg.model_config, self.features, self.labels, device=torch.device("meta"))
            # sequence features carry up to `sequence_length` ids per bag (sizes the peer exchange's wire buffers)
            per_bag = {f.name: int(f.sequence_length) for f in self.features if f.is_sequence and f.sequence_length}
            self.sharded = shard_model(self.model, self.device, default=sharding, group=group,
                                       rw_min_rows=rw_min_rows, constraints=self._table_constraints(),
                                       static_capacity=static_capacity, exchange=exchange, ids_per_bag=per_bag)
        self.model.to(self.device)
        if sharding is not None:
            if exchange == "peer" and self.device.type == "cuda":
                from .peer_exchange import PeerDenseGradSync      # no NCCL call anywhere in the step

                self.grad_sync = PeerDenseGradSync(self.model.dense_parameters(), group)
            else:
                self.grad_sync = DenseGradSync(self.model.dense_parameters(), group)
        self.model.set_sparse_optimizer(sparse_optimizer_from_config(self.cfg.train_config))
        kw = {}
        if self.device.type == "cuda" and capturable:
            kw = dict(capturable=True, fused=True)
        self.dense_optimizer = dense_optimizer_from_config(self.cfg.train_config, self.model.dense_parameters(), **kw)
        tc = self.cfg.train_config
        self.mixed_dtype = mixed_precision_to_dtype(tc.mixed_precision)
        if self.mixed_dtype is not None and tc.HasField("grad_scaler"):
            raise NotImplementedError("train_config.grad_scaler: loss scaling over the fused sparse update is not "
                                      "implemented (mixed_precision without grad_scaler is)")
        self.train_wrapper = TrainWrapper(self.model, self.mixed_dtype, self.device.type)
        torch.backends.cuda.matmul.allow_tf32 = bool(self.cfg.train_config.cuda_matmul_allow_tf32)

    def _table_constraints(self) -> Dict[str, List[str]]:
        """{table: allowed sharding types} from per-feature `embedding_constraints` (features/feature.py:832-845)
        with train_config.global_embedding_constraints as the fallback (tzrec/main.py:788-790)."""
        eg = self.model.embedding_group
        out: Dict[str, List[str]] = {}
        gc = self.cfg.train_config.global_embedding_constraints
        default = list(gc.sharding_types) if self.cfg.train_config.HasField("global_embedding_constraints") else []
        for impl in eg.emb_impls.values():
            if impl.has_sparse:
                for c in impl.ebc.embedding_bag_configs():
                    out[c.name] = default
            for name, pc in impl._emb_bag_constraints.items():
                out[name] = pc.sharding_types or default
        for impl in eg.seq_emb_impls.values():
            for ec in impl.ec_dict.values():
                for c in ec.embedding_configs():
                    out[c.name] = default
            for consts in impl._dim_to_emb_constraints.values():
                for name, pc in consts.items():
                    out[name] = pc.sharding_types or default
        return out

    def synthetic_batch(self, batch_size: int, seed: int = 0, id_dist: str = "uniform") -> Batch:
        b = synthetic_batch(self.features, batch_size, self.labels, seed=seed, id_dist=id_dist)
        for kjt in b.sparse_features.values():
            kjt.length_per_key()  # host-side, before the copy: keeps the device path free of syncs
        return b

    def step_body(self, batch: Batch) -> torch.Tensor:
        """forward + backward (fused sparse update inside) + dense gradient sync + dense optimizer step."""
        if self.grad_sync is not None:
            self.grad_sync.zero()
        # the fused sparse updates stay on their side streams through the dense-gradient sync and the dense optimizer step
        # (neither touches a table); they are joined here, at the end of the step, instead of at the end of backward()
        joiners = self._sparse_joiners() if os.environ.get("TZK_DEFER_JOIN", "1") != "0" else []
        for j in joiners:
            j.defer_join = True
        try:
            loss, _ = self.train_wrapper(batch)
            loss.backward()
            if self.grad_sync is not None:
                self.grad_sync.sync()
            self.dense_optimizer.step()
        finally:
            for j in joiners:
                j.defer_join = False
                j.join_pending()
        return loss.detach()

    def _sparse_joiners(self) -> list:
        """Everything that runs a fused sparse update on a side stream: unsharded collections, peer-exchange states."""
        out = getattr(self, "_joiners", None)
        if out is None:
            from .embedding_modules import _ArenaCollection

            out = [m for m in self.model.modules() if isinstance(m, _ArenaCollection)]
            for sm in self.sharded:
                out += list(getattr(sm, "_peer_states", []) or [])
            self._joiners = out
        return out

    def eager_step(self, batch: Batch) -> torch.Tensor:
        if self.grad_sync is None:
            self.dense_optimizer.zero_grad(set_to_none=True)
        return self.step_body(batch)

    def check_overflow(self) -> None:
        for m in self.sharded:
            m.check_overflow()


def _tensors_of(batch: Batch) -> List[torch.Tensor]:
    out = []
    for k in sorted(batch.sparse_features):
        kjt = batch.sparse_features[k]
        out += [kjt.values(), kjt.lengths()]
        if kjt.weights_or_none() is not None:      # weighted id features: replay must see the new weights too
            out.append(kjt.weights_or_none())
    for k in sorted(batch.dense_features):
        out.append(batch.dense_features[k].values())
    for k in sorted(batch.labels):
        out.append(batch.labels[k])
    return out


class GraphedTrainStep:
    """One CUDA graph per (model, batch shape).  `load()` refreshes the static inputs, `replay()` runs a step."""

    def __init__(self, pipe: Pipeline, example: Batch, warmup: int = 3) -> None:
        assert pipe.device.type == "cuda"
        self.pipe = pipe
        self.static = example.to(pipe.device)
        for k, kjt in example.sparse_features.items():
            self.static.sparse_features[k]._length_per_key = kjt._length_per_key
        self._static_tensors = _tensors_of(self.static)
        self.copy_stream = torch.cuda.Stream()
        self._staging = None
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self._fresh_kjt_caches()
                pipe.eager_step(self.static)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        if pipe.grad_sync is None:
            pipe.dense_optimizer.zero_grad(set_to_none=True)
        self._fresh_kjt_caches()
        with torch.cuda.graph(self.graph):
            self.loss = pipe.step_body(self.static)
        torch.cuda.synchronize()

    def _fresh_kjt_caches(self) -> None:
        # offsets are derived data: recompute them from the (possibly refreshed) lengths inside every step
        for kjt in self.static.sparse_features.values():
            kjt._offsets = None

    def load(self, batch: Batch, non_blocking: bool = True) -> None:
        """Copies a batch (host pinned or device) into the static buffers on the current stream."""
        for dst, src in zip(self._static_tensors, _tensors_of(batch)):
            dst.copy_(src, non_blocking=non_blocking)

    # ---- double-buffered host feed (the memcpy stream of TrainPipelineSparseDist, dist_util.py:221-303) --------
    def prefetch(self, batch: Batch) -> None:
        """Starts the pinned-host -> device copy of the NEXT batch on the copy stream (overlaps the running step)."""
        if self._staging is None:
            self._staging = [torch.empty_like(t) for t in self._static_tensors]
            self._ready = torch.cuda.Event()
            self._consumed = torch.cuda.Event()
            self._consumed.record(torch.cuda.current_stream())
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self._consumed)      # previous staged batch has been committed
            for dst, src in zip(self._staging, _tensors_of(batch)):
                dst.copy_(src, non_blocking=True)
            self._ready.record(self.copy_stream)

    def commit(self) -> None:
        """Moves the staged batch into the graph's static inputs (device-to-device, on the compute stream)."""
        cur = torch.cuda.current_stream()
        cur.wait_event(self._ready)
        for dst, src in zip(self._static_tensors, self._staging):
            dst.copy_(src, non_blocking=True)
        self._consumed.record(cur)

    def replay(self) -> torch.Tensor:
        self.graph.replay()
        return self.loss
