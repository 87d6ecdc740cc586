"""Step driver: builds a model from a tzrec pipeline config and runs train steps (and forward-only eval steps) on one H100.

Replaces the part of tzrec/main.py that surrounds the hot path (model construction :763-781, optimizers
:814-876, the step loop :519-547) and torchrec's TrainPipelineSparseDist (tzrec/utils/dist_util.py:221-303)
with an H100-first design: the whole step (KJT scan, gather, interaction, dense towers, loss, backward incl.
the fused sparse update, dense optimizer) is captured ONCE in a CUDA graph over static device buffers and
replayed; a side stream stages the next host batch (pinned H2D) while the current graph runs.
Variable-shape workloads (sequence features) run the same code eagerly.
"""

import contextlib
import os
from typing import Any, Dict, Iterable, List, Optional, Sequence

import numpy as np
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
        (example_configs.BUILTINS: dlrm_criteo, deepfm_criteo, mmoe_taobao, multi_tower_din_taobao, masknet_criteo,
        ple_taobao, pepnet_taobao, wukong_criteo)."""
        from . import example_configs
        from .config import parse_text

        if config in example_configs.BUILTINS:
            self.cfg = parse_text(example_configs.BUILTINS[config]())
        else:
            self.cfg = load_pipeline_config(config)
        if edits:
            edit_config(self.cfg, edits)
        if max_rows:
            override_num_buckets(self.cfg, max_rows)
        self.device = torch.device(device)
        self.capturable = capturable
        # process group whose ranks' metric states compute_metric sums (sharded pipelines; None = the default group)
        self.metric_group = group
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
        """A seeded host batch (batch.synthetic_batch).  For a model with a jrc_loss tower, the session feature's ids are
        drawn over min(ceil(B / 8), table rows) values, so sessions average 8 samples: uniform ids over a table as large
        as Taobao's users would make almost every session a singleton, whose JRC term is 0."""
        mc = self.cfg.model_config
        pep = mc.pepnet if mc.WhichOneof("model") == "pepnet" else None
        card = ({pep.domain_input_name: pep.task_domain_num}
                if pep is not None and pep.HasField("domain_input_name") else None)
        b = synthetic_batch(self.features, batch_size, self.labels, seed=seed, id_dist=id_dist, label_cardinality=card)
        sessions = {lc.jrc_loss.session_name for tc in getattr(getattr(mc, mc.WhichOneof("model")), "task_towers", None) or []
                    for lc in tc.losses if lc.WhichOneof("loss") == "jrc_loss"}
        if sessions:
            from .features import BASE_DATA_GROUP

            kjt = b.sparse_features[BASE_DATA_GROUP]
            rng = np.random.default_rng(seed + 1)
            lens = kjt.lengths()
            rows = {f.name: f.num_embeddings for f in self.features}
            for name in sorted(sessions):
                f = kjt.keys().index(name)
                hi = min(-(-batch_size // 8), rows.get(name) or -(-batch_size // 8))
                s = int(lens[:f * batch_size].sum())
                n = int(lens[f * batch_size:(f + 1) * batch_size].sum())
                kjt.values()[s:s + n] = torch.from_numpy(rng.integers(0, hi, size=n))
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

    # ---- evaluation (tzrec/main.py:169-233 `_evaluate`) -------------------------------------------------------------
    def _ensure_metrics(self) -> None:
        if getattr(self.model, "_metric_modules", None) is None:
            self.model.init_metric(process_group=self.metric_group, distributed=bool(self.sharded))

    @contextlib.contextmanager
    def _eval_mode(self):
        """model.eval() and no_grad for the block; the model's previous mode comes back even if the block raises."""
        was_training = self.model.training
        self.model.eval()
        try:
            with torch.no_grad():
                yield
        finally:
            self.model.train(was_training)

    def _check_eval_batch(self, batch: Batch) -> None:
        """The peer exchange is sized for the local batch of its first step: an eval batch larger than that is refused
        here, before anything is launched (a smaller one, e.g. the last of an eval set, is gathered at its own size)."""
        B = next(iter(batch.labels.values())).shape[0]
        for sm in self.sharded:
            for st in getattr(sm, "_peer_states", None) or []:
                if B > st.B:
                    raise ValueError(f"eval batch of {B} samples: the peer exchange is sized for local batches of at "
                                     f"most {st.B} (the training batch); split the eval set into batches of that size")

    def _eval_body(self, batch: Batch) -> Dict[str, torch.Tensor]:
        """Forward through train_wrapper (autocast as in training) + update_metric; the caller holds _eval_mode."""
        _, (losses, predictions, _) = self.train_wrapper(batch)
        self.model.update_metric(predictions, batch, {k: v.detach() for k, v in losses.items()})
        return predictions

    def eval_step(self, batch: Batch) -> Dict[str, torch.Tensor]:
        """One eager forward-only step under model.eval() and no_grad: adds `batch` to the metric states and returns the
        predictions."""
        self._ensure_metrics()
        self._check_eval_batch(batch)
        with self._eval_mode():
            return self._eval_body(batch)

    def evaluate(self, batches: Iterable[Batch], num_steps: Optional[int] = None) -> Dict[str, float]:
        """Runs `num_steps` eval steps (default eval_config.num_steps; every batch when it is unset or <= 0), then returns
        {metric name: value} and resets the metric states.  On CUDA with `capturable`, batches shaped like the first one
        replay a GraphedEvalStep (one per batch shape, kept for later evaluations); any other batch, e.g. a shorter last
        one, takes the eager eval_step, and so does every batch of a model with sequence features.  The model's train /
        eval mode is restored afterwards."""
        if num_steps is None:
            num_steps = int(self.cfg.eval_config.num_steps)
        if num_steps <= 0:                 # as main.py:187: unset or 0 evaluates every batch
            num_steps = None
        self._ensure_metrics()
        # captured graphs update the metric state tensors they were captured with: a new init_metric drops them
        mods = self.model._metric_modules
        cache = self.__dict__.get("_eval_graphs")
        if cache is None or cache[0] is not mods:
            cache = self._eval_graphs = (mods, {})
        graphs = cache[1]
        graph = None
        # sequence features vary in shape from batch to batch: those models step eagerly, as in training
        graphable = self.device.type == "cuda" and self.capturable and not any(f.is_sequence for f in self.features)
        try:
            for i, batch in enumerate(batches):
                if num_steps is not None and i >= num_steps:
                    break
                self._check_eval_batch(batch)
                # (a capture needs the per-key id counts on the host: a device batch without them steps eagerly)
                if graphable and all(k._length_per_key is not None or not k.lengths().is_cuda
                                     for k in batch.sparse_features.values()):
                    if graph is None:
                        key = tuple(t.shape for t in _tensors_of(batch))
                        graph = graphs.get(key)
                        if graph is None or not graph.fits(batch):
                            graph = graphs[key] = GraphedEvalStep(self, batch)
                    if graph.fits(batch):
                        graph.load(batch)
                        graph.replay()
                        continue
                self.eval_step(batch.to(self.device))
        except BaseException:
            for m in self.model._metric_modules.values():
                m.reset()
            raise
        return {k: float(v) for k, v in self.model.compute_metric().items()}


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


class _StaticFeed:
    """Static device copies of one example batch (the inputs a captured step reads) and the feed that refreshes them."""

    def __init__(self, pipe: Pipeline, example: Batch) -> None:
        assert pipe.device.type == "cuda"
        self.static = example.to(pipe.device)
        for k, kjt in example.sparse_features.items():
            self.static.sparse_features[k]._length_per_key = kjt._length_per_key
        self._static_tensors = _tensors_of(self.static)
        self.copy_stream = torch.cuda.Stream()
        self._staging = None

    def fits(self, batch: Batch) -> bool:
        """True when `batch` has the static inputs' shapes and per-key id counts, which a replay takes as given."""
        if [t.shape for t in _tensors_of(batch)] != [t.shape for t in self._static_tensors]:
            return False
        for k, kjt in self.static.sparse_features.items():
            other = batch.sparse_features[k]
            lpk = other._length_per_key
            if lpk is None and not other.lengths().is_cuda:
                lpk = other.length_per_key()
            if lpk is None or list(lpk) != list(kjt._length_per_key or []):
                return False
        return True

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


class GraphedTrainStep(_StaticFeed):
    """One CUDA graph per (model, batch shape).  `load()` refreshes the static inputs, `replay()` runs a step."""

    def __init__(self, pipe: Pipeline, example: Batch, warmup: int = 3) -> None:
        super().__init__(pipe, example)
        self.pipe = pipe
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

    def replay(self) -> torch.Tensor:
        self.graph.replay()
        return self.loss


class GraphedEvalStep(_StaticFeed):
    """Pipeline.eval_step captured in one CUDA graph: the forward and the metric update.  `load()` / `prefetch()` +
    `commit()` refresh the static inputs as for GraphedTrainStep; `replay()` adds the loaded batch to the metric states
    and returns the step's (static) predictions.  The warm-up steps' metric updates are undone.  The graph updates the
    metric states that existed at capture: after another `model.init_metric()`, capture a new step.  It keeps no reference
    to the pipeline, which caches it (Pipeline.evaluate): no cycle holds the graph's memory after the pipeline is gone."""

    def __init__(self, pipe: Pipeline, example: Batch, warmup: int = 2) -> None:
        from . import metrics

        super().__init__(pipe, example)
        pipe._ensure_metrics()
        mods = pipe.model._metric_modules
        saved = metrics.snapshot(mods)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self._fresh_kjt_caches()
                pipe.eval_step(self.static)
        torch.cuda.current_stream().wait_stream(side)
        metrics.restore(mods, saved)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        self._fresh_kjt_caches()
        with pipe._eval_mode():
            with torch.cuda.graph(self.graph):
                self.predictions = pipe._eval_body(self.static)
        torch.cuda.synchronize()

    def replay(self) -> Dict[str, torch.Tensor]:
        self.graph.replay()
        return self.predictions
