"""Checkpoints in the reference's on-disk layout (SURVEY §8f N2).

tzrec/utils/checkpoint_util.py:1109-1160 saves `<dir>/model` and `<dir>/optimizer` with torch.distributed.checkpoint
(one `.metadata` + one `__<rank>_0.distcp` per rank) and `<dir>/plan` as json; `restore_model` (:943-1107) loads them
back through DCP, which re-shards by the per-tensor chunk metadata — so a checkpoint written by W ranks under one plan
loads under another world size / plan.  Here:

  * model keys are the reference's: `…ebc.embedding_bags.<table>.weight`, `…ec_dict.<dim>.embeddings.<table>.weight`
    (tzrec/utils/checkpoint_util_test.py:375-396) — a ShardedTensor over the table's global [rows, D] shape whose local
    shard is a VIEW of this rank's arena slice (sharded collections), or the plain [rows, D] view (unsharded);
  * fused sparse optimizer state: `state.<weight key>.<table>.momentum1` (+ `.momentum2` / `.iter` for the Adam and
    LAMB variants [EXT names]); dense optimizer: `state.<param fqn>.exp_avg|exp_avg_sq|step`;
  * `plan`: {module path: {table: {sharding_type, compute_kernel, ranks}}} like checkpoint_util.py:1145-1160.
The arena buffers and the `shards.*` submodules never appear in a key.
"""
import json
import os
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from .distributed import TABLE_WISE, _ShardedBase
from .embedding_modules import ADAM_LIKE_KINDS, ELEMENTWISE_STATE_KINDS, _ArenaCollection
from .kernels import OPT_ADAGRAD, OPT_ADAM, OPT_LAMB, OPT_LARS_SGD, OPT_ROWWISE_ADAGRAD


def _placement(rank: int, device: torch.device) -> str:
    return f"rank:{rank}/cuda:{device.index if device.index is not None else rank}" if device.type == "cuda" else f"rank:{rank}/cpu"


def sharded_rows_tensor(local: Optional[torch.Tensor], row_offset: int, global_shape, group=None):
    """ShardedTensor of `global_shape` whose (only) local shard is `local` placed at row `row_offset`; ranks without
    rows pass None.  Collective (the shard metadata is all-gathered)."""
    from torch.distributed._shard.sharded_tensor import Shard, ShardedTensor, ShardMetadata

    rank = dist.get_rank(group)
    shards = []
    if local is not None and local.shape[0] > 0:
        offs = [row_offset] + [0] * (len(global_shape) - 1)
        shards.append(Shard(local, ShardMetadata(shard_offsets=offs, shard_sizes=list(local.shape),
                                                 placement=_placement(rank, local.device))))
    return ShardedTensor._init_from_local_shards(shards, *global_shape, process_group=group)


def _state_names(kind: int) -> List[str]:
    if kind in (OPT_ADAGRAD, OPT_ROWWISE_ADAGRAD, OPT_LARS_SGD):
        return ["momentum1"]
    if kind in ADAM_LIKE_KINDS:
        return ["momentum1", "momentum2", "iter"]
    return []


def _local_state(coll: _ArenaCollection, t: int, which: str) -> Optional[torch.Tensor]:
    """[rows_local, D] / [rows_local] view of table t's optimizer state (`momentum1` / `momentum2`)."""
    spec = coll.optimizer
    if which == "momentum1" and coll.layout.interleaved and spec is not None and t in coll._table_off:
        return coll.table_state(t)            # [weight row | accumulator row] arena: a strided view
    buf = coll.opt_state if which == "momentum1" else coll.opt_state2
    if spec is None or buf is None or t not in coll._table_off:
        return None
    rows, dim = coll._table_rows[t], coll._table_dim[t]
    if _is_elementwise(spec.kind, which):
        o = coll._table_off[t]
        return buf[o:o + rows * dim].view(rows, dim)
    k = coll._table_key[t]
    return buf[k:k + rows]


def _collections(model):
    """(key prefix, collection) for every arena-backed collection, sharded wrappers as one entry."""
    out = []
    skip = set()
    for name, m in model.named_modules():
        if isinstance(m, _ShardedBase):
            out.append((name + ".", m))
            skip.update(id(g.local) for g in m.groups)
        elif isinstance(m, _ArenaCollection) and id(m) not in skip:
            out.append((name + ".", m))
    return out


def fused_optimizer_state_dict(model, group=None) -> Dict[str, object]:
    """`state.<weight key>.<table>.<name>` for every table (the keys of the reference's `model.fused_optimizer`)."""
    out: Dict[str, object] = {}
    for prefix, m in _collections(model):
        if isinstance(m, _ShardedBase):
            attr = "embedding_bags" if m._pooled else "embeddings"
            for g in m.groups:
                spec = g.local.optimizer
                for t, c in enumerate(g.configs):
                    sh = m.plan[c.name]
                    start = 0 if sh.kind == TABLE_WISE else m.rank * sh.block
                    for nm in _state_names(spec.kind if spec else -1):
                        key = f"state.{prefix}{attr}.{c.name}.weight.{c.name}.{nm}"
                        if nm == "iter":
                            out[key] = g.local.opt_step.reshape(1)
                            continue
                        loc = _local_state(g.local, t, nm)
                        shape = (c.num_embeddings,) + (tuple(loc.shape[1:]) if loc is not None and loc.dim() > 1 else
                                                       ((c.embedding_dim,) if _is_elementwise(spec.kind, nm) else ()))
                        out[key] = sharded_rows_tensor(loc, start, shape, group)
        else:
            spec = m.optimizer
            for t, c in enumerate(m._configs):
                for nm in _state_names(spec.kind if spec else -1):
                    key = f"state.{prefix}{m._table_attr()}.{c.name}.weight.{c.name}.{nm}"
                    out[key] = m.opt_step.reshape(1) if nm == "iter" else _local_state(m, t, nm)
    return out


def _is_elementwise(kind: int, which: str) -> bool:
    return (kind in ELEMENTWISE_STATE_KINDS) if which == "momentum1" else kind in (OPT_ADAM, OPT_LAMB)


def dense_optimizer_state_dict(model, optimizer: torch.optim.Optimizer) -> Dict[str, torch.Tensor]:
    """`state.<param fqn>.<exp_avg|exp_avg_sq|step>` (torch optimizer state keyed by parameter name, as the reference's
    KeyedOptimizer wrapper does)."""
    names = {id(p): n for n, p in model.named_parameters()}
    out = {}
    for group in optimizer.param_groups:
        for p in group["params"]:
            st = optimizer.state.get(p, {})
            for k, v in st.items():
                if isinstance(v, torch.Tensor):
                    out[f"state.{names[id(p)]}.{k}"] = v if v.dim() else v.reshape(1)
    return out


def plan_json(model) -> Dict[str, Dict[str, dict]]:
    out: Dict[str, Dict[str, dict]] = {}
    for prefix, m in _collections(model):
        if isinstance(m, _ShardedBase):
            mod = {}
            for c in m._configs:
                sh = m.plan[c.name]
                ranks = [sh.owner] if sh.kind == TABLE_WISE else \
                    [r for r in range(m.world) if r * sh.block < c.num_embeddings]
                mod[c.name] = {"sharding_type": sh.kind, "compute_kernel": "fused", "ranks": ranks}
            out[prefix[:-1]] = mod
    return out


def save_model(checkpoint_dir: str, model, dense_optimizer: Optional[torch.optim.Optimizer] = None, group=None) -> None:
    """checkpoint_util.save_model: `<dir>/model`, `<dir>/optimizer` (DCP) and `<dir>/plan` (json, rank 0)."""
    import torch.distributed.checkpoint as dcp

    os.makedirs(checkpoint_dir, exist_ok=True)
    dcp.save(dict(model.state_dict()), checkpoint_id=os.path.join(checkpoint_dir, "model"), process_group=group)
    opt = fused_optimizer_state_dict(model, group)
    if dense_optimizer is not None:
        opt.update(dense_optimizer_state_dict(model, dense_optimizer))
    if opt:
        dcp.save(opt, checkpoint_id=os.path.join(checkpoint_dir, "optimizer"), process_group=group)
    if not dist.is_initialized() or dist.get_rank(group) == 0:
        with open(os.path.join(checkpoint_dir, "plan"), "w") as f:
            json.dump(plan_json(model), f)


def _check_dtypes(sd: Dict[str, object], path: str) -> None:
    """Tables are saved in their data_type (FP16 tables as fp16 tensors).  Loading a checkpoint into a model whose table
    has the other data_type would convert every row silently: raise instead, before anything is read."""
    import torch.distributed.checkpoint as dcp

    meta = dcp.FileSystemReader(path).read_metadata().state_dict_metadata
    bad = []
    for k, v in sd.items():
        props = getattr(meta.get(k), "properties", None)
        if isinstance(v, torch.Tensor) and props is not None and props.dtype != v.dtype:
            bad.append(f"{k} (checkpoint {props.dtype}, model {v.dtype})")
    if bad:
        raise ValueError("checkpoint and model disagree on the tables' data_type (FP32 / FP16); loading across "
                         "data_type is not supported: " + ", ".join(bad))


def restore_model(checkpoint_dir: str, model, dense_optimizer: Optional[torch.optim.Optimizer] = None, group=None) -> None:
    """checkpoint_util.restore_model: loads `<dir>/model` (+ `<dir>/optimizer`) into the CURRENT sharding — DCP
    re-shards by chunk metadata, so world size and plan may differ from the run that saved."""
    import torch.distributed.checkpoint as dcp

    sd = dict(model.state_dict())            # table entries view the arenas: DCP writes straight into the shards
    _check_dtypes(sd, os.path.join(checkpoint_dir, "model"))
    dcp.load(sd, checkpoint_id=os.path.join(checkpoint_dir, "model"), process_group=group)
    model.load_state_dict(sd)
    opt_dir = os.path.join(checkpoint_dir, "optimizer")
    if os.path.exists(opt_dir):
        opt = fused_optimizer_state_dict(model, group)
        if dense_optimizer is not None:
            opt.update(dense_optimizer_state_dict(model, dense_optimizer))
        if opt:
            dcp.load(opt, checkpoint_id=opt_dir, process_group=group)   # in place (views / optimizer state tensors)


def list_checkpoint_keys(checkpoint_dir: str) -> List[str]:
    """Tensor names in `<dir>/model` and `<dir>/optimizer` (checkpoint_util.list_distcp_param)."""
    import torch.distributed.checkpoint as dcp

    keys: List[str] = []
    for sub in ("model", "optimizer"):
        p = os.path.join(checkpoint_dir, sub)
        if os.path.exists(p):
            keys += list(dcp.FileSystemReader(p).read_metadata().state_dict_metadata.keys())
    return sorted(keys)
