"""In-process parity check of a sharded model against its unsharded twin (used by tests/ and by `bench.py --verify`).

Every rank builds the same small-table model twice from one seed: `ref` stays unsharded and is stepped on the
concatenation of all ranks' batches, `shd` is sharded (same plan / exchange as the run being verified, seeded from `ref`)
and is stepped on this rank's batch.  Compared: logits before any update, the mean loss, every table after `steps`
fused updates (shards gathered), every dense parameter.  The comparison IS the unsharded CUDA path (itself checked
against the oracle by tests/test_model_gpu.py) — nothing here touches oracle/.

What the reference has instead: nothing at this level (its sharded path lives in torchrec, SURVEY.md §4: shapes only);
the W-invariance it relies on is App. A.5-A.8.
"""
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.distributed as dist

from .batch import Batch
from .sparse import KeyedJaggedTensor, KeyedTensor


def concat_batches(batches: List[Batch]) -> Batch:
    """Key-major concatenation of per-rank batches = the global batch the unsharded twin sees."""
    out = Batch()
    b0 = batches[0]
    for dg, kjt0 in b0.sparse_features.items():
        vals, lens = [], []
        dicts = [b.sparse_features[dg].to_dict() for b in batches]
        for k in kjt0.keys():
            for d in dicts:
                vals.append(d[k].values())
                lens.append(d[k].lengths())
        out.sparse_features[dg] = KeyedJaggedTensor(kjt0.keys(), torch.cat(vals), lengths=torch.cat(lens),
                                                    stride=sum(b.sparse_features[dg].stride() for b in batches))
    for dg, kt0 in b0.dense_features.items():
        out.dense_features[dg] = KeyedTensor(kt0.keys(), kt0.length_per_key(),
                                             torch.cat([b.dense_features[dg].values() for b in batches]))
    for k in b0.labels:
        out.labels[k] = torch.cat([b.labels[k] for b in batches])
    return out


def verify_sharded(name: str, device, sharding: str, rw_min_rows: int = 0, static_capacity: Optional[float] = None,
                   exchange: str = "nccl", sparse_opt: Optional[str] = None, max_rows: int = 300, batch: int = 48,
                   steps: int = 2, bit_exact_logits: bool = False, group=None) -> Dict[str, float]:
    """Raises AssertionError on a mismatch; returns the largest deviations seen.  Collective: every rank calls it."""
    from .distributed import DenseGradSync, shard_model
    from .engine import Pipeline
    from .rank_models import dense_optimizer_from_config

    rank, world = dist.get_rank(group), dist.get_world_size(group)
    dev = torch.device(device)
    B = batch
    ref = Pipeline(name, device=dev, max_rows=max_rows, seed=5, capturable=False)   # unsharded twin
    shd = Pipeline(name, device=dev, max_rows=max_rows, seed=5, capturable=False)
    shd.model.load_state_dict(ref.model.state_dict())
    per_bag = {f.name: int(f.sequence_length) for f in shd.features if f.is_sequence and f.sequence_length}
    sharded = shard_model(shd.model, dev, default=sharding, rw_min_rows=rw_min_rows, source=ref.model,
                          static_capacity=static_capacity, exchange=exchange, ids_per_bag=per_bag, group=group)
    if sparse_opt is not None:     # e.g. "adam": second state + device-side step counter on every shard
        from .embedding_modules import SparseOptimizerSpec

        ref.model.set_sparse_optimizer(SparseOptimizerSpec.from_name(sparse_opt, lr=0.01))
    shd.model.set_sparse_optimizer(ref.model.sparse_collections()[0].optimizer)
    shd.dense_optimizer = dense_optimizer_from_config(shd.cfg.train_config, shd.model.dense_parameters())
    if exchange == "peer" and dev.type == "cuda":
        from .peer_exchange import PeerDenseGradSync

        shd.grad_sync = PeerDenseGradSync(shd.model.dense_parameters(), group)
    else:
        shd.grad_sync = DenseGradSync(shd.model.dense_parameters(), group)
    batches = [ref.synthetic_batch(B, seed=77 + r) for r in range(world)]
    glob = concat_batches(batches).to(dev)
    mine = batches[rank].to(dev)
    worst = {"logits": 0.0, "tables": 0.0, "dense": 0.0, "loss": 0.0}
    # forward parity (before any update)
    with torch.no_grad():
        p_ref = ref.model.predict(glob)
        p_shd = shd.model.predict(mine)
    for k, v in p_shd.items():
        if k.startswith("logits"):
            want = p_ref[k][rank * B:(rank + 1) * B].cpu().numpy()
            got = v.cpu().numpy()
            if bit_exact_logits:
                np.testing.assert_array_equal(got, want)
            else:   # cuBLAS / gemm3x tiles differ between batch B and W*B: not bit-stable across shapes
                np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-6)
            worst["logits"] = max(worst["logits"], float(np.abs(got - want).max()))
    for _ in range(steps):
        loss_ref = ref.eager_step(glob)
        loss_shd = shd.eager_step(mine)
    for sm in sharded:
        sm.check_overflow()
    t = torch.tensor([float(loss_shd)], dtype=torch.float64, device=dev)
    dist.all_reduce(t, group=group)
    np.testing.assert_allclose(t.item() / world, float(loss_ref), rtol=1e-6)
    worst["loss"] = abs(t.item() / world - float(loss_ref))
    # updated tables: gather shards, compare with the unsharded twin
    ref_tables = {}
    for coll in ref.model.sparse_collections():
        for ti, c in enumerate(coll._configs):
            ref_tables[(type(coll).__name__, c.name)] = coll.table_weight(ti)
    for sm in sharded:
        kind = "EmbeddingBagCollection" if sm._pooled else "EmbeddingCollection"
        for c in sm._configs:
            full = sm.gather_full_table(c.name).cpu().numpy()
            want = ref_tables[(kind, c.name)].cpu().numpy()
            # dL/dlogit is 1/B per rank then /W on the owners vs 1/(W*B) in the twin: same value, one more fp32
            # rounding per contribution -> a few ulp after two Adagrad steps
            np.testing.assert_allclose(full, want, rtol=5e-5, atol=1e-6, err_msg=f"{kind}.{c.name}")
            worst["tables"] = max(worst["tables"], float(np.abs(full - want).max()))
    dense = lambda m: sorted((n, p) for n, p in m.named_parameters() if not n.endswith("weights"))
    for (n1, p1), (n2, p2) in zip(dense(ref.model), dense(shd.model)):
        assert n1 == n2
        a, b = p2.detach().cpu().numpy(), p1.detach().cpu().numpy()
        # Adam normalises by sqrt(v): tiny gradient differences (mean over W*B vs mean of W means) are amplified
        np.testing.assert_allclose(a, b, rtol=2e-4, atol=2e-6, err_msg=n1)
        worst["dense"] = max(worst["dense"], float(np.abs(a - b).max()))
    return worst
