"""FP16 tables end to end: a built-in example config with every id feature's `data_type: "FP16"`, sharded against its
unsharded twin (torcheasyrec_b200/verify.py's comparison with the tolerances of half tables).

TEST INFRASTRUCTURE, used by tests/test_fp16_peer_cpu.py (gloo, NCCL-exchange fallback, oracle compute) and
tests/test_fp16_peer_gpu.py (two GPUs, peer exchange)."""
from typing import Dict

import numpy as np
import torch
import torch.distributed as dist


def fp16_edits(name: str) -> Dict[str, str]:
    """Pipeline `edits` that give every id / sequence-id feature of example config `name` FP16 tables."""
    from torcheasyrec_b200 import example_configs
    from torcheasyrec_b200.config import parse_text

    cfg = parse_text(example_configs.GENERATORS[name]())
    edits = {}
    for i, fc in enumerate(cfg.feature_configs):
        for kind in ("id_feature", "sequence_id_feature"):
            if fc.HasField(kind):
                edits[f"feature_configs[{i}].{kind}.data_type"] = "FP16"
    assert edits, name
    return edits


def assert_within_one_ulp(got: np.ndarray, want: np.ndarray, err_msg: str = "") -> None:
    """|got - want| <= one fp16 ulp of the larger magnitude (halfs compared as exact float64 values)."""
    g, w = got.astype(np.float64), want.astype(np.float64)
    ulp = np.spacing(np.maximum(np.abs(g), np.abs(w)).astype(np.float16)).astype(np.float64)
    bad = np.abs(g - w) > ulp
    assert not bad.any(), f"{err_msg}: {int(bad.sum())} elements more than one fp16 ulp apart, e.g. " \
                          f"{g[bad][:4]} vs {w[bad][:4]}"


def verify_fp16_sharded(name: str, device, sharding: str, exchange: str = "nccl", rw_min_rows: int = 0,
                        static_capacity=None, max_rows: int = 300, batch: int = 48, steps: int = 2,
                        bit_exact_logits: bool = False) -> None:
    """Collective.  Every rank: the unsharded FP16 twin stepped on the concatenated batch, the sharded model on this
    rank's batch; logits before any update, the mean loss, every table (halfs, within one ulp) and dense parameter."""
    from torcheasyrec_b200.distributed import DenseGradSync, shard_model
    from torcheasyrec_b200.engine import Pipeline
    from torcheasyrec_b200.rank_models import dense_optimizer_from_config
    from torcheasyrec_b200.verify import concat_batches

    rank, world = dist.get_rank(), dist.get_world_size()
    dev = torch.device(device)
    edits = fp16_edits(name)
    ref = Pipeline(name, device=dev, max_rows=max_rows, seed=5, capturable=False, edits=edits)
    shd = Pipeline(name, device=dev, max_rows=max_rows, seed=5, capturable=False, edits=edits)
    assert all(c.weights.dtype == torch.float16 for c in ref.model.sparse_collections())
    per_bag = {f.name: int(f.sequence_length) for f in shd.features if f.is_sequence and f.sequence_length}
    sharded = shard_model(shd.model, dev, default=sharding, rw_min_rows=rw_min_rows, source=ref.model,
                          static_capacity=static_capacity, exchange=exchange, ids_per_bag=per_bag)
    assert all(g.local.weights.dtype == torch.float16 for sm in sharded for g in sm.groups)
    shd.model.set_sparse_optimizer(ref.model.sparse_collections()[0].optimizer)
    shd.dense_optimizer = dense_optimizer_from_config(shd.cfg.train_config, shd.model.dense_parameters())
    if exchange == "peer" and dev.type == "cuda":
        from torcheasyrec_b200.peer_exchange import PeerDenseGradSync

        shd.grad_sync = PeerDenseGradSync(shd.model.dense_parameters())
    else:
        shd.grad_sync = DenseGradSync(shd.model.dense_parameters())
    B = batch
    batches = [ref.synthetic_batch(B, seed=77 + r) for r in range(world)]
    glob = concat_batches(batches).to(dev)
    mine = batches[rank].to(dev)
    with torch.no_grad():
        p_ref = ref.model.predict(glob)
        p_shd = shd.model.predict(mine)
    for k, v in p_shd.items():
        if k.startswith("logits"):
            want = p_ref[k][rank * B:(rank + 1) * B].cpu().numpy()
            if bit_exact_logits:
                np.testing.assert_array_equal(v.cpu().numpy(), want)
            else:
                np.testing.assert_allclose(v.cpu().numpy(), want, rtol=1e-6, atol=1e-6)
    for _ in range(steps):
        loss_ref = ref.eager_step(glob)
        loss_shd = shd.eager_step(mine)
    for sm in sharded:
        sm.check_overflow()
    t = torch.tensor([float(loss_shd)], dtype=torch.float64, device=dev)
    dist.all_reduce(t)
    np.testing.assert_allclose(t.item() / world, float(loss_ref), rtol=1e-5)
    ref_tables = {}
    for coll in ref.model.sparse_collections():
        for ti, c in enumerate(coll._configs):
            ref_tables[(type(coll).__name__, c.name)] = coll.table_weight(ti)
    for sm in sharded:
        kind = "EmbeddingBagCollection" if sm._pooled else "EmbeddingCollection"
        for c in sm._configs:
            full = sm.gather_full_table(c.name)
            assert full.dtype == torch.float16
            assert_within_one_ulp(full.cpu().numpy(), ref_tables[(kind, c.name)].cpu().numpy(), f"{kind}.{c.name}")
    dense = lambda m: sorted((n, p) for n, p in m.named_parameters() if not n.endswith("weights"))
    for (n1, p1), (n2, p2) in zip(dense(ref.model), dense(shd.model)):
        assert n1 == n2
        np.testing.assert_allclose(p2.detach().cpu().numpy(), p1.detach().cpu().numpy(), rtol=2e-3, atol=2e-5,
                                   err_msg=n1)
