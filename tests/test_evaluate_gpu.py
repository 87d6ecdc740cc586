"""Evaluation on the H100: tzk_binned_auc_update against the numpy restatement (bit-exact counts), the graphed eval step
against the eager one, DLRM-Criteo at full hash sizes (values, untouched state, training unaffected), BF16 probabilities,
and the peer-exchange W = 2 evaluate against the unsharded one."""
import gc
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import auc_ref  # noqa: E402
from test_evaluate_cpu import _all_state, _assert_same_state  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _statement(p, batches, thresholds):
    probs, labels, lsum, n = [], [], 0.0, 0
    p.model.eval()
    with torch.no_grad():
        for b in batches:
            _, (losses, preds, _) = p.train_wrapper(b)
            probs.append(preds["probs"].float().cpu().numpy())
            labels.append(b.labels[p.labels[0]].cpu().numpy())
            lsum += float(losses["binary_cross_entropy"]) * labels[-1].shape[0]
            n += labels[-1].shape[0]
    p.model.train()
    return {"auc": auc_ref.binned_auc(np.concatenate(probs), np.concatenate(labels), thresholds),
            "binary_cross_entropy": lsum / n}


@pytest.mark.parametrize("T", [1, 200, 1000, 10000, 19340, 19369, 20000])
@pytest.mark.parametrize("pdt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("ldt", [torch.float32, torch.int64])
def test_kernel_counts_equal_restatement(kernels, T, pdt, ldt):
    g = torch.Generator().manual_seed(T)
    B = 65536
    p = torch.rand(B, generator=g)
    p[:4096] = torch.linspace(0, 1, 1000)[torch.randint(0, 1000, (4096,), generator=g)]       # on the thresholds
    p[4096:4200] = 1.0
    p[4200:4300] = 0.0
    y = (torch.rand(B, generator=g) < 0.3).to(ldt)
    pk = p.to(pdt)
    thr = torch.linspace(0, 1, T, dtype=torch.float32, device=DEV)
    counts = torch.zeros((T + 1, 2), dtype=torch.int64, device=DEV)
    invalid = torch.zeros(1, dtype=torch.int64, device=DEV)
    for _ in range(2):                                   # accumulates
        kernels.binned_auc_update(pk.to(DEV), y.to(DEV), thr, counts, invalid)
    torch.cuda.synchronize()
    cm = auc_ref.confmat(pk.float().numpy(), y.numpy(), thr.cpu().numpy())
    np.testing.assert_array_equal(counts.cpu().numpy(), 2 * auc_ref.counts_from_confmat(cm))
    assert int(invalid) == 0
    y2 = y.clone()
    y2[5] = 3
    pk2 = pk.clone()
    pk2[6] = float("nan")
    kernels.binned_auc_update(pk2.to(DEV)[1:], y2.to(DEV)[1:], thr, counts.zero_(), invalid)     # unaligned: scalar path
    np.testing.assert_array_equal(counts.cpu().numpy(), auc_ref.counts_from_confmat(
        auc_ref.confmat(pk2[1:].float().numpy(), y2[1:].numpy(), thr.cpu().numpy())))
    assert int(invalid) == 2


def test_graphed_eval_step_equals_eager_and_runs_no_sparse_backward(kernels, monkeypatch):
    from torcheasyrec_b200.engine import GraphedEvalStep, Pipeline

    calls = []
    for m in ("fused_bwd", "fused_bwd_sort", "fused_bwd_apply", "bag_grad_expand"):
        orig = getattr(type(kernels), m)
        monkeypatch.setattr(type(kernels), m, lambda self, *a, _m=m, _o=orig, **kw: (calls.append(_m), _o(self, *a, **kw))[1])
    a = Pipeline("dlrm_criteo", device=DEV, max_rows=20000, seed=5)
    a.eager_step(a.synthetic_batch(2048, seed=1).to(DEV))
    assert calls
    calls.clear()
    batches = [a.synthetic_batch(2048, seed=10 + i) for i in range(4)]
    step = GraphedEvalStep(a, batches[0])
    a._ensure_metrics()
    ma = a.model._metric_modules
    assert all(int(t.abs().sum()) == 0 for m in ma.values() for t in m.state())       # warm-up left no trace
    eager = {k: [t.clone() for t in m.state()] for k, m in ma.items()}
    for b in batches:
        step.load(b.pin_memory())
        got = {k: v.clone() for k, v in step.replay().items()}
        graph_state = {k: [t.clone() for t in m.state()] for k, m in ma.items()}
        for k, m in ma.items():
            for t, e in zip(m.state(), eager[k]):
                t.copy_(e)
        want = a.eval_step(b.to(DEV))
        for k in got:
            assert torch.equal(got[k], want[k]), k
        for k, m in ma.items():
            for t, gs in zip(m.state(), graph_state[k]):
                assert torch.equal(t, gs), k
        eager = graph_state
    assert a.model.training and calls == []


def test_evaluate_after_init_metric_recaptures():
    """The cached eval graph updates the metric states it was captured with: a new init_metric must not leave the next
    evaluate reading fresh, never-updated states."""
    from torcheasyrec_b200.engine import Pipeline

    p = Pipeline("dlrm_criteo", device=DEV, max_rows=20000, seed=5)
    batches = [p.synthetic_batch(1024, seed=20 + i) for i in range(3)]
    first = p.evaluate(batches)
    p.model.init_metric()
    assert p.evaluate(batches) == first
    assert p.evaluate(batches) == first


def _dlrm_full(seed=5, B=16384, edits=None):
    from torcheasyrec_b200.engine import Pipeline

    return Pipeline("dlrm_criteo", device=DEV, seed=seed, edits=edits)


def test_dlrm_full_size_evaluate_and_training_unaffected():
    """Runs in a child process: two full-size pipelines (one after the other) take most of the card, and the process
    exit hands all of it back before the next test."""
    import subprocess

    r = subprocess.run([sys.executable, os.path.abspath(__file__), "full_size"], capture_output=True, text=True,
                       timeout=1200)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]


def _full_size_body():
    from torcheasyrec_b200.engine import GraphedTrainStep

    B = 16384
    a = _dlrm_full()
    train = [a.synthetic_batch(B, seed=i) for i in range(3)]
    evals = [a.synthetic_batch(B, seed=50 + i) for i in range(3)] + [a.synthetic_batch(1000, seed=60)]
    sa = GraphedTrainStep(a, train[0], warmup=2)
    sa.load(train[1].pin_memory())
    sa.replay()
    torch.cuda.synchronize()
    before = _all_state(a)
    got = a.evaluate(evals)
    _assert_same_state(before, _all_state(a))
    del before
    want = _statement(a, [b.to(DEV) for b in evals], 200)
    assert got["auc"] == pytest.approx(want["auc"], abs=1e-12)
    assert got["binary_cross_entropy"] == pytest.approx(want["binary_cross_entropy"], rel=1e-6)
    sa.load(train[2].pin_memory())
    loss_a = float(sa.replay())
    state_a = {k: v.cpu() for k, v in _all_state(a).items() if k.startswith("opt.") or k.startswith("sd.") and
               "weights" not in k}
    rows_a = [c.dense_weights()[:4096].cpu() for c in a.model.sparse_collections()]
    del sa, a
    gc.collect()
    torch.cuda.empty_cache()
    b = _dlrm_full()
    sb = GraphedTrainStep(b, train[0], warmup=2)
    sb.load(train[1].pin_memory())
    sb.replay()
    sb.load(train[2].pin_memory())
    loss_b = float(sb.replay())
    state_b = {k: v.cpu() for k, v in _all_state(b).items() if k in state_a}
    assert loss_a == loss_b
    _assert_same_state(state_a, state_b)
    for ra, c in zip(rows_a, b.model.sparse_collections()):
        assert torch.equal(ra, c.dense_weights()[:4096].cpu())


def test_bf16_probs_binned_exactly(kernels):
    from torcheasyrec_b200.engine import Pipeline

    p = Pipeline("dlrm_criteo", device=DEV, max_rows=20000, seed=5, edits={"train_config.mixed_precision": "BF16"})
    p.eager_step(p.synthetic_batch(4096, seed=1).to(DEV))
    b = p.synthetic_batch(4096, seed=2).to(DEV)
    preds = p.eval_step(b)
    assert preds["probs"].dtype == torch.bfloat16
    m = p.model._metric_modules["auc"]
    cm = auc_ref.confmat(preds["probs"].float().cpu().numpy(), b.labels[p.labels[0]].cpu().numpy(), auc_ref.thresholds(200))
    np.testing.assert_array_equal(m.counts.cpu().numpy(), auc_ref.counts_from_confmat(cm))
    res = p.model.compute_metric()
    assert float(res["auc"]) == pytest.approx(auc_ref.auc_from_confmat(cm), abs=1e-12)


# ---- peer exchange, W = 2 --------------------------------------------------------------------------------------------
def _peer_worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device(f"cuda:{rank}")
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        from torcheasyrec_b200.distributed import shard_model
        from torcheasyrec_b200.engine import Pipeline
        from torcheasyrec_b200.verify import concat_batches

        ref = Pipeline("dlrm_criteo", device=dev, max_rows=300, seed=5, capturable=False)
        shd = Pipeline("dlrm_criteo", device=dev, max_rows=300, seed=5, capturable=False)
        shd.model.load_state_dict(ref.model.state_dict())
        shd.sharded = shard_model(shd.model, dev, default="row_wise", source=ref.model, static_capacity=2.5,
                                  exchange="peer")
        B = 48
        per_rank = [[ref.synthetic_batch(B, seed=100 * s + r) for r in range(world)] for s in range(2)]
        per_rank.append([ref.synthetic_batch(17 + 6 * r, seed=300 + r) for r in range(world)])   # short last batches
        want = ref.evaluate([concat_batches(bs).to(dev) for bs in per_rank])
        got = shd.evaluate([bs[rank].to(dev) for bs in per_rank])
        assert set(got) == set(want)
        assert got["auc"] == want["auc"]
        assert abs(got["binary_cross_entropy"] - want["binary_cross_entropy"]) <= 1e-6
        try:
            shd.evaluate([ref.synthetic_batch(2 * B, seed=7).to(dev)])
            raise AssertionError("a larger eval batch was accepted")
        except ValueError as e:
            assert "sized for local batches" in str(e)
        q.put((rank, "ok"))
    except Exception:
        import traceback

        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_peer_exchange_two_gpus_equals_unsharded():
    import torch.multiprocessing as mp

    from test_evaluate_cpu import _free_port

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_peer_worker, args=(r, 2, port, q)) for r in range(2)]
    for pr in procs:
        pr.start()
    results = [q.get(timeout=600) for _ in procs]
    for pr in procs:
        pr.join(timeout=60)
    bad = [r for r in results if r[1] != "ok"]
    assert not bad, "\n".join(f"rank {r}: {msg}" for r, msg in bad)


if __name__ == "__main__" and sys.argv[1:] == ["full_size"]:
    sys.path.insert(0, os.path.dirname(HERE))
    _full_size_body()
