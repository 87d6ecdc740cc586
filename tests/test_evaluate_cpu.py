"""Pipeline.evaluate on the CPU checker backend: the reference's metric names, each value against a float64 statement
computed from the step's own predictions and losses, model state untouched, train -> evaluate -> train equal to
train -> train, the unsupported metric kinds refused at evaluate (and only there), and a sharded W = 2 evaluate over gloo
equal to the unsharded one on the concatenated batch."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import auc_ref  # noqa: E402
from metric_oracle_backend import MetricOracleKernels  # noqa: E402

from torcheasyrec_b200 import example_configs  # noqa: E402
from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200.engine import Pipeline  # noqa: E402

NAMES = {"dlrm_criteo": {"auc", "binary_cross_entropy"}, "deepfm_criteo": {"auc", "binary_cross_entropy"},
         "multi_tower_din_taobao": {"auc", "binary_cross_entropy"},
         "mmoe_taobao": {"auc_ctr", "auc_cvr", "binary_cross_entropy_ctr", "binary_cross_entropy_cvr"}}
THRESHOLDS = {"auc": 200, "auc_ctr": 200, "auc_cvr": 1000}


def _all_state(p: Pipeline):
    """Every tensor the model and its optimizers own: parameters, buffers (BatchNorm statistics), the sparse
    collections' arenas / optimizer states / device step counters, and the dense optimizer's state."""
    out = {f"sd.{k}": v.detach().clone() for k, v in p.model.state_dict().items()}
    for mn, m in p.model.named_modules():
        for an, v in vars(m).items():
            if isinstance(v, torch.Tensor):
                out[f"attr.{mn}.{an}"] = v.detach().clone()
    for i, st in p.dense_optimizer.state_dict()["state"].items():
        for k, v in st.items():
            if isinstance(v, torch.Tensor):
                out[f"opt.{i}.{k}"] = v.clone()
    return out


def _assert_same_state(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), k


def _statement(p: Pipeline, batches):
    """float64 values from the eval forward's own predictions and losses (model.eval(), no_grad)."""
    probs, labels, loss_sum, n = {}, {}, {}, {}
    p.model.eval()
    with torch.no_grad():
        for b in batches:
            _, (losses, preds, _) = p.train_wrapper(b)
            for metrics, loss_cfgs, label_name, sfx in p.model._metric_heads():
                probs.setdefault(sfx, []).append(preds["probs" + sfx].numpy())
                labels.setdefault(sfx, []).append(b.labels[label_name].numpy())
                for lc in loss_cfgs:
                    name = lc.WhichOneof("loss") + sfx
                    B = b.labels[label_name].shape[0]
                    loss_sum[name] = loss_sum.get(name, 0.0) + float(losses[name]) * B
                    n[name] = n.get(name, 0) + B
    p.model.train()
    out = {name: loss_sum[name] / n[name] for name in loss_sum}
    for sfx in probs:
        name = "auc" + sfx
        out[name] = auc_ref.binned_auc(np.concatenate(probs[sfx]), np.concatenate(labels[sfx]), THRESHOLDS[name])
    return out


@pytest.mark.parametrize("name", sorted(NAMES))
def test_evaluate_matches_statement_and_leaves_state(name):
    p = Pipeline(name, device="cpu", max_rows=200, seed=3)
    with Fn.use_backend(MetricOracleKernels()):
        p.eager_step(p.synthetic_batch(64, seed=0))            # trained state: optimizer states, step counters set
        evals = [p.synthetic_batch(48, seed=10 + i) for i in range(3)] + [p.synthetic_batch(20, seed=20)]
        before = _all_state(p)
        assert p.model.training
        got = p.evaluate(evals)
        assert p.model.training
        _assert_same_state(before, _all_state(p))
        want = _statement(p, evals)
    assert set(got) == NAMES[name] == set(want)
    for k in got:
        assert got[k] == pytest.approx(want[k], abs=1e-12, rel=1e-12), k
    if name == "mmoe_taobao":
        assert p.model._metric_modules["auc_cvr"].counts.shape == (1001, 2)
    # the state was reset: a second evaluation of the same batches gives the same numbers
    with Fn.use_backend(MetricOracleKernels()):
        assert p.evaluate(evals) == got


def test_num_steps_defaults_to_eval_config_and_limits_the_batches():
    p = Pipeline("dlrm_criteo", device="cpu", max_rows=100, seed=2, edits={"eval_config.num_steps": 2})
    evals = [p.synthetic_batch(32, seed=i) for i in range(4)]
    k = MetricOracleKernels()
    with Fn.use_backend(k):
        got = p.evaluate(evals)
        assert k.auc_updates == 2
        assert got == p.evaluate(evals[:2], num_steps=0) == p.evaluate(iter(evals[:3]), num_steps=2)


def test_evaluate_between_train_steps_changes_nothing():
    a = Pipeline("deepfm_criteo", device="cpu", max_rows=100, seed=4)
    b = Pipeline("deepfm_criteo", device="cpu", max_rows=100, seed=4)
    t1, t2 = a.synthetic_batch(32, seed=1), a.synthetic_batch(32, seed=2)
    with Fn.use_backend(MetricOracleKernels()):
        la1 = a.eager_step(t1)
        a.evaluate([a.synthetic_batch(32, seed=9), a.synthetic_batch(7, seed=8)])
        la2 = a.eager_step(t2)
        lb1, lb2 = b.eager_step(t1), b.eager_step(t2)
    assert torch.equal(la1, lb1) and torch.equal(la2, lb2)
    _assert_same_state(_all_state(a), _all_state(b))


def test_eval_enqueues_no_sparse_backward_work():
    k = MetricOracleKernels()
    calls = []
    for m in ("fused_bwd", "fused_bwd_sort", "fused_bwd_apply", "bag_grad_expand"):
        orig = getattr(k, m)
        setattr(k, m, lambda *a, _m=m, _o=orig, **kw: (calls.append(_m), _o(*a, **kw))[1])
    p = Pipeline("dlrm_criteo", device="cpu", max_rows=100, seed=2)
    with Fn.use_backend(k):
        p.eager_step(p.synthetic_batch(16, seed=0))
        assert calls
        calls.clear()
        p.evaluate([p.synthetic_batch(16, seed=1)])
    assert calls == []


def _config_with(tmp_path, metric: str) -> str:
    text = example_configs.dlrm_criteo()
    text = text.replace("    metrics {\n        auc {}\n    }\n", "    metrics {\n        auc {}\n    }\n"
                        f"    metrics {{\n        {metric} {{}}\n    }}\n")
    path = str(tmp_path / f"dlrm_{metric}.config")
    with open(path, "w") as fh:
        fh.write(text)
    return path


@pytest.mark.parametrize("metric", ["grouped_auc", "recall_at_k", "accuracy"])
def test_unsupported_metric_raises_only_at_evaluate(tmp_path, metric):
    p = Pipeline(_config_with(tmp_path, metric), device="cpu", max_rows=100, seed=2)
    assert any(m.WhichOneof("metric") == metric for m in p.cfg.model_config.metrics)
    with Fn.use_backend(MetricOracleKernels()):
        p.eager_step(p.synthetic_batch(16, seed=0))             # training is unaffected
        with pytest.raises(NotImplementedError, match=metric):
            p.evaluate([p.synthetic_batch(16, seed=1)])
        p.eager_step(p.synthetic_batch(16, seed=2))
    assert p.model.training


def test_invalid_labels_raise_at_compute_and_reset():
    p = Pipeline("dlrm_criteo", device="cpu", max_rows=100, seed=2)
    bad = p.synthetic_batch(16, seed=1)
    bad.labels[p.labels[0]][3] = 2.0
    with Fn.use_backend(MetricOracleKernels()):
        with pytest.raises(ValueError, match="1 samples"):
            p.evaluate([bad])
        good = p.synthetic_batch(16, seed=1)
        assert set(p.evaluate([good])) == {"auc", "binary_cross_entropy"}     # the failed evaluation left no state


def test_failing_step_restores_train_mode_and_resets(monkeypatch):
    p = Pipeline("dlrm_criteo", device="cpu", max_rows=100, seed=2)
    evals = [p.synthetic_batch(16, seed=i) for i in range(2)]
    with Fn.use_backend(MetricOracleKernels()):
        want = p.evaluate(evals)
        orig = p.train_wrapper.forward
        n = []

        def flaky(batch):
            n.append(1)
            if len(n) == 2:
                raise RuntimeError("step failed")
            return orig(batch)

        monkeypatch.setattr(p.train_wrapper, "forward", flaky)
        with pytest.raises(RuntimeError, match="step failed"):
            p.evaluate(evals)
        assert p.model.training
        monkeypatch.setattr(p.train_wrapper, "forward", orig)
        assert p.evaluate(evals) == want


# ---- sharded: W = 2 over gloo ----------------------------------------------------------------------------------------
def _free_port():
    import socket

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, name, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    try:
        from torcheasyrec_b200 import metrics
        from torcheasyrec_b200.distributed import shard_model
        from torcheasyrec_b200.verify import concat_batches

        with Fn.use_backend(MetricOracleKernels()):
            ref = Pipeline(name, device="cpu", max_rows=300, seed=5, capturable=False)
            shd = Pipeline(name, device="cpu", max_rows=300, seed=5, capturable=False)
            shd.model.load_state_dict(ref.model.state_dict())
            shard_model(shd.model, torch.device("cpu"), default="row_wise", source=ref.model)
            shd.model.init_metric(distributed=True)
            B = 40
            per_rank = [[ref.synthetic_batch(B, seed=100 * s + r) for r in range(world)] for s in range(2)]
            per_rank.append([ref.synthetic_batch(11 + 6 * r, seed=300 + r) for r in range(world)])   # short last batches
            glob = [concat_batches(bs) for bs in per_rank]
            mine = [bs[rank] for bs in per_rank]
            for g in glob:
                ref.eval_step(g)
            for m in mine:
                shd.eval_step(m)
            metrics.sync_states(shd.model._metric_modules)
            for k, m in ref.model._metric_modules.items():
                if k.startswith("auc"):
                    assert torch.equal(m.counts, shd.model._metric_modules[k].counts), k
                    assert int(m.counts.sum()) == sum(b.labels[next(iter(b.labels))].shape[0] for b in glob)
            for m in ref.model._metric_modules.values():
                m.reset()
            for m in shd.model._metric_modules.values():
                m.reset()
            want = ref.evaluate(glob)
            got = shd.evaluate(mine)
        assert set(got) == set(want)
        for k in got:
            if k.startswith("auc"):
                assert got[k] == want[k], k
            else:
                assert abs(got[k] - want[k]) <= 1e-6, (k, got[k], want[k])
        q.put((rank, "ok"))
    except Exception:
        import traceback

        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("name", ["dlrm_criteo", "mmoe_taobao"])
def test_sharded_two_ranks_equals_unsharded_on_concatenated_batch(name):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, name, q)) for r in range(2)]
    for pr in procs:
        pr.start()
    results = [q.get(timeout=600) for _ in procs]
    for pr in procs:
        pr.join(timeout=60)
    bad = [r for r in results if r[1] != "ok"]
    assert not bad, "\n".join(f"rank {r}: {msg}" for r, msg in bad)
