"""PLE on the H100: the fused gate kernels (csrc/tzk_ple.cuh) against the float64 restatement (tests/ple_ref.py), the
fused model against the torch formulation on the same weights and batches, determinism (two runs, and graphed train
and eval steps against the eager ones, bit for bit), BF16 autocast on the torch formulation, and the fallback outside
the kernels' cover."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ple_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _kern():
    from torcheasyrec_b200.kernels import default_kernels

    return default_kernels()


def _np(t):
    return t.detach().cpu().numpy()


def _close(got, want, r, name=""):
    """|got - want| <= r (|want| + max(1, max |want|)): relative to the tensor's scale."""
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(np.asarray(got, np.float64), want, rtol=r, atol=r * max(1.0, np.abs(want).max()),
                               err_msg=name)


def _layer(T, per, S, final):
    """(gate_input, gate_experts, n_experts) of a layer whose input 0 is the shared input and 1 + i task i's."""
    shared = list(range(T * per, T * per + S))
    gi = [1 + i for i in range(T)] + ([] if final else [0])
    ge = [list(range(i * per, (i + 1) * per)) + shared for i in range(T)] + ([] if final else [list(range(T * per + S))])
    return gi, ge, T * per + S


# (input widths [shared, task 0, ...], H, T, per task, shared, final, all inputs the same tensor)
LAYERS = {
    "taobao1": ([256] * 3, 256, 2, 2, 2, False, True),
    "taobao2": ([256] * 3, 64, 2, 3, 3, False, False),
    "taobao3": ([64] * 3, 32, 2, 4, 4, True, False),
    "extnet": ([13, 16, 15, 14], 4, 3, 3, 4, False, False),       # the reference's module test: a shared gate over 13
    "pletest1": ([25] * 4, 4, 3, 3, 4, False, True),
    "pletest2": ([4] * 4, 8, 3, 3, 3, False, False),
    "e32_odd": ([37, 37], 33, 1, 28, 4, True, False),               # E_g = 32, odd K and H
}


@pytest.mark.parametrize("name", list(LAYERS))
@pytest.mark.parametrize("B", [1, 3, 257, 8192])
def test_kernels_match_restatement(name, B):
    dims, H, T, per, S, final, one = LAYERS[name]
    gi, ge, ne = _layer(T, per, S, final)
    g = torch.Generator().manual_seed(B + H)
    if one:
        inputs, gi = [torch.randn(B, dims[0], generator=g).to(DEV)], [0] * len(gi)
    else:
        inputs = [torch.randn(B, k, generator=g).to(DEV) for k in dims]
    experts = [torch.randn(B, H, generator=g).to(DEV) for _ in range(ne)]
    weights = [(0.3 * torch.randn(len(ids), inputs[gi[j]].shape[1], generator=g)).to(DEV) for j, ids in enumerate(ge)]
    biases = [(0.3 * torch.randn(len(ids), generator=g)).to(DEV) for ids in ge]
    dy = torch.randn(len(gi), B, H, generator=g).to(DEV)
    K = _kern()
    y, p = K.ple_gate_fwd(inputs, gi, weights, biases, experts, ge)
    n = [[_np(t) for t in ts] for ts in (inputs, weights, biases, experts)]
    ry, rp = R.gates_fwd(n[0], gi, n[1], n[2], n[3], ge)
    _close(_np(y), ry, 1e-5, "y")
    _close(_np(p), rp, 1e-5, "p")
    dx, dex, dW, db = K.ple_gate_bwd(inputs, gi, weights, biases, experts, ge, p, dy)
    rdx, rdex, rdW, rdb = R.gates_bwd(n[0], gi, n[1], n[2], n[3], ge, _np(dy))
    for i in range(len(inputs)):
        _close(_np(dx[i]), rdx[i], 2e-5, f"dx{i}")
    _close(_np(dex), rdex, 2e-5, "d_experts")
    for j in range(len(gi)):
        _close(_np(dW[j]), rdW[j], 2e-5, f"dW{j}")
        _close(_np(db[j]), rdb[j], 2e-5, f"db{j}")


def _pipe(seed=7, **kw):
    from torcheasyrec_b200.engine import Pipeline

    return Pipeline("ple_taobao", device=DEV, max_rows=2000, seed=seed, **kw)


def _copy_state(dst, src):
    dst.model.load_state_dict(src.model.state_dict())
    for ca, cb in zip(src.model.sparse_collections(), dst.model.sparse_collections()):
        cb.weights.data.copy_(ca.weights.data)
        if not ca.layout.interleaved and ca.opt_state is not None:
            cb.opt_state.copy_(ca.opt_state)
    dst.dense_optimizer.load_state_dict(copy.deepcopy(src.dense_optimizer.state_dict()))


def _grads(p, batch):
    p.dense_optimizer.zero_grad(set_to_none=True)
    total, (_, preds, _) = p.train_wrapper(batch)
    total.backward()
    torch.cuda.synchronize()
    return ({k: v.clone() for k, v in preds.items() if k.startswith("logits")}, total.detach().clone(),
            {k: v.grad.detach().clone() for k, v in p.model.named_parameters() if v.grad is not None})


def test_fused_model_matches_torch_formulation(monkeypatch):
    """The two paths share every GEMM and differ in the gates' arithmetic order: 1e-5 on logits and loss, 1e-4 on
    gradients; then three steps on each path."""
    from torcheasyrec_b200 import functional as Fn

    a, b = _pipe(), _pipe()
    _copy_state(b, a)
    batch = a.synthetic_batch(4096, seed=3).to(DEV)
    la, lossa, ga = _grads(a, batch)
    with monkeypatch.context() as mp:
        mp.setattr(Fn, "ple_gate_usable", lambda *args, **kw: False)
        lb, lossb, gb = _grads(b, batch)
    for k in la:
        _close(_np(la[k]), _np(lb[k]), 1e-5, k)
    _close(_np(lossa), _np(lossb), 1e-5, "loss")
    assert ga.keys() == gb.keys() and any("_shared_gate" in k for k in ga)
    for k in ga:
        _close(_np(ga[k]), _np(gb[k]), 1e-4, k)
    a2, b2 = _pipe(seed=9), _pipe(seed=9)
    _copy_state(b2, a2)
    batches = [a2.synthetic_batch(4096, seed=20 + i).to(DEV) for i in range(3)]
    la_ = [float(a2.eager_step(bt)) for bt in batches]
    with monkeypatch.context() as mp:
        mp.setattr(Fn, "ple_gate_usable", lambda *args, **kw: False)
        lb_ = [float(b2.eager_step(bt)) for bt in batches]
    np.testing.assert_allclose(la_, lb_, rtol=1e-5)
    lr = max(g["lr"] for g in a2.dense_optimizer.param_groups)
    for (k, pa), pb in zip(a2.model.named_parameters(), b2.model.parameters()):
        diff = float((pa - pb).abs().max())
        assert diff <= 1e-4 * max(1.0, float(pb.abs().max())) + 6 * lr, (k, diff)


def test_two_runs_are_bit_identical():
    outs = []
    for _ in range(2):
        p = _pipe(seed=11)
        batches = [p.synthetic_batch(8192, seed=30 + i).to(DEV) for i in range(2)]
        losses = [float(p.eager_step(bt)) for bt in batches]
        outs.append((losses, [v.detach().clone() for v in p.model.parameters()]))
    assert outs[0][0] == outs[1][0]
    for x, y in zip(outs[0][1], outs[1][1]):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))


def test_graph_replay_equals_eager_step():
    from torcheasyrec_b200.engine import GraphedTrainStep

    a = _pipe(seed=13)
    batches = [a.synthetic_batch(8192, seed=40 + i) for i in range(3)]
    step = GraphedTrainStep(a, batches[0], warmup=2)
    b = _pipe(seed=13, capturable=False)
    _copy_state(b, a)
    for bt in batches[1:]:
        step.load(bt.pin_memory())
        la = float(step.replay())
        lb = float(b.eager_step(bt.to(DEV)))
        assert la == lb
    for pa, pb in zip(a.model.parameters(), b.model.parameters()):
        assert torch.equal(pa.data.view(torch.int32), pb.data.view(torch.int32))


def test_graphed_eval_step_equals_eager():
    from torcheasyrec_b200.engine import GraphedEvalStep

    a = _pipe(seed=19)
    a.eager_step(a.synthetic_batch(2048, seed=1).to(DEV))
    batches = [a.synthetic_batch(2048, seed=50 + i) for i in range(3)]
    step = GraphedEvalStep(a, batches[0])
    a._ensure_metrics()
    ma = a.model._metric_modules
    assert set(ma) == {"auc_ctr", "auc_cvr", "binary_cross_entropy_ctr", "binary_cross_entropy_cvr"}
    eager = {k: [t.clone() for t in m.state()] for k, m in ma.items()}
    for bt in batches:
        step.load(bt.pin_memory())
        got = {k: v.clone() for k, v in step.replay().items()}
        graph_state = {k: [t.clone() for t in m.state()] for k, m in ma.items()}
        for k, m in ma.items():
            for t, e in zip(m.state(), eager[k]):
                t.copy_(e)
        want = a.eval_step(bt.to(DEV))
        for k in got:
            assert torch.equal(got[k], want[k]), k
        for k, m in ma.items():
            for t, gs in zip(m.state(), graph_state[k]):
                assert torch.equal(t, gs), k
        eager = graph_state


def _count(monkeypatch, calls):
    from torcheasyrec_b200 import kernels

    for nm in ("ple_gate_fwd", "ple_gate_bwd"):
        orig = getattr(kernels.CudaKernels, nm)
        monkeypatch.setattr(kernels.CudaKernels, nm,
                            lambda self, *a, _o=orig, _n=nm, **kw: calls.append(_n) or _o(self, *a, **kw))
    for nm in ("stack", "matmul", "bmm"):
        orig = getattr(torch, nm)
        monkeypatch.setattr(torch, nm, lambda *a, _o=orig, _n=nm, **kw: calls.append(_n) or _o(*a, **kw))
    from torcheasyrec_b200 import functional as Fn

    orig = Fn.torch_ple_gate
    monkeypatch.setattr(Fn, "torch_ple_gate", lambda *a, **kw: calls.append("torch_ple_gate") or orig(*a, **kw))


def test_fp32_step_runs_the_fused_gates_and_no_stack_or_bmm(monkeypatch):
    """One fp32 training step calls the forward and the backward gate kernel once per extraction layer, and never the
    torch gate (torch.stack of the experts, torch.matmul / torch.bmm); the one torch.stack is TrainWrapper's sum of the
    two towers' losses."""
    calls = []
    p = _pipe(seed=15)
    batch = p.synthetic_batch(4096, seed=1).to(DEV)
    _count(monkeypatch, calls)
    p.eager_step(batch)
    torch.cuda.synchronize()
    assert sorted(calls) == ["ple_gate_bwd"] * 3 + ["ple_gate_fwd"] * 3 + ["stack"], calls


def test_bf16_autocast_takes_the_torch_formulation_and_trains(monkeypatch):
    calls = []
    p = _pipe(seed=17, edits={"train_config.mixed_precision": "BF16"})
    batch = p.synthetic_batch(2048, seed=2).to(DEV)
    _count(monkeypatch, calls)
    losses = [float(p.eager_step(batch)) for _ in range(3)]
    assert "ple_gate_fwd" not in calls and calls.count("torch_ple_gate") == 3 * 8
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses


def test_shapes_outside_the_cover_fall_back_and_train():
    """H = 1100 (wider than 1024) and a gate over 33 experts take the torch formulation on the GPU, equal to the CPU
    layer, and train."""
    from torcheasyrec_b200.rank_models import ExtractionNet

    for per, S, units, K in [(1, 1, [1100], 8), (16, 17, [4], 8), (2, 2, [8], 1100)]:
        torch.manual_seed(0)
        net = ExtractionNet([K, K], K, "layer", S, per, {"hidden_units": units}, {"hidden_units": units})
        x = torch.randn(300, K)
        outs_cpu, sh_cpu = net([x, x], x)
        net = net.to(DEV)
        xg = x.to(DEV)
        gi, ge = net.gate_layout()
        experts = [torch.zeros(300, units[-1], device=DEV)] * (2 * per + S)
        from torcheasyrec_b200 import functional as Fn

        gates = list(net._task_gates) + [net._shared_gate]
        assert not Fn.ple_gate_usable([xg], [0] * len(gi), [g.weight for g in gates], experts, ge)
        outs, sh = net([xg, xg], xg)
        for o, oc in zip(outs + [sh], outs_cpu + [sh_cpu]):
            np.testing.assert_allclose(_np(o), _np(oc), rtol=1e-4, atol=1e-5)
        (sum(o.sum() for o in outs) + sh.sum()).backward()
        assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in net._task_gates.parameters())


def test_reference_test_shapes_on_the_fused_path(monkeypatch):
    """The reference's ple_test model shapes (3 tasks, group width 25, a 13-expert shared gate) run fused on the GPU
    and match the torch formulation."""
    from torcheasyrec_b200 import functional as Fn
    from torcheasyrec_b200.rank_models import ExtractionNet

    torch.manual_seed(0)
    net = ExtractionNet([25] * 3, 25, "layer1", 4, 3, {"hidden_units": [12, 8, 6, 4]},
                        {"hidden_units": [12, 8, 4]}).to(DEV)
    x = torch.randn(300, 25, device=DEV, requires_grad=True)
    outs, sh = net([x] * 3, x)
    (sum((o * (i + 1)).sum() for i, o in enumerate(outs)) + sh.sum()).backward()
    gx, gp = x.grad.clone(), [p.grad.clone() for p in net.parameters()]
    x.grad = None
    net.zero_grad(set_to_none=True)
    with monkeypatch.context() as mp:
        mp.setattr(Fn, "ple_gate_usable", lambda *a, **k: False)
        outs2, sh2 = net([x] * 3, x)
        (sum((o * (i + 1)).sum() for i, o in enumerate(outs2)) + sh2.sum()).backward()
    for o, o2 in zip(outs + [sh], outs2 + [sh2]):
        _close(_np(o), _np(o2), 1e-5, "y")
    _close(_np(gx), _np(x.grad), 1e-4, "dx")
    for a, p in zip(gp, net.parameters()):
        _close(_np(a), _np(p.grad), 1e-4)
