"""PEPNet on the H100: the fused gate-product kernels (csrc/tzk_pepnet.cuh) against the float64 restatement
(tests/pepnet_ref.py), the fused EPNet / PPNet against the torch formulation on the same weights, determinism (two runs,
and graphed train and eval steps against the eager ones, bit for bit, with dropout 0), pepnet_taobao with its dropout
0.1 training graphed, BF16 autocast on the torch formulation, and the fallback outside the kernels' cover."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pepnet_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NO_DROPOUT = {"model_config.pepnet.ppnet_dropout_ratio": [0.0]}


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


# (segment widths, relu, with bias, gamma): pepnet_taobao's EPNet (256, identity, no bias), its PPNet depths (2 x 512,
# 2 x 256, ReLU + bias), 8 tasks of mixed widths, and the widest segment
SEGMENTS = {
    "taobao_epnet": ([256], False, False, 2.0),
    "taobao_depth0": ([512, 512], True, True, 2.0),
    "taobao_depth1": ([256, 256], True, True, 2.0),
    "eight_tasks": ([4, 8, 12, 16, 96, 128, 384, 1024], True, True, 1.5),
}


@pytest.mark.parametrize("name", list(SEGMENTS))
@pytest.mark.parametrize("B", [1, 3, 257, 8192, 65536])
def test_kernels_match_restatement(name, B):
    """x / z / y of the T segments side by side in [B, T N] buffers (PPNet's layout), so the rows are strided."""
    widths, relu, bias, gamma = SEGMENTS[name]
    if B == 65536 and name == "eight_tasks":
        pytest.skip("pepnet_taobao's widths only at B = 65536")
    g = torch.Generator(device=DEV).manual_seed(B + len(widths))
    W = sum(widths)
    x, z, dy = (torch.randn(B, W, device=DEV, generator=g) for _ in range(3))
    bxs = [torch.randn(n, device=DEV, generator=g) * 0.5 if bias else None for n in widths]
    bzs = [torch.randn(n, device=DEV, generator=g) * 0.5 for n in widths]
    y, dx, dz = torch.full_like(x, float("nan")), torch.full_like(x, float("nan")), torch.full_like(x, float("nan"))
    cols, o = [], 0
    for n in widths:
        cols.append(slice(o, o + n))
        o += n
    segs = [(x[:, c], bxs[i], z[:, c], bzs[i], y[:, c], relu, gamma) for i, c in enumerate(cols)]
    _kern().pepnet_gate_fwd(segs)
    sums = _kern().pepnet_gate_bwd([(s[0], s[1], s[2], s[3], None, relu, gamma) for s in segs],
                                   [dy[:, c] for c in cols], [dx[:, c] for c in cols], [dz[:, c] for c in cols])
    torch.cuda.synchronize()
    d = lambda t: None if t is None else t.double().cpu().numpy()  # noqa: E731
    rsegs = [(d(x[:, c]), d(bxs[i]), d(z[:, c]), d(bzs[i]), relu, gamma) for i, c in enumerate(cols)]
    ys = R.gate_fwd(rsegs)
    bw = R.gate_bwd(rsegs, [d(dy[:, c]) for c in cols])
    for i, c in enumerate(cols):
        _close(_np(y[:, c]), ys[i], 1e-6, f"y{i}")
        _close(_np(dx[:, c]), bw[i][0], 1e-6, f"dx{i}")
        _close(_np(dz[:, c]), bw[i][1], 1e-6, f"dz{i}")
        tol = 1e-6 * max(8.0, np.sqrt(B))
        _close(_np(sums[i][0]), bw[i][2], tol, f"dbx{i}")
        _close(_np(sums[i][1]), bw[i][3], tol, f"dbz{i}")


def _modules(M, Dd, U, eh, T, hidden):
    from torch import nn
    from torcheasyrec_b200.rank_models import EPNet, PPNet

    mods = nn.Module()
    mods.epnet = EPNet(M, Dd, hidden_dim=eh or M) if Dd else None
    mods.ppnet = PPNet(M, U, num_task=T, hidden_units=hidden, dropout_ratio=[0.0]) if U else None
    return mods


def _run_modules(mods, xs, dys):
    x = xs["main"]
    if mods.epnet is not None:
        x = mods.epnet(x, xs["domain"])
    outs = mods.ppnet(x, xs["uia"]) if mods.ppnet is not None else [x]
    torch.autograd.backward(outs, dys)
    torch.cuda.synchronize()
    return ([o.detach().clone() for o in outs], {k: v.grad.clone() for k, v in xs.items()},
            {k: p.grad.clone() for k, p in mods.named_parameters()})


# (main, domain, uia, epnet hidden, tasks, ppnet hidden): pepnet_taobao's modules, and a covered variant of the
# reference test's shapes with epnet_hidden_unit set and three tasks
MODULES = {"taobao": (256, 16, 208, None, 2, [512, 256]), "small": (24, 8, 16, 8, 3, [16, 8])}


@pytest.mark.parametrize("name", list(MODULES))
def test_fused_modules_match_torch_formulation(name, monkeypatch):
    """Fused EPNet + PPNet against the torch formulation on the same weights at B = 8192: outputs, input gradients and
    every parameter gradient.  Both sides run fp32 GEMMs (the fused side cuBLASLt BF16x9, torch's cuBLAS with TF32 off)
    and differ in summation order: 1e-5 on outputs, 1e-4 on gradients."""
    from torcheasyrec_b200 import functional as Fn

    M, Dd, U, eh, T, hidden = MODULES[name]
    torch.manual_seed(0)
    mods = _modules(M, Dd, U, eh, T, hidden).to(DEV)
    B = 8192
    g = torch.Generator(device=DEV).manual_seed(1)
    base = {"main": torch.randn(B, M, device=DEV, generator=g), "domain": torch.randn(B, Dd, device=DEV, generator=g),
            "uia": torch.randn(B, U, device=DEV, generator=g)}
    dys = [torch.randn(B, hidden[-1], device=DEV, generator=g) for _ in range(T)]
    assert mods.ppnet.fused_usable(base["main"], base["uia"])
    res = []
    for fused in (True, False):
        for p in mods.parameters():
            p.grad = None
        xs = {k: v.clone().requires_grad_(True) for k, v in base.items()}
        with monkeypatch.context() as mp:
            if not fused:
                mp.setattr(Fn, "pepnet_usable", lambda *a, **kw: False)
            res.append(_run_modules(mods, xs, dys))
    (oa, da, ga), (ob, db, gb) = res
    for i, (a, b) in enumerate(zip(oa, ob)):
        _close(_np(a), _np(b), 1e-5, f"out{i}")
    for k in da:
        _close(_np(da[k]), _np(db[k]), 1e-4, f"d_{k}")
    assert ga.keys() == gb.keys()
    for k in ga:
        _close(_np(ga[k]), _np(gb[k]), 1e-4, k)


def _pipe(seed=7, edits=NO_DROPOUT, **kw):
    from torcheasyrec_b200.engine import Pipeline

    return Pipeline("pepnet_taobao", device=DEV, max_rows=2000, seed=seed, edits=edits, **kw)


def _copy_state(dst, src):
    dst.model.load_state_dict(src.model.state_dict())
    for ca, cb in zip(src.model.sparse_collections(), dst.model.sparse_collections()):
        cb.weights.data.copy_(ca.weights.data)
        if not ca.layout.interleaved and ca.opt_state is not None:
            cb.opt_state.copy_(ca.opt_state)
    dst.dense_optimizer.load_state_dict(copy.deepcopy(src.dense_optimizer.state_dict()))


def _count(monkeypatch, calls):
    from torcheasyrec_b200 import kernels

    for nm in ("pepnet_gate_fwd", "pepnet_gate_bwd"):
        orig = getattr(kernels.CudaKernels, nm)
        monkeypatch.setattr(kernels.CudaKernels, nm,
                            lambda self, *a, _o=orig, _n=nm, **kw: calls.append(_n) or _o(self, *a, **kw))


def test_fp32_step_runs_the_fused_product_once_per_depth(monkeypatch):
    """One fp32 training step of pepnet_taobao: the product kernels run once each way for EPNet and for each of PPNet's
    two depths, and the loss moves over three steps."""
    calls = []
    p = _pipe(seed=15, edits=None)
    batch = p.synthetic_batch(4096, seed=1).to(DEV)
    _count(monkeypatch, calls)
    losses = [float(p.eager_step(batch)) for _ in range(3)]
    torch.cuda.synchronize()
    assert sorted(calls) == ["pepnet_gate_bwd"] * 9 + ["pepnet_gate_fwd"] * 9, calls
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses


def test_two_runs_are_bit_identical():
    outs = []
    for _ in range(2):
        p = _pipe(seed=11, edits=None)         # dropout 0.1: the seeded generator makes it repeatable too
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


def test_reference_example_with_dropout_trains_graphed():
    """tests/golden/ref_examples/pepnet_taobao.config as stored (dropout 0.1) as a captured step: finite losses that go
    down on a repeated batch, and replays draw fresh dropout masks (two replays on one batch differ)."""
    from torcheasyrec_b200.engine import GraphedTrainStep, Pipeline

    ref = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_examples", "pepnet_taobao.config")
    p = Pipeline(ref, device=DEV, max_rows=2000, seed=21)
    batch = p.synthetic_batch(8192, seed=2)
    step = GraphedTrainStep(p, batch, warmup=2)
    losses = []
    for _ in range(6):
        step.load(batch.pin_memory())
        losses.append(float(step.replay()))
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
    assert len(set(losses)) == len(losses)


def test_bf16_autocast_takes_the_torch_formulation_and_trains(monkeypatch):
    calls = []
    p = _pipe(seed=17, edits={"train_config.mixed_precision": "BF16"})
    batch = p.synthetic_batch(2048, seed=2).to(DEV)
    _count(monkeypatch, calls)
    losses = [float(p.eager_step(batch)) for _ in range(3)]
    assert calls == []
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses


def test_shapes_outside_the_cover_fall_back_and_match_the_cpu():
    """The reference test's group width 25 (EPNet and PPNet), hidden units wider than 1024, and a non-ReLU activation
    take the torch formulation on the GPU, equal to the CPU modules, and train."""
    from torcheasyrec_b200 import functional as Fn
    from torcheasyrec_b200.rank_models import PPNet

    cases = [(_modules(25, 16, 16, None, 2, [16, 8]), 25, 16),
             (_modules(24, 8, 16, None, 2, [1028, 8]), 24, 16)]
    torch.manual_seed(0)
    cases.append((_modules(24, 8, 16, None, 2, [16, 8]), 24, 16))
    cases[-1][0].ppnet = PPNet(24, 16, 2, [16, 8], activation="nn.Sigmoid", dropout_ratio=[0.0])
    for mods, M, U in cases:
        g = torch.Generator().manual_seed(3)
        base = {"main": torch.randn(64, M, generator=g), "domain": torch.randn(64, 16 if M == 25 else 8, generator=g),
                "uia": torch.randn(64, U, generator=g)}
        dys = [torch.randn(64, mods.ppnet.hidden_units[-1], generator=g) for _ in range(2)]
        oc, dc, gc = _run_cpu(mods, base, dys)
        mods = mods.to(DEV)
        xs = {k: v.to(DEV).requires_grad_(True) for k, v in base.items()}
        assert not mods.ppnet.fused_usable(xs["main"], xs["uia"])
        if M == 25:
            assert not Fn.pepnet_usable(xs["main"], xs["domain"], [25], [25])
        for p in mods.parameters():
            p.grad = None
        og, dg, gg = _run_modules(mods, xs, [d.to(DEV) for d in dys])
        for a, b in zip(og, oc):
            _close(_np(a), _np(b), 1e-4, "out")
        for k in gc:
            _close(_np(gg[k]), _np(gc[k]), 1e-4, k)


def _run_cpu(mods, base, dys):
    xs = {k: v.clone().requires_grad_(True) for k, v in base.items()}
    x = xs["main"]
    if mods.epnet is not None:
        x = mods.epnet(x, xs["domain"])
    outs = mods.ppnet(x, xs["uia"])
    torch.autograd.backward(outs, dys)
    res = ([o.detach().clone() for o in outs], {k: v.grad.clone() for k, v in xs.items()},
           {k: p.grad.clone() for k, p in mods.named_parameters()})
    for p in mods.parameters():
        p.grad = None
    return res
