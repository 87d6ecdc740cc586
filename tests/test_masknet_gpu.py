"""MaskNet on the H100: every fused kernel (csrc/tzk_masknet.cuh) against the float64 restatement
(tests/masknet_ref.py), the fused model against the torch formulation on the same weights and batches, determinism
(two runs, and graphed train and eval steps against the eager ones, bit for bit), BF16 autocast and serial mode on the
torch formulation, and the fallback outside the kernels' cover."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import masknet_ref as M  # noqa: E402

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


def _r(g, *s, scale=1.0):
    return (torch.randn(*s, generator=g) * scale).to(DEV)


# (E, H, nb): masknet_criteo, the reference's module test, its model test with one block
@pytest.mark.parametrize("E,H,nb", [(429, 512, 3), (24, 16, 3), (33, 16, 1)])
@pytest.mark.parametrize("B", [1, 3, 257, 8192])
def test_kernels_match_restatement(E, H, nb, B):
    Ep = M.pad4(E)
    g = torch.Generator().manual_seed(B + E)
    e = torch.zeros(B, Ep, device=DEV)
    e[:, :E] = _r(g, B, E)
    m, dv = _r(g, B, nb * Ep), _r(g, B, nb * Ep)
    b2, lw, lb = _r(g, nb * E, scale=0.3), 1 + _r(g, E, scale=0.1), _r(g, E, scale=0.1)
    z, dy = _r(g, B, nb * H), _r(g, B, nb * H)
    b3, fw, fb = _r(g, nb * H, scale=0.3), 1 + _r(g, nb * H, scale=0.1), _r(g, nb * H, scale=0.3)
    K = _kern()
    v, st = K.masknet_mask_fwd(e, m, b2, lw, lb, E, nb)
    rv, rst = M.mask_fwd(_np(e), _np(m), _np(b2), _np(lw), _np(lb), E, nb)
    _close(_np(v), rv, 1e-5, "v")
    _close(_np(st), rst, 1e-5, "mask stats")
    got = K.masknet_mask_bwd(e, m, b2, lw, lb, st, dv, E, nb)
    want = M.mask_bwd(_np(e), _np(m), _np(b2), _np(lw), _np(lb), _np(dv), E, nb)
    for a, w, what in zip(got, want, ("dm", "de", "db2", "dgamma_ln", "dbeta_ln")):
        _close(_np(a), w, 2e-5, what)
    y, st2 = K.masknet_ffn_fwd(z, b3, fw, fb, nb)
    ry, rst2 = M.ffn_fwd(_np(z), _np(b3), _np(fw), _np(fb), nb)
    _close(_np(y), ry, 1e-5, "y")
    _close(_np(st2), rst2, 1e-5, "ffn stats")
    got = K.masknet_ffn_bwd(z, b3, fw, fb, st2, dy, nb)
    want = M.ffn_bwd(_np(z), _np(b3), _np(fw), _np(fb), _np(dy), nb)
    for a, w, what in zip(got, want, ("dz", "dgamma", "dbeta", "db3")):
        _close(_np(a), w, 2e-5, what)


def _pipe(seed=7, **kw):
    from torcheasyrec_b200.engine import Pipeline

    return Pipeline("masknet_criteo", device=DEV, max_rows=2000, seed=seed, **kw)


def _copy_state(dst, src):
    dst.model.load_state_dict(src.model.state_dict())
    for ca, cb in zip(src.model.sparse_collections(), dst.model.sparse_collections()):
        cb.weights.data.copy_(ca.weights.data)
        if not ca.layout.interleaved and ca.opt_state is not None:
            cb.opt_state.copy_(ca.opt_state)
    dst.dense_optimizer.load_state_dict(copy.deepcopy(src.dense_optimizer.state_dict()))


def _grads(p, batch):
    """Logits, loss, every dense parameter's gradient and the group's input gradient of one forward/backward."""
    p.dense_optimizer.zero_grad(set_to_none=True)
    seen = {}
    mod = p.model.mask_net_layer

    def keep(_mod, args):
        args[0].retain_grad()
        seen["e"] = args[0]

    handle = mod.register_forward_pre_hook(keep)
    try:
        total, (_, preds, _) = p.train_wrapper(batch)
        total.backward()
    finally:
        handle.remove()
    torch.cuda.synchronize()
    return preds["logits"].clone(), total.detach().clone(), {
        k: v.grad.detach().clone() for k, v in p.model.named_parameters() if v.grad is not None}, seen["e"].grad.clone()


def test_fused_model_matches_torch_formulation(monkeypatch):
    """Tolerances (DESIGN §5): the two paths run the same GEMMs on cuBLASLt BF16x9 at different row pitches and sum the
    batch reductions in different orders, so they agree to fp32 rounding: 1e-5 on logits and loss, 1e-4 on gradients."""
    from torcheasyrec_b200 import functional as Fn

    calls = []
    orig = type(_kern()).masknet_mask_fwd
    monkeypatch.setattr(type(_kern()), "masknet_mask_fwd", lambda self, *a: calls.append(1) or orig(self, *a))
    a = _pipe()
    b = _pipe()
    _copy_state(b, a)
    batch = a.synthetic_batch(4096, seed=3).to(DEV)
    la, lossa, ga, dea = _grads(a, batch)
    assert calls
    with monkeypatch.context() as mp:
        mp.setattr(Fn, "masknet_usable", lambda *args, **kw: False)
        lb, lossb, gb, deb = _grads(b, batch)
    _close(_np(la), _np(lb), 1e-5, "logits")
    _close(_np(lossa), _np(lossb), 1e-5, "loss")
    _close(_np(dea), _np(deb), 1e-4, "d all_features")
    assert ga.keys() == gb.keys()
    assert any("mask_blocks.2.mask_generator.0.weight" in k for k in ga)
    for k in ga:
        _close(_np(ga[k]), _np(gb[k]), 1e-4, k)
    # three Adagrad (sparse) / Adam (dense) steps on each path
    a2, b2 = _pipe(seed=9), _pipe(seed=9)
    _copy_state(b2, a2)
    batches = [a2.synthetic_batch(4096, seed=20 + i).to(DEV) for i in range(3)]
    la_ = [float(a2.eager_step(bt)) for bt in batches]
    with monkeypatch.context() as mp:
        mp.setattr(Fn, "masknet_usable", lambda *args, **kw: False)
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


def test_fp32_step_runs_the_fused_kernels_and_no_layer_norm(monkeypatch):
    """One fp32 training step calls each of the four MaskNet kernels once and never torch's layer_norm."""
    import torch.nn.functional as F

    from torcheasyrec_b200 import kernels

    calls = []
    for nm in ("masknet_mask_fwd", "masknet_mask_bwd", "masknet_ffn_fwd", "masknet_ffn_bwd"):
        orig = getattr(kernels.CudaKernels, nm)
        monkeypatch.setattr(kernels.CudaKernels, nm,
                            lambda self, *a, _o=orig, _n=nm, **kw: calls.append(_n) or _o(self, *a, **kw))
    ln = F.layer_norm
    monkeypatch.setattr(F, "layer_norm", lambda *a, **kw: calls.append("layer_norm") or ln(*a, **kw))
    p = _pipe(seed=15)
    batch = p.synthetic_batch(4096, seed=1).to(DEV)
    p.eager_step(batch)
    torch.cuda.synchronize()
    assert sorted(calls) == ["masknet_ffn_bwd", "masknet_ffn_fwd", "masknet_mask_bwd", "masknet_mask_fwd"], calls


def test_bf16_autocast_takes_the_torch_formulation_and_trains(monkeypatch):
    from torcheasyrec_b200 import kernels

    calls = []
    for nm in ("masknet_mask_fwd", "masknet_ffn_fwd"):
        orig = getattr(kernels.CudaKernels, nm)
        monkeypatch.setattr(kernels.CudaKernels, nm,
                            lambda self, *a, _o=orig, _n=nm, **kw: calls.append(_n) or _o(self, *a, **kw))
    p = _pipe(seed=17, edits={"train_config.mixed_precision": "BF16"})
    batch = p.synthetic_batch(2048, seed=2).to(DEV)
    losses = [float(p.eager_step(batch)) for _ in range(3)]
    assert calls == []
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses


def test_serial_mode_and_shapes_outside_the_cover_fall_back():
    """Serial blocks, H = 18 (not a multiple of 4) and E = 1100 (pitch above 1024) take the torch formulation on the GPU,
    equal to the CPU module."""
    from torcheasyrec_b200.rank_models import MaskNetModule

    for E, H, nb, par in [(429, 16, 2, False), (40, 18, 2, True), (1100, 8, 1, True)]:
        torch.manual_seed(0)
        mod = MaskNetModule(E, nb, {"reduction_ratio": 0.5, "aggregation_dim": 0, "hidden_dim": H},
                            {"hidden_units": [4]}, par)
        e = torch.randn(300, E)
        assert not mod.to(DEV).fused_usable(e.to(DEV))
        y_gpu = mod(e.to(DEV))
        y_cpu = mod.cpu()(e)
        np.testing.assert_allclose(y_gpu.detach().cpu().numpy(), y_cpu.detach().numpy(), rtol=1e-4, atol=1e-5)


def test_reference_module_test_shape_on_the_fused_path():
    """tzrec/modules/masknet_test.py's module (E = 24, ratio 2, H = 16, top [8, 4, 2], parallel, dropout 0) runs fused on
    the GPU and matches its torch formulation."""
    from torcheasyrec_b200 import functional as Fn
    from torcheasyrec_b200.rank_models import MaskNetModule

    torch.manual_seed(0)
    mod = MaskNetModule(24, 3, {"reduction_ratio": 2.0, "aggregation_dim": 0, "hidden_dim": 16},
                        {"hidden_units": [8, 4, 2]}).to(DEV)
    e = torch.randn(300, 24, device=DEV, requires_grad=True)
    assert mod.fused_usable(e)
    y = mod(e)
    assert y.shape == (300, 2)
    y.sum().backward()
    ge, gp = e.grad.clone(), [p.grad.clone() for p in mod.parameters()]
    e.grad = None
    mod.zero_grad(set_to_none=True)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(Fn, "masknet_usable", lambda *a, **k: False)
        y2 = mod(e)
        y2.sum().backward()
    _close(_np(y), _np(y2), 1e-5, "y")
    _close(_np(ge), _np(e.grad), 1e-4, "de")
    for a, p in zip(gp, mod.parameters()):
        _close(_np(a), _np(p.grad), 1e-4)
