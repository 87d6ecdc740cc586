"""WuKong on the H100: every fused kernel (csrc/tzk_wukong.cuh) against the float64 restatement (tests/wukong_ref.py),
the fused model against the torch formulation on the same weights and batches, determinism (two runs, and a graphed
step against the eager one, bit for bit), BF16 autocast on the torch formulation, and the fallback outside the
kernels' cover."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import wukong_ref as W  # noqa: E402
from test_wukong_cpu import SHAPES, _close  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _kern():
    from torcheasyrec_b200.kernels import default_kernels

    return default_kernels()


def _inputs(shape, B, seed):
    n, d, k, f, l, proj = shape
    m = f + l
    g = torch.Generator().manual_seed(seed)

    def r(*s, scale=1.0):
        return (torch.randn(*s, generator=g) * scale).to(DEV)

    return dict(x=r(B, n, d), wf=r(n, k, scale=0.3), wl=r(n, l, scale=0.3), wr=r(n, m, scale=0.3) if proj else None,
                gf=1 + r(n * k, scale=0.1), bf=r(n * k, scale=0.1), g=1 + r(d, scale=0.1), b=r(d, scale=0.1),
                fmb=r(B, f * d), d_ln_f=r(B, n * k), dy=r(B, m, d))


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


@pytest.mark.parametrize("name", sorted(SHAPES))
@pytest.mark.parametrize("B", [1, 3, 257, 8192])
def test_kernels_match_restatement(name, B):
    n, d, k, f, l, proj = SHAPES[name]
    t = _inputs(SHAPES[name], B, seed=B + n)
    K = _kern()
    ln_f, st, base = K.wukong_mix_fwd(t["x"], t["wf"], t["gf"], t["bf"], t["wl"], t["wr"], f)
    r_ln_f, r_st, r_base = W.mix_fwd(_np(t["x"]), _np(t["wf"]), _np(t["gf"]), _np(t["bf"]), _np(t["wl"]), _np(t["wr"]), f)
    _close(_np(ln_f), r_ln_f, 1e-5, "ln_f")
    _close(_np(st), r_st, 1e-5, "mix stats")
    _close(_np(base), r_base, 1e-5, "base")
    y, ost = K.wukong_out_fwd(t["fmb"], base, t["g"], t["b"], f)
    r_y, r_ost = W.out_fwd(_np(t["fmb"]), _np(base), _np(t["g"]), _np(t["b"]), f)
    _close(_np(y), r_y, 1e-5, "y")
    _close(_np(ost), r_ost, 1e-5, "out stats")
    dx, dwf, dgf, dbf, dwl, dwr = K.wukong_mix_bwd(t["x"], t["wf"], t["gf"], t["wl"], t["wr"], f, st, t["d_ln_f"], t["dy"])
    r = W.mix_bwd(_np(t["x"]), _np(t["wf"]), _np(t["gf"]), _np(t["wl"]), _np(t["wr"]), f, _np(t["d_ln_f"]), _np(t["dy"]))
    for got, want, what in zip((dx, dwf, dgf, dbf, dwl, dwr), r, ("dx", "dw_fmb", "dgamma", "dbeta", "dw_lcb", "dw_res")):
        if want is None:
            assert got is None
            continue
        _close(_np(got), want, 2e-5, what)
    d_fmb, d_base, dg, db = K.wukong_out_bwd(t["fmb"], base, t["g"], f, ost, t["dy"])
    r = W.out_bwd(_np(t["fmb"]), _np(base), _np(t["g"]), f, _np(t["dy"]))
    for got, want, what in zip((d_fmb, d_base, dg, db), r, ("d_fmb", "d_base", "dgamma", "dbeta")):
        _close(_np(got), want, 2e-5, what)


def _pipe(seed=7, **kw):
    from torcheasyrec_b200.engine import Pipeline

    return Pipeline("wukong_criteo", device=DEV, max_rows=2000, seed=seed, **kw)


def _copy_state(dst, src):
    dst.model.load_state_dict(src.model.state_dict())
    for ca, cb in zip(src.model.sparse_collections(), dst.model.sparse_collections()):
        cb.weights.data.copy_(ca.weights.data)
        if not ca.layout.interleaved and ca.opt_state is not None:
            cb.opt_state.copy_(ca.opt_state)
    dst.dense_optimizer.load_state_dict(copy.deepcopy(src.dense_optimizer.state_dict()))


def _grads(p, batch):
    """Logits, loss and every dense parameter's gradient of one forward/backward (the sparse update runs as usual)."""
    p.dense_optimizer.zero_grad(set_to_none=True)
    total, (_, preds, _) = p.train_wrapper(batch)
    total.backward()
    torch.cuda.synchronize()
    return preds["logits"].clone(), total.detach().clone(), {
        k: v.grad.detach().clone() for k, v in p.model.named_parameters() if v.grad is not None}


def test_fused_model_matches_torch_formulation(monkeypatch):
    from torcheasyrec_b200 import functional as Fn

    a = _pipe()
    b = _pipe()
    _copy_state(b, a)
    batch = a.synthetic_batch(4096, seed=3).to(DEV)
    la, lossa, ga = _grads(a, batch)
    with monkeypatch.context() as mp:
        mp.setattr(Fn, "wukong_usable", lambda *args, **kw: False)
        lb, lossb, gb = _grads(b, batch)
    _close(_np(la), _np(lb), 1e-5, "logits")
    _close(_np(lossa), _np(lossb), 1e-5, "loss")
    assert ga.keys() == gb.keys()
    assert any("_wukong_layers.0.fmb.weight" in k for k in ga)
    for k in ga:
        _close(_np(ga[k]), _np(gb[k]), 1e-4, k)
    # three Adagrad (sparse) / Adam (dense) steps on each path
    a2, b2 = _pipe(seed=9), _pipe(seed=9)
    _copy_state(b2, a2)
    batches = [a2.synthetic_batch(4096, seed=20 + i).to(DEV) for i in range(3)]
    la_ = [float(a2.eager_step(bt)) for bt in batches]
    with monkeypatch.context() as mp:
        mp.setattr(Fn, "wukong_usable", lambda *args, **kw: False)
        lb_ = [float(b2.eager_step(bt)) for bt in batches]
    np.testing.assert_allclose(la_, lb_, rtol=1e-5)
    lr = max(g["lr"] for g in a2.dense_optimizer.param_groups)
    for (k, pa), pb in zip(a2.model.named_parameters(), b2.model.parameters()):
        # Adam moves each weight by about lr per step whatever its gradient's size: a gradient near zero may take
        # either sign on the two paths, so the bound is relative to the parameter's scale plus a few lr
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


def test_fp32_step_launches_the_fused_kernels_and_no_bmm_or_layer_norm():
    from torch.profiler import ProfilerActivity, profile

    p = _pipe(seed=15)
    batch = p.synthetic_batch(4096, seed=1).to(DEV)
    p.eager_step(batch)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        p.eager_step(batch)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert any("mix_fwd_kernel" in n for n in names) and any("mix_bwd_kernel" in n for n in names)
    assert any("out_fwd_kernel" in n for n in names) and any("out_bwd_kernel" in n for n in names)
    low = [n.lower() for n in names]
    assert not any("layer_norm" in n or "layernorm" in n for n in low), sorted(set(names))
    assert not any("bmm" in n for n in low), sorted(set(names))


def test_bf16_autocast_takes_the_torch_formulation_and_trains(monkeypatch):
    from torcheasyrec_b200 import kernels

    calls = []
    for nm in ("wukong_mix_fwd", "wukong_out_fwd"):
        orig = getattr(kernels.CudaKernels, nm)
        monkeypatch.setattr(kernels.CudaKernels, nm, lambda self, *a, _o=orig, _n=nm, **kw: calls.append(_n) or _o(self, *a, **kw))
    p = _pipe(seed=17, edits={"train_config.mixed_precision": "BF16"})
    batch = p.synthetic_batch(2048, seed=2).to(DEV)
    losses = [float(p.eager_step(batch)) for _ in range(3)]
    assert calls == []
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses


def test_shapes_outside_the_cover_fall_back():
    """d = 12 (not in {4, 8, 16, 32}) and k = 40 take the torch formulation on the GPU, equal to the CPU module."""
    from torcheasyrec_b200.rank_models import WuKongLayer

    for d, n, l, f, k in [(12, 6, 3, 4, 2), (16, 6, 3, 4, 40)]:
        torch.manual_seed(0)
        layer = WuKongLayer(d, n, l, f, k, {"hidden_units": [8]})
        x = torch.randn(5, n, d)
        assert not layer.to(DEV).fused_usable(x.to(DEV))
        y_gpu = layer(x.to(DEV))
        y_cpu = layer.cpu()(x)
        np.testing.assert_allclose(y_gpu.detach().cpu().numpy(), y_cpu.detach().numpy(), rtol=1e-4, atol=1e-5)
