"""DCN-v2 on the H100: the three fused cross-network kernels against float64 over the corners of their cover up to
B = 65536 + 7, bit-identical reruns and graph replay, the fused model against the torch path, and the dcn_v2_taobao
example trained as captured steps and evaluated."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import dcn_v2_ref as R  # noqa: E402

from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200.engine import Pipeline  # noqa: E402
from torcheasyrec_b200.kernels import default_kernels  # noqa: E402
from torcheasyrec_b200.rank_models import CrossV2  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _close(got, want, r, name):
    got, want = got.detach().double().cpu().numpy(), want.detach().double().cpu().numpy()
    np.testing.assert_allclose(got, want, rtol=r, atol=r * max(1.0, np.abs(want).max() if want.size else 1.0),
                               err_msg=name)


def _run(x0, wu, wv, bias, dy):
    k = default_kernels()
    f = lambda t: t.float().to(DEV).contiguous()  # noqa: E731
    x0, wu, wv, bias, dy = (f(t) for t in (x0, wu, wv, bias, dy))
    y, v = k.dcn_v2_fwd(x0, wu, wv, bias)
    dx0, dwu, dwv, db = k.dcn_v2_bwd(x0, wu, wv, bias, v, dy)
    return y, dx0, dwu, dwv, db


# (B, D, L, r): the cover's corners, the reference's test shapes, the docs example and D = 256 at L = 3
CASES = [(65543, 33, 3, 64), (65536, 128, 2, 32), (65543, 256, 3, 64), (65536, 256, 3, 32), (4103, 512, 8, 64),
         (3001, 512, 1, 1), (777, 1, 1, 1), (1000, 32, 6, 2), (129, 100, 8, 17), (1, 7, 2, 3), (0, 64, 2, 8)]


@pytest.mark.parametrize("B,D,L,r", CASES)
def test_kernels_against_float64(B, D, L, r):
    x0, wu, wv, bias = (t.to(DEV) for t in R.case(B + D, B, D, L, r))
    dy = torch.randn(B, D, dtype=torch.float64, device=DEV, generator=torch.Generator(DEV).manual_seed(1))
    want = R.grads(x0, wu, wv, bias, dy)
    got = _run(x0, wu, wv, bias, dy)
    for name, g, w, tol in zip(("y", "dx0", "d wu", "d wv", "d bias"), got, want, (1e-5, 2e-5, 2e-5, 2e-5, 2e-5)):
        _close(g, w, tol, name)


def test_reruns_and_graph_replay_bit_identical():
    x0, wu, wv, bias = (t.to(DEV) for t in R.case(3, 65536, 256, 3, 32))
    dy = torch.randn(65536, 256, dtype=torch.float64, device=DEV)
    a = _run(x0, wu, wv, bias, dy)
    b = _run(x0, wu, wv, bias, dy)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    f = lambda t: t.float().contiguous()  # noqa: E731
    x0, wu, wv, bias, dy = (f(t) for t in (x0, wu, wv, bias, dy))
    k = default_kernels()

    def body():
        y, v = k.dcn_v2_fwd(x0, wu, wv, bias)
        return (y,) + tuple(k.dcn_v2_bwd(x0, wu, wv, bias, v, dy))

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        body()                                                        # warm the workspaces on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c = body()
    g.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a, c))


def _pipe(seed, **kw):
    return Pipeline("dcn_v2_taobao", device=DEV, max_rows=2000, seed=seed, **kw)


def test_fused_model_matches_torch_path(monkeypatch):
    """dcn_v2_taobao's model on one batch of 4096: the fused cross network against Fn.torch_cross_v2 (the predicate
    patched to refuse) with the same weights: logits and loss to 1e-5, every dense gradient and the group's input
    gradient to 1e-4."""
    from torcheasyrec_b200.embedding_modules import SparseOptimizerSpec
    from torcheasyrec_b200.kernels import OPT_SGD

    p = _pipe(seed=5)
    batch = p.synthetic_batch(4096, seed=1).to(DEV)
    model = p.model
    model.set_sparse_optimizer(SparseOptimizerSpec(kind=OPT_SGD, lr=0.0))
    model.train()
    build, held = model.build_input, {}

    def build_input(b):
        grouped = dict(build(b))
        held["x"] = grouped["features"] = grouped["features"].detach().requires_grad_(True)
        return grouped

    model.build_input = build_input
    outs = []
    for fused in (True, False):
        if not fused:
            monkeypatch.setattr(Fn, "cross_v2_usable", lambda *a, **k: False)
        else:
            x = torch.zeros(8, 128, device=DEV)
            assert Fn.cross_v2_usable(x, model.cross.u_kernels, model.cross.v_kernels)
        model.zero_grad(set_to_none=True)
        preds = model.predict(batch)
        losses = model.loss(preds, batch)
        losses["binary_cross_entropy"].backward()
        outs.append((preds, losses, {n: q.grad.clone() for n, q in model.named_parameters()
                                     if q.grad is not None and "embedding" not in n}, held["x"].grad.clone()))
    (pf, lf, gf, xf), (pt, lt, gt, xt) = outs
    assert set(gf) == set(gt) and any(n.startswith("cross.") for n in gf)
    for k in pt:
        _close(pf[k], pt[k], 1e-5, k)
    for k in lt:
        _close(lf[k], lt[k], 1e-5, k)
    for k in gt:
        _close(gf[k], gt[k], 1e-4, k)
    _close(xf, xt, 1e-4, "d features")


def test_example_trains_captured_and_evaluates():
    from torcheasyrec_b200.engine import GraphedTrainStep

    p = _pipe(seed=21)
    batch = p.synthetic_batch(8192, seed=2)
    step = GraphedTrainStep(p, batch, warmup=2)
    losses = []
    for _ in range(6):
        step.load(batch.pin_memory())
        losses.append(float(step.replay()))
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
    m = p.evaluate([p.synthetic_batch(4096, seed=s) for s in range(3)])
    assert set(m) == {"auc", "binary_cross_entropy"}
    assert 0.0 < m["auc"] < 1.0 and np.isfinite(m["binary_cross_entropy"])


def test_autocast_tf32_and_uncovered_shapes_take_torch_path():
    cross = CrossV2(128, 2, 32).to(DEV)
    x = torch.randn(64, 128, device=DEV)
    assert Fn.cross_v2_usable(x, cross.u_kernels, cross.v_kernels)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        assert not Fn.cross_v2_usable(x, cross.u_kernels, cross.v_kernels)
        y = cross(x)
        want = Fn.torch_cross_v2(x, cross.u_kernels, cross.v_kernels)
    assert torch.equal(y, want)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        assert not Fn.cross_v2_usable(x, cross.u_kernels, cross.v_kernels)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    wide = CrossV2(520, 1, 8).to(DEV)
    assert not Fn.cross_v2_usable(torch.randn(4, 520, device=DEV), wide.u_kernels, wide.v_kernels)
    deep = CrossV2(64, 9, 8).to(DEV)
    assert not Fn.cross_v2_usable(torch.randn(4, 64, device=DEV), deep.u_kernels, deep.v_kernels)
    rank = CrossV2(64, 2, 65).to(DEV)
    xr = torch.randn(4, 64, device=DEV)
    assert not Fn.cross_v2_usable(xr, rank.u_kernels, rank.v_kernels)
    torch.testing.assert_close(rank(xr), Fn.torch_cross_v2(xr, rank.u_kernels, rank.v_kernels))
