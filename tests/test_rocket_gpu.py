"""RocketLaunching's fused head (csrc/tzk_rocket.cuh) on the H100: both kernels against float64 over batch sizes,
class counts and similarity modes, bit-identical reruns, graph replay equal to eager, the fused path against
functional.torch_rocket_head, the example trained as captured steps and evaluated, and the torch path taken under BF16
autocast and outside the cover."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from test_rocket_cpu import ref_head  # noqa: E402

from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200.kernels import default_kernels  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
REF_EXAMPLE = os.path.join(HERE, "golden", "ref_examples", "rocket_launching_criteo.config")


def _case(B, C, seed, widths=(64, 32), Hl=32, Hb=32):
    g = torch.Generator().manual_seed(seed)
    def r(*s, scale=1.0):
        return (torch.randn(*s, generator=g) * scale).float().to(DEV)
    heads = [(torch.relu(r(B, Hl)), r(C, Hl, scale=0.3), r(C, scale=0.1)),
             (torch.relu(r(B, Hb)), r(C, Hb, scale=0.3), r(C, scale=0.1))]
    pairs = [(torch.relu(r(B, d)), r(B, d).abs()) for d in widths]
    if B > 0:
        pairs[0][0][0].zero_()
    labels = torch.randint(0, C, (B,), generator=g).float().to(DEV)
    return heads, labels, pairs


def _run(heads, labels, eps, pairs, sim, dl):
    K = default_kernels()
    logits, probs, losses, stats = K.rocket_head_fwd(heads, labels, eps, pairs, sim)
    if not torch.is_tensor(dl):
        dl = torch.tensor(dl, dtype=torch.float32, device=DEV)
    dhs, dls, dps = K.rocket_head_bwd(heads, logits, probs, labels, eps, pairs, sim, stats, losses, dl)
    return logits, probs, losses, dhs, dls, dps


def _np(t):
    return t.detach().double().cpu().numpy()


def _close(got, want, r, name):
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(got, want, rtol=r, atol=r * max(1.0, np.abs(want).max()), err_msg=name)


@pytest.mark.parametrize("sim", [Fn.ROCKET_COSINE, Fn.ROCKET_EUCLID])
@pytest.mark.parametrize("C", [2, 3, 8])
@pytest.mark.parametrize("B", [1, 7, 8193, 65536])
def test_kernels_match_float64(B, C, sim):
    heads, labels, pairs = _case(B, C, seed=B + C)
    dl = [0.7, 1.3, 0.9, 1.1, 0.5]
    logits, probs, losses, dhs, dls, dps = _run(heads, labels, 0.1, pairs, sim, dl)
    z, p, rl, rdh, rdl, rdp = ref_head([tuple(_np(t) for t in h) for h in heads], _np(labels), 0.1,
                                       [(_np(l), _np(o)) for l, o in pairs], sim, dl)
    r = 2e-5
    for e in range(2):
        _close(_np(logits[e]), z[e], 1e-5, f"logits{e}")
        _close(_np(probs[e]), p[e], 1e-5, f"probs{e}")
        _close(_np(dhs[e]), rdh[e], 1e-5, f"dh{e}")
        _close(_np(dps[e][0]), rdp[e][0], r, f"dW{e}")
        _close(_np(dps[e][1]), rdp[e][1], r, f"db{e}")
    _close(_np(losses), rl, r, "losses")
    for k in range(2):
        _close(_np(dls[k]), rdl[k], 1e-5, f"dlight{k}")


def test_reruns_and_graph_replay_bit_identical():
    heads, labels, pairs = _case(65536, 2, seed=3)
    dl = torch.ones(5, device=DEV)
    a = _run(heads, labels, 0.0, pairs, Fn.ROCKET_COSINE, dl)
    b = _run(heads, labels, 0.0, pairs, Fn.ROCKET_COSINE, dl)
    flat = torch.utils._pytree.tree_leaves
    assert all(torch.equal(x, y) for x, y in zip(flat(a), flat(b)))
    _run(heads, labels, 0.0, pairs, Fn.ROCKET_COSINE, dl)           # warm the workspaces on this stream
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _run(heads, labels, 0.0, pairs, Fn.ROCKET_COSINE, dl)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c = _run(heads, labels, 0.0, pairs, Fn.ROCKET_COSINE, dl)
    g.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(flat(a), flat(c)))


def _pipe(seed, **kw):
    from torcheasyrec_b200.engine import Pipeline

    return Pipeline(REF_EXAMPLE, device=DEV, max_rows=2000, seed=seed, **kw)


def test_fused_model_matches_torch_head(monkeypatch):
    """The example's model on one batch: the fused head against torch_rocket_head (the predicate patched to refuse),
    with every other layer the same: predictions, losses and dense gradients."""
    from torcheasyrec_b200.embedding_modules import SparseOptimizerSpec
    from torcheasyrec_b200.kernels import OPT_SGD

    p = _pipe(seed=5)
    batch = p.synthetic_batch(8192, seed=1).to(DEV)
    model = p.model
    model.set_sparse_optimizer(SparseOptimizerSpec(kind=OPT_SGD, lr=0.0))   # both passes see the same embeddings
    model.train()
    outs = []
    for fused in (True, False):
        if not fused:
            monkeypatch.setattr(Fn, "rocket_head_usable", lambda *a, **k: False)
        model.zero_grad(set_to_none=True)
        preds = model.predict(batch)
        losses = model.loss(preds, batch)
        torch.stack(list(losses.values())).sum().backward()
        outs.append((preds, losses, {n: p_.grad.clone() for n, p_ in model.named_parameters()
                                     if p_.grad is not None and "embedding" not in n}))
    (pf, lf, gf), (pt, lt, gt) = outs
    assert list(pf) == list(pt) and list(lf) == list(lt) and set(gf) == set(gt)
    for k in lt:
        assert abs(float(lf[k]) - float(lt[k])) <= 1e-5 * max(1.0, abs(float(lt[k]))), k
    for k in pt:
        _close(_np(pf[k]), _np(pt[k]), 1e-5, k)
    for k in gt:
        _close(_np(gf[k]), _np(gt[k]), 1e-4, k)


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
    assert set(m) == {"auc_booster", "auc_light", "softmax_cross_entropy_booster", "softmax_cross_entropy_light"}
    assert 0.0 < m["auc_light"] < 1.0 and np.isfinite(m["softmax_cross_entropy_light"])
    assert m["auc_booster"] == 0.0 and np.isnan(m["softmax_cross_entropy_booster"])


def _copy_state(dst, src):
    import copy

    dst.model.load_state_dict(src.model.state_dict())
    for ca, cb in zip(src.model.sparse_collections(), dst.model.sparse_collections()):
        cb.weights.data.copy_(ca.weights.data)
        if not ca.layout.interleaved and ca.opt_state is not None:
            cb.opt_state.copy_(ca.opt_state)
    dst.dense_optimizer.load_state_dict(copy.deepcopy(src.dense_optimizer.state_dict()))


def test_graph_replay_equals_eager_step():
    """Captured steps of the example equal eager steps bit for bit: losses and every dense parameter."""
    from torcheasyrec_b200.engine import GraphedTrainStep

    a = _pipe(seed=13)
    batches = [a.synthetic_batch(4096, seed=40 + i) for i in range(3)]
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


def test_bf16_autocast_and_uncovered_shapes_take_torch_path():
    heads, labels, pairs = _case(64, 2, seed=1)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        assert not Fn.rocket_head_usable([heads[0][0]], 2, [64])
    assert Fn.rocket_head_usable([heads[0][0], heads[1][0]], 2, [64, 32])
    assert not Fn.rocket_head_usable([heads[0][0][:, :30]], 2, [])            # width not a multiple of 4
    assert not Fn.rocket_head_usable([heads[0][0]], 9, [])                     # more than 8 classes
    assert not Fn.rocket_head_usable([heads[0][0]], 2, [32] * 9)               # more than 8 pairs
    p = _pipe(seed=7, edits={"train_config.mixed_precision": "BF16"})
    batch = p.synthetic_batch(2048, seed=3).to(DEV)
    losses = [float(p.eager_step(batch)) for _ in range(4)]
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses


def test_backward_shared_memory_just_under_48k():
    """C = 8 and hidden widths 736: the backward's dW / db accumulator is 47168 B of dynamic shared memory, which with
    its 2 KB of static shared memory needs the opt-in; against float64 like every other shape."""
    heads, labels, pairs = _case(3000, 8, seed=11, widths=(64,), Hl=736, Hb=736)
    dl = [0.7, 1.3, 0.9, 1.1]
    logits, probs, losses, dhs, dls, dps = _run(heads, labels, 0.0, pairs, Fn.ROCKET_COSINE, dl)
    z, p, rl, rdh, rdl, rdp = ref_head([tuple(_np(t) for t in h) for h in heads], _np(labels), 0.0,
                                       [(_np(l), _np(o)) for l, o in pairs], Fn.ROCKET_COSINE, dl)
    _close(_np(losses), rl, 2e-5, "losses")
    for e in range(2):
        _close(_np(dhs[e]), rdh[e], 2e-5, f"dh{e}")
        _close(_np(dps[e][0]), rdp[e][0], 2e-5, f"dW{e}")
        _close(_np(dps[e][1]), rdp[e][1], 2e-5, f"db{e}")
    _close(_np(dls[0]), rdl[0], 2e-5, "dlight")
