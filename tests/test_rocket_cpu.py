"""RocketLaunching and softmax cross-entropy heads on the CPU: the SOURCE of the fused head kernels
(csrc/tzk_rocket.cuh) run on the host through tests/native/cuda_cpu_shim.h against float64, the model with the fused
path (that host build as its backend) against the torch formulation, the detach semantics, the prediction and loss
keys, two-class heads on DeepFM and DLRM, the refusals, and the reference example trained and evaluated."""
import contextlib
import ctypes
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from metric_oracle_backend import MetricOracleKernels  # noqa: E402

from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200._lib import ROCKET_COSINE, ROCKET_EUCLID, TzkRocketArgs  # noqa: E402
from torcheasyrec_b200.config import parse_text  # noqa: E402
from torcheasyrec_b200.engine import Pipeline  # noqa: E402
from torcheasyrec_b200.example_configs import GENERATORS  # noqa: E402
from torcheasyrec_b200.embedding_modules import SparseOptimizerSpec  # noqa: E402
from torcheasyrec_b200.features import create_features  # noqa: E402
from torcheasyrec_b200.kernels import OPT_SGD  # noqa: E402
from torcheasyrec_b200.metrics import BinnedAUC, MeanLoss  # noqa: E402
from torcheasyrec_b200.rank_models import MLP, create_model  # noqa: E402

NATIVE = os.path.join(HERE, "native")
REF_EXAMPLE = os.path.join(HERE, "golden", "ref_examples", "rocket_launching_criteo.config")


# ---- float64 statement of the head ---------------------------------------------------------------------------------
def ref_head(heads, labels, eps, pairs, sim, dlosses=None):
    """heads [(h, w, b)] float64; -> (logits, probs, losses [3 + n_pairs], and with dlosses: dh per head, dlight per
    pair, (dW, db) per head), written out from the definitions (torch's F.normalize / cross_entropy / mse_loss)."""
    B = heads[0][0].shape[0]
    C = heads[0][1].shape[0]
    z = [h @ w.T + b for h, w, b in heads]
    p = [np.exp(x - x.max(1, keepdims=True)) / np.exp(x - x.max(1, keepdims=True)).sum(1, keepdims=True) for x in z]
    q = np.full((B, C), eps / C) + (1 - eps) * np.eye(C)[labels.astype(np.int64)]
    ce = [(-(q * np.log(pp)).sum(1)).mean() for pp in p]
    losses = [ce[0], ce[1] if len(heads) > 1 else 0.0, ((z[0] - z[1]) ** 2).mean() if len(heads) > 1 else 0.0]
    cos = []
    for l, o in pairs:
        nl, nb = np.linalg.norm(l, axis=1), np.linalg.norm(o, axis=1)
        cl, cb = np.maximum(nl, 1e-12), np.maximum(nb, 1e-12)
        dot = (l * o).sum(1)
        if sim == ROCKET_COSINE:
            losses.append(-0.1 * (dot / (cb * cl)).mean())
        else:
            losses.append(np.sqrt(((o - l) ** 2).sum()))
        cos.append((nl, cl, cb, dot))
    if dlosses is None:
        return z, p, np.array(losses)
    dz = [dlosses[e] / B * (p[e] - q) for e in range(len(heads))]
    if len(heads) > 1:
        dz[0] = dz[0] + dlosses[2] * 2.0 / (B * C) * (z[0] - z[1])
    dhs = [d @ w for d, (_, w, _) in zip(dz, heads)]
    dparams = [(d.T @ h, d.sum(0)) for d, (h, _, _) in zip(dz, heads)]
    dls = []
    for k, ((l, o), (nl, cl, cb, dot)) in enumerate(zip(pairs, cos)):
        g = dlosses[3 + k]
        if sim == ROCKET_COSINE:
            beta = np.where(nl >= 1e-12, dot / (cb * cl * cl * np.where(nl > 0, nl, 1.0)), 0.0)
            dls.append(g * -0.1 / B * (o / (cb * cl)[:, None] - beta[:, None] * l))
        else:
            with np.errstate(invalid="ignore", divide="ignore"):
                dls.append(g * (l - o) / losses[3 + k])
    return z, p, np.array(losses), dhs, dls, dparams


# ---- the kernel source on the host ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kern(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("shim") / "librocket_cpu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", NATIVE,
                    "-x", "c++", os.path.join(NATIVE, "rocket_standalone.cu"), "-shared", "-fPIC", "-o", out],
                   check=True)
    L = ctypes.CDLL(out)
    P, I32 = ctypes.c_void_p, ctypes.c_int
    L.rocket_check.argtypes = [P, I32]
    L.rocket_head_fwd.argtypes = [P, I32, P, P]
    L.rocket_head_bwd.argtypes = [P, P, P, I32, P, P]
    return L


class ShimRocket:
    """rocket_head_fwd / _bwd of kernels.CudaKernels on CPU tensors, computed by the host build of the kernel source."""

    def __init__(self, L, grid_fwd=None, grid_bwd=None):
        self.L, self.grid_fwd, self.grid_bwd, self.calls = L, grid_fwd, grid_bwd, 0

    @staticmethod
    def _args(heads, logits, probs, labels, eps, pairs, sim, stats, dhs=None, dls=None):
        a = TzkRocketArgs()
        a.B, a.C = heads[0][0].shape[0], heads[0][1].shape[0]
        a.has_booster, a.n_pairs, a.sim, a.eps = len(heads) - 1, len(pairs), sim, eps
        a.labels = None if labels is None else labels.data_ptr()
        a.pair_stats = None if stats is None else stats.data_ptr()
        for e, (h, w, b) in enumerate(heads):
            g = a.head[e]
            g.h, g.w, g.b, g.H = h.data_ptr(), w.data_ptr(), b.data_ptr(), h.shape[1]
            g.logits, g.probs = logits[e].data_ptr(), probs[e].data_ptr()
            if dhs is not None:
                g.dh = dhs[e].data_ptr()
        for k, (l, o) in enumerate(pairs):
            p = a.pair[k]
            p.light, p.booster, p.d = l.data_ptr(), o.data_ptr(), l.shape[1]
            if dls is not None:
                p.dlight = dls[k].data_ptr()
        return a

    def _grid(self, B, per, fixed):
        return fixed or max(1, min(-(-B // per), 4))

    def rocket_head_fwd(self, heads, labels, eps, pairs, sim):
        self.calls += 1
        heads = [tuple(t.detach().contiguous() for t in h) for h in heads]
        pairs = [(l.detach().contiguous(), o.detach().contiguous()) for l, o in pairs]
        B, C = heads[0][0].shape[0], heads[0][1].shape[0]
        logits = [torch.empty(B, C) for _ in heads]
        probs = [torch.empty(B, C) for _ in heads]
        stats = torch.empty(len(pairs), B, 2) if pairs else None
        grid = self._grid(B, 8, self.grid_fwd)
        losses = partials = None
        if labels is not None:
            losses = torch.empty(3 + len(pairs))
            partials = torch.empty(grid, 3 + len(pairs))
        a = self._args(heads, logits, probs, labels, eps, pairs, sim, stats)
        assert self.L.rocket_head_fwd(ctypes.byref(a), grid, None if partials is None else partials.data_ptr(),
                                      None if losses is None else losses.data_ptr()) == 0
        return logits, probs, losses, stats

    def rocket_head_bwd(self, heads, logits, probs, labels, eps, pairs, sim, stats, losses, dlosses):
        self.calls += 1
        heads = [tuple(t.detach().contiguous() for t in h) for h in heads]
        pairs = [(l.detach().contiguous(), o.detach().contiguous()) for l, o in pairs]
        B, C = heads[0][0].shape[0], heads[0][1].shape[0]
        dhs = [torch.empty_like(h) for h, _, _ in heads]
        dls = [torch.empty_like(l) for l, _ in pairs]
        Pn = sum(C * (h.shape[1] + 1) for h, _, _ in heads)
        grid = self._grid(B, 32, self.grid_bwd)
        partials, dparams = torch.empty(grid, Pn), torch.empty(Pn)
        a = self._args(heads, logits, probs, labels, eps, pairs, sim, stats, dhs, dls)
        assert self.L.rocket_head_bwd(ctypes.byref(a), dlosses.data_ptr(), losses.data_ptr(), grid,
                                      partials.data_ptr(), dparams.data_ptr()) == 0
        out, o = [], 0
        for h, _, _ in heads:
            n = C * h.shape[1]
            out.append((dparams[o:o + n].view(C, h.shape[1]), dparams[o + n:o + n + C]))
            o += n + C
        return dhs, dls, out


class ShimBackend(MetricOracleKernels):
    """The CPU checker backend with the rocket head computed by the host build of its kernel source."""

    def __init__(self, L):
        super().__init__()
        self._rocket = ShimRocket(L)
        self.rocket_head_fwd = self._rocket.rocket_head_fwd
        self.rocket_head_bwd = self._rocket.rocket_head_bwd

    @property
    def rocket_calls(self):
        return self._rocket.calls


def _case(seed, B, C, Hl, Hb, widths, zero_light_row=False, booster=True):
    g = torch.Generator().manual_seed(seed)
    def r(*s, scale=1.0):
        return (torch.randn(*s, generator=g) * scale).float()
    heads = [(torch.relu(r(B, Hl)), r(C, Hl, scale=0.3), r(C, scale=0.1))]
    if booster:
        heads.append((torch.relu(r(B, Hb)), r(C, Hb, scale=0.3), r(C, scale=0.1)))
    pairs = [(torch.relu(r(B, d)), r(B, d).abs()) for d in widths]
    if zero_light_row and B > 0:
        for l, _ in pairs:
            l[0].zero_()
    labels = torch.randint(0, C, (B,), generator=g).float()
    return heads, labels, pairs


def _np(t):
    return t.detach().double().numpy()


def _run_shim(L, heads, labels, eps, pairs, sim, dl, grid_fwd, grid_bwd):
    s = ShimRocket(L, grid_fwd, grid_bwd)
    logits, probs, losses, stats = s.rocket_head_fwd(heads, labels, eps, pairs, sim)
    dhs, dls, dps = s.rocket_head_bwd(heads, logits, probs, labels, eps, pairs, sim, stats, losses,
                                      torch.tensor(dl, dtype=torch.float32))
    return logits, probs, losses, dhs, dls, dps


def _close(got, want, r, name):
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(np.asarray(got, np.float64), want, rtol=r,
                               atol=r * max(1.0, np.abs(want).max() if want.size else 1.0), err_msg=name)


@pytest.mark.parametrize("sim", [ROCKET_COSINE, ROCKET_EUCLID])
@pytest.mark.parametrize("B,C,grids", [(1, 2, (1, 1)), (7, 3, (1, 1)), (7, 8, (3, 2)), (300, 2, (5, 3)),
                                       (300, 5, (40, 10))])
def test_kernel_source_against_float64(kern, B, C, grids, sim):
    """Both heads, three pairs (widths 4, 32 and 64, one light row all zero), eps 0.1, every output of both kernels
    against float64; multi-CTA grids, grids larger than the work, and a CTA with a partial tile."""
    heads, labels, pairs = _case(B * 10 + C, B, C, 32, 64, [4, 32, 64], zero_light_row=True)
    dl = [0.7, 1.3, 0.9, 1.1, 0.5, 2.0]
    logits, probs, losses, dhs, dls, dps = _run_shim(kern, heads, labels, 0.1, pairs, sim, dl, *grids)
    z, p, rl, rdh, rdl, rdp = ref_head([tuple(_np(t) for t in h) for h in heads], _np(labels), 0.1,
                                       [(_np(l), _np(o)) for l, o in pairs], sim, dl)
    for e in range(2):
        _close(_np(logits[e]), z[e], 1e-5, f"logits{e}")
        _close(_np(probs[e]), p[e], 1e-5, f"probs{e}")
        _close(_np(dhs[e]), rdh[e], 1e-5, f"dh{e}")
        _close(_np(dps[e][0]), rdp[e][0], 1e-5, f"dW{e}")
        _close(_np(dps[e][1]), rdp[e][1], 1e-5, f"db{e}")
    _close(_np(losses), rl, 1e-5, "losses")
    for k in range(3):
        _close(_np(dls[k]), rdl[k], 1e-5, f"dlight{k}")
    if sim == ROCKET_COSINE:                     # the all-zero light row: torch's gradient at the clamp
        np.testing.assert_allclose(_np(dls[0][0]), rdl[0][0], rtol=1e-5)
        assert np.abs(_np(dls[0][0])).max() > 1e6


def test_kernel_source_reruns_bit_identical(kern):
    heads, labels, pairs = _case(5, 257, 3, 32, 32, [32, 8])
    a = _run_shim(kern, heads, labels, 0.0, pairs, ROCKET_COSINE, [1.0] * 5, 6, 4)
    b = _run_shim(kern, heads, labels, 0.0, pairs, ROCKET_COSINE, [1.0] * 5, 6, 4)
    for x, y in zip(torch.utils._pytree.tree_leaves(a), torch.utils._pytree.tree_leaves(b)):
        assert torch.equal(x, y)


def test_kernel_source_empty_batch(kern):
    """B = 0: NaN means (torch's mean over no samples), EUCLID 0, zero parameter gradients."""
    heads, labels, pairs = _case(1, 0, 2, 8, 8, [8])
    for sim, want in ((ROCKET_COSINE, True), (ROCKET_EUCLID, False)):
        logits, probs, losses, dhs, dls, dps = _run_shim(kern, heads, labels, 0.0, pairs, sim, [1.0] * 4, 1, 1)
        assert torch.isnan(losses[:3]).all()
        assert bool(torch.isnan(losses[3])) == want and (want or float(losses[3]) == 0.0)
        assert all(float(t.abs().sum()) == 0 for dw, db in dps for t in (dw, db))


def test_kernel_source_euclid_zero_distance_nan(kern):
    """EUCLID with light == booster: loss 0 and a NaN gradient, as torch's autograd of sqrt at 0."""
    heads, labels, pairs = _case(2, 5, 2, 8, 8, [8])
    pairs = [(pairs[0][0], pairs[0][0].clone())]
    _, _, losses, _, dls, _ = _run_shim(kern, heads, labels, 0.0, pairs, ROCKET_EUCLID, [1.0] * 4, 1, 1)
    assert float(losses[3]) == 0.0 and torch.isnan(dls[0]).all()
    l = pairs[0][0].clone().requires_grad_(True)
    Fn.feature_based_sim(l, pairs[0][1], ROCKET_EUCLID).backward()
    assert torch.isnan(l.grad).all()


def test_kernel_source_eval_light_only(kern):
    """Eval: the light head only, no labels -> logits and probs, no losses."""
    heads, labels, _ = _case(3, 9, 4, 16, 16, [], booster=False)
    s = ShimRocket(kern)
    logits, probs, losses, stats = s.rocket_head_fwd(heads, None, 0.0, [], ROCKET_COSINE)
    z, p, _ = ref_head([tuple(_np(t) for t in h) for h in heads], _np(labels), 0.0, [], ROCKET_COSINE)
    _close(_np(logits[0]), z[0], 1e-5, "logits")
    _close(_np(probs[0]), p[0], 1e-5, "probs")
    assert losses is None and stats is None


def test_kernel_source_refuses_outside_cover(kern):
    heads, labels, pairs = _case(4, 4, 2, 8, 8, [8])
    s = ShimRocket(kern)
    bad = [(heads[0][0][:, :6].contiguous(), heads[0][1][:, :6].contiguous(), heads[0][2]), heads[1]]
    a = s._args(bad, [torch.empty(4, 2)] * 2, [torch.empty(4, 2)] * 2, labels, 0.0, pairs, 0, torch.empty(1, 4, 2))
    assert kern.rocket_check(ctypes.byref(a), 0) == 1                  # H = 6 is not a multiple of 4
    a = s._args(heads, [torch.empty(4, 2)] * 2, [torch.empty(4, 2)] * 2, None, 0.0, pairs, 0, torch.empty(1, 4, 2))
    assert kern.rocket_check(ctypes.byref(a), 0) == 1                  # pairs without labels (B > 0)


# ---- MLP hidden layers ---------------------------------------------------------------------------------------------
def test_mlp_return_hidden_layer_feature():
    torch.manual_seed(0)
    m = MLP(8, [6, 4], return_hidden_layer_feature=True)
    x = torch.randn(3, 8)
    out = m(x)
    assert list(out) == ["hidden_layer0", "hidden_layer1", "hidden_layer_end"]
    assert out["hidden_layer_end"] is out["hidden_layer1"]
    m.return_hidden_layer_feature = False
    assert torch.equal(m(x), out["hidden_layer_end"])


# ---- the model -----------------------------------------------------------------------------------------------------
ROCKET_SMALL = """
feature_configs { raw_feature { feature_name: "int_0" } }
feature_configs { raw_feature { feature_name: "int_1" } }
feature_configs { raw_feature { feature_name: "int_2" } }
feature_configs { raw_feature { feature_name: "int_3" } }
feature_configs { id_feature { feature_name: "cat_0" num_buckets: 50 embedding_dim: 8 } }
feature_configs { id_feature { feature_name: "cat_1" num_buckets: 50 embedding_dim: 8 } }
model_config {
  feature_groups { group_name: "deep" feature_names: ["int_0", "int_1", "int_2", "int_3", "cat_0", "cat_1"]
                   group_type: DEEP }
  rocket_launching {
    %SHARE%
    booster_mlp { hidden_units: [32, 16, 8] }
    light_mlp { hidden_units: [16, 16, 8] }
    feature_based_distillation: %DISTILL%
    feature_distillation_function: %SIM%
  }
  num_class: %C%
  metrics { auc {} }
  losses { softmax_cross_entropy { label_smoothing: %EPS% } }
}
"""


def _rocket_cfg(share=False, distill=True, sim="COSINE", C=2, eps=0.0):
    return (ROCKET_SMALL.replace("%SHARE%", "share_mlp { hidden_units: [24] }" if share else "")
            .replace("%DISTILL%", "true" if distill else "false").replace("%SIM%", sim).replace("%C%", str(C))
            .replace("%EPS%", str(eps)))


def _model(text, seed=0):
    cfg = parse_text(text)
    feats = create_features(list(cfg.feature_configs))
    torch.manual_seed(seed)
    m = create_model(cfg.model_config, feats, ["label"], device=torch.device("cpu"))
    m.set_sparse_optimizer(SparseOptimizerSpec(kind=OPT_SGD, lr=0.0))        # tables stay put across steps
    return m, feats


def _batch(feats, B, C, seed):
    from torcheasyrec_b200.batch import synthetic_batch

    b = synthetic_batch(feats, B, ["label"], seed=seed)
    g = torch.Generator().manual_seed(seed)
    b.labels["label"] = torch.randint(0, C, (B,), generator=g).float()
    return b


def _step(model, batch, backend=None):
    """backend None: the checker backend without the rocket kernels, so the heads take the torch formulation."""
    model.zero_grad(set_to_none=True)
    with Fn.use_backend(backend or MetricOracleKernels()):
        preds = model.predict(batch)
        losses = model.loss(preds, batch)
        torch.stack(list(losses.values())).sum().backward()
    grads = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    return preds, losses, grads


MODEL_CASES = {
    "example_cosine": dict(),
    "share_mlp": dict(share=True),
    "distill_off": dict(distill=False),
    "euclid": dict(sim="EUCLID"),
    "inner_product": dict(sim="INNER_PRODUCT"),
    "three_class_eps": dict(C=3, eps=0.1),
}


@pytest.mark.parametrize("case", list(MODEL_CASES))
def test_model_fused_matches_torch(kern, case):
    """The fused head (host build of the kernels) against the reference's torch ops on the same model and batch:
    predictions, every loss and every parameter gradient.  Light layers 0 and 1 (both 16 wide) map to booster layer 1;
    distillation off uses light widths that match no booster layer (the reference needs that in training)."""
    kw = MODEL_CASES[case]
    text = _rocket_cfg(**kw)
    if case == "distill_off":
        text = text.replace("light_mlp { hidden_units: [16, 16, 8] }", "light_mlp { hidden_units: [12, 20] }")
    model, feats = _model(text)
    model.train()
    batch = _batch(feats, 37, kw.get("C", 2), seed=3)
    if case != "distill_off":
        assert model.mlp_index_dict == {0: 1, 1: 1, 2: 2}
    p0, l0, g0 = _step(model, batch)
    be = ShimBackend(kern)
    p1, l1, g1 = _step(model, batch, be)
    assert be.rocket_calls == 2
    assert list(p0) == list(p1) and list(l0) == list(l1)
    for k in p0:
        _close(_np(p1[k]), _np(p0[k]), 2e-5, k)
    for k in l0:
        _close(_np(l1[k]), _np(l0[k]), 2e-5, k)
    assert set(g0) == set(g1)
    for k in g0:
        _close(_np(g1[k]), _np(g0[k]), 5e-5, k)


def test_prediction_and_loss_keys():
    model, feats = _model(_rocket_cfg())
    batch = _batch(feats, 16, 2, seed=1)
    model.train()
    be = MetricOracleKernels()
    with Fn.use_backend(be):
        preds = model.predict(batch)
    assert list(preds) == ["logits_light", "probs_light", "probs1_light", "logits_booster", "probs_booster",
                           "probs1_booster", "light_0", "booster_1", "light_1", "light_2", "booster_2"]
    assert list(model.loss(preds, batch)) == ["softmax_cross_entropy_booster", "softmax_cross_entropy_light",
                                              "similarity_0_1", "similarity_1_1", "similarity_2_2", "hint_l2_loss"]
    model.eval()
    with Fn.use_backend(be), torch.no_grad():
        preds = model.predict(batch)
        assert list(preds) == ["logits_light", "probs_light", "probs1_light"]
        assert list(model.loss(preds, batch)) == ["softmax_cross_entropy_light"]
    sd = list(model.state_dict())
    assert [k.split(".")[0] for k in sd if not k.startswith("embedding_group")] == \
        ["booster_mlp"] * 6 + ["booster_linear"] * 2 + ["light_mlp"] * 6 + ["light_linear"] * 2


def test_light_losses_leave_embeddings_and_share_mlp_alone(kern):
    """The light net reads share_mlp's output detached: its losses put no gradient on share_mlp or the embeddings."""
    model, feats = _model(_rocket_cfg(share=True))
    model.train()
    batch = _batch(feats, 20, 2, seed=2)
    for be in (MetricOracleKernels(), ShimBackend(kern)):
        model.zero_grad(set_to_none=True)
        with Fn.use_backend(be):
            preds = model.predict(batch)
            losses = model.loss(preds, batch)
            light = losses["softmax_cross_entropy_light"] + losses["hint_l2_loss"] + sum(
                v for k, v in losses.items() if k.startswith("similarity"))
            light.backward()
        for n, p in model.named_parameters():
            touched = p.grad is not None and bool(p.grad.abs().sum() > 0)
            assert touched == n.startswith(("light_mlp", "light_linear")), n


def test_refusals():
    with pytest.raises(NotImplementedError, match="softmax_cross_entropy only"):
        _model(_rocket_cfg().replace("softmax_cross_entropy { label_smoothing: 0.0 }", "binary_cross_entropy {}"))
    model, feats = _model(_rocket_cfg(C=3))
    with pytest.raises(ValueError, match="num_class must be at most 2"):
        model.init_metric(device=torch.device("cpu"))
    model, feats = _model(_rocket_cfg(distill=False))
    model.train()
    with pytest.raises(TypeError, match="feature_based_distillation"), Fn.use_backend(MetricOracleKernels()):
        model.predict(_batch(feats, 4, 2, seed=0))


def test_metrics_booster_reported_from_empty_state():
    """Evaluation updates only the light head; the booster's auc and loss mean are reported from their empty state:
    metrics.py gives 0 for an empty binned AUC and NaN for an empty loss mean."""
    model, feats = _model(_rocket_cfg())
    model.init_metric(device=torch.device("cpu"))
    assert list(model._metric_modules) == ["auc_booster", "softmax_cross_entropy_booster", "auc_light",
                                           "softmax_cross_entropy_light"]
    model.eval()
    batch = _batch(feats, 32, 2, seed=4)
    be = MetricOracleKernels()
    with Fn.use_backend(be), torch.no_grad():
        preds = model.predict(batch)
        model.update_metric(preds, batch, model.loss(preds, batch))
        got = model.compute_metric()
    assert float(BinnedAUC(200, torch.device("cpu")).compute()) == float(got["auc_booster"]) == 0.0
    assert np.isnan(float(MeanLoss(torch.device("cpu")).compute())) and np.isnan(float(
        got["softmax_cross_entropy_booster"]))
    assert 0.0 < float(got["auc_light"]) < 1.0 and np.isfinite(float(got["softmax_cross_entropy_light"]))


# ---- softmax cross-entropy heads on other single-task models -------------------------------------------------------
@pytest.mark.parametrize("name", ["deepfm_criteo", "dlrm_criteo"])
def test_two_class_softmax_heads(name):
    text = GENERATORS[name]().replace("binary_cross_entropy {}", "softmax_cross_entropy { label_smoothing: 0.2 }")
    text = text.replace("num_class: 1", "num_class: 2") if "num_class: 1" in text else \
        text.replace("    metrics {", "    num_class: 2\n    metrics {", 1)
    pipe = Pipeline(_write(text), device="cpu", max_rows=100, seed=3, capturable=False)
    model = pipe.model
    batch = pipe.synthetic_batch(24, seed=1)
    model.train()
    with Fn.use_backend(MetricOracleKernels()):
        preds = model.predict(batch)
    assert list(preds) == ["logits", "probs", "probs1"] and tuple(preds["logits"].shape) == (24, 2)
    torch.testing.assert_close(preds["probs"], torch.softmax(preds["logits"], 1), rtol=0, atol=0)
    assert torch.equal(preds["probs1"], preds["probs"][:, 1])
    losses = model.loss(preds, batch)
    want = torch.nn.CrossEntropyLoss(reduction="mean", label_smoothing=0.2)(
        preds["logits"], batch.labels["label"].to(torch.int64))
    assert list(losses) == ["softmax_cross_entropy"]
    torch.testing.assert_close(losses["softmax_cross_entropy"], want, rtol=0, atol=0)
    with Fn.use_backend(MetricOracleKernels()):
        l0 = float(pipe.eager_step(batch))
        l1 = float(pipe.eager_step(batch))
        m = pipe.evaluate([pipe.synthetic_batch(32, seed=s) for s in range(2)])
    assert np.isfinite([l0, l1]).all() and l1 < l0
    assert set(m) == {"auc", "softmax_cross_entropy"} and 0.0 <= m["auc"] <= 1.0


def _write(text):
    import tempfile

    fd, path = tempfile.mkstemp(suffix=".config")
    with os.fdopen(fd, "w") as fh:
        fh.write(text)
    return path


# ---- the reference example ----------------------------------------------------------------------------------------
def test_reference_example_trains_and_evaluates(kern):
    """The reference's file as stored, stepped on the CPU on the fused path (host build of the kernels) and evaluated:
    finite falling losses, the light head's auc and loss mean."""
    pipe = Pipeline(REF_EXAMPLE, device="cpu", max_rows=200, seed=3, capturable=False)
    assert type(pipe.model).__name__ == "RocketLaunching" and pipe.model.mlp_index_dict == {1: 2, 2: 3}
    batch = pipe.synthetic_batch(64, seed=1)
    be = ShimBackend(kern)
    with Fn.use_backend(be):
        ls = [float(pipe.eager_step(batch)) for _ in range(3)]
        m = pipe.evaluate([pipe.synthetic_batch(64, seed=s) for s in range(2)])
    assert np.isfinite(ls).all() and ls[-1] < ls[0]
    assert be.rocket_calls == 3 * 2 + 2
    assert set(m) == {"auc_booster", "auc_light", "softmax_cross_entropy_booster", "softmax_cross_entropy_light"}
    assert 0.0 < m["auc_light"] < 1.0 and np.isfinite(m["softmax_cross_entropy_light"])


# ---- this repo's RocketLaunching against the reference's own (tests/golden/ref_rocket.npz) ---------------------------
import rocket_ref as RR  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "ref_rocket.npz"))


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("tag", list(RR.CASES))
def test_model_matches_reference_fixture(kern, tag, fused):
    """State-dict keys, training and eval predictions and losses (keys in order and values), the input gradient and
    every parameter gradient of the sum of the training losses, against the reference's own RocketLaunching run in
    float64: on the torch formulation and on the fused path (host build of the kernels), fed the case's seeded group
    input in place of the embedding lookup."""
    m, _ = _model(RR.config_text(tag))
    pre = f"{tag}_"
    keys = [k for k in m.state_dict() if not k.startswith("embedding_group")]
    assert keys == list(GOLD[pre + "keys"])
    m.load_state_dict({k: torch.from_numpy(GOLD[pre + "sd__" + k]).float() for k in keys}, strict=False)
    x = torch.from_numpy(GOLD[pre + "x"]).float().requires_grad_(True)
    m.build_input = lambda batch: {"deep": x}
    batch = types.SimpleNamespace(labels={"label": torch.from_numpy(GOLD[pre + "labels"]).float()})
    be = ShimBackend(kern) if fused else None
    def ctx():
        return Fn.use_backend(be) if fused else contextlib.nullcontext()

    m.train()
    with ctx():
        preds = m.predict(batch)
        losses = m.loss(preds, batch)
        torch.stack(list(losses.values())).sum().backward()
    assert list(preds) == list(GOLD[pre + "train_pred_keys"])
    assert list(losses) == list(GOLD[pre + "train_loss_keys"])
    for k, v in preds.items():
        _close(_np(v), GOLD[pre + "train_pred__" + k], 2e-5, k)
    for k, v in losses.items():
        _close(_np(v), GOLD[pre + "train_loss__" + k], 2e-5, k)
    _close(_np(x.grad), GOLD[pre + "dx"], 2e-5, "dx")
    params = dict(m.named_parameters())
    for k in keys:
        _close(_np(params[k].grad), GOLD[pre + "grad__" + k], 5e-5, k)
    m.eval()
    with ctx(), torch.no_grad():
        preds = m.predict(batch)
        losses = m.loss(preds, batch)
    assert list(preds) == list(GOLD[pre + "eval_pred_keys"])
    assert list(losses) == list(GOLD[pre + "eval_loss_keys"])
    for k, v in preds.items():
        _close(_np(v), GOLD[pre + "eval_pred__" + k], 2e-5, k)
    for k, v in losses.items():
        _close(_np(v), GOLD[pre + "eval_loss__" + k], 2e-5, k)
    if fused:
        assert be.rocket_calls == 3                     # training forward and backward, eval forward


# ---- data parallelism over gloo --------------------------------------------------------------------------------------
def _gloo_worker(rank, world, port, lib, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    try:
        from torcheasyrec_b200.verify import verify_sharded

        L = ctypes.CDLL(lib)
        P, I32 = ctypes.c_void_p, ctypes.c_int
        L.rocket_head_fwd.argtypes = [P, I32, P, P]
        L.rocket_head_bwd.argtypes = [P, P, P, I32, P, P]
        be = ShimBackend(L)
        with Fn.use_backend(be):
            verify_sharded(REF_EXAMPLE, "cpu", "mixed", rw_min_rows=250, bit_exact_logits=True)
        assert be.rocket_calls > 0
        q.put((rank, "ok"))
    except Exception:
        import traceback

        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_example_two_ranks_equal_the_unsharded_step(kern):
    """rocket_launching_criteo (COSINE: every loss a batch mean) over gloo W = 2 on the fused path (the host build of
    the kernels): light and booster logits bit-equal to the unsharded model's on the concatenated batch, the mean of the
    ranks' losses equal to its loss, tables and dense weights equal after the steps."""
    import torch.multiprocessing as mp
    from test_distributed_cpu import _free_port

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, kern._name, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    bad = [r for r in res if r[1] != "ok"]
    assert not bad, "\n".join(f"rank {r}: {m}" for r, m in bad)


def test_multi_task_models_refuse_model_level_softmax_ce():
    """A model-level softmax_cross_entropy stays refused at construction on multi-task models (their towers' heads
    are BCE or JRC), as before single-task models accepted it."""
    text = GENERATORS["mmoe_taobao"]().replace("model_config {\n", "model_config {\n    losses {\n        "
                                               "softmax_cross_entropy {}\n    }\n", 1)
    with pytest.raises(NotImplementedError, match="softmax_cross_entropy is outside the hot-path scope of multi-task"):
        cfg = parse_text(text)
        create_model(cfg.model_config, create_features(list(cfg.feature_configs), fg_mode=cfg.data_config.fg_mode),
                     list(cfg.data_config.label_fields), device=torch.device("cpu"))
