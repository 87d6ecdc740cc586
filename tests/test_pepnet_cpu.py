"""PEPNet on the CPU: the float64 restatement (tests/pepnet_ref.py) pinned to the reference's own EPNet and PPNet
(tests/golden/ref_pepnet.npz, made by tests/golden/make_pepnet_golden.py), the SOURCE of the fused gate kernels
(csrc/tzk_pepnet.cuh) run on the host through tests/native/cuda_cpu_shim.h against float64, and the model: reference
parameter names, domain selection, the task-space-weighted loss, the reference example trained unchanged, training and
evaluation with the fused path (checker backend) and with the torch formulation, and a sharded gloo step."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import pepnet_ref as R  # noqa: E402
from oracle_backend import OracleKernels  # noqa: E402
from pepnet_oracle_backend import PepnetOracleKernels  # noqa: E402

from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200._lib import PEPNET_RELU, TzkPepnetGateArgs  # noqa: E402
from torcheasyrec_b200.batch import Batch, synthetic_batch  # noqa: E402
from torcheasyrec_b200.config import parse_text  # noqa: E402
from torcheasyrec_b200.dense_gemm import bce_with_logits  # noqa: E402
from torcheasyrec_b200.embedding_modules import SparseOptimizerSpec  # noqa: E402
from torcheasyrec_b200.engine import Pipeline  # noqa: E402
from torcheasyrec_b200.features import create_features  # noqa: E402
from torcheasyrec_b200.kernels import OPT_ADAGRAD  # noqa: E402
from torcheasyrec_b200.rank_models import EPNet, PPNet, create_model, task_space_weighted_bce  # noqa: E402
from torcheasyrec_b200.sparse import KeyedJaggedTensor, KeyedTensor  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "ref_pepnet.npz"))
CASES = list(R.CASES)
REF_EXAMPLE = os.path.join(HERE, "golden", "ref_examples", "pepnet_taobao.config")
NATIVE = os.path.join(HERE, "native")


def _close(got, want, r, name=""):
    """|got - want| <= r (|want| + max(1, max |want|)): relative to the tensor's scale."""
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(np.asarray(got, np.float64), want, rtol=r, atol=r * max(1.0, np.abs(want).max()),
                               err_msg=name)


def _gold_outs(tag):
    return [GOLD[f"{tag}_out{i}"] for i in range(sum(1 for k in GOLD.files if k.startswith(f"{tag}_out")))]


# ---- the restatement and this repo's modules, pinned to the reference's ----------------------------------------------
@pytest.mark.parametrize("tag", CASES)
def test_restatement_matches_reference_modules(tag):
    sd, inputs, dys = R.seeded_case(tag)
    outs, dxs, grads = R.run(tag, sd, inputs, dys)
    for i, (o, g) in enumerate(zip(outs, _gold_outs(tag))):
        _close(o, g, 1e-6, f"out{i}")
    for k, d in dxs.items():
        _close(d, GOLD[f"{tag}_d_{k}"], 1e-6, f"d_{k}")
    pre = f"{tag}_grad__"
    assert {k[len(pre):] for k in GOLD.files if k.startswith(pre)} == set(grads)
    for name, g in grads.items():
        _close(g, GOLD[pre + name], 1e-6, name)
    assert R.ordered_keys(tag) == list(GOLD[f"{tag}_keys"])


def _modules(tag):
    B, M, Dd, U, eh, T, hidden, g_ep, g_pp = R.CASES[tag]
    mods = nn.Module()
    mods.epnet = EPNet(M, Dd, hidden_dim=eh or M, gamma=g_ep) if Dd is not None else None
    mods.ppnet = PPNet(M, U, num_task=T, hidden_units=hidden, activation="nn.ReLU", dropout_ratio=[0.0],
                       gamma=g_pp) if U is not None else None
    return mods


def _covered(tag):
    """Whether the fused path covers the case: every width a multiple of 4 (pepnet_test.py's group is 25 wide)."""
    B, M, Dd, U, eh, T, hidden, _, _ = R.CASES[tag]
    return M % 4 == 0 and all(h % 4 == 0 for h in hidden) and ((eh or M) % 4 == 0) and (Dd or 0) % 4 == 0


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("tag", CASES)
def test_modules_match_reference_modules(tag, fused):
    """This repo's EPNet / PPNet with the reference's state dict: same keys, same outputs and gradients; with the checker
    backend, covered shapes run the fused autograd path (one product call forward and one backward per EPNet and per
    PPNet depth), the others the torch formulation."""
    B, M, Dd, U, eh, T, hidden, _, _ = R.CASES[tag]
    mods = _modules(tag)
    assert list(mods.state_dict()) == list(GOLD[f"{tag}_keys"])
    sd, inputs, dys = R.seeded_case(tag)
    mods.load_state_dict({k: torch.from_numpy(v).float() for k, v in sd.items()}, strict=True)
    xs = {k: torch.from_numpy(v).float().requires_grad_(True) for k, v in inputs.items()}
    be = PepnetOracleKernels() if fused else OracleKernels()
    with Fn.use_backend(be):
        x = xs["main"]
        if mods.epnet is not None:
            x = mods.epnet(x, xs["domain"])
        outs = mods.ppnet(x, xs["uia"]) if mods.ppnet is not None else [x]
        torch.autograd.backward(outs, [torch.from_numpy(d).float() for d in dys])
    want_calls = 2 * ((Dd is not None) + (len(hidden) if U is not None else 0)) if fused and _covered(tag) else 0
    assert getattr(be, "pepnet_calls", 0) == want_calls
    for i, (o, g) in enumerate(zip(outs, _gold_outs(tag))):
        _close(o.detach().numpy(), g, 2e-5, f"out{i}")
    for k, x in xs.items():
        _close(x.grad.numpy(), GOLD[f"{tag}_d_{k}"], 2e-5, f"d_{k}")
    for name, p in mods.named_parameters():
        _close(p.grad.numpy(), GOLD[f"{tag}_grad__{name}"], 2e-5, name)


def test_ppnet_dropout_ratio_expansion():
    """PPNet expands dropout_ratio as the reference does: empty or None -> 0, one value -> every depth, else per depth."""
    def ratios(d, n=3):
        return [m.p for m in PPNet(8, 4, 2, [4] * n, dropout_ratio=d).dropout_ratios]
    assert ratios([]) == [0.0] * 6 and ratios(None) == [0.0] * 6
    assert ratios([0.2]) == [0.2] * 6
    assert ratios([0.1, 0.2, 0.3]) == [0.1, 0.2, 0.3] * 2
    assert ratios(0.4) == [0.4] * 6
    with pytest.raises(AssertionError, match="length of dropout_ratio"):
        ratios([0.1, 0.2])


# ---- the kernel source on the host ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kern(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("shim") / "libpepnet_cpu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", NATIVE,
                    "-x", "c++", os.path.join(NATIVE, "pepnet_standalone.cu"), "-shared", "-fPIC", "-o", out],
                   check=True)
    L = ctypes.CDLL(out)
    P, I32 = ctypes.c_void_p, ctypes.c_int
    L.pepnet_check.argtypes = [P, I32]
    L.pepnet_gate_fwd.argtypes = [P, I32]
    L.pepnet_gate_bwd.argtypes = [P, I32, P, P]
    return L


def _buf(rng, B, ld):
    return rng.standard_normal((B, ld)).astype(np.float32)


def _run_segments(L, B, specs, grid, seed):
    """specs [(N, relu, has_bias, gamma, ld_extra)]: x / z / y / dy / dx / dz of segment s are [B, N] column windows of
    buffers with a row pitch of N + ld_extra (a multiple of 4), so the kernels see strided rows."""
    rng = np.random.default_rng(seed)
    a = TzkPepnetGateArgs()
    a.B, a.n_segs = B, len(specs)
    keep, segs, ys, dys, dxs, dzs = [], [], [], [], [], []
    for s, (N, relu, has_bias, gamma, extra) in enumerate(specs):
        ld = N + extra
        x, z, dy = _buf(rng, B, ld), _buf(rng, B, ld), _buf(rng, B, ld)
        y, dx, dz = (np.full((B, ld), np.nan, np.float32) for _ in range(3))
        bx = (rng.standard_normal(N).astype(np.float32) * 0.5) if has_bias else None
        bz = rng.standard_normal(N).astype(np.float32) * 0.5
        keep += [x, z, dy, y, dx, dz, bx, bz]
        g = a.seg[s]
        g.x, g.z, g.y, g.dy, g.dx, g.dz = (t.ctypes.data for t in (x, z, y, dy, dx, dz))
        g.bx, g.bz = (None if bx is None else bx.ctypes.data), bz.ctypes.data
        g.ldx = g.ldz = g.ldy = ld
        g.N, g.act, g.gamma = N, PEPNET_RELU if relu else 0, gamma
        segs.append((x[:, :N].astype(np.float64), None if bx is None else bx.astype(np.float64),
                     z[:, :N].astype(np.float64), bz.astype(np.float64), relu, np.float32(gamma)))
        ys.append(y)
        dys.append(dy[:, :N].astype(np.float64))
        dxs.append(dx)
        dzs.append(dz)
    assert L.pepnet_check(ctypes.byref(a), 1) == 0
    assert L.pepnet_gate_fwd(ctypes.byref(a), grid) == 0
    for s, (y, ry) in enumerate(zip(ys, R.gate_fwd(segs))):
        N = specs[s][0]
        _close(y[:, :N], ry, 1e-6, f"y{s}")
        assert np.isnan(y[:, N:]).all()                      # nothing written past the segment's columns
    P_ = sum(2 * sp[0] for sp in specs)
    part, dpar = np.full((grid, P_), np.nan, np.float32), np.full(P_, np.nan, np.float32)
    assert L.pepnet_gate_bwd(ctypes.byref(a), grid, part.ctypes.data, dpar.ctypes.data) == 0
    o = 0
    for s, (rdx, rdz, rdbx, rdbz) in enumerate(R.gate_bwd(segs, dys)):
        N = specs[s][0]
        _close(dxs[s][:, :N], rdx, 1e-6, f"dx{s}")
        _close(dzs[s][:, :N], rdz, 1e-6, f"dz{s}")
        _close(dpar[o:o + N], rdbx, 1e-5, f"dbx{s}")
        _close(dpar[o + N:o + 2 * N], rdbz, 1e-5, f"dbz{s}")
        o += 2 * N
    want = np.zeros(P_, np.float32)
    for row in part:                                          # the partial rows added in CTA order
        want += row
    np.testing.assert_array_equal(dpar, want)


def test_kernel_source_epnet_segment(kern):
    """EPNet: identity, no bias, one segment; odd B."""
    _run_segments(kern, 5, [(16, False, False, 2.0, 0)], grid=2, seed=1)


@pytest.mark.parametrize("n_segs", [1, 3, 8])
def test_kernel_source_ppnet_depth(kern, n_segs):
    """PPNet depth: ReLU with the main linear's bias, one segment per task, strided rows, several widths."""
    widths = [8, 12, 4, 20, 8, 16, 24, 12]
    specs = [(widths[s], True, True, 1.5, 4 * (s % 3)) for s in range(n_segs)]
    _run_segments(kern, 3, specs, grid=2, seed=10 + n_segs)


def test_kernel_source_mixed_activations_and_bias(kern):
    specs = [(8, True, False, 2.0, 0), (12, False, True, 0.5, 4), (4, True, True, 3.0, 8), (8, False, False, 1.0, 0)]
    _run_segments(kern, 7, specs, grid=3, seed=4)


def test_kernel_source_grid_stride(kern):
    """B = 37 on 2 CTAs of a 64-wide segment (16 quads -> 16 rows per step): every CTA walks several steps, the last
    one partial, and the batch sums add 2 partial rows."""
    _run_segments(kern, 37, [(64, True, True, 2.0, 0), (32, False, False, 2.0, 4)], grid=2, seed=5)


def test_kernel_source_widest_segment(kern):
    """N = 1024: one row per step, every thread one quad."""
    _run_segments(kern, 3, [(1024, True, True, 2.0, 0)], grid=2, seed=6)


def test_kernel_source_empty_batch_zeroes_dparams(kern):
    """B = 0: no backward kernel runs and the batch sums add no partial rows, so dparams comes back all zeros."""
    widths, grid = [8, 12, 64], 5
    a = TzkPepnetGateArgs()
    a.B, a.n_segs = 0, len(widths)
    for s, N in enumerate(widths):                            # no rows: the segments' buffers may be null
        g = a.seg[s]
        g.N, g.ldx, g.ldz, g.ldy, g.act, g.gamma = N, N, N, N, PEPNET_RELU, 2.0
    P_ = 2 * sum(widths)
    part, dpar = np.full((grid, P_), np.nan, np.float32), np.full(P_, np.nan, np.float32)
    assert kern.pepnet_gate_bwd(ctypes.byref(a), grid, part.ctypes.data, dpar.ctypes.data) == 0
    np.testing.assert_array_equal(dpar, np.zeros(P_, np.float32))


def test_kernel_source_refuses_uncovered_segments(kern):
    x = np.zeros((2, 2048), np.float32)

    def check(N=8, ld=8, n_segs=1, act=1, off=0, backward=1):
        a = TzkPepnetGateArgs()
        a.B, a.n_segs = 2, n_segs
        for s in range(min(n_segs, 8)):
            g = a.seg[s]
            g.x = g.z = g.y = g.dy = g.dx = g.dz = x.ctypes.data + off
            g.bz = x.ctypes.data
            g.ldx = g.ldz = g.ldy = ld
            g.N, g.act, g.gamma = N, act, 2.0
        return kern.pepnet_check(ctypes.byref(a), backward)

    assert check() == 0 and check(N=1024, ld=1024) == 0 and check(n_segs=8) == 0
    assert check(N=6, ld=8) == 1 and check(N=1028, ld=1028) == 1 and check(N=0, ld=8) == 1   # N % 4, N > 1024
    assert check(ld=10) == 1 and check(N=8, ld=4) == 1                                     # pitch
    assert check(n_segs=9) == 1 and check(n_segs=0) == 1
    assert check(act=2) == 1
    assert check(off=4) == 1                                                                # 16-B alignment


# ---- the model -------------------------------------------------------------------------------------------------------
PEPNET_TEST_CONFIG = """
feature_configs { id_feature { feature_name: "cat_a" embedding_dim: 16 num_buckets: 100 } }
feature_configs { id_feature { feature_name: "cat_b" embedding_dim: 8 num_buckets: 1000 } }
feature_configs { raw_feature { feature_name: "int_a" } }
feature_configs { id_feature { feature_name: "domainf" embedding_dim: 16 num_buckets: 3 } }
feature_configs { id_feature { feature_name: "uia" embedding_dim: 16 num_buckets: 100 } }
model_config {
  feature_groups { group_name: "all" feature_names: "cat_a" feature_names: "cat_b" feature_names: "int_a"
                   group_type: DEEP }
  feature_groups { group_name: "domain" feature_names: "domainf" group_type: DEEP }
  feature_groups { group_name: "uia" feature_names: "uia" group_type: DEEP }
  pepnet {
    task_domain_num: 3 domain_input_name: "domainf"
    ppnet_hidden_units: [16, 8] ppnet_dropout_ratio: [0.1, 0.1]
    task_towers { tower_name: "t1" label_name: "label1" mlp { hidden_units: [8, 4] }
      metrics { auc {} } losses { binary_cross_entropy {} } }
    task_towers { tower_name: "t2" label_name: "label2" mlp { hidden_units: [8, 4] }
      metrics { auc {} } losses { binary_cross_entropy {} } }
  }
}"""
# the same model with the widths the fused path covers: group all 16 + 8 + 4 = 28 wide, dropout 0
COVERED_CONFIG = (PEPNET_TEST_CONFIG.replace('raw_feature { feature_name: "int_a" }',
                                             'raw_feature { feature_name: "int_a" value_dim: 4 }')
                  .replace("ppnet_dropout_ratio: [0.1, 0.1]", ""))


def _model(config=PEPNET_TEST_CONFIG, seed=0, labels=("label1", "label2", "domainf")):
    cfg = parse_text(config)
    torch.manual_seed(seed)
    return create_model(cfg.model_config, create_features(list(cfg.feature_configs)), list(labels),
                        device=torch.device("cpu"))


def _batch(int_dim=1, labels=True, domains=(1.0, 2.0)):
    sparse = KeyedJaggedTensor.from_lengths_sync(
        keys=["cat_a", "cat_b", "domainf", "uia"], values=torch.tensor([1, 2, 3, 4, 5, 6, 7, 1, 2, 3, 4]),
        lengths=torch.tensor([1, 2, 1, 3, 1, 1, 1, 1], dtype=torch.int32))
    dense = KeyedTensor.from_tensor_list(keys=["int_a"], tensors=[torch.arange(2 * int_dim).float().view(2, -1) / 7])
    lab = {"domainf": torch.tensor(domains)}
    if labels:
        lab.update({"label1": torch.tensor([1.0, 0.0]), "label2": torch.tensor([0.0, 1.0])})
    return Batch(dense_features={"__BASE__": dense}, sparse_features={"__BASE__": sparse}, labels=lab)


def test_state_dict_names_are_the_references():
    """The reference's test model (EPNet and PPNet): module names as in the fixture's `test_both` case, then 2 x 3
    domain towers `_task_tower.{i D + j}`."""
    model = _model()
    names = [k for k in model.state_dict() if not k.startswith("embedding_group")]
    towers = [k for k in names if k.startswith("_task_tower.")]
    assert names[:len(names) - len(towers)] == list(GOLD["test_both_keys"])
    assert sorted({int(k.split(".")[1]) for k in towers}) == list(range(6))
    assert towers[:6] == ["_task_tower.0.tower_mlp.mlp.0.perceptron.0.weight",
                          "_task_tower.0.tower_mlp.mlp.0.perceptron.0.bias",
                          "_task_tower.0.tower_mlp.mlp.1.perceptron.0.weight",
                          "_task_tower.0.tower_mlp.mlp.1.perceptron.0.bias",
                          "_task_tower.0.linear.weight", "_task_tower.0.linear.bias"]
    assert model.epnet.gate_nu.dense_layers[0].in_features == 16 + 25
    assert [m.p for m in model.ppnet.dropout_ratios] == [pytest.approx(0.1)] * 4


def test_replay_of_reference_model_test():
    """tzrec/models/pepnet_test.py: every `logits_t{1,2}_{0,1,2}` / `probs_...` has shape (2,), without and with each
    module."""
    for drop in ([], ["domain"], ["uia"], ["domain", "uia"]):
        cfg = PEPNET_TEST_CONFIG
        for g in drop:
            cfg = cfg.replace(f'  feature_groups {{ group_name: "{g}"', "  # ")
        model = _model(cfg)
        assert (model.epnet is None) == ("domain" in drop) and (model.ppnet is None) == ("uia" in drop)
        with Fn.use_backend(OracleKernels()), torch.no_grad():
            preds = model.predict(_batch(labels=False))
        assert sorted(preds) == sorted(f"{k}_t{t}_{j}" for k in ("logits", "probs") for t in (1, 2) for j in range(3))
        assert all(v.size() == (2,) for v in preds.values())


def test_missing_all_group_fails_as_in_the_reference():
    cfg = PEPNET_TEST_CONFIG.replace('group_name: "all"', 'group_name: "main"')
    with pytest.raises(Exception, match="all feature group not found"):
        _model(cfg)


def test_domain_selection_by_comparison():
    """logits_<t> = sum_j [d == j] logits_<t>_<j>, exact; only the selected tower gets a gradient; a label outside
    [0, D) selects 0 (the reference's torch.gather raises there)."""
    model = _model()
    outs = {f"{k}_t{t}_{j}": torch.randn(6, requires_grad=True) for k in ("logits", "probs") for t in (1, 2)
            for j in range(3)}
    d = torch.tensor([0.0, 2.0, 1.0, 1.0, 3.0, -1.0])
    sel = model._select_domain_task_output(outs, Batch(labels={"domainf": d}))
    assert sorted(sel) == ["logits_t1", "logits_t2", "probs_t1", "probs_t2"]
    for name, v in sel.items():
        want = torch.stack([outs[f"{name}_{j}"] for j in range(3)], 1)
        idx = torch.tensor([0, 2, 1, 1])
        assert torch.equal(v[:4], torch.gather(want[:4], 1, idx.unsqueeze(1)).squeeze(1))
        assert torch.equal(v[4:], torch.zeros(2))            # out of range: 0, where the reference raises
    sel["logits_t1"].sum().backward()
    for j in range(3):
        assert torch.equal(outs[f"logits_t1_{j}"].grad, (d == j).float())


def test_loss_and_metrics_see_the_selected_tower():
    model = _model(seed=2)
    batch = _batch()
    with Fn.use_backend(OracleKernels()), torch.no_grad():
        preds = model.predict(batch)
        losses = model.loss(preds, batch)
    for t, lab in (("t1", "label1"), ("t2", "label2")):
        sel = torch.stack([preds[f"logits_{t}_1"][0], preds[f"logits_{t}_2"][1]])
        want = torch.nn.functional.binary_cross_entropy_with_logits(sel, batch.labels[lab])
        torch.testing.assert_close(losses[f"binary_cross_entropy_{t}"], want, rtol=1e-6, atol=1e-7)


def _reference_task_space_loss(logits, label, ind, in_w, out_w, weight):
    """multi_task_rank.py:105-125 + rank_model.py:260-261, as written there."""
    loss_weight = torch.Tensor([1.0])
    in_task_space = (ind > 0).float()
    loss_weight = loss_weight * (in_w * in_task_space + out_w * (1 - in_task_space))
    loss_weight = torch.nan_to_num(torch.div(loss_weight, torch.mean(loss_weight)), nan=0.0, posinf=0.0, neginf=0.0)
    loss_weight *= weight
    losses = torch.nn.BCEWithLogitsLoss(reduction="none")(logits, label)
    return torch.mean(losses * loss_weight)


@pytest.mark.parametrize("ind,in_w,out_w,weight", [
    ([1, 0, 1, 1, 0, 0, 1, 0], 1.0, 0.0, 1.0),         # pepnet_taobao's cvr
    ([1, 0, 1, 1, 0, 0, 1, 0], 2.0, 0.5, 0.7),
    ([0] * 8, 1.0, 0.0, 1.0),                          # no sample in the space: div_no_nan gives weight 0, not NaN
    ([3, -1, 0, 2, 0, 1, 1, 0], 1.0, 1.0, 1.0),
])
def test_task_space_loss_matches_reference_formula(ind, in_w, out_w, weight):
    g = torch.Generator().manual_seed(0)
    logits, label = torch.randn(8, generator=g), (torch.rand(8, generator=g) < 0.5).float()
    ind = torch.tensor(ind, dtype=torch.float32)
    got = task_space_weighted_bce(logits, label, ind, in_w, out_w, weight)
    want = _reference_task_space_loss(logits, label, ind, in_w, out_w, weight)
    assert torch.equal(got, want)
    assert torch.isfinite(got)


def test_pepnet_taobao_cvr_loss_is_task_space_weighted():
    pipe = Pipeline(REF_EXAMPLE, device="cpu", max_rows=200, seed=3)
    batch = pipe.synthetic_batch(32, seed=4)
    with Fn.use_backend(OracleKernels()), torch.no_grad():
        pipe.model.eval()
        preds = pipe.model.predict(batch)
        losses = pipe.model.loss(preds, batch)
    sel = pipe.model._select_domain_task_output(preds, batch)
    want = _reference_task_space_loss(sel["logits_cvr"], batch.labels["buy"], batch.labels["clk"], 1.0, 0.0, 1.0)
    assert torch.equal(losses["binary_cross_entropy_cvr"], want)
    assert torch.equal(losses["binary_cross_entropy_ctr"], bce_with_logits(sel["logits_ctr"], batch.labels["clk"]))


@pytest.mark.parametrize("name", ["mmoe_taobao", "ple_taobao"])
def test_towers_without_task_space_keep_their_loss(name):
    """MMoE and PLE: every tower's loss is cfg.weight * bce_with_logits, bit for bit."""
    pipe = Pipeline(name, device="cpu", max_rows=200, seed=3)
    batch = pipe.synthetic_batch(16, seed=2)
    with Fn.use_backend(OracleKernels()), torch.no_grad():
        preds = pipe.model.predict(batch)
        losses = pipe.model.loss(preds, batch)
    for cfg in pipe.model._task_tower_cfgs:
        want = cfg.weight * bce_with_logits(preds[f"logits_{cfg.tower_name}"], batch.labels[cfg.label_name])
        assert torch.equal(losses[f"binary_cross_entropy_{cfg.tower_name}"], want)


def test_sample_weight_name_and_other_losses_stay_refused():
    with pytest.raises(NotImplementedError, match="sample_weight_name"):
        _model(PEPNET_TEST_CONFIG.replace('tower_name: "t2"', 'tower_name: "t2" sample_weight_name: "w"'))
    with pytest.raises(NotImplementedError, match="l2_loss"):
        _model(PEPNET_TEST_CONFIG.replace("losses { binary_cross_entropy {} } }\n  }", "losses { l2_loss {} } }\n  }"))


@pytest.mark.parametrize("fused", [False, True])
def test_reference_example_trains_unchanged(fused):
    """examples/pepnet_taobao.config as stored: group all 256, domain 16, uia 208; two steps on the same batch give a
    finite loss that goes down; with the checker backend the fused gates run."""
    pipe = Pipeline(REF_EXAMPLE, device="cpu", max_rows=200, seed=3)
    eg = pipe.model.embedding_group
    assert (eg.group_total_dim("all"), eg.group_total_dim("domain"), eg.group_total_dim("uia")) == (256, 16, 208)
    batch = pipe.synthetic_batch(24, seed=1)
    assert set(batch.labels["occupation"].tolist()) <= {0.0, 1.0, 2.0}
    be = PepnetOracleKernels() if fused else OracleKernels()
    with Fn.use_backend(be):
        l0 = float(pipe.eager_step(batch))
        l1 = float(pipe.eager_step(batch))
    assert np.isfinite([l0, l1]).all()
    assert l1 < l0
    assert getattr(be, "pepnet_calls", 0) == (12 if fused else 0)   # (EPNet + 2 PPNet depths) x 2 ways x 2 steps


def test_fused_and_torch_formulations_train_alike():
    """Three Adagrad (sparse) / Adam (dense) steps of the covered test model: the fused autograd path and the torch
    formulation give the same losses, parameters and tables."""
    out = []
    for be in (OracleKernels(), PepnetOracleKernels()):
        model = _model(COVERED_CONFIG, seed=1)
        model.set_sparse_optimizer(SparseOptimizerSpec(kind=OPT_ADAGRAD, lr=0.05))
        opt = torch.optim.Adam(model.dense_parameters(), lr=0.01)
        losses = []
        with Fn.use_backend(be):
            for _ in range(3):
                batch = _batch(int_dim=4)
                loss = sum(model.loss(model.predict(batch), batch).values())
                opt.zero_grad()
                loss.backward()
                opt.step()
                losses.append(float(loss.detach()))
        assert getattr(be, "pepnet_calls", 0) == (18 if isinstance(be, PepnetOracleKernels) else 0)
        state = {k: v.detach().clone() for k, v in model.named_parameters()}
        state["tables"] = model.sparse_collections()[0].dense_weights().clone()
        out.append((losses, state))
    np.testing.assert_allclose(out[0][0], out[1][0], rtol=1e-5)
    for k in out[0][1]:
        np.testing.assert_allclose(out[1][1][k].numpy(), out[0][1][k].numpy(), rtol=1e-4, atol=1e-6, err_msg=k)


def test_evaluate_returns_per_tower_auc_and_loss():
    pipe = Pipeline("pepnet_taobao", device="cpu", max_rows=200, seed=3)
    with Fn.use_backend(PepnetOracleKernels()):
        pipe.eager_step(pipe.synthetic_batch(32, seed=0))
        got = pipe.evaluate([pipe.synthetic_batch(32, seed=5), pipe.synthetic_batch(9, seed=6)])
    assert set(got) == {"auc_ctr", "auc_cvr", "binary_cross_entropy_ctr", "binary_cross_entropy_cvr"}
    for k, v in got.items():
        assert np.isfinite(float(v)), k
    assert 0.0 <= float(got["auc_ctr"]) <= 1.0 and 0.0 <= float(got["auc_cvr"]) <= 1.0


def test_sharded_two_ranks_equal_the_unsharded_twin(tmp_path):
    """pepnet_taobao with two edits that make a sharded step comparable with one step on the whole batch: dropout 0 (the
    masks of the two shapes differ), and the cvr tower's out-of-space weight back to 1, so its task-space weights stay
    1 (mean(v) normalises per rank, as in the reference under data parallelism, so weights that depend on it differ
    between a rank's half and the whole batch; the weighted loss path still runs)."""
    from test_distributed_cpu import _run

    from torcheasyrec_b200 import example_configs

    text = example_configs.pepnet_taobao()
    assert "ppnet_dropout_ratio: [0.1, 0.1]" in text and "out_task_space_weight: 0" in text
    cfg = tmp_path / "pepnet_taobao_sharded.config"
    cfg.write_text(text.replace("ppnet_dropout_ratio: [0.1, 0.1]", "ppnet_dropout_ratio: [0.0]")
                   .replace("out_task_space_weight: 0", "out_task_space_weight: 1"))
    _run(2, str(cfg), "mixed", rw_min_rows=250)


def test_synthetic_batch_labels():
    """Without label_cardinality every label is {0, 1} exactly as before (a feature-less batch pins the draws); a label
    given a cardinality D is drawn over [0, D), and labels before it are unchanged."""
    got = synthetic_batch([], 64, ["a", "b"], seed=9)
    rng = np.random.default_rng(9)
    for name in ("a", "b"):
        assert torch.equal(got.labels[name], torch.from_numpy((rng.random(64) < 0.25).astype(np.float32)))
    pipe = Pipeline("pepnet_taobao", device="cpu", max_rows=200, seed=3)
    plain = synthetic_batch(pipe.features, 300, pipe.labels, seed=4)
    dom = pipe.synthetic_batch(300, seed=4)
    assert pipe.labels == ["clk", "buy", "occupation"]
    for name in ("clk", "buy"):
        assert torch.equal(plain.labels[name], dom.labels[name])
    assert set(dom.labels["occupation"].tolist()) == {0.0, 1.0, 2.0}
    assert set(plain.labels["occupation"].tolist()) == {0.0, 1.0}


def test_usable_predicate():
    m, u = torch.zeros(2, 256), torch.zeros(2, 208)
    with Fn.use_backend(PepnetOracleKernels()):
        assert Fn.pepnet_usable(m, u, [512, 256], [512, 256], 2, "nn.ReLU")
        assert Fn.pepnet_usable(m, torch.zeros(2, 16), [256], [256])                          # EPNet
        assert not Fn.pepnet_usable(m, u, [512, 256], [512, 256], 2, "nn.Sigmoid")
        assert not Fn.pepnet_usable(m.double(), u.double(), [512], [512], 2, "nn.ReLU")
        assert not Fn.pepnet_usable(m, torch.zeros(2, 18), [512], [512], 2, "nn.ReLU")      # 18 + 256 % 4 != 0
        assert not Fn.pepnet_usable(m, u, [510], [510], 2, "nn.ReLU")
        assert not Fn.pepnet_usable(m, u, [2048], [2048], 2, "nn.ReLU")                       # N > 1024
        assert not Fn.pepnet_usable(m, u, [16], [16], 9, "nn.ReLU")                           # > 8 tasks
        assert not Fn.pepnet_usable(torch.zeros(2, 25), torch.zeros(2, 16), [25], [25])       # pepnet_test's group
        with torch.autocast("cpu", dtype=torch.bfloat16):
            assert not Fn.pepnet_usable(m, u, [512], [512], 2, "nn.ReLU")
    with Fn.use_backend(OracleKernels()):     # a CPU backend without the PEPNet kernels: torch formulation
        assert not Fn.pepnet_usable(m, u, [512], [512], 2, "nn.ReLU")
