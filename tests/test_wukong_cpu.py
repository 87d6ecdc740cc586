"""WuKong on the CPU: the float64 restatement (tests/wukong_ref.py) pinned to the reference's own WuKongLayer
(tests/golden/ref_wukong.npz, made by tests/golden/make_wukong_golden.py), the SOURCE of the fused kernels (csrc/tzk_wukong.cuh) run on the host through
tests/native/cuda_cpu_shim.h against the restatement, and the model: reference parameter names, the replay of
tzrec/models/wukong_test.py, the reference example's exception, the built-in config's one edit, training and
evaluation through the Pipeline with the fused path (checker backend) and with the torch formulation."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import wukong_ref as W  # noqa: E402
from oracle_backend import OracleKernels  # noqa: E402
from wukong_oracle_backend import WuKongOracleKernels  # noqa: E402

from torcheasyrec_b200 import example_configs  # noqa: E402
from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200.batch import Batch  # noqa: E402
from torcheasyrec_b200.config import load_pipeline_config, parse_text  # noqa: E402
from torcheasyrec_b200.embedding_modules import SparseOptimizerSpec  # noqa: E402
from torcheasyrec_b200.engine import Pipeline  # noqa: E402
from torcheasyrec_b200.features import create_features  # noqa: E402
from torcheasyrec_b200.kernels import OPT_ADAGRAD  # noqa: E402
from torcheasyrec_b200.rank_models import WuKongLayer, create_model  # noqa: E402
from torcheasyrec_b200.sparse import KeyedJaggedTensor, KeyedTensor  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "ref_wukong.npz"))
CASES = ["criteo1", "criteo2", "small1", "small2", "small3"]
REF_EXAMPLE = os.path.join(HERE, "golden", "ref_examples", "wukong_criteo.config")
NATIVE = os.path.join(HERE, "native")
P, I32, I64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64


def _case(tag):
    """(B, d, n, l, f, k, MLP width), state dict, x, dy of a golden case: the inputs the generator gave the reference's
    layer, regenerated from the stored seed (wukong_ref.seeded_case)."""
    B, d, n, l, f, k, h, seed = (int(v) for v in GOLD[f"{tag}_case"])
    sd, x, dy = W.seeded_case(B, d, n, l, f, k, [h], seed)
    return (B, d, n, l, f, k, h), sd, x, dy


def _close(got, want, r, name=""):
    """|got - want| <= r (|want| + max(1, max |want|)): relative to the tensor's scale (fp32 sums of O(scale) terms)."""
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(np.asarray(got, np.float64), want, rtol=r, atol=r * max(1.0, np.abs(want).max()),
                               err_msg=name)


# ---- the restatement, pinned to the reference's module -------------------------------------------------------------
@pytest.mark.parametrize("tag", CASES)
def test_restatement_matches_reference_layer(tag):
    (B, d, n, l, f, k, h), sd, x, dy = _case(tag)
    y, dx, grads = W.layer(sd, x, dy, f)
    _close(y, GOLD[f"{tag}_y"], 1e-5, "y")
    _close(dx, GOLD[f"{tag}_dx"], 2e-5, "dx")
    pre = f"{tag}_grad__"
    names = {k[len(pre):] for k in GOLD.files if k.startswith(pre)}
    assert names == set(grads)
    for name in names:
        _close(grads[name], GOLD[pre + name], 2e-5, name)


@pytest.mark.parametrize("tag", CASES)
def test_layer_module_matches_reference_layer(tag):
    """This repo's WuKongLayer (torch formulation on the CPU) with the reference's state dict: same names, same values."""
    (B, d, n, l, f, k, h), sd_np, x_np, dy_np = _case(tag)
    layer = WuKongLayer(d, n, l, f, k, {"hidden_units": [h]})
    sd = {name: torch.from_numpy(v) for name, v in sd_np.items()}
    assert set(layer.state_dict()) == set(sd) == {k[len(f"{tag}_grad__"):] for k in GOLD.files
                                                  if k.startswith(f"{tag}_grad__")}
    layer.load_state_dict(sd)
    x = torch.from_numpy(x_np).requires_grad_(True)
    y = layer(x)
    y.backward(torch.from_numpy(dy_np))
    _close(y.detach().numpy(), GOLD[f"{tag}_y"], 1e-5, "y")
    _close(x.grad.numpy(), GOLD[f"{tag}_dx"], 2e-5, "dx")
    for name, p in layer.named_parameters():
        _close(p.grad.numpy(), GOLD[f"{tag}_grad__{name}"], 2e-5, name)


# ---- the kernel source on the host -----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kern(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("shim") / "libwukong_cpu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", NATIVE,
                    "-x", "c++", os.path.join(NATIVE, "wukong_standalone.cu"), "-shared", "-fPIC", "-o", out],
                   check=True)
    L = ctypes.CDLL(out)
    L.wk_mix_fwd.argtypes = [P] * 6 + [I64] + [I32] * 6 + [P] * 3
    L.wk_mix_bwd.argtypes = [P] * 8 + [I64] + [I32] * 6 + [P] * 3
    L.wk_out_fwd.argtypes = [P] * 4 + [I64] + [I32] * 4 + [P] * 2
    L.wk_out_bwd.argtypes = [P] * 5 + [I64] + [I32] * 4 + [P] * 4
    return L


def _p(a):
    return None if a is None else a.ctypes.data


def _f32(rng, *shape, scale=1.0):
    return (rng.standard_normal(shape) * scale).astype(np.float32)


# (n, d, k, f, l, projection): the wukong_criteo layers, the wukong_test.py layers, n k = 15 (not a multiple of 4) at
# d = 4 with the identity residual, and the widest shape the kernels cover
SHAPES = {"criteo1": (27, 16, 24, 16, 16, True), "criteo2": (32, 16, 24, 16, 16, False),
          "small1": (3, 8, 2, 4, 3, True), "small2": (7, 8, 2, 2, 3, True), "small3": (5, 8, 2, 2, 2, True),
          "odd_d4": (5, 4, 3, 2, 3, False), "max": (64, 32, 32, 40, 24, False)}


def _run_shim(L, shape, B, grid, seed):
    n, d, k, f, l, proj = shape
    m = f + l
    rng = np.random.default_rng(seed)
    x = _f32(rng, B, n, d)
    wf, wl = _f32(rng, n, k, scale=0.3), _f32(rng, n, l, scale=0.3)
    wr = _f32(rng, n, m, scale=0.3) if proj else None
    gf, bf = 1 + _f32(rng, n * k, scale=0.1), _f32(rng, n * k, scale=0.1)
    g, b = 1 + _f32(rng, d, scale=0.1), _f32(rng, d, scale=0.1)
    fmb = _f32(rng, B, f * d)
    d_ln_f, dy = _f32(rng, B, n * k), _f32(rng, B, m, d)
    # forward
    ln_f, st, base = np.empty((B, n * k), np.float32), np.empty((B, 2), np.float32), np.empty((B, m, d), np.float32)
    assert L.wk_mix_fwd(_p(x), _p(wf), _p(gf), _p(bf), _p(wl), _p(wr), B, n, d, k, f, l, grid, _p(ln_f), _p(st),
                        _p(base)) == 0
    r_ln_f, r_st, r_base = W.mix_fwd(x, wf, gf, bf, wl, wr, f)
    _close(ln_f, r_ln_f, 1e-5, "ln_f")
    _close(st, r_st, 1e-5, "mix stats")
    _close(base, r_base, 1e-5, "base")
    y, ost = np.empty((B, m, d), np.float32), np.empty((B, m, 2), np.float32)
    assert L.wk_out_fwd(_p(fmb), _p(base), _p(g), _p(b), B, d, f, l, grid, _p(y), _p(ost)) == 0
    r_y, r_ost = W.out_fwd(fmb, base, g, b, f)
    _close(y, r_y, 1e-5, "y")
    _close(ost, r_ost, 1e-5, "out stats")
    # backward
    Pm = 3 * n * k + n * l + (n * m if proj else 0)
    dx, part, dpar = np.empty_like(x), np.full((grid, Pm), np.nan, np.float32), np.empty(Pm, np.float32)
    assert L.wk_mix_bwd(_p(x), _p(wf), _p(gf), _p(wl), _p(wr), _p(st), _p(d_ln_f), _p(dy), B, n, d, k, f, l, grid,
                        _p(dx), _p(part), _p(dpar)) == 0
    r = W.mix_bwd(x, wf, gf, wl, wr, f, d_ln_f, dy)
    nk, nl = n * k, n * l
    o = [0, nk, nk + nl, nk + nl + (n * m if proj else 0)]
    _close(dx, r[0], 2e-5, "dx")
    _close(dpar[o[0]:o[1]].reshape(n, k), r[1], 2e-5, "dw_fmb")
    _close(dpar[o[1]:o[2]].reshape(n, l), r[4], 2e-5, "dw_lcb")
    if proj:
        _close(dpar[o[2]:o[3]].reshape(n, m), r[5], 2e-5, "dw_res")
    _close(dpar[o[3]:o[3] + nk], r[2], 2e-5, "dgamma_fmb")
    _close(dpar[o[3] + nk:], r[3], 2e-5, "dbeta_fmb")
    d_fmb, d_base = np.empty_like(fmb), np.empty((B, m, d), np.float32)
    opart, odpar = np.full((grid, 2 * d), np.nan, np.float32), np.empty(2 * d, np.float32)
    assert L.wk_out_bwd(_p(fmb), _p(base), _p(g), _p(ost), _p(dy), B, d, f, l, grid, _p(d_fmb), _p(d_base), _p(opart),
                        _p(odpar)) == 0
    rd_fmb, rd_base, rdg, rdb = W.out_bwd(fmb, base, g, f, dy)
    _close(d_fmb, rd_fmb, 2e-5, "d_fmb")
    _close(d_base, rd_base, 2e-5, "d_base")
    _close(odpar[:d], rdg, 2e-5, "dgamma")
    _close(odpar[d:], rdb, 2e-5, "dbeta")
    # the reduction over the CTAs' partial sums is exactly the fixed-order sum of the partials
    want = np.zeros(Pm, np.float32)
    for row in part:
        want += row
    np.testing.assert_array_equal(dpar, want)


@pytest.mark.parametrize("name", sorted(SHAPES))
@pytest.mark.parametrize("B", [1, 3])
def test_kernel_source_matches_restatement(kern, name, B):
    _run_shim(kern, SHAPES[name], B, grid=B, seed=B)


@pytest.mark.parametrize("name", ["criteo1", "odd_d4"])
def test_kernel_source_matches_restatement_grid_stride(kern, name):
    """B = 257 on 5 CTAs: every CTA walks ~51 samples and the weight gradients add 5 partial rows."""
    _run_shim(kern, SHAPES[name], 257, grid=5, seed=11)


def test_kernel_source_is_deterministic(kern):
    """The same launch twice gives the same bits (the partials and their reduce have a fixed order)."""
    outs = []
    for _ in range(2):
        n, d, k, f, l = 27, 16, 24, 16, 16
        rng = np.random.default_rng(5)
        B, grid = 19, 4
        x, wf, wl, wr = _f32(rng, B, n, d), _f32(rng, n, k), _f32(rng, n, l), _f32(rng, n, f + l)
        gf = 1 + _f32(rng, n * k, scale=0.1)
        st = np.stack([np.zeros(B, np.float32), np.ones(B, np.float32)], -1)
        d_ln_f, dy = _f32(rng, B, n * k), _f32(rng, B, f + l, d)
        P_ = 3 * n * k + n * l + n * (f + l)
        dx, part, dpar = np.empty_like(x), np.empty((grid, P_), np.float32), np.empty(P_, np.float32)
        assert kern.wk_mix_bwd(_p(x), _p(wf), _p(gf), _p(wl), _p(wr), _p(st), _p(d_ln_f), _p(dy), B, n, d, k, f, l,
                               grid, _p(dx), _p(part), _p(dpar)) == 0
        outs.append((dx.copy(), dpar.copy()))
    np.testing.assert_array_equal(outs[0][0], outs[1][0])
    np.testing.assert_array_equal(outs[0][1], outs[1][1])


def test_kernel_source_empty_batch_zeroes_dparams(kern):
    """B = 0: no backward kernel runs and the batch sums add no partial rows, so dparams comes back all zeros."""
    n, d, k, f, l, grid = 27, 16, 24, 16, 16, 5
    z = np.zeros(1, np.float32)                               # inputs: never read
    P_ = 3 * n * k + n * l + n * (f + l)
    part, dpar = np.full((grid, P_), np.nan, np.float32), np.full(P_, np.nan, np.float32)
    assert kern.wk_mix_bwd(_p(z), _p(z), _p(z), _p(z), _p(z), _p(z), _p(z), _p(z), 0, n, d, k, f, l, grid, _p(z),
                           _p(part), _p(dpar)) == 0
    np.testing.assert_array_equal(dpar, np.zeros(P_, np.float32))
    opart, odpar = np.full((grid, 2 * d), np.nan, np.float32), np.full(2 * d, np.nan, np.float32)
    assert kern.wk_out_bwd(_p(z), _p(z), _p(z), _p(z), _p(z), 0, d, f, l, grid, _p(z), _p(z), _p(opart),
                           _p(odpar)) == 0
    np.testing.assert_array_equal(odpar, np.zeros(2 * d, np.float32))


def test_kernel_source_refuses_uncovered_shapes(kern):
    z = np.zeros(4096, np.float32)
    for n, d, k, f, l in [(65, 16, 8, 8, 8), (8, 12, 8, 4, 4), (8, 16, 33, 4, 4), (8, 16, 8, 40, 25), (8, 16, 8, 0, 8)]:
        assert kern.wk_mix_fwd(_p(z), _p(z), _p(z), _p(z), _p(z), _p(z), 1, n, d, k, f, l, 1, _p(z), _p(z), _p(z)) == 1


# ---- the model ---------------------------------------------------------------------------------------------------------
WUKONG_TEST_CONFIG = """
feature_configs { id_feature { feature_name: "cat_a" embedding_dim: 8 num_buckets: 100 } }
feature_configs { id_feature { feature_name: "cat_b" embedding_dim: 8 num_buckets: 1000 } }
feature_configs { raw_feature { feature_name: "int_a" } }
model_config {
  feature_groups { group_name: "dense" feature_names: "int_a" group_type: DEEP }
  feature_groups { group_name: "sparse" feature_names: "cat_a" feature_names: "cat_b" group_type: DEEP }
  wukong {
    dense_mlp { hidden_units: [8] }
    wukong_layers { lcb_feature_num: 3 fmb_feature_num: 4 compressed_feature_num: 2 feature_num_mlp { hidden_units: [4] } }
    wukong_layers { lcb_feature_num: 3 fmb_feature_num: 2 compressed_feature_num: 2 feature_num_mlp { hidden_units: [4] } }
    wukong_layers { lcb_feature_num: 2 fmb_feature_num: 2 compressed_feature_num: 2 feature_num_mlp { hidden_units: [4] } }
    final { hidden_units: [4, 2] }
  }
  losses { binary_cross_entropy {} }
}"""


def _wukong_test_model(seed=0):
    cfg = parse_text(WUKONG_TEST_CONFIG)
    torch.manual_seed(seed)
    features = create_features(list(cfg.feature_configs))
    return create_model(cfg.model_config, features, ["label"], device=torch.device("cpu"))


def _wukong_test_batch(labels=False):
    sparse = KeyedJaggedTensor.from_lengths_sync(keys=["cat_a", "cat_b"], values=torch.tensor([1, 2, 3, 4, 5, 6, 7]),
                                                 lengths=torch.tensor([1, 2, 1, 3], dtype=torch.int32))
    dense = KeyedTensor.from_tensor_list(keys=["int_a"], tensors=[torch.tensor([[0.2], [0.3]])])
    lab = {"label": torch.tensor([1.0, 0.0])} if labels else {}
    return Batch(dense_features={"__BASE__": dense}, sparse_features={"__BASE__": sparse}, labels=lab)


def test_state_dict_names_are_the_references():
    model = _wukong_test_model()
    names = [k for k in model.state_dict() if not k.startswith("embedding_group")]
    layer_names = {k[len("small1_grad__"):] for k in GOLD.files if k.startswith("small1_grad__")}
    want = ["dense_mlp.mlp.0.perceptron.0.weight", "dense_mlp.mlp.0.perceptron.0.bias"]
    for i in range(3):
        want += [f"_wukong_layers.{i}.{n}" for n in sorted(layer_names)]
    want += [f"final_mlp.mlp.{j}.perceptron.0.{p}" for j in range(2) for p in ("weight", "bias")]
    want += ["output_mlp.weight", "output_mlp.bias"]
    assert sorted(names) == sorted(want)
    # the residual projection exists exactly when n != f + l (3 -> 7 -> 5 -> 4: all three layers)
    assert all(f"_wukong_layers.{i}.residual_projection.weight" in names for i in range(3))


def test_replay_of_reference_model_test():
    """tzrec/models/wukong_test.py: logits and probs of shape [2]; the fused path (checker backend) equals the torch
    formulation on the same weights."""
    model = _wukong_test_model()
    batch = _wukong_test_batch()
    with Fn.use_backend(OracleKernels()), torch.no_grad():
        ref = model.predict(batch)
    be = WuKongOracleKernels()
    with Fn.use_backend(be), torch.no_grad():
        got = model.predict(batch)
    assert be.wukong_calls == 6            # mix + out per layer
    assert ref["logits"].size() == (2,) and ref["probs"].size() == (2,)
    np.testing.assert_allclose(got["logits"].numpy(), ref["logits"].numpy(), rtol=1e-5, atol=1e-6)


def test_fused_and_torch_formulations_train_alike():
    """Three Adagrad (sparse) / Adam (dense) steps of the reference's test model with a label: the fused autograd path
    and the torch formulation give the same losses, parameters and tables."""
    out = []
    for be in (OracleKernels(), WuKongOracleKernels()):
        model = _wukong_test_model(seed=1)
        model.set_sparse_optimizer(SparseOptimizerSpec(kind=OPT_ADAGRAD, lr=0.05))
        opt = torch.optim.Adam(model.dense_parameters(), lr=0.01)
        losses = []
        with Fn.use_backend(be):
            for _ in range(3):
                batch = _wukong_test_batch(labels=True)
                loss = model.loss(model.predict(batch), batch)["binary_cross_entropy"]
                opt.zero_grad()
                loss.backward()
                opt.step()
                losses.append(float(loss.detach()))
        state = {k: v.detach().clone() for k, v in model.named_parameters()}
        state["tables"] = model.sparse_collections()[0].dense_weights().clone()
        out.append((losses, state))
    np.testing.assert_allclose(out[0][0], out[1][0], rtol=1e-5)
    for k in out[0][1]:
        np.testing.assert_allclose(out[1][1][k].numpy(), out[0][1][k].numpy(), rtol=1e-4, atol=1e-6, err_msg=k)


def test_reference_example_raises_the_references_exception():
    with pytest.raises(Exception, match="dense mlp last hidden_unit must be the same sparse feature dim"):
        Pipeline(REF_EXAMPLE, device="cpu", max_rows=200)


def test_builtin_example_is_the_reference_file_with_one_edit():
    ref = load_pipeline_config(REF_EXAMPLE)
    ours = parse_text(example_configs.BUILTINS["wukong_criteo"]())
    assert list(ours.model_config.wukong.dense_mlp.hidden_units) == [512, 256, 16]
    assert list(ref.model_config.wukong.dense_mlp.hidden_units) == [512, 256, 128]
    ref.model_config.wukong.dense_mlp.hidden_units = [512, 256, 16]
    assert ours.to_dict() == ref.to_dict()
    assert "wukong_criteo" not in example_configs.GENERATORS      # GENERATORS: the configs equal to their examples


@pytest.mark.parametrize("fused", [False, True])
def test_pipeline_steps_and_the_loss_drops(fused):
    pipe = Pipeline("wukong_criteo", device="cpu", max_rows=200, seed=3)
    batch = pipe.synthetic_batch(24, seed=1)
    be = WuKongOracleKernels() if fused else OracleKernels()
    with Fn.use_backend(be):
        l0 = float(pipe.eager_step(batch))
        l1 = float(pipe.eager_step(batch))
    assert np.isfinite([l0, l1]).all()
    assert l1 < l0
    assert (getattr(be, "wukong_calls", 0) > 0) == fused


def test_evaluate_returns_auc_and_loss():
    pipe = Pipeline("wukong_criteo", device="cpu", max_rows=200, seed=3)
    with Fn.use_backend(WuKongOracleKernels()):
        pipe.eager_step(pipe.synthetic_batch(32, seed=0))
        got = pipe.evaluate([pipe.synthetic_batch(32, seed=5), pipe.synthetic_batch(9, seed=6)])
    assert set(got) == {"auc", "binary_cross_entropy"}
    assert 0.0 <= float(got["auc"]) <= 1.0 and np.isfinite(float(got["binary_cross_entropy"]))


def test_usable_predicate():
    x = torch.zeros(2, 27, 16)
    with Fn.use_backend(WuKongOracleKernels()):
        assert Fn.wukong_usable(x, 27, 16, 24, 16, 16)
        assert not Fn.wukong_usable(x.double(), 27, 16, 24, 16, 16)
        assert not Fn.wukong_usable(torch.zeros(2, 27, 12), 27, 12, 24, 16, 16)
        assert not Fn.wukong_usable(x, 27, 16, 33, 16, 16)
        assert not Fn.wukong_usable(torch.zeros(2, 65, 16), 65, 16, 24, 16, 16)
        assert not Fn.wukong_usable(x, 27, 16, 24, 40, 25)
        with torch.autocast("cpu", dtype=torch.bfloat16):
            assert not Fn.wukong_usable(x, 27, 16, 24, 16, 16)
    with Fn.use_backend(OracleKernels()):     # a CPU backend without the WuKong kernels: torch formulation
        assert not Fn.wukong_usable(x, 27, 16, 24, 16, 16)
