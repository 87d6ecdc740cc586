"""MaskNet on the CPU: the float64 restatement (tests/masknet_ref.py) pinned to the reference's own MaskNetModule
(tests/golden/ref_masknet.npz, made by tests/golden/make_masknet_golden.py), the SOURCE of the fused kernels
(csrc/tzk_masknet.cuh) run on the host through tests/native/cuda_cpu_shim.h against the restatement, the reference's
construction rules and checks, the GEMM row pitches of the fused path, and the model: reference parameter names, the
replay of tzrec/models/masknet_test.py, the reference example trained unchanged, and training and evaluation through
the Pipeline with the fused path (checker backend) and with the torch formulation."""
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
import masknet_ref as M  # noqa: E402
from masknet_oracle_backend import MaskNetOracleKernels  # noqa: E402
from oracle_backend import OracleKernels  # noqa: E402

from torcheasyrec_b200 import dense_gemm  # noqa: E402
from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200.batch import Batch  # noqa: E402
from torcheasyrec_b200.config import parse_text  # noqa: E402
from torcheasyrec_b200.embedding_modules import SparseOptimizerSpec  # noqa: E402
from torcheasyrec_b200.engine import Pipeline  # noqa: E402
from torcheasyrec_b200.features import create_features  # noqa: E402
from torcheasyrec_b200.kernels import OPT_ADAGRAD  # noqa: E402
from torcheasyrec_b200.rank_models import MaskBlock, MaskNetModule, create_model, proto_float32  # noqa: E402
from torcheasyrec_b200.sparse import KeyedJaggedTensor, KeyedTensor  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "ref_masknet.npz"))
CASES = ["criteo_par", "criteo_ser", "ratio03", "modtest_par", "modtest_ser", "modeltest"]
REF_EXAMPLE = os.path.join(HERE, "golden", "ref_examples", "masknet_criteo.config")
NATIVE = os.path.join(HERE, "native")
P, I32, I64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64


def _case(tag):
    """(B, E, ratio, agg, H, nb, top, parallel), state dict, e, dy of a golden case, regenerated from its seed."""
    c = GOLD[f"{tag}_case"]
    B, E, agg, H, nb, parallel, seed = int(c[0]), int(c[1]), int(c[3]), int(c[4]), int(c[5]), bool(c[6]), int(c[7])
    ratio, top = float(c[2]), [int(u) for u in c[8:]]
    sd, e, dy = M.seeded_case(B, E, ratio, agg, H, nb, top, parallel, seed)
    return (B, E, ratio, agg, H, nb, top, parallel), sd, e, dy


def _close(got, want, r, name=""):
    """|got - want| <= r (|want| + max(1, max |want|)): relative to the tensor's scale (fp32 sums of O(scale) terms)."""
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(np.asarray(got, np.float64), want, rtol=r, atol=r * max(1.0, np.abs(want).max()),
                               err_msg=name)


def _module(tag):
    (B, E, ratio, agg, H, nb, top, parallel), sd, e, dy = _case(tag)
    mod = MaskNetModule(E, nb, {"reduction_ratio": ratio, "aggregation_dim": agg, "hidden_dim": H},
                        {"hidden_units": top}, parallel)
    mod.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    return mod, e, dy


# ---- the restatement and this repo's module, pinned to the reference's module ------------------------------------------
@pytest.mark.parametrize("tag", CASES)
def test_restatement_matches_reference_module(tag):
    (B, E, ratio, agg, H, nb, top, parallel), sd, e, dy = _case(tag)
    y, de, grads = M.module(sd, e, dy, nb, parallel, len(top))
    _close(y, GOLD[f"{tag}_y"], 1e-5, "y")
    _close(de, GOLD[f"{tag}_de"], 2e-5, "de")
    pre = f"{tag}_grad__"
    names = {k[len(pre):] for k in GOLD.files if k.startswith(pre)}
    assert names == set(grads)
    for name in names:
        _close(grads[name], GOLD[pre + name], 2e-5, name)


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("tag", CASES)
def test_module_matches_reference_module(tag, fused):
    """This repo's MaskNetModule with the reference's state dict: same keys, same values; parallel cases also through
    the fused autograd path (checker backend for the kernels, the padded GEMM layout on the CPU)."""
    mod, e_np, dy_np = _module(tag)
    assert list(mod.state_dict()) == list(GOLD[f"{tag}_keys"])
    be = MaskNetOracleKernels() if fused else OracleKernels()
    e = torch.from_numpy(e_np).requires_grad_(True)
    with Fn.use_backend(be):
        assert mod.fused_usable(e) == (fused and mod.use_parallel)
        y = mod(e)
        y.backward(torch.from_numpy(dy_np))
    assert (be.masknet_calls == 4) if (fused and mod.use_parallel) else not getattr(be, "masknet_calls", 0)
    _close(y.detach().numpy(), GOLD[f"{tag}_y"], 1e-5, "y")
    _close(e.grad.numpy(), GOLD[f"{tag}_de"], 2e-5, "de")
    for name, p in mod.named_parameters():
        _close(p.grad.numpy(), GOLD[f"{tag}_grad__{name}"], 2e-5, name)


# ---- the reference's construction rules ----------------------------------------------------------------------------
def test_reduction_ratio_overrides_aggregation_dim():
    assert MaskBlock(33, 33, 16, reduction_ratio=2.0, aggregation_dim=32).aggregation_dim == 66
    assert MaskBlock(33, 33, 16, reduction_ratio=0.0, aggregation_dim=32).aggregation_dim == 32
    # config_to_kwargs includes the proto default reduction_ratio = 1.0, so aggregation_dim alone never wins
    cfg = parse_text(MODEL_TEST_CONFIG.replace("reduction_ratio: 2 ", ""))
    torch.manual_seed(0)
    model = create_model(cfg.model_config, create_features(list(cfg.feature_configs)), ["label"],
                         device=torch.device("cpu"))
    assert model.mask_net_layer.mask_blocks[0].aggregation_dim == 33


def test_ratio_is_the_float32_proto_value_as_printed():
    """0.3 and 0.7 are not float32-exact; MessageToDict prints them as 0.3 / 0.7, so int(E * ratio) is the float64
    product of the printed value (int(10 * float32(0.7)) would be 6)."""
    assert proto_float32(0.3) == 0.3 and proto_float32(0.7) == 0.7 and proto_float32(3) == 3.0
    assert proto_float32(0.1 + 0.2) == 0.3
    mod = MaskNetModule(10, 1, {"reduction_ratio": 0.7, "aggregation_dim": 0, "hidden_dim": 4})
    assert mod.mask_blocks[0].aggregation_dim == 7
    mod = MaskNetModule(429, 1, {"reduction_ratio": 0.3, "aggregation_dim": 0, "hidden_dim": 4})
    assert mod.mask_blocks[0].aggregation_dim == 128


def test_serial_blocks_take_the_previous_hidden_and_the_raw_mask_input():
    mod = MaskNetModule(429, 3, {"reduction_ratio": 0.25, "aggregation_dim": 0, "hidden_dim": 64}, None, False)
    dims = [(b.mask_generator[0].in_features, b.aggregation_dim, b.mask_generator[2].out_features,
             b.ffn[0].in_features) for b in mod.mask_blocks]
    assert dims == [(429, 107, 429, 429), (429, 16, 64, 64), (429, 16, 64, 64)]
    assert mod.output_dim() == 64
    assert M.block_dims(429, 64, 3, 0.25, 0, False) == [(429, 107), (64, 16), (64, 16)]


def test_the_references_checks_fire():
    with pytest.raises(ValueError, match="Either aggregation_dim or reduction_ratio must be provided."):
        MaskBlock(8, 8, 4, reduction_ratio=0.0, aggregation_dim=0)
    with pytest.raises(AssertionError, match="aggregation_dim must be > 0"):
        MaskBlock(8, 8, 4, reduction_ratio=0.1)
    with pytest.raises(AssertionError, match="hidden_dim must be > 0."):
        MaskBlock(8, 8, 0)
    with pytest.raises(AssertionError, match="aggregation_dim must be > 0"):      # serial: int(hidden_dim * ratio) == 0
        MaskNetModule(64, 2, {"reduction_ratio": 0.1, "aggregation_dim": 0, "hidden_dim": 8}, None, False)


# ---- the kernel source on the host ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kern(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("shim") / "libmasknet_cpu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", NATIVE,
                    "-x", "c++", os.path.join(NATIVE, "masknet_standalone.cu"), "-shared", "-fPIC", "-o", out],
                   check=True)
    L = ctypes.CDLL(out)
    L.mn_mask_fwd.argtypes = [P, I32, P, P, P, P, I64, I32, I32, I32, P, P]
    L.mn_mask_bwd.argtypes = [P, I32, P, P, P, P, P, P, I64, I32, I32, I32, P, P, P, P]
    L.mn_ffn_fwd.argtypes = [P, P, P, P, I64, I32, I32, I32, P, P]
    L.mn_ffn_bwd.argtypes = [P, P, P, P, P, P, I64, I32, I32, I32, P, P, P]
    return L


def _p(a):
    return None if a is None else a.ctypes.data


def _f32(rng, *shape, scale=1.0):
    return (rng.standard_normal(shape) * scale).astype(np.float32)


def _run_mask(L, E, nb, B, grid, seed):
    Ep = M.pad4(E)
    rng = np.random.default_rng(seed)
    e = np.zeros((B, Ep), np.float32)
    e[:, :E] = _f32(rng, B, E)
    m, dv = _f32(rng, B, nb * Ep), _f32(rng, B, nb * Ep)
    b2, g, b = _f32(rng, nb * E, scale=0.3), 1 + _f32(rng, E, scale=0.1), _f32(rng, E, scale=0.1)
    v, st = np.full((B, nb * Ep), np.nan, np.float32), np.empty((B, 2), np.float32)
    assert L.mn_mask_fwd(_p(e), Ep, _p(m), _p(b2), _p(g), _p(b), B, E, nb, grid, _p(v), _p(st)) == 0
    rv, rst = M.mask_fwd(e, m, b2, g, b, E, nb)
    _close(v, rv, 1e-5, "v")
    _close(st, rst, 1e-5, "mask stats")
    P_ = (nb + 2) * E
    dm, de = np.full((B, nb * Ep), np.nan, np.float32), np.full((B, Ep), np.nan, np.float32)
    part, dpar = np.full((grid, P_), np.nan, np.float32), np.empty(P_, np.float32)
    assert L.mn_mask_bwd(_p(e), Ep, _p(m), _p(b2), _p(g), _p(b), _p(st), _p(dv), B, E, nb, grid, _p(dm), _p(de),
                         _p(part), _p(dpar)) == 0
    rdm, rde, rdb2, rdg, rdb = M.mask_bwd(e, m, b2, g, b, dv, E, nb)
    _close(dm, rdm, 2e-5, "dm")
    _close(de, rde, 2e-5, "de")
    _close(dpar[:nb * E], rdb2, 2e-5, "db2")
    _close(dpar[nb * E:(nb + 1) * E], rdg, 2e-5, "dgamma_ln")
    _close(dpar[(nb + 1) * E:], rdb, 2e-5, "dbeta_ln")
    want = np.zeros(P_, np.float32)
    for row in part[:min(grid, B)]:
        want += row
    np.testing.assert_array_equal(dpar, want)


def _run_ffn(L, H, nb, B, grid, seed):
    rng = np.random.default_rng(seed)
    z, dy = _f32(rng, B, nb * H), _f32(rng, B, nb * H)
    b3, g, b = _f32(rng, nb * H, scale=0.3), 1 + _f32(rng, nb * H, scale=0.1), _f32(rng, nb * H, scale=0.3)
    y, st = np.empty((B, nb * H), np.float32), np.empty((B, nb, 2), np.float32)
    assert L.mn_ffn_fwd(_p(z), _p(b3), _p(g), _p(b), B, H, nb, grid, _p(y), _p(st)) == 0
    ry, rst = M.ffn_fwd(z, b3, g, b, nb)
    _close(y, ry, 1e-5, "y")
    _close(st, rst, 1e-5, "ffn stats")
    dz = np.empty((B, nb * H), np.float32)
    part, dpar = np.full((nb, grid, 3 * H), np.nan, np.float32), np.empty((nb, 3, H), np.float32)
    assert L.mn_ffn_bwd(_p(z), _p(b3), _p(g), _p(b), _p(st), _p(dy), B, H, nb, grid, _p(dz), _p(part),
                        _p(dpar)) == 0
    rdz, rdg, rdb, rdb3 = M.ffn_bwd(z, b3, g, b, dy, nb)
    _close(dz, rdz, 2e-5, "dz")
    _close(dpar[:, 0], rdg, 2e-5, "dgamma")
    _close(dpar[:, 1], rdb, 2e-5, "dbeta")
    _close(dpar[:, 2], rdb3, 2e-5, "db3")
    want = np.zeros((nb, 3 * H), np.float32)
    for j in range(min(grid, B)):
        want += part[:, j]
    np.testing.assert_array_equal(dpar.reshape(nb, 3 * H), want)


# E: masknet_criteo's 429 (pitch 432), the module test's 24, the model test's 33 (pitch 36)
@pytest.mark.parametrize("E", [429, 24, 33])
@pytest.mark.parametrize("nb", [1, 3])
@pytest.mark.parametrize("B", [1, 3])
def test_mask_kernels_source_matches_restatement(kern, E, nb, B):
    _run_mask(kern, E, nb, B, grid=B, seed=E + nb + B)


@pytest.mark.parametrize("H", [16, 512])
@pytest.mark.parametrize("nb", [1, 3])
@pytest.mark.parametrize("B", [1, 3])
def test_ffn_kernels_source_matches_restatement(kern, H, nb, B):
    _run_ffn(kern, H, nb, B, grid=B, seed=H + nb + B)


@pytest.mark.parametrize("E,H,nb", [(429, 512, 3), (33, 16, 1)])
def test_kernels_source_grid_stride(kern, E, H, nb):
    """B = 257 on 5 CTAs: every CTA walks ~51 samples and the batch sums add 5 partial rows."""
    _run_mask(kern, E, nb, 257, grid=5, seed=11)
    _run_ffn(kern, H, nb, 257, grid=5, seed=12)


def test_kernel_source_empty_batch_zeroes_dparams(kern):
    """B = 0: no backward kernel runs and the batch sums add no partial rows, so dparams comes back all zeros (the FFN's
    for every mask block)."""
    E, H, nb, grid = 33, 16, 3, 5
    z = np.zeros(1, np.float32)                               # inputs: never read
    P_ = (nb + 2) * E
    part, dpar = np.full((grid, P_), np.nan, np.float32), np.full(P_, np.nan, np.float32)
    assert kern.mn_mask_bwd(_p(z), M.pad4(E), _p(z), _p(z), _p(z), _p(z), _p(z), _p(z), 0, E, nb, grid, _p(z), _p(z),
                            _p(part), _p(dpar)) == 0
    np.testing.assert_array_equal(dpar, np.zeros(P_, np.float32))
    part, dpar = np.full((nb, grid, 3 * H), np.nan, np.float32), np.full((nb, 3, H), np.nan, np.float32)
    assert kern.mn_ffn_bwd(_p(z), _p(z), _p(z), _p(z), _p(z), _p(z), 0, H, nb, grid, _p(z), _p(part), _p(dpar)) == 0
    np.testing.assert_array_equal(dpar, np.zeros((nb, 3, H), np.float32))


def test_kernel_source_refuses_uncovered_shapes(kern):
    z = np.zeros(1 << 16, np.float32)
    for E, nb in [(1025, 1), (0, 1), (24, 0), (24, 9)]:
        assert kern.mn_mask_fwd(_p(z), max(E, 1), _p(z), _p(z), _p(z), _p(z), 1, E, nb, 1, _p(z), _p(z)) == 1
    assert kern.mn_mask_fwd(_p(z), 20, _p(z), _p(z), _p(z), _p(z), 1, 24, 1, 1, _p(z), _p(z)) == 1   # lde < E
    for H, nb in [(18, 1), (1028, 1), (16, 9), (0, 1)]:
        assert kern.mn_ffn_fwd(_p(z), _p(z), _p(z), _p(z), 1, H, nb, 1, _p(z), _p(z)) == 1


# ---- GEMM row pitches of the fused path ------------------------------------------------------------------------------
def test_every_gemm_row_pitch_is_a_multiple_of_4_floats(monkeypatch):
    """A masknet_criteo-shaped module step (E = 429, A = 1287, H = 512, 3 blocks) through the fused path: every GEMM
    operand and result of the blocks has a row pitch (and a column offset) that is a multiple of 4 floats."""
    calls = []
    real = dense_gemm.gemm

    def recording(a, ta, b, tb, out=None, beta=0.0):
        r = real(a, ta, b, tb, out=out, beta=beta)
        for t in (a, b, r):
            calls.append((t.stride(0), t.stride(1), t.storage_offset()))
        return r

    monkeypatch.setattr(dense_gemm, "gemm", recording)
    torch.manual_seed(0)
    mod = MaskNetModule(429, 3, {"reduction_ratio": 3.0, "aggregation_dim": 0, "hidden_dim": 512},
                        {"hidden_units": [256, 128, 64]})
    e = torch.randn(4, 429, requires_grad=True)
    with Fn.use_backend(MaskNetOracleKernels()):
        mod(e).sum().backward()
    assert len(calls) == 3 * (1 + 3 + 3 + 2 * 3 + 2 * 3 + 2)
    for stride0, stride1, off in calls:
        assert stride1 == 1 and stride0 % 4 == 0 and off % 4 == 0, (stride0, stride1, off)
    assert e.grad is not None and torch.isfinite(e.grad).all()


# ---- the model -------------------------------------------------------------------------------------------------------
MODEL_TEST_CONFIG = """
feature_configs { id_feature { feature_name: "cat_a" embedding_dim: 16 num_buckets: 100 } }
feature_configs { id_feature { feature_name: "cat_b" embedding_dim: 16 num_buckets: 1000 } }
feature_configs { raw_feature { feature_name: "int_a" } }
model_config {
  feature_groups { group_name: "all_features" feature_names: "cat_a" feature_names: "cat_b" feature_names: "int_a"
                   group_type: DEEP }
  mask_net { mask_net_module { n_mask_blocks: 3
      mask_block { reduction_ratio: 2 aggregation_dim: 32 hidden_dim: 16 }
      use_parallel: true top_mlp { hidden_units: [8, 4] } } }
  losses { binary_cross_entropy {} }
}"""


def _masknet_test_model(seed=0):
    cfg = parse_text(MODEL_TEST_CONFIG)
    torch.manual_seed(seed)
    features = create_features(list(cfg.feature_configs))
    return create_model(cfg.model_config, features, ["label"], device=torch.device("cpu"))


def _masknet_test_batch(labels=False):
    sparse = KeyedJaggedTensor.from_lengths_sync(keys=["cat_a", "cat_b"], values=torch.tensor([1, 2, 3, 4, 5, 6, 7]),
                                                 lengths=torch.tensor([1, 2, 1, 3], dtype=torch.int32))
    dense = KeyedTensor.from_tensor_list(keys=["int_a"], tensors=[torch.tensor([[0.2], [0.3]])])
    lab = {"label": torch.tensor([1.0, 0.0])} if labels else {}
    return Batch(dense_features={"__BASE__": dense}, sparse_features={"__BASE__": sparse}, labels=lab)


def test_state_dict_names_are_the_references():
    model = _masknet_test_model()
    names = [k for k in model.state_dict() if not k.startswith("embedding_group")]
    assert names == ["mask_net_layer." + k for k in GOLD["modeltest_keys"]] + ["output_linear.weight"]
    assert model.mask_net_layer.mask_blocks[0].aggregation_dim == 66       # 33 * 2; aggregation_dim 32 is overridden
    assert model.output_linear.bias is None


def test_replay_of_reference_model_test():
    """tzrec/models/masknet_test.py: logits and probs of shape (2,); the fused path (checker backend) equals the torch
    formulation on the same weights."""
    model = _masknet_test_model()
    batch = _masknet_test_batch()
    with Fn.use_backend(OracleKernels()), torch.no_grad():
        ref = model.predict(batch)
    be = MaskNetOracleKernels()
    with Fn.use_backend(be), torch.no_grad():
        got = model.predict(batch)
    assert be.masknet_calls == 2            # mask_fwd + ffn_fwd
    assert ref["logits"].size() == (2,) and ref["probs"].size() == (2,)
    assert got["logits"].size() == (2,) and got["probs"].size() == (2,)
    np.testing.assert_allclose(got["logits"].numpy(), ref["logits"].numpy(), rtol=1e-5, atol=1e-6)


def test_fused_and_torch_formulations_train_alike():
    """Three Adagrad (sparse) / Adam (dense) steps of the reference's test model with a label: the fused autograd path
    and the torch formulation give the same losses, parameters and tables."""
    out = []
    for be in (OracleKernels(), MaskNetOracleKernels()):
        model = _masknet_test_model(seed=1)
        model.set_sparse_optimizer(SparseOptimizerSpec(kind=OPT_ADAGRAD, lr=0.05))
        opt = torch.optim.Adam(model.dense_parameters(), lr=0.01)
        losses = []
        with Fn.use_backend(be):
            for _ in range(3):
                batch = _masknet_test_batch(labels=True)
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


@pytest.mark.parametrize("fused", [False, True])
def test_reference_example_trains_unchanged(fused):
    """examples/masknet_criteo.config as stored: one DEEP group of width 26 * 16 + 13 = 429, two steps on the same
    batch, the loss goes down; with the checker backend the fused path runs."""
    pipe = Pipeline(REF_EXAMPLE, device="cpu", max_rows=200, seed=3)
    assert pipe.model.embedding_group.group_total_dim("all_features") == 429
    batch = pipe.synthetic_batch(24, seed=1)
    be = MaskNetOracleKernels() if fused else OracleKernels()
    with Fn.use_backend(be):
        l0 = float(pipe.eager_step(batch))
        l1 = float(pipe.eager_step(batch))
    assert np.isfinite([l0, l1]).all()
    assert l1 < l0
    assert (getattr(be, "masknet_calls", 0) > 0) == fused


def test_evaluate_returns_auc_and_loss():
    pipe = Pipeline("masknet_criteo", device="cpu", max_rows=200, seed=3)
    with Fn.use_backend(MaskNetOracleKernels()):
        pipe.eager_step(pipe.synthetic_batch(32, seed=0))
        got = pipe.evaluate([pipe.synthetic_batch(32, seed=5), pipe.synthetic_batch(9, seed=6)])
    assert set(got) == {"auc", "binary_cross_entropy"}
    assert 0.0 <= float(got["auc"]) <= 1.0 and np.isfinite(float(got["binary_cross_entropy"]))


def test_usable_predicate():
    e = torch.zeros(2, 429)
    with Fn.use_backend(MaskNetOracleKernels()):
        assert Fn.masknet_usable(e, 429, 512, 3, True)
        assert not Fn.masknet_usable(e, 429, 512, 3, False)          # serial: torch formulation
        assert not Fn.masknet_usable(e.double(), 429, 512, 3, True)
        assert not Fn.masknet_usable(e, 429, 510, 3, True)           # H % 4 != 0
        assert not Fn.masknet_usable(e, 429, 1028, 3, True)
        assert not Fn.masknet_usable(e, 429, 512, 9, True)
        assert not Fn.masknet_usable(torch.zeros(2, 1025), 1025, 512, 3, True)
        with torch.autocast("cpu", dtype=torch.bfloat16):
            assert not Fn.masknet_usable(e, 429, 512, 3, True)
    with Fn.use_backend(OracleKernels()):     # a CPU backend without the MaskNet kernels: torch formulation
        assert not Fn.masknet_usable(e, 429, 512, 3, True)
