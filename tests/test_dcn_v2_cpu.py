"""DCN-v2 on the CPU: the SOURCE of the fused cross-network kernels (csrc/tzk_dcn_v2.cuh) run on the host through
tests/native/cuda_cpu_shim.h with the emulated mma.sync of sm90_cpu_emu.h, against the float64 restatement
(tests/dcn_v2_ref.py); that restatement, this repo's CrossV2 on both paths and its DCNV2 against the reference's own
(tests/golden/ref_dcn_v2.npz); the dcn_v2_taobao config trained and evaluated; and two gloo ranks."""
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
import dcn_v2_ref as R  # noqa: E402
from metric_oracle_backend import MetricOracleKernels  # noqa: E402

from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200._lib import TzkDcnV2Args  # noqa: E402
from torcheasyrec_b200.config import parse_text  # noqa: E402
from torcheasyrec_b200.embedding_modules import SparseOptimizerSpec  # noqa: E402
from torcheasyrec_b200.engine import Pipeline  # noqa: E402
from torcheasyrec_b200.example_configs import BUILTINS, EDITED_GENERATORS, GENERATORS  # noqa: E402
from torcheasyrec_b200.features import create_features  # noqa: E402
from torcheasyrec_b200.kernels import OPT_SGD  # noqa: E402
from torcheasyrec_b200.rank_models import CrossV2, create_model  # noqa: E402

NATIVE = os.path.join(HERE, "native")
GOLD = np.load(os.path.join(HERE, "golden", "ref_dcn_v2.npz"))
MULTI_TOWER_EXAMPLE = os.path.join(HERE, "golden", "ref_examples", "multi_tower_taobao.config")


# ---- the kernel source on the host ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kern(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("shim") / "libdcn_v2_cpu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", NATIVE,
                    "-x", "c++", os.path.join(NATIVE, "dcn_v2_standalone.cu"), "-shared", "-fPIC", "-o", out],
                   check=True)
    L = ctypes.CDLL(out)
    P, I32 = ctypes.c_void_p, ctypes.c_int
    L.dcn_v2_check.argtypes = [P, I32]
    for f in ("dcn_v2_work_floats", "dcn_v2_param_floats"):
        getattr(L, f).argtypes = [P]
        getattr(L, f).restype = ctypes.c_int64
    L.dcn_v2_fwd.argtypes = [P, I32]
    L.dcn_v2_bwd_data.argtypes = [P, I32]
    L.dcn_v2_bwd_weight.argtypes = [P, I32, P, P]
    return L


class ShimDcnV2:
    """dcn_v2_fwd / dcn_v2_bwd of kernels.CudaKernels on CPU tensors, computed by the host build of the kernel
    source.  Grids: fixed ones, or min(work, 3) tiles and min(work, 2) chunks as a small stand-in for the device's."""

    def __init__(self, L, grid=None, chunks=None):
        self.L, self.grid, self.chunks, self.calls = L, grid, chunks, 0

    def _args(self, x0, wu, wv, bias):
        a = TzkDcnV2Args()
        a.B, a.D = x0.shape
        a.L, a.r = wu.shape[:2]
        self._keep = [t.detach().float().contiguous() for t in (x0, wu, wv, bias)]
        a.x0, a.wu, a.wv, a.bias = (t.data_ptr() for t in self._keep)
        self._work = torch.zeros(self.L.dcn_v2_work_floats(ctypes.byref(a)))
        a.work = self._work.data_ptr()
        return a

    def _grid(self, B):
        return self.grid or max(1, min(-(-B // 16), 3))

    def dcn_v2_fwd(self, x0, wu, wv, bias):
        self.calls += 1
        a = self._args(x0, wu, wv, bias)
        y, v = torch.empty(a.B, a.D), torch.empty(a.B, a.L * a.r)
        a.y, a.v = y.data_ptr(), v.data_ptr()
        assert self.L.dcn_v2_fwd(ctypes.byref(a), self._grid(a.B)) == 0
        return y, v

    def dcn_v2_bwd(self, x0, wu, wv, bias, v, dy):
        self.calls += 1
        a = self._args(x0, wu, wv, bias)
        v, dy = v.float().contiguous(), dy.float().contiguous()
        dx0, dv = torch.empty(a.B, a.D), torch.empty(a.B, a.L * a.r)
        a.v, a.dy, a.dx0, a.dv = v.data_ptr(), dy.data_ptr(), dx0.data_ptr(), dv.data_ptr()
        assert self.L.dcn_v2_bwd_data(ctypes.byref(a), self._grid(a.B)) == 0
        Pn = self.L.dcn_v2_param_floats(ctypes.byref(a))
        chunks = self.chunks or max(1, min(-(-a.B // 64), 2))
        partials, dparams = torch.empty(chunks, Pn), torch.empty(Pn)
        assert self.L.dcn_v2_bwd_weight(ctypes.byref(a), chunks, partials.data_ptr(), dparams.data_ptr()) == 0
        n = a.L * a.r * a.D
        return (dx0, dparams[:n].view(a.L, a.r, a.D), dparams[n:2 * n].view(a.L, a.D, a.r),
                dparams[2 * n:].view(a.L, a.D))


class ShimBackend(MetricOracleKernels):
    """The CPU checker backend with the cross network computed by the host build of its kernel source."""

    def __init__(self, L):
        super().__init__()
        self._dcn = ShimDcnV2(L)
        self.dcn_v2_fwd = self._dcn.dcn_v2_fwd
        self.dcn_v2_bwd = self._dcn.dcn_v2_bwd

    @property
    def dcn_v2_calls(self):
        return self._dcn.calls


def _close(got, want, r, name):
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(np.asarray(got, np.float64), want, rtol=r,
                               atol=r * max(1.0, np.abs(want).max() if want.size else 1.0), err_msg=name)


def _np(t):
    return t.detach().double().numpy()


def _run_shim(L, x0, wu, wv, bias, dy, grid=None, chunks=None):
    s = ShimDcnV2(L, grid, chunks)
    y, v = s.dcn_v2_fwd(x0, wu, wv, bias)
    return (y,) + s.dcn_v2_bwd(x0, wu, wv, bias, v, dy)


# (B, D, L, r, grid, chunks)
KERNEL_CASES = {
    "empty_batch": (0, 33, 3, 64, 1, 1),
    "one_row": (1, 33, 3, 64, 1, 1),
    "b17_model_test_shape": (17, 33, 3, 64, 2, 1),
    "multi_cta": (150, 64, 2, 32, 3, 2),
    "eight_layers_r64": (9, 40, 8, 64, 1, 1),
    "rank_two_d512": (5, 512, 1, 2, 1, 1),
    "module_test_shape": (20, 32, 6, 2, 2, 2),
    "d1_l1_r1": (33, 1, 1, 1, 2, 1),
}


@pytest.mark.parametrize("tag", list(KERNEL_CASES))
def test_kernel_source_against_float64(kern, tag):
    """y, dx0 and every weight gradient of the three kernels against float64, over B = 0, 1, 17 and several CTAs and
    chunks, L = 1 and 8, r = 1, 2 and 64, D = 1, 33 and 512: 1e-5 (forward) and 2e-5 (gradients) of each tensor's
    scale."""
    B, D, L, r, grid, chunks = KERNEL_CASES[tag]
    x0, wu, wv, bias = (t.float().double() for t in R.case(len(tag), B, D, L, r))
    dy = torch.from_numpy(np.random.default_rng(1).standard_normal((B, D))).float().double()
    want = R.grads(x0, wu, wv, bias, dy)
    got = _run_shim(kern, x0, wu, wv, bias, dy, grid, chunks)
    for name, g, w, tol in zip(("y", "dx0", "d wu", "d wv", "d bias"), got, want, (1e-5, 2e-5, 2e-5, 2e-5, 2e-5)):
        assert tuple(g.shape) == tuple(w.shape), name
        _close(_np(g), w.numpy(), tol, name)
    if B == 0:
        assert all(float(g.abs().sum()) == 0 for g in got[2:])


@pytest.mark.parametrize("grid,chunks", [(2, 2), (3, 3)])
def test_kernel_source_reruns_bit_identical(kern, grid, chunks):
    x0, wu, wv, bias = R.case(5, 140, 24, 3, 8)
    dy = torch.from_numpy(np.random.default_rng(2).standard_normal((140, 24)))
    a = _run_shim(kern, x0, wu, wv, bias, dy, grid, chunks)
    b = _run_shim(kern, x0, wu, wv, bias, dy, grid, chunks)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def _args(D, L, r):
    a = TzkDcnV2Args()
    a.B, a.D, a.L, a.r = 4, D, L, r
    a.x0 = a.wu = a.wv = a.bias = a.v = a.y = a.dy = a.dx0 = a.dv = 16
    a.work = 64
    return a


def test_kernel_source_refuses_outside_cover(kern):
    for D, L, r in ((512, 8, 64), (1, 1, 1), (33, 3, 64)):
        assert all(kern.dcn_v2_check(ctypes.byref(_args(D, L, r)), p) == 0 for p in range(3))
    for D, L, r in ((0, 2, 8), (513, 2, 8), (64, 0, 8), (64, 9, 8), (64, 2, 0), (64, 2, 65)):
        for p in range(3):
            assert kern.dcn_v2_check(ctypes.byref(_args(D, L, r)), p) == 1, (D, L, r, p)
    a = _args(64, 2, 8)
    a.work = 68                                          # the fragments are read as 16-B vectors
    assert kern.dcn_v2_check(ctypes.byref(a), 0) == 1
    a = _args(64, 2, 8)
    a.y = None
    assert kern.dcn_v2_check(ctypes.byref(a), 0) == 1
    assert kern.dcn_v2_check(ctypes.byref(a), 3) == 1


def test_torch_path_outside_cover(kern):
    """Shapes outside the cover, and a v kernel without bias, run the reference's loop even with the kernels
    available; inside the cover the fused path runs."""
    be = ShimBackend(kern)
    with Fn.use_backend(be):
        for D, L, r in ((520, 1, 4), (16, 9, 4), (16, 2, 65)):
            m = CrossV2(D, L, r)
            x = torch.randn(3, D)
            assert not Fn.cross_v2_usable(x, m.u_kernels, m.v_kernels)
            torch.testing.assert_close(m(x), Fn.torch_cross_v2(x, m.u_kernels, m.v_kernels))
        m = CrossV2(16, 2, 4)
        x = torch.randn(3, 16)
        assert Fn.cross_v2_usable(x, m.u_kernels, m.v_kernels)
        assert not Fn.cross_v2_usable(x.double(), m.u_kernels, m.v_kernels)
        m.v_kernels[1].bias = None
        assert not Fn.cross_v2_usable(x, m.u_kernels, m.v_kernels)
    assert be.dcn_v2_calls == 0
    with Fn.use_backend(MetricOracleKernels()):
        assert not Fn.cross_v2_usable(x, CrossV2(16).u_kernels, CrossV2(16).v_kernels)


# ---- the float64 restatement and this repo's CrossV2 against the reference's own ------------------------------------
MOD_TAGS = sorted({k[len("mod_"):-len("_keys")] for k in GOLD.files if k.startswith("mod_") and k.endswith("_keys")})
MODEL_TAGS = sorted({k[len("model_"):-len("_keys")] for k in GOLD.files
                     if k.startswith("model_") and k.endswith("_keys")})


def test_fixture_covers_the_issue_cases():
    assert {tuple(GOLD[f"mod_{t}_shape"]) for t in MOD_TAGS} == {(32, 6, 2), (33, 3, 64), (128, 2, 32), (256, 3, 32)}
    assert set(MODEL_TAGS) == {"test_config", "backbone", "no_deep", "softmax2"}


def _mod_module(tag):
    """CrossV2 of a module case with the reference's initialisation: nn.Linear's default draws after
    torch.manual_seed(0), which the fixture pins by each state entry's sum."""
    pre = f"mod_{tag}_"
    D, L, r = (int(v) for v in GOLD[pre + "shape"])
    torch.manual_seed(0)
    m = CrossV2(D, L, r)
    assert list(m.state_dict()) == list(GOLD[pre + "keys"])
    for k, v in m.state_dict().items():
        np.testing.assert_allclose(float(v.double().sum()), GOLD[pre + "sdsum__" + k], rtol=1e-12, atol=1e-12,
                                   err_msg=k)
    return D, L, r, m


def _mod_weights(tag):
    D, L, r, m = _mod_module(tag)
    sd = lambda k: m.state_dict()[k].double()  # noqa: E731
    wu = torch.stack([sd(f"u_kernels.{i}.weight") for i in range(L)])
    wv = torch.stack([sd(f"v_kernels.{i}.weight") for i in range(L)])
    bias = torch.stack([sd(f"v_kernels.{i}.bias") for i in range(L)])
    return D, L, r, wu, wv, bias


@pytest.mark.parametrize("tag", MOD_TAGS)
def test_restatement_matches_fixture(tag):
    D, L, r, wu, wv, bias = _mod_weights(tag)
    y, dx, dwu, dwv, db = R.grads(torch.from_numpy(GOLD[f"mod_{tag}_x"]).double(), wu, wv, bias,
                                  torch.from_numpy(GOLD[f"mod_{tag}_dout"]).double())
    pre = f"mod_{tag}_"
    np.testing.assert_allclose(y.numpy(), GOLD[pre + "out"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(dx.numpy(), GOLD[pre + "dx"], rtol=1e-12, atol=1e-12)
    for i in range(L):                               # the fixture holds parameter gradients rounded to float32
        for got, k in ((dwu[i], f"u_kernels.{i}.weight"), (dwv[i], f"v_kernels.{i}.weight"),
                       (db[i], f"v_kernels.{i}.bias")):
            _close(got.numpy(), GOLD[pre + "grad__" + k], 1e-7, k)


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("tag", MOD_TAGS)
def test_module_matches_fixture(kern, tag, fused):
    """State-dict keys, output, input gradient and every parameter gradient of this repo's CrossV2 on the torch loop
    and on the fused path (host build of the kernels)."""
    pre = f"mod_{tag}_"
    D, L, r, m = _mod_module(tag)
    assert m.output_dim() == D
    x = torch.from_numpy(GOLD[pre + "x"]).float().requires_grad_(True)
    be = ShimBackend(kern) if fused else MetricOracleKernels()
    with Fn.use_backend(be):
        y = m(x)
        y.backward(torch.from_numpy(GOLD[pre + "dout"]).float())
    if fused:
        assert be.dcn_v2_calls == 2
    _close(_np(y), GOLD[pre + "out"], 1e-5, "out")
    _close(_np(x.grad), GOLD[pre + "dx"], 2e-5, "dx")
    for k, p in m.named_parameters():
        _close(_np(p.grad), GOLD[pre + "grad__" + k], 2e-5, k)


def test_default_init_is_the_reference_linear_init():
    """Linear's default init, as the reference (no reset of its own): same draws for the same seed."""
    torch.manual_seed(0)
    m = CrossV2(33, 3, 64)
    torch.manual_seed(0)
    ref = [torch.nn.Linear(33, 64, bias=False) for _ in range(3)] + [torch.nn.Linear(64, 33) for _ in range(3)]
    for a, b in zip(list(m.u_kernels) + list(m.v_kernels), ref):
        assert torch.equal(a.weight, b.weight)


# ---- the model against the reference's DCNV2 ------------------------------------------------------------------------
def _model_text(D, backbone, cross, deep, final, num_class):
    a = D // 2
    mlp = lambda name, units: f"    {name} {{ hidden_units: {list(units)} }}\n" if units else ""  # noqa: E731
    loss = "binary_cross_entropy {}" if num_class == 1 else "softmax_cross_entropy {}"
    return f"""
feature_configs {{ id_feature {{ feature_name: "f0" num_buckets: 20 embedding_dim: {a} }} }}
feature_configs {{ id_feature {{ feature_name: "f1" num_buckets: 20 embedding_dim: {D - a} }} }}
model_config {{
  feature_groups {{ group_name: "all" feature_names: ["f0", "f1"] group_type: DEEP }}
  dcn_v2 {{
{mlp("backbone", backbone)}    cross {{ cross_num: {cross["cross_num"]} low_rank: {cross["low_rank"]} }}
{mlp("deep", deep)}{mlp("final", final)}  }}
  num_class: {num_class}
  metrics {{ auc {{}} }}
  losses {{ {loss} }}
}}
"""


MODEL_CASES = {
    "test_config": (33, None, dict(cross_num=3, low_rank=64), [8, 4], [2], 1),
    "backbone": (40, [24, 16], dict(cross_num=2, low_rank=8), [12], [8], 1),
    "no_deep": (24, None, dict(cross_num=2, low_rank=4), None, [8, 4], 1),
    "softmax2": (20, [16], dict(cross_num=1, low_rank=6), [8], [6], 2),
}


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("tag", MODEL_TAGS)
def test_model_matches_reference_fixture(kern, tag, fused):
    """State-dict keys, predictions, the loss and every parameter and input gradient of this repo's DCNV2 against
    the reference's DCNV2 in float64, fed the fixture's group features in place of the embedding lookup."""
    cfg = parse_text(_model_text(*MODEL_CASES[tag]))
    feats = create_features(list(cfg.feature_configs))
    torch.manual_seed(0)
    m = create_model(cfg.model_config, feats, ["clk"], device=torch.device("cpu"))
    m.set_sparse_optimizer(SparseOptimizerSpec(kind=OPT_SGD, lr=0.0))
    pre = f"model_{tag}_"
    keys = [k for k in m.state_dict() if not k.startswith("embedding_group")]
    assert keys == list(GOLD[pre + "keys"])
    sd = m.state_dict()
    m.load_state_dict({k: torch.from_numpy(GOLD[pre + "sd__" + k]).to(sd[k].dtype) for k in keys}, strict=False)
    x = torch.from_numpy(GOLD[pre + "x"]).float().requires_grad_(True)
    m.build_input = lambda batch: {"all": x}
    batch = types.SimpleNamespace(labels={"clk": torch.from_numpy(GOLD[pre + "labels"]).float()})
    be = ShimBackend(kern) if fused else MetricOracleKernels()
    m.train()
    with Fn.use_backend(be):
        preds = m.predict(batch)
        losses = m.loss(preds, batch)
        (loss,) = losses.values()
        loss.backward()
    if fused:
        assert be.dcn_v2_calls == 2
    assert set(preds) == {k[len(pre + "pred__"):] for k in GOLD.files if k.startswith(pre + "pred__")}
    for k, v in preds.items():
        _close(_np(v), GOLD[pre + "pred__" + k], 2e-5, k)
    _close(_np(loss), GOLD[pre + "loss"], 2e-5, "loss")
    _close(_np(x.grad), GOLD[pre + "dx"], 5e-5, "d features")
    params = dict(m.named_parameters())
    for k in keys:
        _close(_np(params[k].grad), GOLD[pre + "grad__" + k], 5e-5, k)


# ---- the dcn_v2_taobao config ---------------------------------------------------------------------------------------
DOCS_MODEL_CONFIG = """
model_config {
    feature_groups {
        group_name: "features"
        feature_names: "user_id"
        feature_names: "cms_segid"
        feature_names: "cms_group_id"
        feature_names: "final_gender_code"
        feature_names: "age_level"
        feature_names: "pvalue_level"
        feature_names: "shopping_level"
        feature_names: "occupation"
        feature_names: "new_user_class_level"
        feature_names: "pid"
        feature_names: "adgroup_id"
        feature_names: "cate_id"
        feature_names: "campaign_id"
        feature_names: "customer"
        feature_names: "brand"
        feature_names: "price"
        group_type: DEEP
    }
    dcn_v2 {
        backbone {
            hidden_units: 512
            hidden_units: 256
            hidden_units: 128
        }
        cross {
            cross_num: 2
            low_rank: 32
        }
        deep {
            hidden_units: 512
            hidden_units: 256
        }
        final {
            hidden_units: 128
            hidden_units: 32
        }
    }
    num_class: 1
    metrics {
        auc {}
    }
    losses {
        binary_cross_entropy {}
    }
}
"""


def test_dcn_v2_taobao_is_multi_tower_taobao_with_the_docs_model():
    """The built-in config is examples/multi_tower_taobao.config with its model_config replaced by the block of the
    reference's docs/source/models/dcn_v2.md (above, verbatim), so it is an edited generator."""
    from torcheasyrec_b200.config import load_pipeline_config

    assert "dcn_v2_taobao" in EDITED_GENERATORS and "dcn_v2_taobao" not in GENERATORS
    ours = parse_text(BUILTINS["dcn_v2_taobao"]()).to_dict()
    ref = load_pipeline_config(MULTI_TOWER_EXAMPLE).to_dict()
    docs = parse_text(DOCS_MODEL_CONFIG).to_dict()
    assert ours == dict(ref, model_config=docs["model_config"])


def test_dcn_v2_taobao_trains_and_evaluates(kern):
    """The built-in config stepped on the CPU on the fused path (host build of the kernels): the cross network runs at
    D = 128 (after the backbone), finite falling losses, then evaluate() reports auc and the loss."""
    pipe = Pipeline("dcn_v2_taobao", device="cpu", max_rows=200, seed=3, capturable=False)
    assert type(pipe.model).__name__ == "DCNV2"
    assert pipe.model.cross.output_dim() == 128 and pipe.model.cross.cross_num == 2
    assert pipe.model.embedding_group.group_total_dim("features") == 256
    batch = pipe.synthetic_batch(64, seed=1)
    be = ShimBackend(kern)
    with Fn.use_backend(be):
        ls = [float(pipe.eager_step(batch)) for _ in range(3)]
        m = pipe.evaluate([pipe.synthetic_batch(64, seed=s) for s in range(2)])
    assert np.isfinite(ls).all() and ls[-1] < ls[0], ls
    assert be.dcn_v2_calls == 2 * 3 + 2
    assert set(m) == {"auc", "binary_cross_entropy"}
    assert 0.0 <= m["auc"] <= 1.0 and np.isfinite(m["binary_cross_entropy"])


def test_dcn_v2_taobao_two_ranks_equal_the_unsharded_twin():
    """The config over gloo W = 2 against the unsharded model on the concatenated batch: logits, losses, tables and
    dense weights."""
    from test_distributed_cpu import _run

    _run(2, "dcn_v2_taobao", "mixed", rw_min_rows=250)
