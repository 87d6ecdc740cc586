"""TDM on the CPU: the SOURCE of the fused multi-window DIN kernels (csrc/tzk_tdm.cuh) run on the host through
tests/native/cuda_cpu_shim.h against the float64 restatement (tests/tdm_ref.py), that restatement and this repo's
encoder and model against the reference's own (tests/golden/ref_tdm.npz), the stored example trained and evaluated,
the generated config, and the synthetic batch's shared behaviour-list lengths."""
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
import tdm_ref as R  # noqa: E402
from metric_oracle_backend import MetricOracleKernels  # noqa: E402

from torcheasyrec_b200 import batch as batch_mod  # noqa: E402
from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200._lib import TDM_PRELU, TDM_RELU, TzkTdmArgs  # noqa: E402
from torcheasyrec_b200.config import parse_text  # noqa: E402
from torcheasyrec_b200.engine import Pipeline  # noqa: E402
from torcheasyrec_b200.example_configs import BUILTINS, GENERATORS  # noqa: E402
from torcheasyrec_b200.embedding_modules import SparseOptimizerSpec  # noqa: E402
from torcheasyrec_b200.features import create_features  # noqa: E402
from torcheasyrec_b200.kernels import OPT_SGD  # noqa: E402
from torcheasyrec_b200.rank_models import MultiWindowDINEncoder, create_model  # noqa: E402

NATIVE = os.path.join(HERE, "native")
REF_EXAMPLE = os.path.join(HERE, "golden", "ref_examples", "tdm_taobao.config")
GOLD = np.load(os.path.join(HERE, "golden", "ref_tdm.npz"))
EXAMPLE_WINDOWS = [1, 1, 1, 2, 2, 2, 5, 6, 10, 20]


# ---- the kernel source on the host ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kern(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("shim") / "libtdm_cpu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", NATIVE,
                    "-x", "c++", os.path.join(NATIVE, "tdm_standalone.cu"), "-shared", "-fPIC", "-o", out],
                   check=True)
    L = ctypes.CDLL(out)
    P, I32 = ctypes.c_void_p, ctypes.c_int
    L.tdm_check.argtypes = [P, I32]
    L.tdm_param_floats.argtypes = [P]
    L.tdm_param_floats.restype = ctypes.c_int64
    L.tdm_fwd.argtypes = [P, I32]
    L.tdm_bwd.argtypes = [P, I32, P, P]
    return L


class ShimTdm:
    """tdm_fwd / tdm_bwd of kernels.CudaKernels on CPU tensors, computed by the host build of the kernel source.
    Grids: fixed ones, or min(work, 3) as a small stand-in for the device's."""

    def __init__(self, L, grid_fwd=None, grid_bwd=None):
        self.L, self.grid_fwd, self.grid_bwd, self.calls = L, grid_fwd, grid_bwd, 0

    @staticmethod
    def args(query, seq, offsets, layers, lin_w, lin_b, act_w, windows, prelu):
        a = TzkTdmArgs()
        a.B, a.Dq = query.shape
        a.N, a.C = seq.shape
        a.L, a.n_layers, a.act = len(windows), len(layers), TDM_PRELU if prelu else TDM_RELU
        for w, n in enumerate(windows):
            a.windows[w] = int(n)
        for l, (W, b, s) in enumerate(layers):
            a.hidden[l], a.w[l], a.b[l] = W.shape[0], W.data_ptr(), b.data_ptr()
            if s is not None:
                a.slope[l] = s.data_ptr()
        a.seq, a.offsets, a.query = seq.data_ptr(), offsets.data_ptr(), query.data_ptr()
        a.lin_w, a.lin_b, a.act_w = lin_w.data_ptr(), lin_b.data_ptr(), act_w.data_ptr()
        return a

    @staticmethod
    def _prep(query, seq, layers, lin_w, lin_b, act_w):
        f = lambda t: None if t is None else t.detach().float().contiguous()  # noqa: E731
        return (f(query), f(seq), [tuple(f(t) for t in l) for l in layers], f(lin_w), f(lin_b), f(act_w))

    def tdm_fwd(self, query, seq, offsets, layers, lin_w, lin_b, act_w, windows, prelu):
        self.calls += 1
        query, seq, layers, lin_w, lin_b, act_w = self._prep(query, seq, layers, lin_w, lin_b, act_w)
        self._keep = (query, seq, layers, lin_w, lin_b, act_w)
        a = self.args(query, seq, offsets, layers, lin_w, lin_b, act_w, windows, prelu)
        out = torch.empty(a.B, (a.L + 1) * a.C)
        z = torch.empty(a.N)
        a.out, a.z = out.data_ptr(), z.data_ptr()
        grid = self.grid_fwd or max(1, min(-(-a.B // 8), 3))
        assert self.L.tdm_fwd(ctypes.byref(a), grid) == 0
        return out, z

    def tdm_bwd(self, query, seq, offsets, layers, lin_w, lin_b, act_w, windows, prelu, z, d_out):
        self.calls += 1
        query, seq, layers, lin_w, lin_b, act_w = self._prep(query, seq, layers, lin_w, lin_b, act_w)
        d_out = d_out.float().contiguous()
        a = self.args(query, seq, offsets, layers, lin_w, lin_b, act_w, windows, prelu)
        d_query, d_seq = torch.empty_like(query), torch.empty_like(seq)
        a.z, a.d_out, a.d_seq, a.d_query = z.data_ptr(), d_out.data_ptr(), d_seq.data_ptr(), d_query.data_ptr()
        Pn = self.L.tdm_param_floats(ctypes.byref(a))
        grid = self.grid_bwd or max(1, min(a.B, 3))
        partials, dparams = torch.empty(grid, Pn), torch.empty(Pn)
        assert self.L.tdm_bwd(ctypes.byref(a), grid, partials.data_ptr(), dparams.data_ptr()) == 0
        grads, o = [], 0
        for W, b, s in layers:
            n = W.numel()
            grads.append((dparams[o:o + n].view_as(W), dparams[o + n:o + n + b.numel()],
                          dparams[o + n + b.numel():o + n + b.numel() + 1] if prelu else None))
            o += n + b.numel() + int(prelu)
        H = lin_w.numel()
        return d_query, d_seq, grads, dparams[o:o + H].view_as(lin_w), dparams[o + H:o + H + 1], \
            dparams[o + H + 1:o + H + 2]


class ShimBackend(MetricOracleKernels):
    """The CPU checker backend with the TDM attention computed by the host build of its kernel source."""

    def __init__(self, L):
        super().__init__()
        self._tdm = ShimTdm(L)
        self.tdm_fwd = self._tdm.tdm_fwd
        self.tdm_bwd = self._tdm.tdm_bwd

    @property
    def tdm_calls(self):
        return self._tdm.calls


def _close(got, want, r, name):
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(np.asarray(got, np.float64), want, rtol=r,
                               atol=r * max(1.0, np.abs(want).max() if want.size else 1.0), err_msg=name)


def _np(t):
    return t.detach().double().numpy()


def _reference(case, dout_seed=0):
    """float64 padded formulation of a tdm_ref.case: (out, dout, d_query, d_seq rows, [param grads in dparams order])."""
    q, seq, off, layers, lw, lb, aw = case
    seqp, lens = R.pad_rows(seq, off, T=max(int((off[1:] - off[:-1]).max()) if len(off) > 1 else 0, 1))
    kind = "relu" if layers[0][2] is None else "prelu"
    leaves = [q, seqp, lw, lb, aw] + [t for l in layers for t in l if t is not None]
    for t in leaves:
        t.requires_grad_(True)
    out = R.multiwindow_din(q, seqp, lens, WINDOWS[0], layers, kind, lw, lb, aw)
    dout = torch.from_numpy(np.random.default_rng(dout_seed).standard_normal(tuple(out.shape)))
    out.backward(dout)
    d_rows = torch.cat([seqp.grad[b, :int(off[b + 1] - off[b])] for b in range(len(off) - 1)] +
                       [torch.zeros(0, seq.shape[1], dtype=torch.float64)])
    grads = []
    for W, b, s in layers:
        grads += [W.grad, b.grad] + ([s.grad] if s is not None else [])
    grads += [lw.grad, lb.grad, aw.grad]
    for t in leaves:
        t.requires_grad_(False)
    return out.detach(), dout, q.grad, d_rows, grads


WINDOWS = [None]


def _run_shim(L, case, dout, windows, gf, gb):
    q, seq, off, layers, lw, lb, aw = case
    prelu = layers[0][2] is not None
    s = ShimTdm(L, gf, gb)
    offs = torch.from_numpy(np.asarray(off, np.int64))
    out, z = s.tdm_fwd(q, seq, offs, layers, lw.reshape(1, -1), lb, aw, windows, prelu)
    d_q, d_seq, grads, d_lw, d_lb, d_aw = s.tdm_bwd(q, seq, offs, layers, lw.reshape(1, -1), lb, aw, windows, prelu,
                                                     z, dout.float())
    flat = []
    for dw, db, ds in grads:
        flat += [dw, db] + ([ds] if prelu else [])
    return out, z, d_q, d_seq, flat + [d_lw.reshape(-1), d_lb, d_aw]


# (C, Dq, hidden, kind, windows, B, max_len, lengths, grids)
KERNEL_CASES = {
    "example_prelu": (48, 48, [36], "prelu", EXAMPLE_WINDOWS, 11, 70, None, (2, 3)),
    "one_layer_relu": (16, 16, [8], "relu", [1, 2, 5], 9, 12, None, (1, 1)),
    "two_layers_relu_dq": (16, 12, [8, 4], "relu", [1, 2, 5], 10, 11, None, (3, 4)),
    "three_layers_prelu": (8, 8, [8, 4, 2], "prelu", [2, 3], 12, 9, None, (5, 12)),
    "wide_units": (32, 20, [64, 33], "prelu", [3, 1, 4], 6, 10, None, (1, 2)),
    "crop_beyond_s": (12, 12, [6], "relu", [1, 2], 5, 0, [7, 3, 0, 3, 9], (2, 5)),
    "all_zero_lengths": (8, 8, [4], "prelu", [1, 1], 6, 0, [0] * 6, (2, 3)),
    "empty_batch": (8, 8, [4], "relu", [2], 0, 0, [], (1, 1)),
}


@pytest.mark.parametrize("tag", list(KERNEL_CASES))
def test_kernel_source_against_float64(kern, tag):
    """Forward and every gradient of both kernels against the padded formulation in float64, over the cover's
    corners: 1/2/3 layers, ReLU and PReLU, Dq < C, 64-unit layers, rows cropped beyond S, all-zero lengths, an empty
    batch; grids of one CTA, of several, and larger than the work."""
    C, Dq, hidden, kind, windows, B, mx, lengths, grids = KERNEL_CASES[tag]
    case = R.case(len(tag), B, C, Dq, hidden, windows, kind, mx, lengths)
    WINDOWS[0] = windows
    out_r, dout, dq_r, dseq_r, grads_r = _reference(case)
    out, _, dq, dseq, grads = _run_shim(kern, case, dout, windows, *grids)
    _close(_np(out), out_r, 1e-5, "out")
    _close(_np(dq), dq_r, 1e-5, "d_query")
    _close(_np(dseq), dseq_r, 1e-5, "d_seq")
    assert len(grads) == len(grads_r)
    for i, (g, r) in enumerate(zip(grads, grads_r)):
        _close(_np(g).reshape(-1), _np(r).reshape(-1), 2e-5, f"dparam{i}")
    if tag == "empty_batch":
        assert all(float(g.abs().sum()) == 0 for g in grads)


@pytest.mark.parametrize("grids", [(2, 3), (4, 7)])
def test_kernel_source_reruns_bit_identical(kern, grids):
    case = R.case(9, 23, 16, 16, [8, 4], EXAMPLE_WINDOWS[:5], "prelu", 9)
    dout = torch.randn(23, 6 * 16, generator=torch.Generator().manual_seed(1))
    a = _run_shim(kern, case, dout, EXAMPLE_WINDOWS[:5], *grids)
    b = _run_shim(kern, case, dout, EXAMPLE_WINDOWS[:5], *grids)
    for x, y in zip(torch.utils._pytree.tree_leaves(a), torch.utils._pytree.tree_leaves(b)):
        assert torch.equal(x, y)


def test_kernel_source_refuses_outside_cover(kern):
    q, seq, off, layers, lw, lb, aw = R.case(1, 4, 16, 16, [8], [1, 2], "relu", 3)
    f = lambda t: t.float().contiguous()  # noqa: E731
    layers = [(f(W), f(b), None) for W, b, _ in layers]
    offs = torch.from_numpy(off)
    ok = ShimTdm.args(f(q), f(seq), offs, layers, f(lw), f(lb), f(aw), [1, 2], False)
    ok.out, ok.z = 1, 1
    assert kern.tdm_check(ctypes.byref(ok), 0) == 0
    for field, value in (("C", 18), ("C", 132), ("Dq", 20), ("n_layers", 4), ("L", 33)):
        a = ShimTdm.args(f(q), f(seq), offs, layers, f(lw), f(lb), f(aw), [1, 2], False)
        a.out, a.z = 1, 1
        setattr(a, field, value)
        assert kern.tdm_check(ctypes.byref(a), 0) == 1, field
    a = ShimTdm.args(f(q), f(seq), offs, layers, f(lw), f(lb), f(aw), [200, 57], False)     # S = 257
    a.out, a.z = 1, 1
    assert kern.tdm_check(ctypes.byref(a), 0) == 1
    a.hidden[0] = 65
    assert kern.tdm_check(ctypes.byref(a), 0) == 1


# ---- the float64 restatement and this repo's encoder against the reference's own ------------------------------------
ENC_TAGS = sorted({k.split("_keys")[0][len("enc_"):] for k in GOLD.files if k.startswith("enc_") and
                   k.endswith("_keys")})


def _gold_case(tag):
    pre = f"enc_{tag}_"
    lengths = GOLD[pre + "lengths"]
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    seqp = GOLD[pre + "seq"]
    rows = np.concatenate([seqp[b, :n] for b, n in enumerate(lengths)] + [np.zeros((0, seqp.shape[2]))])
    return pre, lengths, off, rows


def test_fixture_covers_the_issue_cases():
    assert set(ENC_TAGS) == {"example", "w125_relu84", "relu842", "dq_lt_c"}
    lens = GOLD["enc_example_lengths"]
    assert {0, 1, 50}.issubset(set(lens.tolist())) and lens.max() > 50


@pytest.mark.parametrize("tag", ENC_TAGS)
def test_restatement_matches_fixture(tag):
    pre, lengths, off, _ = _gold_case(tag)
    t = lambda k: torch.from_numpy(GOLD[pre + k])  # noqa: E731
    kind = "prelu" if str(GOLD[pre + "act"]) == "nn.PReLU" else "relu"
    n = len(GOLD[pre + "hidden"])
    layers = [(t(f"sd__mlp.mlp.{i}.perceptron.0.weight"), t(f"sd__mlp.mlp.{i}.perceptron.0.bias"),
               t(f"sd__mlp.mlp.{i}.perceptron.1.weight") if kind == "prelu" else None) for i in range(n)]
    out = R.multiwindow_din(t("query"), t("seq"), torch.from_numpy(lengths), list(GOLD[pre + "windows"]), layers, kind,
                            t("sd__linear.weight"), t("sd__linear.bias"), t("sd__active.weight"))
    np.testing.assert_allclose(out.numpy(), GOLD[pre + "out"], rtol=1e-12, atol=1e-12)


def _encoder(tag):
    pre = f"enc_{tag}_"
    C, Dq = GOLD[pre + "seq"].shape[2], GOLD[pre + "query"].shape[1]
    enc = MultiWindowDINEncoder(C, Dq, "seq", list(GOLD[pre + "windows"]),
                                dict(hidden_units=list(GOLD[pre + "hidden"]), activation=str(GOLD[pre + "act"])))
    assert list(enc.state_dict()) == list(GOLD[pre + "keys"])
    enc.load_state_dict({k: torch.from_numpy(GOLD[pre + "sd__" + k]).to(v.dtype) for k, v in enc.state_dict().items()})
    return enc


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("tag", ENC_TAGS)
def test_encoder_matches_fixture(kern, tag, fused):
    """State-dict keys (buffers included), output, d query, d sequence rows and every parameter gradient of this
    repo's encoder over jagged rows, on the torch formulation and on the fused path (host build of the kernels)."""
    pre, lengths, off, rows = _gold_case(tag)
    enc = _encoder(tag)
    q = torch.from_numpy(GOLD[pre + "query"]).float().requires_grad_(True)
    seq = torch.from_numpy(rows).float().requires_grad_(True)
    emb = {"seq.query": q, "seq.sequence": seq, "seq.sequence_length": torch.from_numpy(lengths),
           "seq.sequence_offsets": torch.from_numpy(off)}
    be = ShimBackend(kern) if fused else MetricOracleKernels()
    with Fn.use_backend(be):
        out = enc(emb)
        out.backward(torch.from_numpy(GOLD[pre + "dout"]).float())
    if fused:
        assert be.tdm_calls == 2
    _close(_np(out), GOLD[pre + "out"], 2e-5, "out")
    _close(_np(q.grad), GOLD[pre + "dquery"], 2e-5, "d_query")
    dseq = GOLD[pre + "dseq"]
    _close(_np(seq.grad), np.concatenate([dseq[b, :n] for b, n in enumerate(lengths)]), 2e-5, "d_seq")
    for k, p in enc.named_parameters():
        _close(_np(p.grad), GOLD[pre + "grad__" + k], 5e-5, k)


def test_padded_form_matches_fixture():
    """The encoder's padded [B, T, C] path (no offsets) is the reference's formulation."""
    tag = "example"
    pre = f"enc_{tag}_"
    enc = _encoder(tag).double()
    out = enc({"seq.query": torch.from_numpy(GOLD[pre + "query"]), "seq.sequence": torch.from_numpy(GOLD[pre + "seq"]),
               "seq.sequence_length": torch.from_numpy(GOLD[pre + "lengths"])})
    np.testing.assert_allclose(out.detach().numpy(), GOLD[pre + "out"], rtol=1e-10, atol=1e-10)


def test_query_wider_than_sequence_raises():
    with pytest.raises(ValueError, match="query_dim > sequence_dim"):
        MultiWindowDINEncoder(8, 12, "seq", [1, 2], dict(hidden_units=[4]))


# ---- the model against the reference's TDM ------------------------------------------------------------------------
TDM_SMALL = """
feature_configs { id_feature { feature_name: "user_id" num_buckets: 20 embedding_dim: 8 } }
feature_configs { id_feature { feature_name: "pid" num_buckets: 20 embedding_dim: 8 } }
feature_configs { sequence_id_feature { feature_name: "click_seq__item" sequence_length: 20 num_buckets: 30
                                        embedding_dim: 8 embedding_name: "item_emb" } }
feature_configs { sequence_id_feature { feature_name: "click_seq__cate" sequence_length: 20 num_buckets: 10
                                        embedding_dim: 8 embedding_name: "cate_emb" } }
feature_configs { id_feature { feature_name: "item" num_buckets: 30 embedding_dim: 8 embedding_name: "item_emb" } }
feature_configs { id_feature { feature_name: "cate" num_buckets: 10 embedding_dim: 8 embedding_name: "cate_emb" } }
feature_configs { id_feature { feature_name: "price" num_buckets: 10 embedding_dim: 8 } }
model_config {
  feature_groups { group_name: "seq" feature_names: ["click_seq__item", "click_seq__cate", "item", "cate"]
                   group_type: SEQUENCE }
  feature_groups { group_name: "user" feature_names: ["user_id", "pid"] group_type: DEEP }
  feature_groups { group_name: "item" feature_names: ["price"] group_type: DEEP }
  tdm {
    multiwindow_din { windows_len: [1, 2, 5] attn_mlp { hidden_units: [12] activation: "nn.PReLU" } }
    final { hidden_units: [16, 8] use_bn: true }
  }
  num_class: 2
  metrics { auc {} }
  losses { softmax_cross_entropy {} }
}
"""


def _model(text):
    cfg = parse_text(text)
    feats = create_features(list(cfg.feature_configs))
    torch.manual_seed(0)
    m = create_model(cfg.model_config, feats, ["clk"], device=torch.device("cpu"))
    m.set_sparse_optimizer(SparseOptimizerSpec(kind=OPT_SGD, lr=0.0))
    return m, feats


@pytest.mark.parametrize("fused", [False, True])
def test_model_matches_reference_fixture(kern, fused):
    """State-dict keys, logits / probs / probs1, the softmax cross-entropy and every parameter and input gradient of
    this repo's TDM against the reference's TDM in float64, fed the fixture's grouped features (the sequence as jagged
    rows) in place of the embedding lookup."""
    m, _ = _model(TDM_SMALL)
    keys = [k for k in m.state_dict() if not k.startswith("embedding_group")]
    assert keys == list(GOLD["tdm_keys"])
    sd = m.state_dict()
    m.load_state_dict({k: torch.from_numpy(GOLD["tdm_sd__" + k]).to(sd[k].dtype) for k in keys}, strict=False)
    lengths = GOLD["tdm_in__seq.sequence_length"]
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    seqp = GOLD["tdm_in__seq.sequence"]
    ins = {"seq.query": torch.from_numpy(GOLD["tdm_in__seq.query"]).float().requires_grad_(True),
           "seq.sequence": torch.from_numpy(np.concatenate([seqp[b, :n] for b, n in enumerate(lengths)])).float()
           .requires_grad_(True),
           "user": torch.from_numpy(GOLD["tdm_in__user"]).float().requires_grad_(True),
           "item": torch.from_numpy(GOLD["tdm_in__item"]).float().requires_grad_(True)}
    grouped = dict(ins, **{"seq.sequence_length": torch.from_numpy(lengths),
                           "seq.sequence_offsets": torch.from_numpy(off)})
    m.build_input = lambda batch: grouped
    batch = types.SimpleNamespace(labels={"clk": torch.from_numpy(GOLD["tdm_labels"]).float()})
    be = ShimBackend(kern) if fused else MetricOracleKernels()
    m.train()
    with Fn.use_backend(be):
        preds = m.predict(batch)
        losses = m.loss(preds, batch)
        losses["softmax_cross_entropy"].backward()
    assert list(preds) == ["logits", "probs", "probs1"] and list(losses) == ["softmax_cross_entropy"]
    for k, v in preds.items():
        _close(_np(v), GOLD["tdm_pred__" + k], 2e-5, k)
    _close(_np(losses["softmax_cross_entropy"]), GOLD["tdm_loss"], 2e-5, "loss")
    for k, v in ins.items():
        want = GOLD["tdm_din__" + k]
        if k == "seq.sequence":
            want = np.concatenate([want[b, :n] for b, n in enumerate(lengths)])
        _close(_np(v.grad), want, 5e-5, "d " + k)
    params = dict(m.named_parameters())
    for k in keys:
        if k in params:
            _close(_np(params[k].grad), GOLD["tdm_grad__" + k], 5e-5, k)
    if fused:
        assert be.tdm_calls == 2


# ---- the reference example ----------------------------------------------------------------------------------------
def test_generated_config_equals_the_stored_example():
    from torcheasyrec_b200.config import load_pipeline_config

    ours = parse_text(GENERATORS["tdm_taobao"]())
    ref = load_pipeline_config(REF_EXAMPLE)
    assert ours.to_dict() == ref.to_dict()
    assert ref.data_config.tdm_sampler.item_id_field == "adgroup_id"


def test_reference_example_trains_and_evaluates(kern):
    """The stored example stepped on the CPU on the fused path (host build of the kernels): finite falling losses,
    then evaluate() reports auc and the softmax cross-entropy."""
    pipe = Pipeline(REF_EXAMPLE, device="cpu", max_rows=200, seed=3, capturable=False)
    assert type(pipe.model).__name__ == "TDM"
    assert pipe.model.multiwindow_din.output_dim() == 48 * 11
    batch = pipe.synthetic_batch(64, seed=1)
    be = ShimBackend(kern)
    with Fn.use_backend(be):
        ls = [float(pipe.eager_step(batch)) for _ in range(2)]
        m = pipe.evaluate([pipe.synthetic_batch(64, seed=s) for s in range(2)])
    assert np.isfinite(ls).all() and ls[-1] < ls[0]
    assert be.tdm_calls == 2 * 2 + 2
    assert set(m) == {"auc", "softmax_cross_entropy"}
    assert 0.0 <= m["auc"] <= 1.0 and np.isfinite(m["softmax_cross_entropy"])


def test_reference_example_steps_with_the_oracle_backend():
    pipe = Pipeline(REF_EXAMPLE, device="cpu", max_rows=200, seed=3, capturable=False)
    batch = pipe.synthetic_batch(64, seed=2)
    with Fn.use_backend(MetricOracleKernels()):
        ls = [float(pipe.eager_step(batch)) for _ in range(2)]
    assert np.isfinite(ls).all() and ls[1] < ls[0]


# ---- the synthetic batch: one length per behaviour list -------------------------------------------------------------
def test_example_sequences_share_one_length():
    pipe = Pipeline(REF_EXAMPLE, device="cpu", max_rows=50, seed=3, capturable=False)
    b = pipe.synthetic_batch(300, seed=4)
    lens = {}
    for kjt in b.sparse_features.values():
        for k, jt in kjt.to_dict().items():
            if k.startswith("click_50_seq__"):
                lens[k] = jt.lengths()
    assert len(lens) == 3
    first = next(iter(lens.values()))
    assert all(torch.equal(first, v) for v in lens.values())
    assert int(first.max()) == 50 and int(first.min()) == 0


@pytest.mark.parametrize("name", sorted(n for n in BUILTINS if n != "tdm_taobao"))
def test_existing_synthetic_batches_unchanged(name, monkeypatch):
    """Every other built-in config's batch is bit-identical to the one drawn with each sequence feature on its own,
    as before behaviour lists shared a draw."""
    pipe = Pipeline(name, device="cpu", max_rows=50, seed=3, capturable=False)
    new = pipe.synthetic_batch(64, seed=5)
    monkeypatch.setattr(batch_mod, "_behaviour_list", lambda n, feats: n)
    old = pipe.synthetic_batch(64, seed=5)
    for dg in old.sparse_features:
        a, b = old.sparse_features[dg], new.sparse_features[dg]
        assert a.keys() == b.keys()
        assert torch.equal(a.values(), b.values()) and torch.equal(a.lengths(), b.lengths())
    for k in old.labels:
        assert torch.equal(old.labels[k], new.labels[k])


# ---- data parallelism over gloo --------------------------------------------------------------------------------------
def test_tdm_taobao_two_ranks_equal_the_unsharded_twin(tmp_path):
    """The example over gloo W = 2 against the unsharded model on the concatenated batch: logits, losses, tables and
    dense weights.  deep_mlp's BatchNorm normalises over each rank's own samples in data-parallel training (as under
    the reference's DDP), which no single-process twin reproduces, so this runs the example with use_bn off."""
    from test_distributed_cpu import _run

    text = open(REF_EXAMPLE).read()
    assert "use_bn: True" in text
    path = tmp_path / "tdm_taobao_no_bn.config"
    path.write_text(text.replace("use_bn: True", "use_bn: False"))
    _run(2, str(path), "mixed", rw_min_rows=250)
