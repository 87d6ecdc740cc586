"""PLE on the CPU: the float64 restatement (tests/ple_ref.py) pinned to the reference's own ExtractionNet stacked as PLE
stacks it (tests/golden/ref_ple.npz, made by tests/golden/make_ple_golden.py), the SOURCE of the fused gate kernels
(csrc/tzk_ple.cuh) run on the host through tests/native/cuda_cpu_shim.h against the restatement, and the model:
reference parameter names, the replay of tzrec/models/ple_test.py, the reference example trained unchanged, training and
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
import ple_ref as R  # noqa: E402
from oracle_backend import OracleKernels  # noqa: E402
from ple_oracle_backend import PleOracleKernels  # noqa: E402

from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200._lib import TzkPleGateArgs  # noqa: E402
from torcheasyrec_b200.batch import Batch  # noqa: E402
from torcheasyrec_b200.config import parse_text  # noqa: E402
from torcheasyrec_b200.embedding_modules import SparseOptimizerSpec  # noqa: E402
from torcheasyrec_b200.engine import Pipeline  # noqa: E402
from torcheasyrec_b200.features import create_features  # noqa: E402
from torcheasyrec_b200.kernels import OPT_ADAGRAD  # noqa: E402
from torcheasyrec_b200.rank_models import ExtractionNet, create_model  # noqa: E402
from torcheasyrec_b200.sparse import KeyedJaggedTensor, KeyedTensor  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "ref_ple.npz"))
CASES = list(R.CASES)
REF_EXAMPLE = os.path.join(HERE, "golden", "ref_examples", "ple_taobao.config")
NATIVE = os.path.join(HERE, "native")


def _close(got, want, r, name=""):
    """|got - want| <= r (|want| + max(1, max |want|)): relative to the tensor's scale."""
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(np.asarray(got, np.float64), want, rtol=r, atol=r * max(1.0, np.abs(want).max()),
                               err_msg=name)


def _gold(tag, what):
    n = sum(1 for k in GOLD.files if k.startswith(f"{tag}_{what}"))
    return [GOLD[f"{tag}_{what}{i}"] for i in range(n)]


# ---- the restatement and this repo's layers, pinned to the reference's ------------------------------------------------
@pytest.mark.parametrize("tag", CASES)
def test_restatement_matches_reference_module(tag):
    sd, inputs, dys = R.seeded_case(tag)
    outs, dxs, grads = R.stack(tag, sd, inputs, dys)
    for i, (o, g) in enumerate(zip(outs, _gold(tag, "out"))):
        _close(o, g, 1e-5, f"out{i}")
    for i, (d, g) in enumerate(zip(dxs, _gold(tag, "dx"))):
        _close(d, g, 1e-5, f"dx{i}")
    pre = f"{tag}_grad__"
    assert {k[len(pre):] for k in GOLD.files if k.startswith(pre)} == set(grads)
    for name, g in grads.items():
        _close(g, GOLD[pre + name], 1e-5, name)
    assert R.ordered_keys(tag) == list(GOLD[f"{tag}_keys"])


def _layers(tag):
    case = R.CASES[tag]
    nets = nn.ModuleList()
    for (per, S, tu, su), (ins, shared_dim, final) in zip(case[4], R.layer_dims(case)):
        nets.append(ExtractionNet(ins, shared_dim, network_name="layer", share_num=S, expert_num_per_task=per,
                                  share_expert_net={"hidden_units": su}, task_expert_net={"hidden_units": tu},
                                  final_flag=final))
    return nets


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("tag", CASES)
def test_layers_match_reference_module(tag, fused):
    """This repo's ExtractionNet stack with the reference's state dict: same keys, same outputs and gradients; with the
    checker backend the gates run through the fused autograd path (one forward and one backward call per layer)."""
    case = R.CASES[tag]
    nets = _layers(tag)
    assert list(nets.state_dict()) == list(GOLD[f"{tag}_keys"])
    sd, inputs, dys = R.seeded_case(tag)
    nets.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    xs = [torch.from_numpy(x).requires_grad_(True) for x in inputs]
    T = len(case[1])
    task_in, shared_in = ([xs[0]] * T, xs[0]) if case[3] else (xs[:T], xs[T])
    be = PleOracleKernels() if fused else OracleKernels()
    with Fn.use_backend(be):
        for net in nets:
            task_in, shared_in = net(task_in, shared_in)
        outs = list(task_in) + ([] if shared_in is None else [shared_in])
        torch.autograd.backward(outs, [torch.from_numpy(d) for d in dys])
    assert getattr(be, "ple_calls", 0) == (2 * len(nets) if fused else 0)
    assert (shared_in is None) == case[5]
    for i, (o, g) in enumerate(zip(outs, _gold(tag, "out"))):
        _close(o.detach().numpy(), g, 1e-5, f"out{i}")
    for i, (x, g) in enumerate(zip(xs, _gold(tag, "dx"))):
        _close(x.grad.numpy(), g, 1e-5, f"dx{i}")
    for name, p in nets.named_parameters():
        _close(p.grad.numpy(), GOLD[f"{tag}_grad__{name}"], 1e-5, name)


def test_missing_share_expert_net_fails_as_in_the_reference():
    cfg = parse_text(PLE_TEST_CONFIG.replace("share_expert_net { hidden_units: [12, 6] }", ""))
    with pytest.raises(TypeError, match="share_expert_net"):
        create_model(cfg.model_config, create_features(list(cfg.feature_configs)), ["label1", "label2"],
                     device=torch.device("cpu"))


# ---- the kernel source on the host ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kern(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("shim") / "libple_cpu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", NATIVE,
                    "-x", "c++", os.path.join(NATIVE, "ple_standalone.cu"), "-shared", "-fPIC", "-o", out],
                   check=True)
    L = ctypes.CDLL(out)
    P, I32 = ctypes.c_void_p, ctypes.c_int
    L.ple_smem_bytes.argtypes = [P, I32]
    L.ple_smem_bytes.restype = ctypes.c_int64
    L.ple_gate_fwd.argtypes = [P, I32, P, P]
    L.ple_gate_bwd.argtypes = [P, P, P, I32, P, P, P]
    return L


def _f32(rng, *shape, scale=1.0):
    return (rng.standard_normal(shape) * scale).astype(np.float32)


def _args(B, H, inputs, gate_input, weights, biases, experts, gate_experts, d_inputs=()):
    a = TzkPleGateArgs()
    a.B, a.H, a.n_experts, a.n_inputs, a.n_gates = B, H, len(experts), len(inputs), len(gate_input)
    for i, x in enumerate(inputs):
        a.in_dim[i], a.inputs[i] = x.shape[1], x.ctypes.data
    for i, d in enumerate(d_inputs):
        a.d_inputs[i] = d.ctypes.data
    for j, e in enumerate(experts):
        a.experts[j] = e.ctypes.data
    for g, ids in enumerate(gate_experts):
        a.gate_input[g], a.gate_num_experts[g] = gate_input[g], len(ids)
        for e, x in enumerate(ids):
            a.gate_experts[g][e] = x
        a.weight[g], a.bias[g] = weights[g].ctypes.data, biases[g].ctypes.data
    return a


def _run_layer(L, B, H, in_dims, gate_input, gate_experts, n_experts, grid, seed):
    rng = np.random.default_rng(seed)
    inputs = [_f32(rng, B, k) for k in in_dims]
    experts = [_f32(rng, B, H) for _ in range(n_experts)]
    weights = [_f32(rng, len(ids), in_dims[gate_input[g]], scale=0.3) for g, ids in enumerate(gate_experts)]
    biases = [_f32(rng, len(ids), scale=0.3) for ids in gate_experts]
    G, sumE = len(gate_input), sum(len(ids) for ids in gate_experts)
    a = _args(B, H, inputs, gate_input, weights, biases, experts, gate_experts)
    y, p = np.full((G, B, H), np.nan, np.float32), np.full((B, sumE), np.nan, np.float32)
    assert L.ple_gate_fwd(ctypes.byref(a), grid, y.ctypes.data, p.ctypes.data) == 0
    ry, rp = R.gates_fwd(inputs, gate_input, weights, biases, experts, gate_experts)
    _close(y, ry, 1e-5, "y")
    _close(p, rp, 1e-5, "p")
    dy = _f32(rng, G, B, H)
    dx = [np.full((B, k), np.nan, np.float32) for k in in_dims]
    a = _args(B, H, inputs, gate_input, weights, biases, experts, gate_experts, dx)
    P_ = sum(w.size for w in weights) + sumE
    dex = np.full((n_experts, B, H), np.nan, np.float32)
    part, dpar = np.full((grid, P_), np.nan, np.float32), np.empty(P_, np.float32)
    assert L.ple_gate_bwd(ctypes.byref(a), p.ctypes.data, dy.ctypes.data, grid, dex.ctypes.data, part.ctypes.data,
                          dpar.ctypes.data) == 0
    rdx, rdex, rdW, rdb = R.gates_bwd(inputs, gate_input, weights, biases, experts, gate_experts, dy)
    for i in range(len(in_dims)):
        _close(dx[i], rdx[i], 2e-5, f"dx{i}")
    _close(dex, rdex, 2e-5, "d_experts")
    _close(dpar, np.concatenate([w.ravel() for w in rdW] + rdb), 2e-5, "dW | db")
    want = np.zeros(P_, np.float32)
    for row in part:
        want += row
    np.testing.assert_array_equal(dpar, want)


def _taobao_layer(l, T=2):
    """ple_taobao layer l's gates: (in_dims, gate_input, gate_experts, n_experts, H); one input in layer 1."""
    per, K, H = [(2, 256, 256), (3, 256, 64), (4, 64, 32)][l]
    S = per
    task = [list(range(i * per, (i + 1) * per)) + list(range(T * per, T * per + S)) for i in range(T)]
    if l == 0:
        return [K], [0, 0, 0], task + [list(range(T * per + S))], T * per + S, H
    if l == 1:
        return [K] * (T + 1), [1, 2, 0], task + [list(range(T * per + S))], T * per + S, H
    return [K] * T, [0, 1], task, T * per + S, H


@pytest.mark.parametrize("layer", [0, 1, 2])
@pytest.mark.parametrize("B", [1, 3])
def test_kernel_source_taobao_layers(kern, layer, B):
    in_dims, gi, ge, ne, H = _taobao_layer(layer)
    _run_layer(kern, B, H, in_dims, gi, ge, ne, grid=B, seed=10 * layer + B)


def test_kernel_source_odd_widths_distinct_inputs(kern):
    """The reference's module test: task inputs 16 / 15 / 14, shared 13, H = 4 (here 5: odd), a shared gate over 13."""
    task = [list(range(i * 3, i * 3 + 3)) + list(range(9, 13)) for i in range(3)]
    _run_layer(kern, 3, 5, [13, 16, 15, 14], [1, 2, 3, 0], task + [list(range(13))], 13, grid=2, seed=3)


def test_kernel_source_32_experts_per_gate(kern):
    """E_g = 32 (the lane-per-logit limit) next to a gate of 1, odd K and H, aliased input."""
    _run_layer(kern, 3, 33, [37], [0, 0], [list(range(32)), [31]], 32, grid=3, seed=4)


def test_kernel_source_grid_stride(kern):
    """B = 257 on 5 CTAs: every CTA walks several 16-sample tiles and the batch sums add 5 partial rows."""
    in_dims, gi, ge, ne, _ = _taobao_layer(1)
    _run_layer(kern, 257, 7, [19] * 3, gi, ge, ne, grid=5, seed=5)


def test_kernel_source_empty_batch_zeroes_dparams(kern):
    """B = 0: no backward kernel runs and the batch sums add no partial rows, so dparams comes back all zeros."""
    in_dims, gi, ge, ne, H = _taobao_layer(1)
    grid = 5
    inputs = [np.zeros((0, k), np.float32) for k in in_dims]
    weights = [np.zeros((len(ids), in_dims[gi[g]]), np.float32) for g, ids in enumerate(ge)]
    biases = [np.zeros(len(ids), np.float32) for ids in ge]
    experts = [np.zeros((0, H), np.float32) for _ in range(ne)]
    a = _args(0, H, inputs, gi, weights, biases, experts, ge, [np.zeros((0, k), np.float32) for k in in_dims])
    P_ = sum(w.size for w in weights) + sum(len(ids) for ids in ge)
    z = np.zeros(1, np.float32)                               # p, dy, d_experts: never touched
    part, dpar = np.full((grid, P_), np.nan, np.float32), np.full(P_, np.nan, np.float32)
    assert kern.ple_gate_bwd(ctypes.byref(a), z.ctypes.data, z.ctypes.data, grid, z.ctypes.data, part.ctypes.data,
                             dpar.ctypes.data) == 0
    np.testing.assert_array_equal(dpar, np.zeros(P_, np.float32))


def test_kernel_source_refuses_uncovered_layers(kern):
    z = np.zeros(4, np.float32)

    def smem(B=1, H=8, K=8, ges=((0, 1),), n_experts=2, gi=None, edit=None):
        ins = [np.zeros((B, K), np.float32)]
        ws = [np.zeros((len(g), K), np.float32) for g in ges]
        a = _args(B, H, ins, gi or [0] * len(ges), ws, [z] * len(ges), [z] * n_experts, [list(g) for g in ges])
        for k, v in (edit or {}).items():   # fields set past what a well-formed description can hold
            if k == "gate_num_experts":
                a.gate_num_experts[0] = v
            else:
                setattr(a, k, v)
        return kern.ple_smem_bytes(ctypes.byref(a), 1)

    assert smem() > 0
    assert smem(H=1025) == 0 and smem(H=0) == 0 and smem(K=1025) == 0
    assert smem(ges=[tuple(range(32))], n_experts=32) > 0
    assert smem(ges=[tuple(range(32))], n_experts=32, edit={"gate_num_experts": 33}) == 0     # E_g > 32
    assert smem(ges=[(0, 0)]) == 0                                  # an expert twice in one gate
    assert smem(ges=[(0, 2)]) == 0                                  # expert index out of range
    assert smem(ges=[(0, 1)] * 9) > 0 and smem(ges=[(0, 1)] * 9, edit={"n_gates": 10}) == 0      # > 9 gates
    assert smem(n_experts=64) > 0 and smem(edit={"n_experts": 65}) == 0     # > 64 experts
    assert smem(gi=[1]) == 0                                        # input index out of range
    assert smem(K=1024, ges=[tuple(range(20))], n_experts=20) > 0   # sum E K = 20480: the budget
    assert smem(K=1024, ges=[tuple(range(21))], n_experts=21) == 0


# ---- the model -------------------------------------------------------------------------------------------------------
PLE_TEST_CONFIG = """
feature_configs { id_feature { feature_name: "cat_a" embedding_dim: 16 num_buckets: 100 } }
feature_configs { id_feature { feature_name: "cat_b" embedding_dim: 8 num_buckets: 1000 } }
feature_configs { raw_feature { feature_name: "int_a" } }
model_config {
  feature_groups { group_name: "t1" feature_names: "cat_a" feature_names: "cat_b" feature_names: "int_a"
                   group_type: DEEP }
  ple {
    extraction_networks { network_name: "layer1" expert_num_per_task: 3 share_num: 4
      task_expert_net { hidden_units: [12, 8, 4] } share_expert_net { hidden_units: [12, 8, 6, 4] } }
    extraction_networks { network_name: "layer2" expert_num_per_task: 3 share_num: 3
      task_expert_net { hidden_units: [8, 12, 8] } share_expert_net { hidden_units: [8, 12, 8] } }
    extraction_networks { network_name: "layer3" expert_num_per_task: 2 share_num: 2
      task_expert_net { hidden_units: [12, 6] } share_expert_net { hidden_units: [12, 6] } }
    task_towers { tower_name: "is_click" label_name: "label1" mlp { hidden_units: [8, 4] }
      metrics { auc {} } losses { binary_cross_entropy {} } }
    task_towers { tower_name: "is_buy" label_name: "label2"
      metrics { auc {} } losses { binary_cross_entropy {} } }
  }
}"""
L2_TOWER = """    task_towers { tower_name: "cost_price" label_name: "label3" mlp { hidden_units: [12, 6] }
      losses { l2_loss {} } }
  }
}"""


def _ple_test_model(seed=0, config=PLE_TEST_CONFIG, labels=("label1", "label2")):
    cfg = parse_text(config)
    torch.manual_seed(seed)
    return create_model(cfg.model_config, create_features(list(cfg.feature_configs)), list(labels),
                        device=torch.device("cpu"))


def _ple_test_batch(labels=False):
    sparse = KeyedJaggedTensor.from_lengths_sync(keys=["cat_a", "cat_b"], values=torch.tensor([1, 2, 3, 4, 5, 6, 7]),
                                                 lengths=torch.tensor([1, 2, 1, 3], dtype=torch.int32))
    dense = KeyedTensor.from_tensor_list(keys=["int_a"], tensors=[torch.tensor([[0.2], [0.3]])])
    lab = {"label1": torch.tensor([1.0, 0.0]), "label2": torch.tensor([0.0, 1.0])} if labels else {}
    return Batch(dense_features={"__BASE__": dense}, sparse_features={"__BASE__": sparse}, labels=lab)


def test_state_dict_names_are_the_references():
    """The reference's test model with its third tower's l2_loss swapped for BCE (3 tasks, as in the fixture's case)."""
    model = _ple_test_model(config=PLE_TEST_CONFIG[:PLE_TEST_CONFIG.rindex("  }\n}")]
                            + L2_TOWER.replace("l2_loss", "binary_cross_entropy"),
                            labels=("label1", "label2", "label3"))
    names = [k for k in model.state_dict() if not k.startswith("embedding_group")]
    towers = [k for k in names if k.startswith("_task_tower.")]
    assert names[:len(names) - len(towers)] == ["_extraction_nets." + k for k in GOLD["pletest_keys"]]
    assert towers == ["_task_tower.0.tower_mlp.mlp.0.perceptron.0.weight", "_task_tower.0.tower_mlp.mlp.0.perceptron.0.bias",
                      "_task_tower.0.tower_mlp.mlp.1.perceptron.0.weight", "_task_tower.0.tower_mlp.mlp.1.perceptron.0.bias",
                      "_task_tower.0.linear.weight", "_task_tower.0.linear.bias",
                      "_task_tower.1.linear.weight", "_task_tower.1.linear.bias",
                      "_task_tower.2.tower_mlp.mlp.0.perceptron.0.weight", "_task_tower.2.tower_mlp.mlp.0.perceptron.0.bias",
                      "_task_tower.2.tower_mlp.mlp.1.perceptron.0.weight", "_task_tower.2.tower_mlp.mlp.1.perceptron.0.bias",
                      "_task_tower.2.linear.weight", "_task_tower.2.linear.bias"]
    nets = model._extraction_nets
    assert nets[0]._shared_gate.out_features == 13 and nets[1]._shared_gate.out_features == 12
    assert nets[2]._shared_gate is None
    assert [g.out_features for g in nets[0]._task_gates] == [7, 7, 7]
    assert [g.in_features for g in nets[1]._task_gates] == [4, 4, 4] and nets[1]._shared_gate.in_features == 4


def test_replay_of_reference_model_test():
    """tzrec/models/ple_test.py: the two BCE towers give logits and probs of shape (2,); the fused path (checker
    backend) equals the torch formulation on the same weights.  The l2_loss tower is refused as MMoE refuses it."""
    model = _ple_test_model()
    batch = _ple_test_batch()
    with Fn.use_backend(OracleKernels()), torch.no_grad():
        ref = model.predict(batch)
    be = PleOracleKernels()
    with Fn.use_backend(be), torch.no_grad():
        got = model.predict(batch)
    assert be.ple_calls == 3
    for t in ("is_click", "is_buy"):
        assert ref[f"logits_{t}"].size() == (2,) and ref[f"probs_{t}"].size() == (2,)
        np.testing.assert_allclose(got[f"logits_{t}"].numpy(), ref[f"logits_{t}"].numpy(), rtol=1e-5, atol=1e-6)
    with pytest.raises(NotImplementedError, match="cost_price: loss l2_loss"):
        _ple_test_model(config=PLE_TEST_CONFIG[:PLE_TEST_CONFIG.rindex("  }\n}")] + L2_TOWER,
                        labels=("label1", "label2", "label3"))


def test_fused_and_torch_formulations_train_alike():
    """Three Adagrad (sparse) / Adam (dense) steps of the reference's test model with labels: the fused autograd path
    and the torch formulation give the same losses, parameters and tables."""
    out = []
    for be in (OracleKernels(), PleOracleKernels()):
        model = _ple_test_model(seed=1)
        model.set_sparse_optimizer(SparseOptimizerSpec(kind=OPT_ADAGRAD, lr=0.05))
        opt = torch.optim.Adam(model.dense_parameters(), lr=0.01)
        losses = []
        with Fn.use_backend(be):
            for _ in range(3):
                batch = _ple_test_batch(labels=True)
                loss = sum(model.loss(model.predict(batch), batch).values())
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
    """examples/ple_taobao.config as stored: group `all` of width 16 x 16 = 256, two steps on the same batch, the loss
    goes down; with the checker backend the fused gates run."""
    pipe = Pipeline(REF_EXAMPLE, device="cpu", max_rows=200, seed=3)
    assert pipe.model.embedding_group.group_total_dim("all") == 256
    batch = pipe.synthetic_batch(24, seed=1)
    be = PleOracleKernels() if fused else OracleKernels()
    with Fn.use_backend(be):
        l0 = float(pipe.eager_step(batch))
        l1 = float(pipe.eager_step(batch))
    assert np.isfinite([l0, l1]).all()
    assert l1 < l0
    assert getattr(be, "ple_calls", 0) == (12 if fused else 0)     # 3 layers x (forward + backward) x 2 steps


def test_evaluate_returns_per_tower_auc_and_loss():
    pipe = Pipeline("ple_taobao", device="cpu", max_rows=200, seed=3)
    with Fn.use_backend(PleOracleKernels()):
        pipe.eager_step(pipe.synthetic_batch(32, seed=0))
        got = pipe.evaluate([pipe.synthetic_batch(32, seed=5), pipe.synthetic_batch(9, seed=6)])
    assert set(got) == {"auc_ctr", "auc_cvr", "binary_cross_entropy_ctr", "binary_cross_entropy_cvr"}
    for k, v in got.items():
        assert np.isfinite(float(v)), k
    assert 0.0 <= float(got["auc_ctr"]) <= 1.0 and 0.0 <= float(got["auc_cvr"]) <= 1.0


def test_sharded_two_ranks_equal_the_unsharded_twin():
    from test_distributed_cpu import _run

    _run(2, "ple_taobao", "mixed", rw_min_rows=250)


def test_usable_predicate():
    x, e = torch.zeros(2, 16), torch.zeros(2, 8)
    w4 = torch.zeros(4, 16)
    with Fn.use_backend(PleOracleKernels()):
        assert Fn.ple_gate_usable([x], [0, 0], [w4, w4], [e] * 4, [[0, 1, 2, 3], [3, 2, 1, 0]])
        assert not Fn.ple_gate_usable([x.double()], [0], [w4], [e] * 4, [[0, 1, 2, 3]])
        assert not Fn.ple_gate_usable([x], [0], [w4], [e, e, e, torch.zeros(2, 9)], [[0, 1, 2, 3]])    # H differs
        assert not Fn.ple_gate_usable([x], [0], [torch.zeros(33, 16)], [e] * 33, [list(range(33))])   # E_g > 32
        assert not Fn.ple_gate_usable([torch.zeros(2, 1025)], [0], [torch.zeros(4, 1025)], [e] * 4, [[0, 1, 2, 3]])
        assert not Fn.ple_gate_usable([torch.zeros(2, 1024)], [0], [torch.zeros(21, 1024)], [e] * 21,
                                      [list(range(21))])                                             # weight budget
        assert not Fn.ple_gate_usable([x], [0] * 10, [w4] * 10, [e] * 4, [[0, 1, 2, 3]] * 10)          # > 9 gates
        with torch.autocast("cpu", dtype=torch.bfloat16):
            assert not Fn.ple_gate_usable([x], [0], [w4], [e] * 4, [[0, 1, 2, 3]])
    with Fn.use_backend(OracleKernels()):     # a CPU backend without the PLE kernels: torch formulation
        assert not Fn.ple_gate_usable([x], [0], [w4], [e] * 4, [[0, 1, 2, 3]])
