"""The CPU checker backend (metric_oracle_backend.MetricOracleKernels) with the PLE gate kernels added.

TEST INFRASTRUCTURE.  ple_gate_* are the float64 restatement (tests/ple_ref.py) rounded to fp32, with the CUDA
backend's signatures, so the fused autograd path of a PLE model runs on a box without a GPU.
"""
import torch

import ple_ref as R
from metric_oracle_backend import MetricOracleKernels


def _np(t):
    return t.detach().cpu().double().numpy()


def _t(a, like):
    return torch.from_numpy(a).to(dtype=torch.float32, device=like.device)


class PleOracleKernels(MetricOracleKernels):
    def __init__(self, use_c: bool = False) -> None:
        super().__init__(use_c)
        self.ple_calls = 0

    def ple_gate_fwd(self, inputs, gate_input, weights, biases, experts, gate_experts):
        self.ple_calls += 1
        y, p = R.gates_fwd([_np(x) for x in inputs], gate_input, [_np(w) for w in weights], [_np(b) for b in biases],
                           [_np(e) for e in experts], gate_experts)
        return _t(y, experts[0]), _t(p, experts[0])

    def ple_gate_bwd(self, inputs, gate_input, weights, biases, experts, gate_experts, p, dy):
        self.ple_calls += 1
        dx, dex, dW, db = R.gates_bwd([_np(x) for x in inputs], gate_input, [_np(w) for w in weights],
                                      [_np(b) for b in biases], [_np(e) for e in experts], gate_experts, _np(dy))
        like = experts[0]
        return [_t(a, like) for a in dx], _t(dex, like), [_t(a, like) for a in dW], [_t(a, like) for a in db]
