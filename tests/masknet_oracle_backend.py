"""The CPU checker backend (metric_oracle_backend.MetricOracleKernels) with the MaskNet kernels added.

TEST INFRASTRUCTURE.  masknet_* are the float64 restatement (tests/masknet_ref.py) rounded to fp32, with the CUDA
backend's signatures, so the fused autograd path of a MaskNet model runs on a box without a GPU.
"""
import torch

import masknet_ref as M
from metric_oracle_backend import MetricOracleKernels


def _np(t):
    return t.detach().cpu().double().numpy()


def _t(a, like):
    return torch.from_numpy(a).to(dtype=torch.float32, device=like.device)


class MaskNetOracleKernels(MetricOracleKernels):
    def __init__(self, use_c: bool = False) -> None:
        super().__init__(use_c)
        self.masknet_calls = 0

    def masknet_mask_fwd(self, e, m, b2, gamma, beta, E, nb):
        self.masknet_calls += 1
        return tuple(_t(a, e) for a in M.mask_fwd(*map(_np, (e, m, b2, gamma, beta)), E, nb))

    def masknet_mask_bwd(self, e, m, b2, gamma, beta, stats, dv, E, nb):
        self.masknet_calls += 1
        return tuple(_t(a, e) for a in M.mask_bwd(*map(_np, (e, m, b2, gamma, beta, dv)), E, nb))

    def masknet_ffn_fwd(self, z, b3, gamma, beta, nb):
        self.masknet_calls += 1
        return tuple(_t(a, z) for a in M.ffn_fwd(*map(_np, (z, b3, gamma, beta)), nb))

    def masknet_ffn_bwd(self, z, b3, gamma, beta, stats, dy, nb):
        self.masknet_calls += 1
        return tuple(_t(a, z) for a in M.ffn_bwd(*map(_np, (z, b3, gamma, beta, dy)), nb))
