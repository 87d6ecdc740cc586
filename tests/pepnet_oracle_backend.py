"""The CPU checker backend (metric_oracle_backend.MetricOracleKernels) with the PEPNet gate kernels added.

TEST INFRASTRUCTURE.  pepnet_gate_* are the float64 restatement (tests/pepnet_ref.py) rounded to fp32, with the CUDA
backend's signatures (outputs written into the given views), so the fused autograd path of a PEPNet model runs on a box
without a GPU.
"""
import torch

import pepnet_ref as R
from metric_oracle_backend import MetricOracleKernels


def _np(t):
    return None if t is None else t.detach().cpu().double().numpy()


def _segs(segs):
    return [(_np(x), _np(bx), _np(z), _np(bz), relu, gamma) for x, bx, z, bz, _, relu, gamma in segs]


class PepnetOracleKernels(MetricOracleKernels):
    def __init__(self, use_c: bool = False) -> None:
        super().__init__(use_c)
        self.pepnet_calls = 0

    def pepnet_gate_fwd(self, segs):
        self.pepnet_calls += 1
        for s, y in zip(segs, R.gate_fwd(_segs(segs))):
            s[4].copy_(torch.from_numpy(y))

    def pepnet_gate_bwd(self, segs, dys, dxs, dzs):
        self.pepnet_calls += 1
        out = []
        for (dx, dz, dbx, dbz), tdx, tdz in zip(R.gate_bwd(_segs(segs), [_np(d) for d in dys]), dxs, dzs):
            tdx.copy_(torch.from_numpy(dx))
            tdz.copy_(torch.from_numpy(dz))
            out.append((torch.from_numpy(dbx).float(), torch.from_numpy(dbz).float()))
        return out
