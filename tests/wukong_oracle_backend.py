"""The CPU checker backend (metric_oracle_backend.MetricOracleKernels) with the WuKong layer's kernels added.

TEST INFRASTRUCTURE.  wukong_* are the float64 restatement (tests/wukong_ref.py) rounded to fp32, with the CUDA
backend's signatures, so the fused autograd path of a WuKong model runs on a box without a GPU.
"""
import torch

import wukong_ref as W
from metric_oracle_backend import MetricOracleKernels


def _np(t):
    return None if t is None else t.detach().cpu().double().numpy()


def _t(a, like):
    return None if a is None else torch.from_numpy(a).to(dtype=torch.float32, device=like.device)


class WuKongOracleKernels(MetricOracleKernels):
    def __init__(self, use_c: bool = False) -> None:
        super().__init__(use_c)
        self.wukong_calls = 0

    def wukong_mix_fwd(self, x, w_fmb, gamma, beta, w_lcb, w_res, f):
        self.wukong_calls += 1
        return tuple(_t(a, x) for a in W.mix_fwd(*map(_np, (x, w_fmb, gamma, beta, w_lcb, w_res)), f))

    def wukong_mix_bwd(self, x, w_fmb, gamma, w_lcb, w_res, f, stats, d_ln_f, d_base):
        self.wukong_calls += 1
        out = W.mix_bwd(_np(x), _np(w_fmb), _np(gamma), _np(w_lcb), _np(w_res), f, _np(d_ln_f), _np(d_base))
        return tuple(_t(a, x) for a in out)

    def wukong_out_fwd(self, fmb_out, base, gamma, beta, f):
        self.wukong_calls += 1
        return tuple(_t(a, base) for a in W.out_fwd(*map(_np, (fmb_out, base, gamma, beta)), f))

    def wukong_out_bwd(self, fmb_out, base, gamma, f, stats, dy):
        self.wukong_calls += 1
        return tuple(_t(a, base) for a in W.out_bwd(_np(fmb_out), _np(base), _np(gamma), f, _np(dy)))
