"""functional.dot_interact_usable: which DLRM interaction calls the kernels of csrc/tzk_dense.cu cover, and the torch
formulation that dot_interaction / dlrm_interaction take outside that cover (no GPU needed)."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle_backend import OracleKernels  # noqa: E402

from torcheasyrec_b200 import functional as Fn  # noqa: E402


def _rows(B, n, off=0):
    """[B, n] fp32 as a column slice at float offset `off` of a 16-B aligned buffer whose rows are a multiple of 4 wide."""
    ld = -(-(n + off) // 4) * 4
    return torch.randn(B, ld)[:, off:off + n]


@pytest.mark.parametrize("D,ok", [(4, True), (8, True), (12, True), (128, True), (2, False), (10, False), (132, False)])
def test_embedding_dim_edges(D, ok):
    with Fn.use_backend(OracleKernels()):
        assert Fn.dot_interact_usable(_rows(3, D), _rows(3, 5 * D), 5, D) is ok


@pytest.mark.parametrize("Ns,with_dense,ok", [(64, False, True), (63, True, True), (65, False, False), (64, True, False)])
def test_feature_count_edges(Ns, with_dense, ok):
    with Fn.use_backend(OracleKernels()):
        dense = _rows(2, 8) if with_dense else None
        assert Fn.dot_interact_usable(dense, _rows(2, Ns * 8), Ns, 8) is ok


def test_row_alignment_and_layout():
    with Fn.use_backend(OracleKernels()):
        assert Fn.dot_interact_usable(_rows(4, 8), _rows(4, 24, off=4), 3, 8)       # 16-B aligned column slice
        assert not Fn.dot_interact_usable(None, _rows(4, 24, off=1), 3, 8)          # misaligned start
        assert not Fn.dot_interact_usable(_rows(4, 8, off=2), _rows(4, 24), 3, 8)   # misaligned dense
        odd = torch.randn(4, 26)[:, :24]                                            # row stride 26: rows 2 and 3 misaligned
        assert not Fn.dot_interact_usable(None, odd, 3, 8)
        assert not Fn.dot_interact_usable(None, torch.randn(24, 4).t(), 3, 8)       # column-major
        assert not Fn.dot_interact_usable(None, _rows(4, 24).double(), 3, 8)
        assert not Fn.dot_interact_usable(None, _rows(4, 24), 2, 8)                 # width is not Ns * D
        with torch.autocast("cpu", dtype=torch.bfloat16):
            assert not Fn.dot_interact_usable(None, _rows(4, 24), 3, 8)
    # on the CPU the kernels exist only under a test backend that implements them
    assert not Fn.dot_interact_usable(None, _rows(4, 24), 3, 8)


def _fp64(dense, sparse, Ns, D):
    f = sparse.double().reshape(-1, Ns, D)
    if dense is not None:
        f = torch.cat([dense.double()[:, None], f], 1)
    iu = torch.triu_indices(f.shape[1], f.shape[1], 1)
    z = (f @ f.transpose(1, 2))[:, iu[0], iu[1]]
    return torch.cat([z, dense.double(), sparse.double()], 1) if dense is not None else z


def test_outside_the_cover_takes_the_torch_formulation():
    """D = 10: dlrm_interaction and dot_interaction never reach the backend and equal float64 in the reference's
    layout; aligned=True returns no column map.  Gradients flow through the torch formulation."""

    class NoInteract(OracleKernels):
        def dot_interact_fwd(self, *a, **kw):
            raise AssertionError("the kernel does not cover D = 10")

    B, Ns, D = 5, 6, 10
    dense = torch.randn(B, D, requires_grad=True)
    sparse = torch.randn(B, Ns * D, requires_grad=True)
    with Fn.use_backend(NoInteract()):
        x = Fn.dlrm_interaction(dense, sparse, Ns, D)
        xa, in_map = Fn.dlrm_interaction(dense, sparse, Ns, D, aligned=True)
        z = Fn.dot_interaction(sparse.reshape(B, Ns, D))
    assert in_map is None and torch.equal(xa, x)
    np.testing.assert_allclose(x.detach().double().numpy(), _fp64(dense, sparse, Ns, D).detach().numpy(), rtol=1e-5,
                               atol=1e-5)
    np.testing.assert_allclose(z.detach().double().numpy(), _fp64(None, sparse, Ns, D).detach().numpy(), rtol=1e-5,
                               atol=1e-5)
    x.sum().backward()
    assert dense.grad is not None and sparse.grad is not None and torch.isfinite(sparse.grad).all()
