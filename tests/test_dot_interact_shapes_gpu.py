"""The FFMA dot-interaction kernels and the FM kernels of csrc/tzk_dense.cu against float64 over the shapes they accept.

The interaction reference is float64 torch on the GPU: feat = cat(dense[:, None], sparse.view(B, Ns, D)), the strict
upper triangle of feat @ feat^T (row-major), laid out [P | p_pad zeros | dense | sparse | zeros up to pad_to]; the
backward is (G + G^T) feat plus the pass-through slices of d_out.  The bounds are the fp32 rounding of the sums the
kernels form (u = 2^-24), with a factor 2 to spare:
  forward pair (i, j):  2 D u sum_k |x_ik x_jk|
  backward entry:       2 (N + 1) u (sum_j |S_ij x_jk| + |pass-through|)
A wrong swizzle, block decode or triangle index is off by O(|x|^2), far outside them.  Copied columns must be the
input's bits and pad columns exactly zero.

The kernel sweeps pin TZK_INTERACT_TC=0 so that the DLRM-Criteo shape (27 x 16 with the dense row) runs the FFMA
kernels too; the tensor-core kernels have their own float64 test in test_kernels_gpu.py."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24


@pytest.fixture
def ffma(kernels, monkeypatch):
    monkeypatch.setenv("TZK_INTERACT_TC", "0")
    return kernels


def _wide(B, n, off, gen, ld=None):
    """[B, n] fp32 on the GPU as a column slice at `off` of a wider [B, ld] buffer (off = 0, ld = n: contiguous)."""
    ld = n + off if ld is None else ld
    buf = torch.randn(B, ld, generator=gen).to(DEV)
    return buf[:, off:off + n]


def _inputs(B, N, D, with_dense, seed, sparse_off=0, dense_off=0):
    g = torch.Generator().manual_seed(seed)
    Ns = N - int(with_dense)
    sparse = _wide(B, Ns * D, sparse_off, g, Ns * D + sparse_off + (8 if sparse_off else 0))
    dense = _wide(B, D, dense_off, g, D + dense_off + (8 if dense_off else 0)) if with_dense else None
    return dense, sparse, Ns


def _layout(N, D, Ns, has_dense, cd, cs, p_pad, pad_to):
    P = N * (N - 1) // 2
    o_dense = P + p_pad
    o_sparse = o_dense + (D if (cd and has_dense) else 0)
    width = o_sparse + (Ns * D if cs else 0)
    return P, o_dense, o_sparse, width, -(-width // pad_to) * pad_to


def _feat(dense, sparse, Ns, D):
    f = sparse.double().reshape(sparse.shape[0], Ns, D)
    return f if dense is None else torch.cat([dense.double()[:, None], f], 1)


def _check_fwd(out, dense, sparse, Ns, D, cd, cs, p_pad, pad_to, what=""):
    B = sparse.shape[0]
    feat = _feat(dense, sparse, Ns, D)
    N = feat.shape[1]
    P, o_d, o_s, width, wp = _layout(N, D, Ns, dense is not None, cd, cs, p_pad, pad_to)
    assert tuple(out.shape) == (B, wp), (what, tuple(out.shape), (B, wp))
    iu = torch.triu_indices(N, N, 1, device=DEV)
    ref = (feat @ feat.transpose(1, 2))[:, iu[0], iu[1]]
    bound = 2 * D * U * (feat.abs() @ feat.abs().transpose(1, 2))[:, iu[0], iu[1]]
    err = (out[:, :P].double() - ref).abs()
    bad = err > bound
    assert not bad.any(), (what, "pairs", int(bad.sum()), float((err - bound).max()))
    assert torch.equal(out[:, P:o_d], torch.zeros_like(out[:, P:o_d])), (what, "p_pad columns")
    if cd and dense is not None:
        assert torch.equal(out[:, o_d:o_d + D], dense), (what, "dense copy")
    if cs:
        assert torch.equal(out[:, o_s:o_s + Ns * D], sparse), (what, "sparse copy")
    assert torch.equal(out[:, width:], torch.zeros_like(out[:, width:])), (what, "tail columns")


def _check_bwd(d_dense, d_sparse, dense, sparse, d_out, Ns, D, cd, cs, p_pad, what=""):
    B = sparse.shape[0]
    feat = _feat(dense, sparse, Ns, D)
    N = feat.shape[1]
    P, o_d, o_s, _, _ = _layout(N, D, Ns, dense is not None, cd, cs, p_pad, 1)
    iu = torch.triu_indices(N, N, 1, device=DEV)
    G = torch.zeros(B, N, N, dtype=torch.float64, device=DEV)
    G[:, iu[0], iu[1]] = d_out[:, :P].double()
    S = G + G.transpose(1, 2)
    passthru = torch.zeros_like(feat)
    doff = int(dense is not None)
    if cd and dense is not None:
        passthru[:, 0] = d_out[:, o_d:o_d + D].double()
    if cs:
        passthru[:, doff:] = d_out[:, o_s:o_s + Ns * D].double().reshape(B, Ns, D)
    ref = S @ feat + passthru
    bound = 2 * (N + 1) * U * (S.abs() @ feat.abs() + passthru.abs())
    got = d_sparse.double().reshape(B, Ns, D)
    if dense is not None:
        assert d_dense is not None and tuple(d_dense.shape) == (B, D)
        got = torch.cat([d_dense.double()[:, None], got], 1)
    else:
        assert d_dense is None
    err = (got - ref).abs()
    bad = err > bound
    assert not bad.any(), (what, "gradient entries", int(bad.sum()), float((err - bound).max()))


def _run(k, dense, sparse, Ns, D, cd, cs, p_pad, pad_to, seed, what=""):
    out = k.dot_interact_fwd(dense, sparse, Ns, D, cd, cs, pad_to=pad_to, p_pad=p_pad)
    _check_fwd(out, dense, sparse, Ns, D, cd, cs, p_pad, pad_to, what)
    # every column of d_out carries a value, pad columns included: the kernel must ignore those
    d_out = torch.randn(out.shape, generator=torch.Generator().manual_seed(seed + 1)).to(DEV)
    d_dense, d_sparse = k.dot_interact_bwd(dense, sparse, d_out, Ns, D, cd, cs, p_pad=p_pad)
    _check_bwd(d_dense, d_sparse, dense, sparse, d_out, Ns, D, cd, cs, p_pad, what)
    return out, d_dense, d_sparse, d_out


def _model_layout(N):
    return 4, (-(N * (N - 1) // 2)) % 4


# ---- every compile-time specialisation: D in {8, 16, 32, 64} and runtime D (power-of-two D/4 or not), one block per lane
# (N <= 28) or a loop over blocks, the NT = 27 kernels, with and without the dense row -----------------------------------
@pytest.mark.parametrize("with_dense", [True, False])
@pytest.mark.parametrize("N", [2, 5, 8, 27, 28, 29, 33, 64])
@pytest.mark.parametrize("D", [4, 8, 12, 16, 20, 32, 64, 128])
def test_specialisation_grid_matches_fp64(ffma, D, N, with_dense):
    pad_to, p_pad = _model_layout(N)
    for B in (1, 7, 257):
        dense, sparse, Ns = _inputs(B, N, D, with_dense, seed=1000 * D + 10 * N + B)
        _run(ffma, dense, sparse, Ns, D, True, True, p_pad, pad_to, seed=B, what=(D, N, with_dense, B))


# ---- output layouts: both store paths (aligned 128-bit and scalar), every copy combination and p_pad ------------------------
LAYOUT_SHAPES = {          # (N, D, dense row, sparse column offset, dense column offset)
    "27x16": (27, 16, True, 0, 0),     # the NT = 27 kernels
    "13x8": (13, 8, True, 0, 4),       # dense as a column slice
    "29x32": (29, 32, True, 4, 0),     # sparse as a 16-B aligned column slice of a wider buffer
    "64x128": (64, 128, True, 0, 0),
}


@pytest.mark.parametrize("pad_to", [1, 4])
@pytest.mark.parametrize("p_pad", [0, 1, 2, 3])
@pytest.mark.parametrize("cd,cs", [(0, 0), (1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("shape", sorted(LAYOUT_SHAPES))
def test_layout_variants_match_fp64(ffma, shape, cd, cs, p_pad, pad_to):
    N, D, with_dense, s_off, d_off = LAYOUT_SHAPES[shape]
    dense, sparse, Ns = _inputs(37, N, D, with_dense, seed=N + D + p_pad, sparse_off=s_off, dense_off=d_off)
    _run(ffma, dense, sparse, Ns, D, bool(cd), bool(cs), p_pad, pad_to, seed=p_pad, what=(shape, cd, cs, p_pad, pad_to))


# ---- the persistent sample loop: B = 20000 is more than one grid pass (1056 CTAs of at most 8 samples) -----------------
@pytest.mark.parametrize("N,D,with_dense", [(5, 12, True), (28, 16, False), (64, 128, True)])
def test_persistent_loop_matches_fp64_and_is_deterministic(ffma, N, D, with_dense):
    dense, sparse, Ns = _inputs(20000, N, D, with_dense, seed=N * D)
    pad_to, p_pad = _model_layout(N)
    out, d_dense, d_sparse, d_out = _run(ffma, dense, sparse, Ns, D, True, True, p_pad, pad_to, seed=3, what=(N, D))
    out2 = ffma.dot_interact_fwd(dense, sparse, Ns, D, True, True, pad_to=pad_to, p_pad=p_pad)
    d_dense2, d_sparse2 = ffma.dot_interact_bwd(dense, sparse, d_out, Ns, D, True, True, p_pad=p_pad)
    assert torch.equal(out.view(torch.int32), out2.view(torch.int32))
    assert torch.equal(d_sparse.view(torch.int32), d_sparse2.view(torch.int32))
    if with_dense:
        assert torch.equal(d_dense.view(torch.int32), d_dense2.view(torch.int32))


# ---- shapes whose eight per-warp shared-memory slabs exceed the 227 KB one CTA may opt into: fewer warps per CTA --------
@pytest.mark.parametrize("N,D", [(64, 36), (64, 64), (64, 128), (48, 128), (41, 108)])
@pytest.mark.parametrize("with_dense", [True, False])
def test_shared_memory_edge_shapes_launch_and_match_fp64(ffma, N, D, with_dense):
    pad_to, p_pad = _model_layout(N)
    for B in (3, 9000):
        dense, sparse, Ns = _inputs(B, N, D, with_dense, seed=N + D + B)
        _run(ffma, dense, sparse, Ns, D, True, True, p_pad, pad_to, seed=B, what=(N, D, with_dense, B))


# ---- nothing outside a row is written: outputs with 8 spare floats per row, filled with a NaN sentinel ------------------
@pytest.mark.parametrize("N,D,with_dense,cd,cs,p_pad", [
    (27, 16, True, 1, 1, 1), (13, 8, True, 1, 0, 2), (5, 12, False, 0, 1, 0), (64, 128, True, 0, 1, 3),
    (29, 32, True, 1, 1, 0), (8, 20, False, 0, 0, 1),
])
def test_kernels_write_nothing_outside_the_row(ffma, N, D, with_dense, cd, cs, p_pad):
    from torcheasyrec_b200.kernels import _ptr, _stream, check

    B = 300
    dense, sparse, Ns = _inputs(B, N, D, with_dense, seed=7 * N + D)
    P, o_d, o_s, width, _ = _layout(N, D, Ns, with_dense, cd, cs, p_pad, 1)
    ld_out = -(-width // 4) * 4 + 8
    out = torch.full((B, ld_out), float("nan"), device=DEV)
    ld_d = dense.stride(0) if with_dense else 0
    check(ffma._lib.tzk_dot_interact_fwd(_ptr(dense), ld_d, _ptr(sparse), sparse.stride(0), B, Ns, D, cd, cs, p_pad,
                                         _ptr(out), ld_out, _stream()), "tzk_dot_interact_fwd")
    torch.cuda.synchronize()
    assert out[:, width:].isnan().all(), "forward wrote past the row"
    _check_fwd(out[:, :width], dense, sparse, Ns, D, cd, cs, p_pad, 1)
    d_out = torch.randn(B, ld_out, generator=torch.Generator().manual_seed(5)).to(DEV)
    ld_ds, ld_dd = Ns * D + 8, D + 8
    d_sparse = torch.full((B, ld_ds), float("nan"), device=DEV)
    d_dense = torch.full((B, ld_dd), float("nan"), device=DEV) if with_dense else None
    check(ffma._lib.tzk_dot_interact_bwd(_ptr(dense), ld_d, _ptr(sparse), sparse.stride(0), _ptr(d_out), ld_out, B, Ns,
                                         D, cd, cs, p_pad, _ptr(d_dense), ld_dd, _ptr(d_sparse), ld_ds, _stream()),
          "tzk_dot_interact_bwd")
    torch.cuda.synchronize()
    assert d_sparse[:, Ns * D:].isnan().all(), "backward wrote past the sparse gradient row"
    if with_dense:
        assert d_dense[:, D:].isnan().all(), "backward wrote past the dense gradient row"
    _check_bwd(d_dense[:, :D] if with_dense else None, d_sparse[:, :Ns * D], dense, sparse, d_out, Ns, D, cd, cs, p_pad)


# ---- FM: y = 0.5 ((sum_n x)^2 - sum_n x^2), dx = dy (sum_n x - x) -------------------------------------------------------
@pytest.mark.parametrize("B", [1, 20000])
@pytest.mark.parametrize("D", [1, 3, 16, 128])
@pytest.mark.parametrize("N", [1, 2, 26, 100])
def test_fm_matches_fp64(kernels, N, D, B):
    """x and dy are column slices (at a float offset of 1) of wider buffers.  s^2 - q cancels, so the bound is on the
    scale of (sum_n |x|)^2: s is off by at most (N - 1) u sum|x|, q by N u sum x^2 <= N u (sum|x|)^2."""
    g = torch.Generator().manual_seed(N * 1000 + D + B)
    x = _wide(B, N * D, 1, g, N * D + 5)
    dy = _wide(B, D, 1, g, D + 3)
    y = kernels.fm_fwd(x, N, D)
    dx = kernels.fm_bwd(x, dy, N, D)
    x64 = x.double().reshape(B, N, D)
    s = x64.sum(1)
    ref_y = 0.5 * (s * s - (x64 * x64).sum(1))
    a = x64.abs().sum(1)
    err = (y.double() - ref_y).abs()
    assert not (err > 2 * (N + 2) * U * a * a).any(), float(err.max())
    ref_dx = dy.double()[:, None] * (s[:, None] - x64)
    err = (dx.double().reshape(B, N, D) - ref_dx).abs()
    assert not (err > 2 * (N + 2) * U * dy.double().abs()[:, None] * a[:, None]).any(), float(err.max())
    assert torch.equal(kernels.fm_fwd(x, N, D).view(torch.int32), y.view(torch.int32))


# ---- the model: DLRM-Criteo with other embedding dims --------------------------------------------------------------------
def _dlrm(dim, seed=7, arch_with_sparse=True, **kw):
    from torcheasyrec_b200.engine import Pipeline

    edits = {f"feature_configs[{13 + i}].id_feature.embedding_dim": dim for i in range(26)}
    edits["model_config.dlrm.dense_mlp.hidden_units"] = [64, dim]
    edits["model_config.dlrm.arch_with_sparse"] = arch_with_sparse
    return Pipeline("dlrm_criteo", device=DEV, max_rows=2000, seed=seed, edits=edits, **kw)


def _count_interact_calls(monkeypatch):
    from torcheasyrec_b200 import kernels

    calls = []
    for nm in ("dot_interact_fwd", "dot_interact_bwd"):
        orig = getattr(kernels.CudaKernels, nm)
        monkeypatch.setattr(kernels.CudaKernels, nm,
                            lambda self, *a, _o=orig, _n=nm, **kw: calls.append(_n) or _o(self, *a, **kw))
    return calls


@pytest.mark.parametrize("dim,arch_with_sparse", [(8, True), (12, True), (16, False)])
def test_dlrm_kernel_path_matches_torch_formulation(monkeypatch, dim, arch_with_sparse):
    """Embedding dims 8 and 12 (runtime D with D/4 = 3), and arch_with_sparse: false (copy_sparse = 0 on the 27 x 16
    kernels): logits, loss and every dense gradient equal the same model on the torch formulation."""
    from test_wukong_cpu import _close
    from test_wukong_gpu import _copy_state, _grads, _np

    from torcheasyrec_b200 import functional as Fn

    calls = _count_interact_calls(monkeypatch)
    a = _dlrm(dim, arch_with_sparse=arch_with_sparse)
    b = _dlrm(dim, arch_with_sparse=arch_with_sparse)
    _copy_state(b, a)
    batch = a.synthetic_batch(4096, seed=3).to(DEV)
    la, lossa, ga = _grads(a, batch)
    assert calls == ["dot_interact_fwd", "dot_interact_bwd"], calls
    with monkeypatch.context() as mp:
        mp.setattr(Fn, "dot_interact_usable", lambda *args, **kw: False)
        lb, lossb, gb = _grads(b, batch)
    assert len(calls) == 2, calls
    _close(_np(la), _np(lb), 1e-5, "logits")
    _close(_np(lossa), _np(lossb), 1e-5, "loss")
    assert ga.keys() == gb.keys() and any("dense_mlp" in k for k in ga)
    for k in ga:
        _close(_np(ga[k]), _np(gb[k]), 1e-4, k)


def test_dlrm_embedding_dim_outside_the_cover_trains_on_the_torch_formulation(monkeypatch):
    """An embedding dim of 10 is not a multiple of 4: the interaction takes the torch formulation and the model trains."""
    calls = _count_interact_calls(monkeypatch)
    p = _dlrm(10, seed=5)
    batch = p.synthetic_batch(2048, seed=2).to(DEV)
    losses = [float(p.eager_step(batch)) for _ in range(4)]
    assert calls == []
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
    assert all(math.isfinite(float(v.abs().max())) for v in p.model.parameters())
