"""The fused forward of DLRM-Criteo's interaction + first final-MLP layer (tzk_interact_wide_fwd) and the weight gradient
read from the pairs, dense and sparse instead of X (tzk_interact_wide_wgrad), both in
torcheasyrec_b200/csrc/tzk_interact_wide.cu, and the autograd glue dense_gemm.InteractWideFn.

CPU: the kernels' source runs under tests/native/cuda_cpu_shim.h + sm90_cpu_emu.h and is compared bit for bit with the
unfused chain it replaces (tensor-core interaction forward, then gemm3x; wgrad3x on the materialised X), and with a
float64 composite.  GPU: the autograd function against the layer-by-layer path, bit for bit, eagerly and replayed from
a CUDA graph."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "tests", "native")
CSRC = os.path.join(ROOT, "torcheasyrec_b200", "csrc")
P, I64, I32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32
CHILD = os.environ.get("TZK_EMU_CHILD") == "1"
TOL = 2e-5
IN_MAP = ((0, 0, 351), (351, 352, 432))


def _compile(src, out):
    subprocess.run(["g++", "-std=c++20", "-O2", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", EXP, "-x", "c++",
                    src, "-shared", "-fPIC", "-o", out], check=True)


def _declare(fused, g3, itc):
    fused.tzk_interact_wide_fwd.argtypes = [P, I64, P, I64, P, I64, P, I64, P, I64, P, I64, P, P, P]
    fused.tzk_interact_wide_wgrad.argtypes = [P, I64, P, I64, P, I64, P, I64, I64, I32, P, P, I64, P]
    g3.tzk_gemm3x.argtypes = [P, I64, P, I64, P, I64, I32, I32, I32, P, I64, P, P, P]
    g3.tzk_wgrad3x.argtypes = [P, I64, P, I64, I64, I32, I32, P, P, I64, P]
    g3.tzk_wgrad3x_partial_floats.restype = I64
    g3.tzk_wgrad3x_partial_floats.argtypes = [I32, I32]
    itc.tzk_itc_fwd.argtypes = [P, I64, P, I64, I64, P, I64, I32]
    return fused, g3, itc


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    """Parent: compiles the host builds once and hands their paths to the children.  Child: loads them."""
    if CHILD:
        return _declare(*(ctypes.CDLL(p) for p in os.environ["TZK_EMU_LIBS"].split(os.pathsep)))
    d = tmp_path_factory.mktemp("emu")
    paths = (str(d / "libinteract_wide_cpu.so"), str(d / "libtzk_gemm3x_cpu.so"), str(d / "libitc_cpu.so"))
    for src, out in zip((os.path.join(CSRC, "tzk_interact_wide.cu"), os.path.join(CSRC, "tzk_gemm3x.cu"),
                         os.path.join(EXP, "interact_tc_standalone.cu")), paths):
        _compile(src, out)
    return paths


def _delegate(request, libs) -> bool:
    """Each case runs in a child pytest process: the emulation aborts its process on a protocol violation or a deadlock,
    and that must fail one test, not the suite."""
    if CHILD:
        return False
    env = {**os.environ, "TZK_EMU_CHILD": "1", "TZK_EMU_LIBS": os.pathsep.join(libs)}
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", request.node.nodeid]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=900, cwd=ROOT)
    if r.returncode != 0:
        pytest.fail(f"child exited with {r.returncode}:\n{r.stdout[-3000:]}\n{r.stderr[-2000:]}")
    return True


def _p(a):
    return a.ctypes.data


def _data(M, seed):
    rng = np.random.default_rng(seed)
    dense = rng.standard_normal((M, 16)).astype(np.float32)
    sparse = rng.standard_normal((M, 416)).astype(np.float32)
    w = (rng.standard_normal((64, 784)) / 28).astype(np.float32)
    w[:, 351] = 0.0                                                          # the zero column's weight
    bias = (rng.standard_normal(64) / 4).astype(np.float32)
    dz = (rng.standard_normal((M, 64)) / 8).astype(np.float32)
    return dense, sparse, w, bias, dz


def _chain_x(itc, dense, sparse):
    """X [M, 784] from the tensor-core interaction kernel (the layer-by-layer path's forward)."""
    M = dense.shape[0]
    x = np.full((M, 784), np.nan, np.float32)
    assert itc.tzk_itc_fwd(_p(dense), 16, _p(sparse), 416, M, _p(x), 784, 2) == 0
    return x


def _fused_fwd(fused, dense, sparse, w, bias):
    M = dense.shape[0]
    y = np.full((M + 1, 64), np.nan, np.float32)                             # one guard row each
    pairs = np.full((M + 1, 352), np.nan, np.float32)
    wh, wl = np.empty((64, 784), np.float32), np.empty((64, 784), np.float32)
    assert fused.tzk_interact_wide_fwd(_p(dense), 16, _p(sparse), 416, _p(w), 784, _p(bias), M, _p(y), 64, _p(pairs),
                                       352, _p(wh), _p(wl), None) == 0
    assert np.isnan(y[M]).all() and np.isnan(pairs[M]).all()
    return y[:M], pairs[:M]


def reference_fwd(dense, sparse, w, bias):
    """float64: X = [pairs | 0 | dense | sparse], relu(X W^T + b)."""
    E = np.concatenate([dense[:, None, :], sparse.reshape(-1, 26, 16)], axis=1).astype(np.float64)
    Z = np.einsum("bid,bjd->bij", E, E)
    iu = np.triu_indices(27, 1)
    x = np.concatenate([Z[:, iu[0], iu[1]], np.zeros((dense.shape[0], 1)), dense, sparse], axis=1)
    return np.maximum(x @ w.astype(np.float64).T + bias, 0.0), x


@pytest.mark.parametrize("M", [1, 63, 64, 65, 129, 200])
def test_fused_fwd_matches_the_unfused_kernels_and_fp64(request, libs, M):
    """Sample tiles of 128 with a short last tile; chunk 11 straddles dense and sparse, chunk 24 reads past sparse."""
    if _delegate(request, libs):
        return
    fused, g3, itc = libs
    dense, sparse, w, bias, _ = _data(M, M)
    y, pairs = _fused_fwd(fused, dense, sparse, w, bias)
    # the chain it replaces: the interaction kernel, then gemm3x with bias and ReLU -> the same bits
    x = _chain_x(itc, dense, sparse)
    y_chain = np.empty((M, 64), np.float32)
    wh, wl = np.empty_like(w), np.empty_like(w)
    assert g3.tzk_gemm3x(_p(x), 784, _p(w), 784, _p(bias), M, 64, 784, 1, _p(y_chain), 64, _p(wh), _p(wl), None) == 0
    np.testing.assert_array_equal(pairs, x[:, :352])
    np.testing.assert_array_equal(y, y_chain)
    ref_y, ref_x = reference_fwd(dense, sparse, w, bias)
    np.testing.assert_allclose(pairs, ref_x[:, :352], rtol=0, atol=TOL * max(1.0, np.abs(ref_x).max()))
    np.testing.assert_allclose(y, ref_y, rtol=0, atol=TOL * max(1.0, np.abs(ref_y).max()))


@pytest.mark.parametrize("M,slabs", [(45, 2), (200, 3), (257, 37)])
def test_multi_source_wgrad_matches_wgrad3x_on_x(request, libs, M, slabs):
    """M not a multiple of 32, a short last slab, more slabs than 32-row chunks."""
    if _delegate(request, libs):
        return
    fused, g3, itc = libs
    dense, sparse, _, _, dz = _data(M, 1000 + M)
    x = _chain_x(itc, dense, sparse)
    pairs = np.ascontiguousarray(x[:, :352])
    part = np.full(slabs * 896 * 64, np.nan, np.float32)
    dw = np.full((64, 784), np.nan, np.float32)
    assert fused.tzk_interact_wide_wgrad(_p(dz), 64, _p(pairs), 352, _p(dense), 16, _p(sparse), 416, M, slabs, _p(part),
                                         _p(dw), 784, None) == 0
    part_x = np.zeros(g3.tzk_wgrad3x_partial_floats(784, slabs), np.float32)
    dw_x = np.empty((64, 784), np.float32)
    assert g3.tzk_wgrad3x(_p(x), 784, _p(dz), 64, M, 784, slabs, _p(part_x), _p(dw_x), 784, None) == 0
    np.testing.assert_array_equal(dw, dw_x)
    ref = dz.astype(np.float64).T @ x.astype(np.float64)
    np.testing.assert_allclose(dw, ref, rtol=0, atol=TOL * max(1.0, np.abs(ref).max()))


def test_fused_fwd_and_wgrad_reject_bad_arguments(libs):
    if CHILD:
        pytest.skip("parent only")
    fused = _declare(*(ctypes.CDLL(p) for p in libs))[0]
    M = 4
    dense, sparse, w, bias, dz = _data(M, 0)
    y, pairs = np.empty((M, 64), np.float32), np.empty((M, 352), np.float32)
    wh = np.empty((64, 784), np.float32)
    buf = np.empty(M * 800 + 4, np.float32)
    odd = buf[1:].ctypes.data                                                # 4-B aligned, not 16-B
    fwd = fused.tzk_interact_wide_fwd
    for ld_d, ld_s, ld_w, ld_p in ((18, 416, 784, 352), (16, 414, 784, 352), (16, 416, 780, 352), (16, 416, 784, 350)):
        assert fwd(_p(dense), ld_d, _p(sparse), ld_s, _p(w), ld_w, _p(bias), M, _p(y), 64, _p(pairs), ld_p, _p(wh), _p(wh),
                   None) == 1
    assert fwd(_p(dense), 16, _p(sparse), 416, _p(w), 784, _p(bias), M, odd, 64, _p(pairs), 352, _p(wh), _p(wh), None) == 1
    assert fwd(_p(dense), 16, odd, 416, _p(w), 784, _p(bias), M, _p(y), 64, _p(pairs), 352, _p(wh), _p(wh), None) == 1
    assert fwd(_p(dense), 16, _p(sparse), 416, _p(w), 784, _p(bias), 0, _p(y), 64, _p(pairs), 352, _p(wh), _p(wh),
               None) == 1
    part = np.empty(896 * 64, np.float32)
    dw = np.empty((64, 784), np.float32)
    wg = fused.tzk_interact_wide_wgrad
    for ld_z, ld_p, ld_dw in ((62, 352, 784), (64, 350, 784), (64, 352, 780)):
        assert wg(_p(dz), ld_z, _p(pairs), ld_p, _p(dense), 16, _p(sparse), 416, M, 1, _p(part), _p(dw), ld_dw, None) == 1
    assert wg(_p(dz), 64, odd, 352, _p(dense), 16, _p(sparse), 416, M, 1, _p(part), _p(dw), 784, None) == 1
    assert wg(_p(dz), 64, _p(pairs), 352, _p(dense), 16, _p(sparse), 416, M, 0, _p(part), _p(dw), 784, None) == 1


# ---- GPU ---------------------------------------------------------------------------------------------------------------
def _gpu_case(M, seed):
    import torch

    g = torch.Generator().manual_seed(seed)
    dense = torch.randn(M, 16, generator=g)
    sparse = torch.randn(M, 416, generator=g)
    w = torch.randn(64, 783, generator=g) / 28
    b = torch.randn(64, generator=g) / 4
    dy = torch.randn(M, 64, generator=g)
    return [t.cuda() for t in (dense, sparse, w, b, dy)]


def _leaves(dense, sparse, w, b):
    return [t.detach().clone().requires_grad_(True) for t in (dense, sparse, w, b)]


def _fused(dense, sparse, w, b, dy):
    from torcheasyrec_b200 import dense_gemm as G

    ins = _leaves(dense, sparse, w, b)
    assert G.interact_wide_usable(ins[0], ins[1], ins[2], 26, 16)
    y = G.InteractWideFn.apply(G._gemm3x_lib(), *ins, IN_MAP)
    y.backward(dy)
    return [y.detach()] + [t.grad for t in ins]


def _layer_by_layer(dense, sparse, w, b, dy):
    from torcheasyrec_b200 import dense_gemm as G
    from torcheasyrec_b200 import functional as Fn

    ins = _leaves(dense, sparse, w, b)
    x, in_map = Fn.dlrm_interaction(ins[0], ins[1], 26, 16, aligned=True)
    assert tuple(in_map) == IN_MAP
    y = G.Gemm3xLinearFn.apply(G._gemm3x_lib(), x, ins[2], ins[3], True, in_map)
    y.backward(dy)
    return [y.detach()] + [t.grad for t in ins]


NAMES = ["y", "d_dense", "d_sparse", "dW", "db"]


@pytest.mark.gpu
@pytest.mark.parametrize("M", [300, 65536 + 5])
def test_interact_wide_fn_equals_the_layer_by_layer_path_bitwise(M):
    import torch

    from torcheasyrec_b200 import dense_gemm as G

    if G._gemm3x_lib() is None or not G.available():
        pytest.fail("libtzk_gemm3x.so / cuBLASLt not available")
    case = _gpu_case(M, M)
    got = _fused(*case)
    ref = _layer_by_layer(*case)
    for name, a, r in zip(NAMES, got, ref):
        assert torch.equal(a, r), (name, (a - r).abs().max().item())
    again = _fused(*case)
    assert torch.equal(got[3], again[3]) and torch.equal(got[4], again[4])


@pytest.mark.gpu
def test_interact_wide_fn_graph_replay_equals_eager():
    import torch

    from torcheasyrec_b200 import dense_gemm as G

    case = _gpu_case(4096 + 17, 5)
    eager = _fused(*case)
    ins = _leaves(*case[:4])
    dy = case[4]

    def step():
        for t in ins:
            t.grad = None
        y = G.InteractWideFn.apply(G._gemm3x_lib(), *ins, IN_MAP)
        y.backward(dy)
        return y

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    for t in ins:
        t.grad = None
    with torch.cuda.graph(graph):
        y = G.InteractWideFn.apply(G._gemm3x_lib(), *ins, IN_MAP)
        y.backward(dy)
    graph.replay()
    torch.cuda.synchronize()
    for name, a, r in zip(NAMES, [y.detach()] + [t.grad for t in ins], eager):
        assert torch.equal(a, r), name
