"""The 3xTF32 GEMMs of the wide tower layer (torcheasyrec_b200/csrc/tzk_gemm3x.cu) executed on the CPU from their actual
source.

`cuda_cpu_shim.h` runs the kernels with one std::thread per CUDA thread (256 per CTA) and `sm90_cpu_emu.h` stands in
for the hardware: mbarriers with transaction counts, TMA box loads with SWIZZLE_128B and out-of-bounds zero fill, and
mma.sync m16n8k8 TF32 with the fragment layouts of the PTX ISA and TF32 operand truncation.  What this proves: control
flow, barrier protocol, swizzled shared-memory addressing, fragment -> (row, column) mapping, K-tail and M-tail handling
and the epilogues are consistent with those semantics and produce fp32-accurate results.  What it cannot prove: that
the hardware agrees with the emulation (tests/test_kernels_gpu.py checks that on the GPU)."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

EXP = os.path.join(os.path.dirname(os.path.abspath(__file__)), "native")
P, I64, I32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32


CHILD = os.environ.get("TZK_EMU_CHILD") == "1"


def _declare(L):
    L.tzk_gemm3x.argtypes = [P, I64, P, I64, P, I64, I32, I32, I32, P, I64, P, P, P]
    L.tzk_wgrad3x.argtypes = [P, I64, P, I64, I64, I32, I32, P, P, I64, P]
    L.tzk_wgrad3x_partial_floats.restype = I64
    L.tzk_wgrad3x_partial_floats.argtypes = [I32, I32]
    return L


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    """Parent: compiles the host build once and hands its path to the children.  Child: loads it."""
    if CHILD:
        return _declare(ctypes.CDLL(os.environ["TZK_EMU_LIB"]))
    out = str(tmp_path_factory.mktemp("emu") / "libtzk_gemm3x_cpu.so")
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "torcheasyrec_b200", "csrc")
    subprocess.run(["g++", "-std=c++20", "-O2", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", EXP, "-x", "c++",
                    os.path.join(csrc, "tzk_gemm3x.cu"), "-shared", "-fPIC", "-o", out], check=True)
    return out


def _delegate(request, lib) -> bool:
    """Every case runs in a child pytest process: the emulation aborts the process on a protocol violation or a
    deadlock (256 real threads per emulated CTA), and that must fail ONE test, not take the whole suite down.
    An abnormal exit is retried once (thread-scheduling artefacts of the emulation have been seen once in thousands of
    CTAs); an ordinary assertion failure is not."""
    if CHILD:
        return False
    env = {**os.environ, "TZK_EMU_CHILD": "1", "TZK_EMU_LIB": lib}
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", request.node.nodeid]
    for attempt in (1, 2):
        r = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=900,
                           cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
        if r.returncode == 0:
            return True
        crashed = r.returncode < 0 or r.returncode > 5        # pytest's own exit codes are 0..5
        if not crashed or attempt == 2:
            pytest.fail(f"child exited with {r.returncode} (attempt {attempt}):\n{r.stdout[-3000:]}\n{r.stderr[-2000:]}")
    return True


def _p(a):
    return None if a is None else a.ctypes.data


# error budget: the emulated tensor core adds the products of a 32-column chunk one after another (a plain running sum),
# which costs more than the split itself; numpy's blocked fp32 matmul sits at ~2e-6 on the same data
TOL = 2e-5


@pytest.fixture
def stack():
    """One configuration is built: W arrives split into W_hi / W_lo (the scratch the forward writes), X is split in
    registers."""
    return ("1", "4", "0", "1", "0", "0")


@pytest.mark.parametrize("M,relu,bias", [(200, 1, True), (1, 0, False), (128, 1, True)])
def test_forward_784_to_64(request, lib, stack, M, relu, bias):
    """K = 784 = 24.5 chunks of 32 (zero-filled tail), rows past M zero-filled and not stored, bias + ReLU epilogue."""
    if _delegate(request, lib):
        return
    rng = np.random.default_rng(M)
    K, N = 784, 64
    x = rng.standard_normal((M, K)).astype(np.float32)
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32) if bias else None
    y = np.full((M + 1, N), np.nan, np.float32)                  # one guard row
    wh, wl = np.empty_like(w), np.empty_like(w)
    assert lib.tzk_gemm3x(_p(x), K, _p(w), K, _p(b), M, N, K, relu, _p(y), N, _p(wh), _p(wl), None) == 0
    ref = x.astype(np.float64) @ w.astype(np.float64).T + (b if bias else 0.0)
    ref = np.maximum(ref, 0) if relu else ref
    np.testing.assert_allclose(y[:M], ref, rtol=0, atol=TOL)
    assert np.isnan(y[M]).all()
    if stack[2] == "0":     # the split really is hi + lo with hi on the TF32 grid
        assert (wh.view(np.uint32) & 0x1FFF == 0).all() and (wl.view(np.uint32) & 0x1FFF == 0).all()
        np.testing.assert_allclose(wh.astype(np.float64) + wl, w, rtol=2 ** -21)
    # plain TF32 (hi x hi only) would be ~1000x worse: the lo terms are doing their job
    tf = lambda a: (a.view(np.uint32) & 0xFFFFE000).view(np.float32)
    plain = np.abs(tf(x).astype(np.float64) @ tf(w).astype(np.float64).T + (b if bias else 0.0) -
                   (x.astype(np.float64) @ w.astype(np.float64).T + (b if bias else 0.0))).max()
    assert plain > 20 * TOL or M == 1


def test_dgrad_64_to_784(request, lib, stack):
    """The input-gradient pass: BN = 56, fourteen column tiles per row tile, two k-chunks, three stages."""
    if _delegate(request, lib):
        return
    rng = np.random.default_rng(1)
    M, K, N = 130, 64, 784
    dz = rng.standard_normal((M, K)).astype(np.float32)
    wt = (rng.standard_normal((N, K)) / 8).astype(np.float32)     # W^T [784, 64]
    dx = np.full((M, N), np.nan, np.float32)
    wh, wl = np.empty_like(wt), np.empty_like(wt)
    assert lib.tzk_gemm3x(_p(dz), K, _p(wt), K, None, M, N, K, 0, _p(dx), N, _p(wh), _p(wl), None) == 0
    np.testing.assert_allclose(dx, dz.astype(np.float64) @ wt.astype(np.float64).T, rtol=0, atol=TOL)


@pytest.mark.parametrize("M,slabs", [(200, 2), (70, 3), (31, 1), (520, 1)])
def test_wgrad_mn_major(request, lib, M, slabs):
    """dW = dZ^T X with both operands MN-major straight from the row-major tensors; row slabs (the last one short or
    empty), 7 column tiles (the last one 16 of 128 columns), fixed-order slab reduction + transpose."""
    if _delegate(request, lib):
        return
    rng = np.random.default_rng(M + slabs)
    K = 784
    x = rng.standard_normal((M, K)).astype(np.float32)
    dz = (rng.standard_normal((M, 64)) / np.sqrt(M)).astype(np.float32)
    dw = np.full((64, K), np.nan, np.float32)
    part = np.zeros(lib.tzk_wgrad3x_partial_floats(K, slabs), np.float32)
    assert lib.tzk_wgrad3x(_p(x), K, _p(dz), 64, M, K, slabs, _p(part), _p(dw), K, None) == 0
    np.testing.assert_allclose(dw, dz.astype(np.float64).T @ x.astype(np.float64), rtol=0, atol=TOL)
    dw2 = np.empty_like(dw)
    assert lib.tzk_wgrad3x(_p(x), K, _p(dz), 64, M, K, slabs, _p(part), _p(dw2), K, None) == 0
    np.testing.assert_array_equal(dw, dw2)


def test_autograd_wiring_of_the_wide_layer(request, lib, monkeypatch):
    """dense_gemm.Gemm3xLinearFn (the drop-in for dense_gemm._LinearFn on DLRM's 783 -> 64 layer) on CPU
    tensors through the emulated kernels: forward, input gradient, weight gradient (column-mapped 783 -> 784 input)
    and bias gradient against torch autograd."""
    if _delegate(request, lib):
        return
    import sys

    import torch

    import torcheasyrec_b200.dense_gemm as G

    G._declare_gemm3x(lib)
    import torcheasyrec_b200.dense_gemm as DG
    monkeypatch.setattr(DG, "SLABS", 2)
    torch.manual_seed(0)
    M, K, Kx, N = 150, 783, 784, 64
    in_map = ((0, 0, 16), (16, 17, 767))          # dense block, one zero column, the pair block (as DLRM lays it out)
    xs = torch.randn(M, K)
    x = torch.zeros(M, Kx)
    for src, dst, n in in_map:
        x[:, dst:dst + n] = xs[:, src:src + n]
    x.requires_grad_(True)
    xr = xs.clone().requires_grad_(True)
    w = (torch.randn(N, K) / K ** 0.5).requires_grad_(True)
    b = torch.randn(N, requires_grad=True)
    wr, br = w.detach().clone().requires_grad_(True), b.detach().clone().requires_grad_(True)
    y = G.Gemm3xLinearFn.apply(lib, x, w, b, True, in_map)
    ref = torch.relu(torch.nn.functional.linear(xr.double(), wr.double(), br.double()))
    g = torch.randn(M, N)
    y.backward(g)
    ref.backward(g.double())
    np.testing.assert_allclose(y.detach().numpy(), ref.detach().numpy(), atol=TOL)
    np.testing.assert_allclose(b.grad.numpy(), br.grad.numpy(), atol=1e-4)
    np.testing.assert_allclose(w.grad.numpy(), wr.grad.numpy(), atol=1e-4)
    dx = torch.cat([x.grad[:, dst:dst + n] for _, dst, n in in_map], dim=1)
    np.testing.assert_allclose(dx.numpy(), xr.grad.numpy(), atol=TOL)
    assert float(x.grad[:, 16].abs().max()) == 0.0       # the padding column's weight is zero -> zero gradient
