"""The fused input gradient of DLRM-Criteo's interaction + first final-MLP layer (tzk_interact_wide_bwd in
torcheasyrec_b200/csrc/tzk_interact_wide.cu, autograd glue dense_gemm.InteractWideFn).

CPU: the kernel's source runs under tests/native/cuda_cpu_shim.h + sm90_cpu_emu.h (as in test_gemm3x_emu.py) and is
compared with a float64 composite and, bit for bit, with the unfused chain it replaces (the gemm3x input-gradient kernel
followed by the tensor-core interaction backward, both emulated).  GPU: the autograd function against float64 and against
the layer-by-layer path."""
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
    fused.tzk_interact_wide_bwd.argtypes = [P, I64, P, I64, P, I64, P, I64, I64, P, I64, P, I64, P, P, P]
    g3.tzk_gemm3x.argtypes = [P, I64, P, I64, P, I64, I32, I32, I32, P, I64, P, P, P]
    itc.tzk_itc_bwd.argtypes = [P, I64, P, I64, P, I64, I64, P, I64, P, I64, I32]
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


def _pairs():
    return [(i, j) for i in range(27) for j in range(i + 1, 27)]


def reference_bwd(dz, w, dense, sparse):
    """float64: dX = dz W, then the interaction backward of X = [pairs | 0 | dense | sparse]."""
    dx = dz.astype(np.float64) @ w.astype(np.float64)                       # [M, 784]
    E = np.concatenate([dense[:, None, :], sparse.reshape(-1, 26, 16)], axis=1).astype(np.float64)
    S = np.zeros((dz.shape[0], 27, 27))
    for p, (i, j) in enumerate(_pairs()):
        S[:, i, j] = S[:, j, i] = dx[:, p]
    dE = np.einsum("bij,bjd->bid", S, E) + dx[:, 352:].reshape(-1, 27, 16)
    return dE[:, 0], dE[:, 1:].reshape(-1, 416)


def _data(M, seed):
    rng = np.random.default_rng(seed)
    dense = rng.standard_normal((M, 16)).astype(np.float32)
    sparse = rng.standard_normal((M, 416)).astype(np.float32)
    dz = (rng.standard_normal((M, 64)) / 8).astype(np.float32)
    w = (rng.standard_normal((64, 784)) / 28).astype(np.float32)
    w[:, 351] = 0.0                                                          # the zero column's weight
    return dense, sparse, dz, w


@pytest.mark.parametrize("M", [1, 63, 64, 65, 200])
def test_fused_bwd_matches_fp64_and_the_unfused_kernels(request, libs, M):
    """Sample tiles of 64 with a short last tile; 25 column chunks of 32, the last half past the weight."""
    if _delegate(request, libs):
        return
    fused, g3, itc = libs
    dense, sparse, dz, w = _data(M, M)
    dd = np.full((M, 16), np.nan, np.float32)
    ds = np.full((M + 1, 416), np.nan, np.float32)                            # one guard row
    wh, wl = np.empty((784, 64), np.float32), np.empty((784, 64), np.float32)
    assert fused.tzk_interact_wide_bwd(_p(dz), 64, _p(w), 784, _p(dense), 16, _p(sparse), 416, M, _p(dd), 16, _p(ds),
                                       416, _p(wh), _p(wl), None) == 0
    assert np.isnan(ds[M]).all()
    ref_d, ref_s = reference_bwd(dz, w, dense, sparse)
    np.testing.assert_allclose(dd, ref_d, rtol=0, atol=TOL)
    np.testing.assert_allclose(ds[:M], ref_s, rtol=0, atol=TOL)
    # the chain it replaces: dX = gemm3x(dz, W^T), then the tensor-core interaction backward -> the same bits
    wt = np.ascontiguousarray(w.T)
    dx = np.empty((M, 784), np.float32)
    th, tl = np.empty_like(wt), np.empty_like(wt)
    assert g3.tzk_gemm3x(_p(dz), 64, _p(wt), 64, None, M, 784, 64, 0, _p(dx), 784, _p(th), _p(tl), None) == 0
    cd, cs = np.empty((M, 16), np.float32), np.empty((M, 416), np.float32)
    itc.tzk_itc_bwd(_p(dense), 16, _p(sparse), 416, _p(dx), 784, M, _p(cd), 16, _p(cs), 416, 2)
    np.testing.assert_array_equal(dd, cd)
    np.testing.assert_array_equal(ds[:M], cs)


def test_fused_bwd_rejects_misaligned_rows(libs):
    if CHILD:
        pytest.skip("parent only")
    fused = _declare(*(ctypes.CDLL(p) for p in libs))[0]
    dense, sparse, dz, w = _data(4, 0)
    out = np.empty((4, 432), np.float32)
    wh = np.empty((784, 64), np.float32)
    for ld_dz, ld_w in ((63, 784), (64, 780)):
        assert fused.tzk_interact_wide_bwd(_p(dz), ld_dz, _p(w), ld_w, _p(dense), 16, _p(sparse), 416, 4, _p(out), 16,
                                           _p(out), 416, _p(wh), _p(wh), None) == 1


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


def _fused(dense, sparse, w, b, dy):
    import torch

    from torcheasyrec_b200 import dense_gemm as G

    ins = [t.detach().clone().requires_grad_(True) for t in (dense, sparse, w, b)]
    assert G.interact_wide_usable(ins[0], ins[1], ins[2], 26, 16)
    y = G.InteractWideFn.apply(G._gemm3x_lib(), *ins, IN_MAP)
    y.backward(dy)
    torch.cuda.synchronize()
    return [y.detach()] + [t.grad for t in ins]


def _unfused(dense, sparse, w, b, dy):
    from torcheasyrec_b200 import dense_gemm as G
    from torcheasyrec_b200 import functional as Fn

    ins = [t.detach().clone().requires_grad_(True) for t in (dense, sparse, w, b)]
    x, in_map = Fn.dlrm_interaction(ins[0], ins[1], 26, 16, aligned=True)
    assert tuple(in_map) == IN_MAP
    y = G.Gemm3xLinearFn.apply(G._gemm3x_lib(), x, ins[2], ins[3], True, in_map)
    y.backward(dy)
    return [y.detach()] + [t.grad for t in ins]


def _fp64(dense, sparse, w, b, dy):
    import torch

    d, s, w_, b_ = [t.double().cpu().requires_grad_(True) for t in (dense, sparse, w, b)]
    E = torch.cat([d[:, None, :], s.view(-1, 26, 16)], dim=1)
    Z = E @ E.transpose(1, 2)
    iu = torch.triu_indices(27, 27, 1)
    x = torch.cat([Z[:, iu[0], iu[1]], d, s], dim=1)
    y = torch.relu(x @ w_.T + b_)
    y.backward(dy.double().cpu())
    return [y.detach(), d.grad, s.grad, w_.grad, b_.grad]


@pytest.mark.gpu
@pytest.mark.parametrize("M", [300, 65536 + 5])
def test_interact_wide_fn_matches_fp64_and_the_layer_by_layer_path(M):
    import torch

    from torcheasyrec_b200 import dense_gemm as G

    if G._gemm3x_lib() is None or not G.available():
        pytest.fail("libtzk_gemm3x.so / cuBLASLt not available")
    case = _gpu_case(M, M)
    got = _fused(*case)
    ref = _fp64(*case)
    names = ["y", "d_dense", "d_sparse", "dW", "db"]
    for name, a, r in zip(names, got, ref):
        scale = M ** 0.5 if name in ("dW", "db") else 1.0
        err = (a.double().cpu() - r).abs().max().item()
        assert err <= 2e-5 * scale * max(1.0, r.abs().max().item() / 16), (name, err)
    again = _fused(*case)
    assert torch.equal(got[3], again[3]) and torch.equal(got[4], again[4])
    old = _unfused(*case)
    for name, a, o in zip(names, got, old):
        torch.testing.assert_close(a, o, rtol=1e-5, atol=1e-6 * max(1.0, o.abs().max().item()), msg=name)
