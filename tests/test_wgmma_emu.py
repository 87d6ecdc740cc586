"""The host emulation of wgmma m64nNk8 TF32 (tests/native/sm90_wgmma_emu.h), which the CPU tests of the fused wide-layer
kernels run on, against a plain loop: D = (scale-d ? C : 0) + sum over k in order of A[r, k] B[k, c], in fp32.  The
emulation decodes the SWIZZLE_128B descriptor of tzk_wgmma.cuh and reads A from mma.sync's fragment layout, so this
pins the descriptor, the swizzle of a k-step inside the 128-B row and the fragment mapping for N = 8, 32 and 64."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "tests", "native")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("wgmma_emu") / "libwgmma_emu.so")
    subprocess.run(["g++", "-std=c++20", "-O2", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", EXP, "-x",
                    "c++", os.path.join(EXP, "wgmma_emu_standalone.cu"), "-shared", "-fPIC", "-o", out], check=True)
    L = ctypes.CDLL(out)
    P, I = ctypes.c_void_p, ctypes.c_int
    L.wgmma_emu.argtypes = [P, P, P, I, I, I, P]
    return L


def _tf32(x):
    """Values on the TF32 grid (10 explicit mantissa bits), so every product is exact in fp32."""
    return (x.astype(np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


@pytest.mark.parametrize("n", [8, 32, 64])
@pytest.mark.parametrize("ks", [0, 3])
@pytest.mark.parametrize("scale_d", [0, 1])
def test_emulated_wgmma_matches_a_plain_loop(lib, n, ks, scale_d):
    rng = np.random.default_rng(100 * n + 10 * ks + scale_d)
    spread = lambda *s: rng.standard_normal(s) * np.exp2(rng.integers(-8, 9, s))  # noqa: E731
    a, b = _tf32(spread(64, 8)), _tf32(spread(n, 32))
    c = spread(64, n).astype(np.float32)
    out = np.full((64, n), np.nan, np.float32)
    assert lib.wgmma_emu(a.ctypes.data, b.ctypes.data, c.ctypes.data, n, ks, scale_d, out.ctypes.data) == 0
    ref = c.copy() if scale_d else np.zeros((64, n), np.float32)
    for k in range(8):
        ref = ref + a[:, k:k + 1] * b[None, :, 8 * ks + k]
    assert ref.dtype == np.float32
    np.testing.assert_array_equal(out.view(np.uint32), ref.view(np.uint32))
