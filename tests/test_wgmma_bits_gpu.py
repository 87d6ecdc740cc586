"""The fused wide-layer kernels (torcheasyrec_b200/csrc/tzk_interact_wide.cu) run their 3xTF32 k-steps on wgmma, while the
layer-by-layer chain they are compared with bit for bit runs on mma.sync m16n8k8.  That rests on one k8 wgmma giving the
bits of the n / 8 mma.sync it replaces for the same operands and C.  tests/native/wgmma_bits.cu computes 1000 random
operand sets both ways, with C = 0, C != 0 and scale-d = 0, and with the hi / lo split operands of the 3xTF32 k-step."""
import ctypes
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
SETS = 1000


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("wgmma") / "libwgmma_bits.so")
    subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                    "-shared", "-I", os.path.join(ROOT, "torcheasyrec_b200", "csrc"),
                    os.path.join(ROOT, "tests", "native", "wgmma_bits.cu"), "-o", out], check=True)
    L = ctypes.CDLL(out)
    P = ctypes.c_void_p
    L.wgmma_bits.argtypes = [P, P, P, ctypes.c_int, ctypes.c_int, P, P]
    return L


@pytest.mark.gpu
def test_wgmma_k8_gives_the_bits_of_mma_sync(lib):
    import torch

    n = 64
    g = torch.Generator(device="cuda").manual_seed(n)

    def spread(*shape):   # magnitudes over 2^-8 .. 2^8, so the products' exponents differ within a k-step
        e = torch.randint(-8, 9, shape, device="cuda", generator=g).float()
        return torch.randn(*shape, device="cuda", generator=g) * torch.exp2(e)

    a, b, c = spread(SETS, 64, 8), spread(SETS, n, 32), spread(SETS, 64, n)
    c[(torch.arange(SETS, device="cuda") // 4) % 2 == 0] = 0.0       # C = 0 under scale-d = 1 as well
    out_wg = torch.full((SETS, 2, 64, n), float("nan"), device="cuda")
    out_mma = torch.full_like(out_wg, float("nan"))
    assert lib.wgmma_bits(a.data_ptr(), b.data_ptr(), c.data_ptr(), SETS, n, out_wg.data_ptr(),
                          out_mma.data_ptr()) == 0
    assert not torch.isnan(out_mma).any()
    diff = out_wg.view(torch.int32) != out_mma.view(torch.int32)
    per_variant = diff.flatten(2).any(2).sum(0).tolist()
    assert not diff.any(), f"sets whose bits differ, per variant (C / scale-d, 3xTF32): {per_variant}"
