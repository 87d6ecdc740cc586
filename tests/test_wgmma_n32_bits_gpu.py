"""The input gradient of the fused wide layer (interact_wide_bwd_kernel) runs its k-steps as m64n32k8 wgmma against the
mma.sync m16n8k8 chain it is compared with bit for bit.  As tests/test_wgmma_bits_gpu.py does for n = 64: 1000 random
operand sets through tests/native/wgmma_bits.cu with C = 0, C != 0 and scale-d = 0, and the hi / lo chain of the 3xTF32
k-step, at n = 32 (tests/native/wgmma_bits_n32.cu)."""
import ctypes
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
SETS = 1000


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("wgmma_n32") / "libwgmma_bits_n32.so")
    subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                    "-shared", "-I", os.path.join(ROOT, "torcheasyrec_b200", "csrc"),
                    os.path.join(ROOT, "tests", "native", "wgmma_bits_n32.cu"), "-o", out], check=True)
    L = ctypes.CDLL(out)
    P = ctypes.c_void_p
    L.wgmma_bits_n32.argtypes = [P, P, P, ctypes.c_int, P, P]
    return L


@pytest.mark.gpu
def test_wgmma_m64n32k8_gives_the_bits_of_mma_sync(lib):
    import torch

    n = 32
    g = torch.Generator(device="cuda").manual_seed(n)

    def spread(*shape):   # magnitudes over 2^-8 .. 2^8, so the products' exponents differ within a k-step
        e = torch.randint(-8, 9, shape, device="cuda", generator=g).float()
        return torch.randn(*shape, device="cuda", generator=g) * torch.exp2(e)

    a, b, c = spread(SETS, 64, 8), spread(SETS, n, 32), spread(SETS, 64, n)
    c[(torch.arange(SETS, device="cuda") // 4) % 2 == 0] = 0.0       # C = 0 under scale-d = 1 as well
    out_wg = torch.full((SETS, 2, 64, n), float("nan"), device="cuda")
    out_mma = torch.full_like(out_wg, float("nan"))
    assert lib.wgmma_bits_n32(a.data_ptr(), b.data_ptr(), c.data_ptr(), SETS, out_wg.data_ptr(),
                              out_mma.data_ptr()) == 0
    assert not torch.isnan(out_mma).any()
    diff = out_wg.view(torch.int32) != out_mma.view(torch.int32)
    per_variant = diff.flatten(2).any(2).sum(0).tolist()
    assert not diff.any(), f"sets whose bits differ, per variant (C / scale-d, 3xTF32): {per_variant}"
