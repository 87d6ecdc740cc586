"""The persistent tile loop and the stage ring of the fused interaction + wide-layer input gradient
(interact_wide_bwd_kernel in torcheasyrec_b200/csrc/tzk_interact_wide.cu), run on the CPU under tests/native/
cuda_cpu_shim.h, sm90_cpu_emu.h and sm90_wgmma_emu.h with the SM count the grid is sized by set through TZK_EMU_SMS.
Each case must give the bits of the unfused chain (gemm3x dgrad, then the tensor-core interaction backward):
  - more tiles than CTAs, so that each CTA's ring runs on from one tile into the next;
  - M = 64 k + 1, a last tile of one sample;
  - M below one tile;
  - a grid of one CTA that walks every tile."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from test_interact_wide_fused import CSRC, EXP, _compile, _data, _p

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P, I64, I32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32
CHILD = os.environ.get("TZK_RING_CHILD") == "1"

# (M, SMs): tiles of 64 samples, grid = min(tiles, SMs)
CASES = [(64 * 6 + 17, 2), (64 * 2 + 1, 2), (40, 132), (64 * 3 + 5, 1)]


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    if CHILD:
        return os.environ["TZK_RING_LIBS"].split(os.pathsep)
    d = tmp_path_factory.mktemp("ring")
    paths = [str(d / "libinteract_wide_cpu.so"), str(d / "libtzk_gemm3x_cpu.so"), str(d / "libitc_cpu.so")]
    for src, out in zip((os.path.join(CSRC, "tzk_interact_wide.cu"), os.path.join(CSRC, "tzk_gemm3x.cu"),
                         os.path.join(EXP, "interact_tc_standalone.cu")), paths):
        _compile(src, out)
    return paths


@pytest.mark.parametrize("M,sms", CASES)
def test_ring_and_tile_loop_give_the_chains_bits(request, libs, M, sms):
    if not CHILD:   # a child process per case: the emulation aborts its process on a protocol violation or a deadlock
        env = {**os.environ, "TZK_RING_CHILD": "1", "TZK_RING_LIBS": os.pathsep.join(libs), "TZK_EMU_SMS": str(sms)}
        r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", request.node.nodeid],
                           capture_output=True, text=True, env=env, timeout=900, cwd=ROOT)
        if r.returncode != 0:
            pytest.fail(f"child exited with {r.returncode}:\n{r.stdout[-3000:]}\n{r.stderr[-2000:]}")
        return
    fused, g3, itc = (ctypes.CDLL(p) for p in libs)
    fused.tzk_interact_wide_bwd.argtypes = [P, I64, P, I64, P, I64, P, I64, I64, P, I64, P, I64, P, P, P]
    g3.tzk_gemm3x.argtypes = [P, I64, P, I64, P, I64, I32, I32, I32, P, I64, P, P, P]
    itc.tzk_itc_bwd.argtypes = [P, I64, P, I64, P, I64, I64, P, I64, P, I64, I32]
    dense, sparse, dz, w = _data(M, 1000 + M)
    dd = np.full((M, 16), np.nan, np.float32)
    ds = np.full((M + 1, 416), np.nan, np.float32)                            # one guard row
    wh, wl = np.empty((784, 64), np.float32), np.empty((784, 64), np.float32)
    assert fused.tzk_interact_wide_bwd(_p(dz), 64, _p(w), 784, _p(dense), 16, _p(sparse), 416, M, _p(dd), 16, _p(ds),
                                       416, _p(wh), _p(wl), None) == 0
    assert np.isnan(ds[M]).all()
    wt = np.ascontiguousarray(w.T)
    dx = np.empty((M, 784), np.float32)
    th, tl = np.empty_like(wt), np.empty_like(wt)
    assert g3.tzk_gemm3x(_p(dz), 64, _p(wt), 64, None, M, 784, 64, 0, _p(dx), 784, _p(th), _p(tl), None) == 0
    cd, cs = np.empty((M, 16), np.float32), np.empty((M, 416), np.float32)
    itc.tzk_itc_bwd(_p(dense), 16, _p(sparse), 416, _p(dx), 784, M, _p(cd), 16, _p(cs), 416, 2)
    np.testing.assert_array_equal(dd, cd)
    np.testing.assert_array_equal(ds[:M], cs)
