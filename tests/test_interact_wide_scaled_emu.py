"""The dZ scale of the fused interaction + wide-layer input gradient and weight gradient (tzk_interact_wide_bwd_scaled,
tzk_interact_wide_wgrad_scaled in torcheasyrec_b200/csrc/tzk_interact_wide.cu), run on the CPU under tests/native/
cuda_cpu_shim.h, sm90_cpu_emu.h and sm90_wgmma_emu.h: with dz_scale = [s] both give the bits of the unscaled entry
points fed dz * s, for s = 1 and s = 2.5, through the bwd kernel's ring across tiles (TZK_EMU_SMS) and the weight
gradient's slabs."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from test_interact_wide_fused import CSRC, _compile, _data, _p

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P, I64, I32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32
CHILD = os.environ.get("TZK_SCALE_CHILD") == "1"


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    if CHILD:
        return os.environ["TZK_SCALE_LIB"]
    out = str(tmp_path_factory.mktemp("scaled") / "libinteract_wide_cpu.so")
    _compile(os.path.join(CSRC, "tzk_interact_wide.cu"), out)
    return out


def _delegate(request, lib, sms) -> bool:
    """A child pytest process per case: the emulation aborts its process on a protocol violation or a deadlock."""
    if CHILD:
        return False
    env = {**os.environ, "TZK_SCALE_CHILD": "1", "TZK_SCALE_LIB": lib, "TZK_EMU_SMS": str(sms)}
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", request.node.nodeid],
                       capture_output=True, text=True, env=env, timeout=900, cwd=ROOT)
    if r.returncode != 0:
        pytest.fail(f"child exited with {r.returncode}:\n{r.stdout[-3000:]}\n{r.stderr[-2000:]}")
    return True


def _load(path):
    L = ctypes.CDLL(path)
    L.tzk_interact_wide_bwd.argtypes = [P, I64, P, I64, P, I64, P, I64, I64, P, I64, P, I64, P, P, P]
    L.tzk_interact_wide_bwd_scaled.argtypes = [P, I64, P, P, I64, P, I64, P, I64, I64, P, I64, P, I64, P, P, P]
    L.tzk_interact_wide_wgrad.argtypes = [P, I64, P, I64, P, I64, P, I64, I64, I32, P, P, I64, P]
    L.tzk_interact_wide_wgrad_scaled.argtypes = [P, I64, P, P, I64, P, I64, P, I64, I64, I32, P, P, I64, P]
    return L


@pytest.mark.parametrize("scale", [1.0, 2.5])
@pytest.mark.parametrize("M,sms", [(64 * 3 + 5, 2), (40, 132)])
def test_scaled_bwd_is_bwd_of_scaled_dz(request, lib, M, sms, scale):
    if _delegate(request, lib, sms):
        return
    L = _load(lib)
    dense, sparse, dz, w = _data(M, 2000 + M)
    dz[::7, ::5] = 0.0                                                       # masked entries of a ReLU backward
    s = np.array([scale], np.float32)
    wh, wl = np.empty((784, 64), np.float32), np.empty((784, 64), np.float32)
    dd, ds = np.full((M, 16), np.nan, np.float32), np.full((M, 416), np.nan, np.float32)
    assert L.tzk_interact_wide_bwd_scaled(_p(dz), 64, _p(s), _p(w), 784, _p(dense), 16, _p(sparse), 416, M, _p(dd), 16,
                                          _p(ds), 416, _p(wh), _p(wl), None) == 0
    dzs = dz * s[0]                                                          # float32 products
    rd, rs = np.full((M, 16), np.nan, np.float32), np.full((M, 416), np.nan, np.float32)
    assert L.tzk_interact_wide_bwd(_p(dzs), 64, _p(w), 784, _p(dense), 16, _p(sparse), 416, M, _p(rd), 16, _p(rs), 416,
                                   _p(wh), _p(wl), None) == 0
    np.testing.assert_array_equal(dd.view(np.uint32), rd.view(np.uint32))
    np.testing.assert_array_equal(ds.view(np.uint32), rs.view(np.uint32))


@pytest.mark.parametrize("scale", [1.0, 2.5])
@pytest.mark.parametrize("M,slabs", [(200, 3), (45, 2)])
def test_scaled_wgrad_is_wgrad_of_scaled_dz(request, lib, M, slabs, scale):
    if _delegate(request, lib, 132):
        return
    L = _load(lib)
    dense, sparse, dz, _ = _data(M, 3000 + M)
    dz[::5, ::3] = 0.0
    rng = np.random.default_rng(M)
    pairs = rng.standard_normal((M, 352)).astype(np.float32)
    pairs[:, 351] = 0.0
    s = np.array([scale], np.float32)
    part = np.full(slabs * 896 * 64, np.nan, np.float32)
    dw, rw = np.full((64, 784), np.nan, np.float32), np.full((64, 784), np.nan, np.float32)
    assert L.tzk_interact_wide_wgrad_scaled(_p(dz), 64, _p(s), _p(pairs), 352, _p(dense), 16, _p(sparse), 416, M, slabs,
                                            _p(part), _p(dw), 784, None) == 0
    dzs = dz * s[0]
    assert L.tzk_interact_wide_wgrad(_p(dzs), 64, _p(pairs), 352, _p(dense), 16, _p(sparse), 416, M, slabs, _p(part),
                                     _p(rw), 784, None) == 0
    np.testing.assert_array_equal(dw.view(np.uint32), rw.view(np.uint32))
