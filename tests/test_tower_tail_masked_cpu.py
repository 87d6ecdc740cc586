"""The fused tower tail's masked mode (csrc/tzk_tower_tail.cuh, kMask), its SOURCE executed on the host
(tests/native/cuda_cpu_shim.h): dy1 is replaced by dZ = dy1 * [y1 > 0] with act_bwd_colsum's predicate, and each
128-row tile's column sums of dZ land in the workspace in act_bwd_colsum_kernel's order at 64 columns (rows r0, r0 + 4,
.. for r0 = 0 .. 3, then the four sums in order), bit for bit against a float32 restatement.  Everything else the
kernel computes is unchanged by the mode."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

EXP = os.path.join(os.path.dirname(os.path.abspath(__file__)), "native")
P, I32, I64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64


@pytest.fixture(scope="module")
def tail(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("shim") / "libtail_masked_cpu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", EXP, "-x", "c++",
                    os.path.join(EXP, "tower_tail_masked_standalone.cu"), "-shared", "-fPIC", "-o", out], check=True)
    L = ctypes.CDLL(out)
    for f in (L.tzk_tail_ws, L.tzk_tail_colsum_offset):
        f.restype = ctypes.c_size_t
        f.argtypes = [I64, I32, I32]
    L.tzk_tail_run_mode.argtypes = [P, I64, P, P, P, P, P, I64, I32, I32, P, P, I64, P, P, ctypes.c_size_t, I32]
    return L


def colsum_partials(dz):
    """act_bwd_colsum_kernel's per-slab sums in float32: [ceil(M / 128), K]."""
    M, K = dz.shape
    parts = []
    for lo in range(0, M, 128):
        s = [np.zeros(K, np.float32) for _ in range(4)]
        for r in range(lo, min(M, lo + 128)):
            s[(r - lo) % 4] = s[(r - lo) % 4] + dz[r]
        v = np.zeros(K, np.float32)
        for r0 in range(4):
            v = v + s[r0]
        parts.append(v)
    return np.stack(parts)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


@pytest.mark.parametrize("K,N,M,pad", [(64, 32, 300, 0), (64, 32, 100, 4), (64, 64, 1, 0), (32, 16, 129, 0),
                                       (13, 7, 257, 3), (60, 33, 128, 0)])
def test_masked_mode_gives_act_bwd_colsum_bits(tail, K, N, M, pad):
    rng = np.random.default_rng(K * 1000 + N * 10 + M)
    y1 = np.maximum(rng.standard_normal((M, K + pad)), 0).astype(np.float32)     # a ReLU output: exact zeros
    y1[rng.random((M, K + pad)) < 0.05] = -0.0
    y1[rng.random((M, K + pad)) < 0.02] = np.nan
    w1 = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    b1 = (0.1 * rng.standard_normal(N)).astype(np.float32)
    w2 = (rng.standard_normal(N) / np.sqrt(N)).astype(np.float32)
    b2 = np.array([0.05], dtype=np.float32)
    lab = (rng.random(M) < 0.3).astype(np.float32)
    nb = tail.tzk_tail_ws(M, K, N)
    off = tail.tzk_tail_colsum_offset(M, K, N)
    tiles = (M + 127) // 128
    assert nb >= (off + tiles * K) * 4

    def run(mask):
        logits = np.full(M, np.nan, dtype=np.float32)
        dy1 = np.full((M, K + pad), np.nan, dtype=np.float32)
        out = np.full(N * K + 2 * N + 2, np.nan, dtype=np.float32)
        ws = np.full(nb // 4, np.nan, dtype=np.float32)
        assert tail.tzk_tail_run_mode(y1.ctypes.data, K + pad, w1.ctypes.data, b1.ctypes.data, w2.ctypes.data,
                                      b2.ctypes.data, lab.ctypes.data, M, K, N, logits.ctypes.data, dy1.ctypes.data,
                                      K + pad, out.ctypes.data, ws.ctypes.data, nb, int(mask)) == 0
        return logits, dy1, out, ws

    logits0, dy1, out0, _ = run(False)
    logits, dz, out, ws = run(True)
    np.testing.assert_array_equal(_bits(logits), _bits(logits0))
    np.testing.assert_array_equal(_bits(out), _bits(out0))
    y = y1[:, :K]
    want = np.where(y > 0, dy1[:, :K], np.float32(0.0))                          # !(y > 0), NaN and -0 included: +0
    np.testing.assert_array_equal(_bits(dz[:, :K]), _bits(want))
    if pad:
        assert np.isnan(dz[:, K:]).all()
    parts = ws[off:off + tiles * K].reshape(tiles, K)
    np.testing.assert_array_equal(_bits(parts), _bits(colsum_partials(want)))
