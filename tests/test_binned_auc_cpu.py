"""The binned AUC: the numpy restatement of torchmetrics' binned AUROC pinned on hand-derived and reference values, the
package's histogram compute (metrics.binned_auc) against it, and the SOURCE of tzk_binned_auc_update
(csrc/tzk_metrics.cuh) executed on the host (tests/native/cuda_cpu_shim.h) against the restatement, count for count."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import auc_ref
from torcheasyrec_b200.metrics import binned_auc

EXP = os.path.join(os.path.dirname(os.path.abspath(__file__)), "native")
P, I32, I64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64


def _compute(preds, target, T):
    thr = auc_ref.thresholds(T)
    counts = auc_ref.counts_from_confmat(auc_ref.confmat(preds, target, thr))
    return float(binned_auc(torch.from_numpy(counts)))


# ---- the restatement, pinned ---------------------------------------------------------------------------------------
def test_reference_vector():
    """tzrec/metrics/decay_auc_test.py, first compute: these predictions and targets at 10 thresholds give 0.5625."""
    preds = np.array([0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8], dtype=np.float32)
    target = np.array([1, 0, 1, 0, 0, 0, 1, 1])
    assert auc_ref.binned_auc(preds, target, 10) == pytest.approx(0.5625, abs=1e-12)
    assert _compute(preds, target, 10) == pytest.approx(0.5625, abs=1e-12)


def test_ties_at_five_thresholds():
    """thr = [0, .25, .5, .75, 1].  bins: 0.1 -> 1, 0.3 -> 2, 0.6 -> 3, 0.8 -> 4.
    positives {0.6, 0.3}, negatives {0.3, 0.1}: pairs (0.6 > 0.3), (0.6 > 0.1), (0.3 ~ 0.3 half), (0.3 > 0.1) -> 3.5 / 4."""
    preds = np.array([0.6, 0.3, 0.3, 0.1], dtype=np.float32)
    target = np.array([1, 1, 0, 0])
    assert auc_ref.binned_auc(preds, target, 5) == pytest.approx(0.875, abs=1e-15)
    # same bin, different values: 0.26 and 0.49 both land in bin 2 -> a tie
    assert auc_ref.binned_auc(np.array([0.49, 0.26], np.float32), np.array([0, 1]), 5) == pytest.approx(0.5, abs=1e-15)
    assert _compute(preds, target, 5) == pytest.approx(0.875, abs=1e-15)


def test_predictions_on_thresholds_and_the_ends():
    """p >= thr[k] is inclusive: 0.25 counts at thr 0.25 (bin 2), 0.0 is in bin 1, 1.0 in the top bin (5)."""
    thr = auc_ref.thresholds(5)
    p = np.array([0.0, 0.25, 0.5, 0.75, 1.0], dtype=np.float32)
    cm = auc_ref.confmat(p, np.ones(5, np.int64), thr)
    counts = auc_ref.counts_from_confmat(cm)
    np.testing.assert_array_equal(counts[:, 1], [0, 1, 1, 1, 1, 1])
    # positives at 0.5 / 1.0, negatives at 0.25 / 0.75 -> pairs: (0.5 > 0.25), (1 > 0.25), (1 > 0.75) -> 3 / 4
    assert auc_ref.binned_auc(np.array([0.5, 1.0, 0.25, 0.75], np.float32), np.array([1, 1, 0, 0]), 5) == 0.75


@pytest.mark.parametrize("lab", [0, 1])
def test_degenerate_single_class(lab):
    p = np.random.default_rng(1).random(50).astype(np.float32)
    assert auc_ref.binned_auc(p, np.full(50, lab), 200) == 0.0
    assert _compute(p, np.full(50, lab), 200) == 0.0


def test_missing_half_credit_in_the_top_bin():
    """One positive and one negative both at p = 1.0 (fp32 sigmoid of a logit above ~17), plus a positive at 0.5 and a
    negative at 0.0, T = 5.  The curve's first point is thr = 1 with tpr = fpr = 1/2: the segment from there to the next
    point is the only one, so the top-bin tie gets no half credit.
    Points (fpr, tpr) by flipped threshold: 1 -> (.5, .5), .75 -> (.5, .5), .5 -> (.5, 1), .25 -> (.5, 1), 0 -> (1, 1)
    AUC = (1 - .5) * (1 + 1) / 2 = 0.5; the Mann-Whitney value with the tie half-credited would be 0.625."""
    preds = np.array([1.0, 1.0, 0.5, 0.0], dtype=np.float32)
    target = np.array([1, 0, 1, 0])
    assert auc_ref.binned_auc(preds, target, 5) == 0.5
    assert _compute(preds, target, 5) == 0.5
    assert auc_ref.mann_whitney_binned(preds, target, 5) == 0.5


@pytest.mark.parametrize("T", [200, 10000])
def test_equals_mann_whitney_with_half_ties(T):
    rng = np.random.default_rng(T)
    n = 20000
    y = (rng.random(n) < 0.3).astype(np.int64)
    p = np.clip(rng.normal(0.4 + 0.2 * y, 0.2), 0, 0.999).astype(np.float32)
    want = auc_ref.mann_whitney_binned(p, y, T)
    assert auc_ref.binned_auc(p, y, T) == pytest.approx(want, abs=1e-12)
    assert _compute(p, y, T) == pytest.approx(want, abs=1e-12)


# ---- the kernel source on the host ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kern(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("shim") / "libauc_cpu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", EXP, "-x", "c++",
                    os.path.join(EXP, "binned_auc_standalone.cu"), "-shared", "-fPIC", "-o", out], check=True)
    L = ctypes.CDLL(out)
    L.tzk_auc_run.argtypes = [P, I32, P, I32, I64, P, I32, P, P]
    L.tzk_auc_fits_shared.argtypes = [I32]
    return L


def _bf16(x: np.ndarray) -> np.ndarray:
    return torch.from_numpy(x).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)


def _run(kern, p, y, T, offset=0):
    """p: fp32 or uint16 (bf16 bits); y: fp32 or int64.  offset shifts both arrays off 16-B alignment (scalar path)."""
    thr = auc_ref.thresholds(T)
    pb = np.zeros(len(p) + 8, dtype=p.dtype)
    yb = np.zeros(len(y) + 8, dtype=y.dtype)
    pa, ya = pb[offset:offset + len(p)], yb[offset:offset + len(y)]
    pa[:], ya[:] = p, y
    counts = np.full((T + 1) * 2, 7, dtype=np.int64)          # accumulated into
    invalid = np.array([3], dtype=np.int64)
    rc = kern.tzk_auc_run(pa.ctypes.data, int(p.dtype == np.uint16), ya.ctypes.data, int(y.dtype == np.int64), len(p),
                          thr.ctypes.data, T, counts.ctypes.data, invalid.ctypes.data)
    assert rc == 0
    return counts.reshape(T + 1, 2) - 7, int(invalid[0]) - 3


def _want(p_f32, y, T):
    cm = auc_ref.confmat(p_f32, y, auc_ref.thresholds(T))
    return auc_ref.counts_from_confmat(cm), auc_ref.invalid_count(p_f32, y)


def _data(n, seed, ties=True):
    rng = np.random.default_rng(seed)
    p = rng.random(n).astype(np.float32)
    if ties and n >= 8:       # values on the thresholds and at the ends
        p[: n // 8] = auc_ref.thresholds(1000)[rng.integers(0, 1000, n // 8)]
        p[0], p[-1] = 0.0, 1.0
    y = (rng.random(n) < 0.3)
    return p, y


@pytest.mark.parametrize("n", [0, 1, 3, 4, 5, 1000, 65541])
@pytest.mark.parametrize("T", [1, 2, 200, 1000, 10000])
def test_kernel_counts_fp32_preds_fp32_labels(kern, n, T):
    p, y = _data(n, n + T)
    got, bad = _run(kern, p, y.astype(np.float32), T)
    want, wbad = _want(p, y.astype(np.float32), T)
    np.testing.assert_array_equal(got, want)
    assert bad == wbad == 0


@pytest.mark.parametrize("pdt,ldt", [("bf16", "f32"), ("bf16", "i64"), ("f32", "i64")])
@pytest.mark.parametrize("n,T", [(5, 2), (1000, 200), (65541, 10000), (4099, 1000)])
def test_kernel_counts_dtypes(kern, pdt, ldt, n, T):
    p, y = _data(n, 11 * n + T)
    y = y.astype(np.int64) if ldt == "i64" else y.astype(np.float32)
    pk = _bf16(p) if pdt == "bf16" else p
    p_exact = torch.from_numpy(p).to(torch.bfloat16).float().numpy() if pdt == "bf16" else p
    got, bad = _run(kern, pk, y, T)
    want, _ = _want(p_exact, y, T)
    np.testing.assert_array_equal(got, want)
    assert bad == 0


@pytest.mark.parametrize("offset", [1, 3])
def test_kernel_unaligned_inputs_take_the_scalar_path(kern, offset):
    p, y = _data(1001, offset)
    got, _ = _run(kern, p, y.astype(np.float32), 200, offset=offset)
    np.testing.assert_array_equal(got, _want(p, y.astype(np.float32), 200)[0])


def test_kernel_global_atomic_path(kern):
    """A T whose thresholds and histogram exceed one CTA's shared memory takes the global-atomic instantiation."""
    T = 20000
    assert not kern.tzk_auc_fits_shared(T) and kern.tzk_auc_fits_shared(10000)
    # 12 T + 8 B of tables must leave room for the kernel's static shared memory under the 227 KB opt-in limit
    assert kern.tzk_auc_fits_shared(19340) and not kern.tzk_auc_fits_shared(19369)
    p, y = _data(5003, 5)
    got, bad = _run(kern, p, y.astype(np.int64), T)
    np.testing.assert_array_equal(got, _want(p, y.astype(np.int64), T)[0])
    assert bad == 0


@pytest.mark.parametrize("T", [200, 20000])
def test_kernel_counts_invalid_inputs(kern, T):
    p, y = _data(1000, 9)
    y = y.astype(np.float32)
    p[[3, 10, 11]] = [np.nan, -0.5, 1.5]
    y[[20, 21]] = [2.0, 0.5]
    y[3] = 2.0                 # one sample with both defects counts once
    got, bad = _run(kern, p, y, T)
    want, wbad = _want(p, y, T)
    np.testing.assert_array_equal(got, want)
    assert bad == wbad == 5
    yi = (np.arange(1000) % 2).astype(np.int64)
    yi[7] = -1
    got, bad = _run(kern, np.full(1000, 0.5, np.float32), yi, T)
    assert bad == 1 and got.sum() == 999


def test_kernel_rejects_bad_arguments(kern):
    thr = auc_ref.thresholds(4)
    c = np.zeros(10, np.int64)
    inv = np.zeros(1, np.int64)
    p = np.zeros(4, np.float32)
    assert kern.tzk_auc_run(p.ctypes.data, 0, p.ctypes.data, 0, 4, thr.ctypes.data, 0, c.ctypes.data, inv.ctypes.data) == 1
    assert kern.tzk_auc_run(p.ctypes.data, 2, p.ctypes.data, 0, 4, thr.ctypes.data, 4, c.ctypes.data, inv.ctypes.data) == 1
    assert kern.tzk_auc_run(p.ctypes.data, 0, p.ctypes.data, 0, -1, thr.ctypes.data, 4, c.ctypes.data, inv.ctypes.data) == 1
