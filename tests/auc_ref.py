"""numpy restatement of torchmetrics' binned binary AUROC (the `auc` metric of tzrec/models/rank_model.py:296-302), the
yardstick of tzk_binned_auc_update (csrc/tzk_metrics.cuh) and of metrics.binned_auc.

TEST INFRASTRUCTURE.  Written the way torchmetrics states it: `(p >= thr)` comparisons counted per threshold and label,
not as a histogram, so the histogram the kernel builds is checked against the definition it replaces.
"""
import numpy as np
import torch


def thresholds(T: int) -> np.ndarray:
    return torch.linspace(0, 1, T, dtype=torch.float32).numpy()


def confmat(preds, target, thr) -> np.ndarray:
    """[T, 2, 2] int64: [k, y, (p >= thr[k])], over the valid samples (y in {0, 1}, p in [0, 1])."""
    p = np.asarray(preds, dtype=np.float32).reshape(-1)
    y = np.asarray(target).reshape(-1)
    ok = ((y == 0) | (y == 1)) & (p >= 0) & (p <= 1)
    p, y = p[ok], y[ok].astype(np.int64)
    above = p[:, None] >= thr[None, :]                               # [n, T]
    out = np.zeros((len(thr), 2, 2), dtype=np.int64)
    for lab in (0, 1):
        a = above[y == lab]
        out[:, lab, 1] = a.sum(axis=0)
        out[:, lab, 0] = a.shape[0] - out[:, lab, 1]
    return out


def invalid_count(preds, target) -> int:
    p = np.asarray(preds, dtype=np.float32).reshape(-1)
    y = np.asarray(target).reshape(-1)
    return int((~(((y == 0) | (y == 1)) & (p >= 0) & (p <= 1))).sum())


def counts_from_confmat(cm: np.ndarray) -> np.ndarray:
    """The [T + 1, 2] histogram a confusion matrix determines: bin b holds the samples with p >= thr[k] exactly for k < b,
    so (label y) counts[b, y] = cm[b-1, y, 1] - cm[b, y, 1] with cm[-1] = all and cm[T] = none."""
    T = cm.shape[0]
    pos_at = np.concatenate([[cm[0, :, :].sum(axis=1)], cm[:, :, 1], [np.zeros(2, np.int64)]])   # [T + 2, 2]
    return (pos_at[:-1] - pos_at[1:]).astype(np.int64).reshape(T + 1, 2)


def auc_from_confmat(cm: np.ndarray) -> float:
    """torchmetrics' _binary_roc_compute + _auc_compute_without_check, in float64: tpr = tps / (tps + fns) and
    fpr = fps / (fps + tns) (0 where the denominator is 0), flipped, trapezoid."""
    tps, fns = cm[:, 1, 1].astype(np.float64), cm[:, 1, 0].astype(np.float64)
    fps, tns = cm[:, 0, 1].astype(np.float64), cm[:, 0, 0].astype(np.float64)
    d1, d0 = tps + fns, fps + tns
    tpr = np.where(d1 > 0, tps / np.where(d1 > 0, d1, 1), 0.0)[::-1]
    fpr = np.where(d0 > 0, fps / np.where(d0 > 0, d0, 1), 0.0)[::-1]
    return float(np.sum((fpr[1:] - fpr[:-1]) * (tpr[1:] + tpr[:-1])) * 0.5)


def binned_auc(preds, target, T: int) -> float:
    return auc_from_confmat(confmat(preds, target, thresholds(T)))


def mann_whitney_binned(preds, target, T: int) -> float:
    """The same AUC as a float64 rank statistic over the bins: a positive beats a negative in a lower bin, and a pair in
    the same bin counts 1/2 — except in the top bin (p >= thr[T-1]), where the curve has no point above it and such a
    pair gets no credit."""
    thr = thresholds(T)
    p = np.asarray(preds, dtype=np.float32)
    y = np.asarray(target).astype(np.int64)
    b = (p[:, None] >= thr[None, :]).sum(axis=1)
    pos = np.bincount(b[y == 1], minlength=T + 1).astype(np.float64)
    neg = np.bincount(b[y == 0], minlength=T + 1).astype(np.float64)
    P, N = pos.sum(), neg.sum()
    if P == 0 or N == 0:
        return 0.0
    neg_below = np.concatenate([[0.0], np.cumsum(neg)[:-1]])
    ties = pos * neg * 0.5
    ties[T] = 0.0
    return float((np.sum(pos * neg_below) + np.sum(ties)) / (P * N))
