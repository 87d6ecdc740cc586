"""Evaluation metrics of the rank models, with their state on the device.

The reference evaluates with torchmetrics (tzrec/models/rank_model.py:289-398, model.py:207-223):
- `auc`: `AUROC(task="binary", thresholds=T)` on the probabilities.  Its state is a [T, 2, 2] confusion matrix over
  `thr = linspace(0, 1, T)`, which is a function of the histogram of bin(p) = #{k : p >= thr[k]} by label; `BinnedAUC`
  keeps that histogram ([T + 1, 2] int64, built by `tzk_binned_auc_update`) and computes the same curve from it.
- every loss: `MeanMetric` updated with (loss, batch size), i.e. sum(loss_b * B_b) / sum(B_b); `MeanLoss` keeps the two
  sums (float64, int64).
`update` only enqueues device work (it can be captured in a CUDA graph); `compute` reads nothing back from the device.
"""

from typing import Dict, List, Optional

import torch

from . import functional as Fn


class BinnedAUC:
    """torchmetrics.AUROC(task="binary", thresholds=T).  Predictions fp32 or bf16 in [0, 1], labels 0 / 1 (fp32 or int64;
    other dtypes are converted).  A sample outside that domain is counted in `invalid`, and `check_valid` raises for it:
    torchmetrics would re-map such a batch (sigmoid) or raise, and a silently different AUC is worse than either."""

    def __init__(self, thresholds: int, device) -> None:
        T = int(thresholds)
        if T < 1:
            raise ValueError(f"auc: thresholds must be >= 1, got {T}")
        self.thresholds = torch.linspace(0, 1, T, dtype=torch.float32, device=device)    # as torchmetrics builds them
        if T > 1 and not bool((self.thresholds[1:] >= self.thresholds[:-1]).all()):
            raise ValueError("auc: thresholds are not nondecreasing")
        self.counts = torch.zeros((T + 1, 2), dtype=torch.int64, device=device)
        self.invalid = torch.zeros(1, dtype=torch.int64, device=device)

    def update(self, preds: torch.Tensor, target: torch.Tensor) -> None:
        if preds.dtype == torch.float16:          # (FP16 autocast) exact in fp32
            preds = preds.float()
        if target.dtype not in (torch.float32, torch.int64):
            target = target.to(torch.float32 if target.is_floating_point() else torch.int64)
        Fn.backend().binned_auc_update(preds.reshape(-1).contiguous(), target.reshape(-1).contiguous(),
                                       self.thresholds, self.counts, self.invalid)

    def state(self) -> List[torch.Tensor]:
        return [self.counts, self.invalid]

    def check_valid(self, name: str) -> None:
        bad = int(self.invalid.item())
        if bad:
            raise ValueError(f"{name}: {bad} samples had a label outside {{0, 1}} or a prediction that is NaN or outside "
                             "[0, 1]; the binned AUC is undefined for them")

    def compute(self) -> torch.Tensor:
        return binned_auc(self.counts)

    def reset(self) -> None:
        self.counts.zero_()
        self.invalid.zero_()


def binned_auc(counts: torch.Tensor) -> torch.Tensor:
    """AUROC from the [T + 1, 2] histogram (column 0 negatives, column 1 positives), in float64: tps[k] / fps[k] are the
    positives / negatives with bin > k; tpr = tps / P and fpr = fps / N (0 when P or N is 0, torchmetrics' _safe_divide),
    both flipped so the curve runs from thr = 1 to thr = 0, then the trapezoid rule.  No (0, 0) point is prepended: the
    samples in the top bin (p >= thr[T-1] = 1) enter at the first point, without the half credit ties get elsewhere."""
    suffix = counts.flip(0).cumsum(0).flip(0)             # suffix[b] = samples with bin >= b
    total = suffix[0].to(torch.float64).clamp_min(1.0)
    above = suffix[1:].to(torch.float64)                  # [T, 2]: bin > k
    fpr = (above[:, 0] / total[0]).flip(0)
    tpr = (above[:, 1] / total[1]).flip(0)
    return ((fpr[1:] - fpr[:-1]) * (tpr[1:] + tpr[:-1])).sum() * 0.5


class MeanLoss:
    """torchmetrics.MeanMetric updated with (loss, batch size)."""

    def __init__(self, device) -> None:
        self.total = torch.zeros(1, dtype=torch.float64, device=device)
        self.weight = torch.zeros(1, dtype=torch.int64, device=device)

    def update(self, loss: torch.Tensor, n: int) -> None:
        self.total.add_(loss.detach().to(torch.float64) * n)
        self.weight.add_(n)

    def state(self) -> List[torch.Tensor]:
        return [self.total, self.weight]

    def check_valid(self, name: str) -> None:
        pass

    def compute(self) -> torch.Tensor:
        return (self.total / self.weight.to(torch.float64))[0]

    def reset(self) -> None:
        self.total.zero_()
        self.weight.zero_()


def sync_states(metrics: Dict[str, object], group=None) -> None:
    """Sums every metric's state over the ranks of `group` in place, with one all_reduce of the packed
    [counts | invalid | loss sums | batch sums ...] (float64: the counts stay exact below 2**53).  torchmetrics does the
    same sum at compute()."""
    import torch.distributed as dist

    states = [t for m in metrics.values() for t in m.state()]
    if not states:
        return
    packed = torch.cat([t.reshape(-1).to(torch.float64) for t in states])
    if dist.get_backend(group) == "gloo":
        packed = packed.cpu()
    dist.all_reduce(packed, group=group)
    o = 0
    for t in states:
        n = t.numel()
        part = packed[o:o + n].to(t.device)
        t.copy_((part.round() if not t.is_floating_point() else part).to(t.dtype).view_as(t))
        o += n


def snapshot(metrics: Dict[str, object]) -> List[torch.Tensor]:
    return [t.clone() for m in metrics.values() for t in m.state()]


def restore(metrics: Dict[str, object], saved: List[torch.Tensor]) -> None:
    for t, s in zip([t for m in metrics.values() for t in m.state()], saved):
        t.copy_(s)


def compute_all(metrics: Dict[str, object], group: Optional[object] = None, distributed: bool = False
                ) -> Dict[str, torch.Tensor]:
    """{name: value} of every metric (optionally summed over `group` first), then every state reset."""
    try:
        if distributed:
            sync_states(metrics, group)
        for name, m in metrics.items():
            m.check_valid(name)
        return {name: m.compute() for name, m in metrics.items()}
    finally:
        for m in metrics.values():
            m.reset()
