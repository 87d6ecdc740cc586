"""The CPU checker backend (oracle_backend.OracleKernels) with the evaluation metrics' device update added.

TEST INFRASTRUCTURE.  binned_auc_update is restated from its definition (tests/auc_ref.py: `p >= thr` comparisons and
counting), so evaluation host logic runs on a box without a GPU and is checked against an independent statement.
"""
import numpy as np
import torch

import auc_ref
from oracle_backend import OracleKernels


class MetricOracleKernels(OracleKernels):
    def __init__(self, use_c: bool = False) -> None:
        super().__init__(use_c)
        self.auc_updates = 0

    def binned_auc_update(self, preds, labels, thresholds, counts, invalid):
        p = preds.detach().float().cpu().numpy()
        y = labels.detach().cpu().numpy()
        cm = auc_ref.confmat(p, y, thresholds.cpu().numpy())
        counts += torch.from_numpy(auc_ref.counts_from_confmat(cm)).to(counts.device)
        invalid += auc_ref.invalid_count(p, y)
        self.auc_updates += 1
