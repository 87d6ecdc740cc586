"""Generates tests/golden/ref_dlrm_bf16.npz from the REFERENCE's own modules (run in the build container only): the DLRM
predict glue (tzrec/models/dlrm.py:113-131) and its BCE loss under torch.autocast("cpu", torch.bfloat16), the way
tzrec/models/model.py:271-297 runs a train step with train_config.mixed_precision "BF16".  The modules are loaded file by
file as in make_golden_from_reference.py; the tests read only the fixture.

    TZREC_REFERENCE=<checkout of alibaba/TorchEasyRec> python tests/golden/make_golden_mixed_precision.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden_from_reference import _stub_packages  # noqa: E402


def main():
    _stub_packages()
    from tzrec.modules.interaction import InteractionArch  # tzrec/modules/interaction.py:57
    from tzrec.modules.mlp import MLP  # tzrec/modules/mlp.py:86

    torch.manual_seed(20261015)
    out = {}
    B, Ns, D = 48, 26, 16
    dense_mlp = MLP(13, [64, 16])
    final_mlp = MLP(351 + 16 + Ns * D, [64, 32])
    head = torch.nn.Linear(32, 1)
    dense_in = torch.rand(B, 13)
    sparse = torch.randn(B, Ns * D, requires_grad=True)
    labels = (torch.rand(B) < 0.25).float()
    with torch.autocast("cpu", torch.bfloat16):
        dense_feat = dense_mlp(dense_in)
        feat = torch.cat([dense_feat.unsqueeze(1), sparse.reshape(-1, Ns, D)], dim=1)
        all_feat = InteractionArch(Ns + 1)(feat)
        all_feat = torch.cat([all_feat, dense_feat], dim=-1)
        all_feat = torch.cat([all_feat, sparse], dim=-1)
        logits = head(final_mlp(all_feat)).squeeze(1)
        loss = torch.nn.functional.binary_cross_entropy_with_logits(logits, labels)
    loss.backward()
    assert dense_feat.dtype == torch.bfloat16 and feat.dtype == torch.float32 and all_feat.dtype == torch.float32
    assert logits.dtype == torch.bfloat16 and loss.dtype == torch.float32
    out["dense_in"], out["sparse"], out["labels"] = dense_in.numpy(), sparse.detach().numpy(), labels.numpy()
    out["all_feat"] = all_feat.detach().numpy()
    out["logits"] = logits.detach().float().numpy()
    out["loss"] = loss.detach().numpy()
    out["dsparse"] = sparse.grad.numpy()
    for prefix, mod in [("dense_mlp", dense_mlp), ("final_mlp", final_mlp), ("output_mlp", head)]:
        for k, v in mod.state_dict().items():
            out[f"sd__{prefix}.{k}"] = v.numpy()
        for k, p in mod.named_parameters():
            out[f"grad__{prefix}.{k}"] = p.grad.numpy()
    np.savez_compressed(os.path.join(HERE, "ref_dlrm_bf16.npz"), **out)
    print("wrote", os.path.join(HERE, "ref_dlrm_bf16.npz"), len(out), "arrays")


if __name__ == "__main__":
    main()
