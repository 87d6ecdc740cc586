"""Generates tests/golden/ref_masknet.npz from the REFERENCE's own MaskNetModule (run in the build container only).

tzrec/modules/masknet.py is plain PyTorch: it is loaded file by file through the stub parent packages of
make_golden_from_reference.py and run on seeded parameters and inputs (tests/masknet_ref.py `seeded_case`, which the
tests call again); the fixture stores only what the reference computes: output, input gradient, every parameter
gradient, and the module's state-dict key list.

    TZREC_REFERENCE=<checkout of alibaba/TorchEasyRec @ 54cac316> python tests/golden/make_masknet_golden.py

Cases: E = 429 (masknet_criteo's group width) with a small ratio and small H, parallel and serial; a non-dyadic ratio
(0.3); the shapes of tzrec/modules/masknet_test.py (E = 24, ratio 2, H = 16, top [8, 4, 2], dropout 0 here) in both
modes; the shapes of tzrec/models/masknet_test.py (E = 33, ratio 2 overriding aggregation_dim 32, H = 16, top [8, 4]).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_golden_from_reference import _stub_packages  # noqa: E402
from masknet_ref import seeded_case  # noqa: E402

# tag: (B, E, reduction_ratio, aggregation_dim, hidden_dim, n_mask_blocks, top_mlp units, use_parallel, seed)
CASES = {"criteo_par": (3, 429, 0.02, 0, 8, 3, [4], True, 1),
         "criteo_ser": (3, 429, 0.02, 0, 64, 2, [4], False, 2),
         "ratio03": (5, 40, 0.3, 0, 12, 2, [6, 3], True, 3),
         "modtest_par": (4, 24, 2.0, 0, 16, 3, [8, 4, 2], True, 4),
         "modtest_ser": (4, 24, 2.0, 0, 16, 3, [8, 4, 2], False, 5),
         "modeltest": (2, 33, 2.0, 32, 16, 3, [8, 4], True, 6)}


def case_array(B, E, ratio, agg, H, nb, top, parallel, seed):
    return np.array([B, E, ratio, agg, H, nb, parallel, seed] + list(top), np.float64)


def main():
    _stub_packages()
    from tzrec.modules.masknet import MaskNetModule  # tzrec/modules/masknet.py:88

    out = {}
    for tag, (B, E, ratio, agg, H, nb, top, parallel, seed) in CASES.items():
        mod = MaskNetModule(E, nb, dict(reduction_ratio=ratio, aggregation_dim=agg, hidden_dim=H),
                            dict(hidden_units=top, activation="nn.ReLU", use_bn=False, dropout_ratio=0.0), parallel)
        sd, e, dy = seeded_case(B, E, ratio, agg, H, nb, top, parallel, seed)
        mod.load_state_dict({name: torch.from_numpy(v) for name, v in sd.items()}, strict=True)
        et = torch.from_numpy(e).requires_grad_(True)
        y = mod(et)
        y.backward(torch.from_numpy(dy))
        out.update({f"{tag}_y": y.detach().numpy(), f"{tag}_de": et.grad.numpy(),
                    f"{tag}_case": case_array(B, E, ratio, agg, H, nb, top, parallel, seed),
                    f"{tag}_keys": np.array(list(mod.state_dict()))})
        for name, p in mod.named_parameters():
            out[f"{tag}_grad__{name}"] = p.grad.numpy()
    path = os.path.join(HERE, "ref_masknet.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
