"""Generates tests/golden/ref_wukong.npz from the REFERENCE's own WuKongLayer (run in the build container only).

tzrec/modules/interaction.py is plain PyTorch: it is loaded file by file through the stub parent packages of
make_golden_from_reference.py and run on seeded parameters and inputs (tests/wukong_ref.py `seeded_case`, which the
tests call again); the fixture stores only what the reference computes: output, input gradient, parameter gradients.

    TZREC_REFERENCE=<checkout of alibaba/TorchEasyRec @ 54cac316> python tests/golden/make_wukong_golden.py

Cases: the wukong_criteo layers (n = 27 with the residual projection, n = 32 with the identity residual; d = 16,
k = 24, f = l = 16; FMB MLP width reduced from 512 to 2 to keep the fixture small) and the three layers of
tzrec/models/wukong_test.py (d = 8, n = 3 -> 7 -> 5 -> 4, k = 2, MLP [4]).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_golden_from_reference import _stub_packages  # noqa: E402
from wukong_ref import seeded_case  # noqa: E402

# tag: (B, d, n, lcb_feature_num, fmb_feature_num, compressed_feature_num, FMB MLP width (one layer), seed)
CASES = {"criteo1": (2, 16, 27, 16, 16, 24, 2, 1), "criteo2": (2, 16, 32, 16, 16, 24, 2, 2),
         "small1": (5, 8, 3, 3, 4, 2, 4, 3), "small2": (5, 8, 7, 3, 2, 2, 4, 4), "small3": (5, 8, 5, 2, 2, 2, 4, 5)}


def main():
    _stub_packages()
    from tzrec.modules.interaction import WuKongLayer  # tzrec/modules/interaction.py:324

    out = {}
    for tag, (B, d, n, l, f, k, h, seed) in CASES.items():
        layer = WuKongLayer(d, n, l, f, k, {"hidden_units": [h]})
        sd, x, dy = seeded_case(B, d, n, l, f, k, [h], seed)
        layer.load_state_dict({name: torch.from_numpy(v) for name, v in sd.items()}, strict=True)
        xt = torch.from_numpy(x).requires_grad_(True)
        y = layer(xt)
        y.backward(torch.from_numpy(dy))
        out.update({f"{tag}_y": y.detach().numpy(), f"{tag}_dx": xt.grad.numpy(),
                    f"{tag}_case": np.array([B, d, n, l, f, k, h, seed])})
        for name, p in layer.named_parameters():
            out[f"{tag}_grad__{name}"] = p.grad.numpy()
    path = os.path.join(HERE, "ref_wukong.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
